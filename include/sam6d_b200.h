/*
 * sam6d_b200.h -- C ABI of libsam6d_b200.so: the H100 (sm_90a) kernels behind SAM-6D's data-parallel hot path.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (the Python host passes torch storage);
 *     nothing is allocated, freed or synchronised inside the library;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream); calls are asynchronous;
 *   - return value: 0 on success, a positive cudaError_t if a launch / runtime call failed, -22 (EINVAL) if an
 *     argument violates the documented contract.  The library never calls exit() (the reference's native layer
 *     does: PEM/model/pointnet2/_ext_src/include/cuda_utils.h:35-44);
 *   - tensors are dense row-major fp32 unless stated; index tensors are int32 (as in the reference's _ext).
 *
 * Reference paths: PEM = SAM-6D/Pose_Estimation_Model, ISM = SAM-6D/Instance_Segmentation_Model,
 *                  PN2 = PEM/model/pointnet2.
 */
#ifndef SAM6D_B200_H
#define SAM6D_B200_H

#ifdef __cplusplus
extern "C" {
#endif

/* ---- point-cloud ops: replace the pybind module pointnet2._ext (PN2/_ext_src/src/bindings.cpp:11-24) ---------- */

/* _ext.furthest_point_sampling (PN2/_ext_src/src/sampling.cpp:67-91, sampling_gpu.cu:75-178).
 * xyz (b,n,3) -> idx (b,m); idx[:,0] = 0; ties resolved exactly like the reference kernel.
 * temp: scratch (b,n) f32, required only when n > 4096. */
int sam6d_fps(const float* xyz, int b, int n, int m, float* temp, int* idx, void* stream);
/* the single-CTA general-n FPS kernel on its own (comparator of the cluster kernel that sam6d_fps uses for 4096 < n <= 212 992) */
int sam6d_fps_single_cta(const float* xyz, int b, int n, int m, float* temp, int* idx, void* stream);

/* _ext.gather_points (PN2/_ext_src/src/sampling.cpp:18-41, sampling_gpu.cu:13-25): points (b,c,n), idx (b,m) -> (b,c,m) */
int sam6d_gather_points(const float* points, const int* idx, int b, int c, int n, int m, float* out, void* stream);

/* channel-last form used inside the model: out[b,j,:] = src[b, idx[b,j], :] (zeros where idx < 0), src batch stride in elements
 * (sample_pts_feats PEM/utils/model_utils.py:53-66; SparseToDenseTransformer._sample_feats PEM/model/transformer.py:651-658) */
int sam6d_gather_rows(const float* src, const int* idx, int b, int n, int m, int c, long long src_bstride, float* out,
                      void* stream);
/* same gather from a bf16 token matrix, widened to fp32 (c % 8 == 0) */
int sam6d_gather_rows_bf16_f32(const void* src, const int* idx, int b, int n, int m, int c, long long src_bstride, float* out,
                               void* stream);

/* _ext.ball_query (PN2/_ext_src/src/ball_query.cpp:11-35, ball_query_gpu.cu:14-49): new_xyz (b,m,3), xyz (b,n,3)
 * -> idx (b,m,nsample): first nsample hits with d2 < r*r in ascending index order, padded with the first hit,
 * all zero when empty.  cnt (b,m), optional: number of distinct hits kept. */
int sam6d_ball_query(const float* new_xyz, const float* xyz, int b, int n, int m, float radius, int nsample, int* idx,
                     int* cnt, void* stream);
/* two concentric queries (radius_a <= radius_b) of the same clouds in one sweep; outputs as from two sam6d_ball_query calls
 * (PositionalEncoding groups at r1/ns1 and r2/ns2, PEM/model/fine_point_matching.py:104-109) */
int sam6d_ball_query_pair(const float* new_xyz, const float* xyz, int b, int n, int m, float radius_a, int nsample_a,
                          float radius_b, int nsample_b, int* idx_a, int* idx_b, int* cnt_a, int* cnt_b, void* stream);

/* _ext.group_points (PN2/_ext_src/src/group_points.cpp:13-38, group_points_gpu.cu:13-33): points (b,c,n), idx (b,np,ns) -> (b,c,np,ns) */
int sam6d_group_points(const float* points, const int* idx, int b, int c, int n, int np, int ns, float* out, void* stream);

/* ---- dense linear algebra ------------------------------------------------------------------------------------ */

/* C[z] = alpha * A[z] W[z]^T (+ bias) (act) (+ R[z]) for z < batch; `relu` is the activation code 0 none / 1 ReLU / 2 GELU(erf).  A (M,K) lda; W (N,K) ldw (nn.Linear layout);
 * C (M,N) ldc; R (M,N) ldr or NULL; sA..sR batch strides in elements (0 = shared).  fp32 CUDA-core path
 * (every nn.Linear / 1x1 conv of PEM/model/transformer.py, coarse/fine_point_matching.py; the score matrix
 * compute_feature_similarity PEM/utils/model_utils.py:114-136 as a batched call with alpha = 1/temp). */
int sam6d_gemm_f32(const float* A, const float* W, const float* bias, const float* R, float* C, int M, int N, int K,
                   long long lda, long long ldw, long long ldc, long long ldr, int batch, long long sA, long long sW,
                   long long sC, long long sR, float alpha, int relu, void* stream);

/* Same contract on the tensor cores: bf16 operands (dtype code 0 = fp32 converted while staging, 1 = bf16), fp32
 * accumulation in registers (wgmma m64n256k16), C fp32 (0) or bf16 (1).  K % 8 == 0, 16-byte aligned operand rows. */
int sam6d_gemm_bf16(const void* A, int a_dtype, const void* W, int w_dtype, const float* bias, const float* R, void* C,
                    int c_dtype, int M, int N, int K, long long lda, long long ldw, long long ldc, long long ldr, int batch,
                    long long sA, long long sW, long long sC, long long sR, float alpha, int relu, void* stream);

/* Persistent TMA-fed version for plain (non-batched) bf16 operands: cp.async.bulk.tensor boxes with SWIZZLE_128B feed a
 * 4-stage ring consumed by two wgmma warpgroups.  A (M,K) bf16, W (N,K) bf16, C fp32 (0) / bf16 (1).
 * act: 0 none, 1 ReLU, 2 GELU(erf), 3 SwiGLU -- W holds a w12 whose rows are interleaved in blocks of 128 (gate rows of hidden
 * units [128t, 128t+128), then their up rows), bias packed alike; C (M, N/2) bf16 = silu(gate) * up; N % 256 == 0, bias, no
 * residual. */
int sam6d_gemm_tma(const void* A, const void* W, const float* bias, const void* R, void* C, int c_dtype, int M, int N, int K,
                   long long lda, long long ldw, long long ldc, long long ldr, float alpha, int act, void* stream);
/* `batch` independent problems stacked along the rows of A and W (problem z: rows [z*a_rpb, +M) of A, [z*w_rpb, +N) of W,
 * output at C + z*c_bs elements): the per-proposal cosine score matrices (PEM/utils/model_utils.py:114-136). */
int sam6d_gemm_tma_batched(const void* A, const void* W, const float* bias, const void* R, void* C, int c_dtype, int M, int N, int K,
                           long long lda, long long ldw, long long ldc, long long ldr, int batch, long long a_rpb, long long w_rpb,
                           long long c_bs, long long r_bs, float alpha, int act, void* stream);
/* fused QKV / KV projection (bf16 out, bias): output columns [vt_col0, N) are written transposed per cloud of vt_S token rows
 * into Vt[(cloud * (N - vt_col0) + c) * vt_N1 + token] (the V^T operand of sam6d_attn_tc) instead of C; the key-padding columns
 * [vt_S, vt_N1) of Vt are left untouched and must be finite. */
int sam6d_gemm_tma_vt(const void* A, const void* W, const float* bias, void* C, int M, int N, int K, long long lda, long long ldw,
                      long long ldc, void* Vt, int vt_col0, int vt_S, int vt_N1, void* stream);
/* sam6d_gemm_tma_vt with a third column range: [0, vt_col0) -> C, [vt_col0, vt_col1) -> Vt, [vt_col1, N) -> C2 (M, N - vt_col1)
 * bf16, row stride ldc2: one launch for the q | k | v | u projections of an RPE self-attention layer */
int sam6d_gemm_tma_vt2(const void* A, const void* W, const float* bias, void* C, int M, int N, int K, long long lda, long long ldw,
                       long long ldc, void* Vt, int vt_col0, int vt_col1, int vt_S, int vt_N1, void* C2, long long ldc2,
                       void* stream);

/* ---- token-row ops (row r lives at base + (r / rpb) * bstride + (r % rpb) * ld) ----------------------------------- */

/* nn.LayerNorm(C) (PEM/model/transformer.py:156,188,423,572) */
int sam6d_layernorm(const float* x, long long x_rpb, long long x_bstride, long long x_ld, float* y, long long y_rpb,
                    long long y_bstride, long long y_ld, const float* gamma, const float* beta, long long rows, int C,
                    float eps, void* stream);
/* same, writing bf16 rows (the A operand of the next tensor-core GEMM) */
int sam6d_layernorm_bf16(const float* x, long long x_rpb, long long x_bstride, long long x_ld, void* y, long long y_rpb,
                         long long y_bstride, long long y_ld, const float* gamma, const float* beta, long long rows, int C,
                         float eps, void* stream);
/* bf16 rows in and out, statistics in fp32 */
int sam6d_layernorm_bf16io(const void* x, long long x_rpb, long long x_bstride, long long x_ld, void* y, long long y_rpb,
                           long long y_bstride, long long y_ld, const float* gamma, const float* beta, long long rows, int C,
                           float eps, void* stream);
/* F.normalize(x, p=2, dim=-1) (PEM/utils/model_utils.py:124-126; ISM/model/loss.py:32-33) */
int sam6d_l2norm_rows(const float* x, long long x_rpb, long long x_bstride, long long x_ld, float* y, long long y_rpb,
                      long long y_bstride, long long y_ld, long long rows, int C, void* stream);
int sam6d_l2norm_rows_bf16(const float* x, long long x_rpb, long long x_bstride, long long x_ld, void* y, long long y_rpb,
                           long long y_bstride, long long y_ld, long long rows, int C, void* stream);
/* focused-linear-attention feature map (PEM/model/transformer.py:541-550); softplus_scale (C) = softplus(scale) */
int sam6d_focus_rows(const float* x, long long x_rpb, long long x_bstride, long long x_ld, float* y, long long y_rpb,
                     long long y_bstride, long long y_ld, const float* softplus_scale, long long rows, int C, void* stream);
/* out = (p - t) @ R per proposal (PEM/model/fine_point_matching.py:44) */
int sam6d_rigid_warp(const float* p, const float* R, const float* t, int b, int n, float* out, void* stream);
/* radius[b] = max_i ||po[b,i]|| and x / (radius + 1e-6) (PEM/model/feature_extraction.py:139-142) */
int sam6d_cloud_radius(const float* po, int b, int n, float* radius, void* stream);
int sam6d_scale_by_radius(const float* src, const float* radius, int b, long long per_batch, float* dst, void* stream);

/* ---- geometric structure embedding (PEM/model/transformer.py:286-349) -------------------------------------------- */

/* pts (b,S,3) -> T (b,S,S,4) = {angle index k=0..2, distance index} (get_embedding_indices, :302-332) */
int sam6d_geo_indices(const float* pts, int b, int S, float sigma_d, float factor_a, float* T, void* stream);
/* T (npairs,4) -> E (npairs,256) = proj_d(sin_emb(d)) + max_k proj_a(sin_emb(a_k)) (forward, :334-349); WaT/WdT are
 * (in,out) transposes of the nn.Linear weights, bias = proj_a.bias + proj_d.bias, div_term the module buffer. */
int sam6d_geo_embed_f32(const float* T, long long npairs, const float* div_term, const float* WaT, const float* WdT,
                        const float* bias, float* E, void* stream);

/* tensor-core version (wgmma, bf16 operands, fp32 accumulate): Wa/Wd are the (out,in) weights in bf16, E fp32 (0) or bf16 (1) */
int sam6d_geo_embed_tc(const float* T, long long npairs, const float* div_term, const void* Wa_bf16, const void* Wd_bf16,
                       const float* bias, void* E, int e_is_bf16, void* stream);
/* the distance projection of sam6d_geo_embed_tc alone: T (npairs,4) f32 -> E (npairs,256) bf16 = proj_d(emb(T[:,3])) + bias */
int sam6d_geo_embed_dist_tc(const float* T, long long npairs, const float* div_term, const void* Wd_bf16, const float* bias, void* E,
                            void* stream);
/* GeometricStructureEmbedding by table interpolation (csrc/geo_lut.cu; transformer.py:334-349): g_a(x) = W_a emb(x) and
 * g_d(x) = W_d emb(x) + bias are functions of ONE scalar, tabulated on a uniform grid (tabA (na,256) bf16 at step 1/inv_ha from 0,
 * tabD (nd,256) bf16 at step 1/inv_hd) -> E (clouds*S*S,256) bf16 = lerp(tabD, d) + max_k lerp(tabA, a_k), written once.
 * Distances outside tabD: row 0 / column 0 of a cloud read far (clouds,2,S,256) bf16 (exact g_d of those 2 S distances, from
 * sam6d_geo_embed_dist_tc); any other pair is evaluated exactly from div_term (128 f32), WdT (256 in, 256 out) bf16 and bias.
 * Interpolation, maximum and sum in fp32 with one rounding at the store. */
int sam6d_geo_embed_lut(const float* T, long long clouds, int S, const void* tabA, int na, float inv_ha, const void* tabD, int nd,
                        float inv_hd, const void* far, const float* div_term, const void* WdT_bf16, const float* bias, void* E,
                        void* stream);

/* ---- PEM input builder (PEM/run_inference_custom.py:165-253 get_test_data; PEM/utils/data_utils.py:73-160) ----------- */

/* Stage A, all P detections of a frame: uncompressed COCO RLE (column-major runs; rle_cum = cumulative run ends of every
 * detection concatenated, rle_off (P+1) offsets) -> mask AND depth > 0 (P,H,W) u8; stats (P,12) i32 = [0..3] raw extremes,
 * [4] pixel count, [5..8] get_bbox y1,y2,x1,x2, [9] points that survive the radius filter ||p - mean|| < thr;
 * choose2 (P,cap) i32 crop-linear pixel indices and cloud2 (P,cap,3) f32 camera-frame points of the survivors, in the
 * reference's order.  depth (H,W) f32 metres; fx, fy, cx, cy float64 intrinsics; cap >= min(H,W)^2; choose1 scratch. */
int sam6d_inputs_stage_a(const int* rle_cum, const int* rle_off, int P, int H, int W, const float* depth, double fx, double fy,
                         double cx, double cy, double thr, unsigned char* mask, int* stats, int cap, int* choose1, int* choose2,
                         float* cloud2, void* stream);
/* Stage B, the Q kept detections keep[q]: choose_idx (Q,ns) i32 sample indices (drawn by the host like the reference's
 * np.random.choice) -> pts (Q,ns,3) f32, rgb_choose (Q,ns) i64 (get_resize_rgb_choose), rgb (Q,3,S,S) f32 = crop, channel
 * flip, mask, cv2.INTER_LINEAR resize (uint8 fixed point, bit exact), ToTensor + Normalize; rgb_u8 (Q,S,S,3) or NULL. */
int sam6d_inputs_stage_b(const int* stats, const int* keep, int Q, int H, int W, int cap, const int* choose2, const float* cloud2,
                         const int* choose_idx, int ns, int S, const unsigned char* image, const unsigned char* mask, int mask_flag,
                         float* pts, long long* rgb_choose, float* rgb, unsigned char* rgb_u8, void* stream);

/* crop, channel flip, mask, cv2.INTER_LINEAR resize (uint8 fixed point, bit exact), ToTensor + Normalize for Q images of their
 * own (the template renderings of _get_template, run_inference_custom.py:117-136): images (Q,H,W,3) u8, masks (Q,H,W) u8,
 * bbox (Q,4) i32 = y1,y2,x1,x2 (square) -> rgb (Q,3,S,S) f32, rgb_u8 (Q,S,S,3) or NULL */
int sam6d_crop_resize_normalize(const unsigned char* images, const unsigned char* masks, const int* bbox, int Q, int H, int W, int S,
                                int mask_flag, float* rgb, unsigned char* rgb_u8, void* stream);

/* ---- ISM proposal descriptors around the DINOv2 trunk (ISM/model/dinov2.py:131-258, ISM/utils/bbox_utils.py:89-126,
 *      ISM/model/loss.py:46-77) ---------------------------------------------------------------------------------------- */

/* process_rgb_proposals / process_masks_proposals for all P proposals: image (H,W,3) u8 RGB, masks (P,H,W) f32, boxes (P,4) i32
 * xyxy -> rgb (P,3,T,T) f32 (ToTensor + Normalize, x mask, box crop, nearest resize to longer side T, centre pad) and / or
 * pmask (P,T,T) f32 (same geometry); either output may be NULL */
int sam6d_crop_resize_pad(const unsigned char* image, const float* masks, const int* boxes, int P, int H, int W, int T, float* rgb,
                          float* pmask, void* stream);
/* compute_cls_and_patch_features tail: patch token (p,t) = tokens + p*tok_bs + t*tok_ld (C f32); kept when the mean of its
 * patch x patch block of pmask (P, G*patch, G*patch) exceeds thresh, then L2-normalised, else zero -> out_f32 / out_bf16
 * (P, G*G, C) (either NULL), valid (P, G*G) u8 or NULL */
int sam6d_masked_patch_normalize(const float* tokens, long long tok_ld, long long tok_bs, const float* pmask, int P, int G, int patch,
                                 int C, float thresh, float* out_f32, void* out_bf16, unsigned char* valid, void* stream);
/* MaskedPatch_MatrixSimilarity.compute_straight + compute_visible_ratio on sim (P,N,N) f32 = query patches x best-template
 * patches^T (row stride sim_ld, batch stride sim_bs, N <= 256); qvalid (P,N) u8 -> appe (P) f32, vis (P) f32 */
int sam6d_appearance_reduce(const float* sim, long long sim_ld, long long sim_bs, int P, int N, const unsigned char* qvalid, float thred,
                            float* appe, float* vis, void* stream);

/* ---- ISM geometric score (ISM/model/detector.py:209-258, 311-323; ISM/utils/trimesh_utils.py:77-105; ISM/utils/bbox_utils.py:197-221) */

/* Calculate_the_query_translation -> depth_image_to_pointcloud_translate_torch: masks (N,H,W) f32 0/1, depth (H,W) i32, K (3,3) f64
 * row-major ON THE DEVICE, depth_scale -> translate (N,3) f32 = mean back-projected point of the masked depth (float64 sums) */
int sam6d_query_translation(const float* masks, const int* depth, int N, int H, int W, const double* K, double depth_scale,
                            float* translate, void* stream);
/* project_template_to_image + the IoU of compute_geometric_score: poses (T,4,4) f32, pointcloud (O,npc,3) f32, best_pose / pred_obj
 * (N) i64, translate (N,3) f32, K (3,3) f64 on the device, boxes (N,4) i64 xyxy -> image_vu (N,npc,2) i32 or NULL, xyxy (N,4) i32
 * (box of the projected samples), iou (N) f32, ok (N) u8 (non-empty intersection; the reference scores the batch 0 unless all are) */
int sam6d_project_template_iou(const float* poses, int T, const float* pointcloud, int O, int npc, const long long* best_pose,
                               const long long* pred_obj, const float* translate, const double* K, int N, int H, int W,
                               const long long* boxes, int* image_vu, int* xyxy, float* iou, unsigned char* ok, void* stream);

/* ---- ISM -> PEM hand-off: proposal masks -> uncompressed COCO RLE (ISM/model/utils.py:25-43 mask_to_rle) ------------- */

/* masks (n,H,W) f32, a pixel set iff value > 0 -> the cumulative run ends of every mask's column-major RLE in the
 * (rle_cum, rle_off) layout of sam6d_inputs_stage_a: the positions k = x*H + y where the pixel differs from position k-1
 * (k = 0 when pixel (0,0) is set), then H*W.  Two calls: sam6d_mask_rle_count (2 launches) fills col_cnt (n,W) i32 scratch,
 * band_off (n, ceil(W/32)) i32 and rle_off (n+1) i32, rle_off[n] = total run ends; the host sizes rle_cum from rle_off[n] and
 * sam6d_mask_rle_write fills it.  n <= 65535, H*W < 2^31. */
int sam6d_mask_rle_count(const float* masks, int n, int H, int W, int* col_cnt, int* band_off, int* rle_off, void* stream);
int sam6d_mask_rle_write(const float* masks, int n, int H, int W, const int* col_cnt, const int* band_off, const int* rle_off,
                         int* rle_cum, void* stream);

/* ---- SAM prompt encoder / mask decoder / automatic mask generator: everything that is not a GEMM
 *      (ISM/segment_anything/modeling/{prompt_encoder,mask_decoder,transformer}.py, automatic_mask_generator.py:225-321,
 *       utils/amg.py:156-176,303-345, modeling/sam.py:133-162) ------------------------------------------------------------ */

/* PositionEmbeddingRandom._pe_encoding: coords (rows,2) f32 in [0,1], G (2,128) f32 -> out (rows,256) f32 = [sin | cos] */
int sam6d_sam_pe_encode(const float* coords, const float* G, int rows, float* out, void* stream);
/* PromptEncoder.mask_downscaling (Conv2d 1->4 k2 s2, LayerNorm2d, GELU, Conv2d 4->16 k2 s2, LayerNorm2d, GELU, Conv2d 16->256 1x1;
 * fp32, erf GELU, eps 1e-6): masks (B,256,256) f32 (16-byte aligned) -> out (B,4096,256) f32 token rows (row = y*64 + x).
 * params (4684) f32 = conv1 w (4,1,2,2) | conv1 b (4) | ln1 w (4) | ln1 b (4) | conv2 w (16,4,2,2) | conv2 b (16) | ln2 w (16) |
 * ln2 b (16) | conv3 w (256,16) | conv3 b (256) */
int sam6d_sam_mask_embed(const float* masks, const float* params, int B, float* out, void* stream);
/* prompt-token self attention core (8 heads x 32): q, k, v, out (B,T,256) f32, T <= 32 */
int sam6d_sam_self_attn(const float* q, const float* k, const float* v, int B, int T, float* out, void* stream);
/* tokens attend to the image (8 heads x 16): Q (B,T,128) f32; K, V bf16 (L,128) shared (kv_bs = 0) or (B,L,128) -> out (B,T,128) f32;
 * T <= 32, min(T, 8) * L * 4 <= 200 KB */
int sam6d_sam_tok2img_attn(const float* Q, const void* K, const void* V, long long kv_bs, int B, int T, int L, float* out, void* stream);
/* image attends to the tokens: Q bf16 (L,128) shared (q_bs = 0) or (B,L,128); Kt, Vt (B,T,128) f32 -> out (B,L,128) bf16; T <= 32 */
int sam6d_sam_img2tok_attn(const void* Q, long long q_bs, const float* Kt, const float* Vt, int B, int T, int L, void* out, void* stream);
/* LayerNorm2d (eps 1e-6) + GELU over rows of 64 bf16 channels (output_upscaling.1, .2) */
int sam6d_sam_ln2d_gelu(const void* x, const float* gamma, const float* beta, long long rows, void* y, void* stream);
/* mask logits: up (B*G*G*4 rows = (b,y,x,i,j), 128 cols = (i',j',o)) bf16, hyper (B,4,32) f32 -> masks (B,3,4G,4G) f32 (mask
 * tokens 1..3), the pixel shuffles of both transposed convolutions folded into the output index */
int sam6d_sam_mask_dot(const void* up, const float* hyper, int B, int G, float* masks, void* stream);
/* the same product for mask tokens m0 .. m0+nm-1 (0 <= m0, m0 + nm <= 4) -> masks (B,nm,4G,4G) f32; sam6d_sam_mask_dot is (1, 3) */
int sam6d_sam_mask_dot_range(const void* up, const float* hyper, int B, int G, int m0, int nm, float* masks, void* stream);
/* Sam.postprocess_masks evaluated per output pixel (S -> big bilinear, crop to (in_h,in_w), -> (H,W) bilinear) + statistics:
 * low (N,S,S) f32 -> stats (N,8) i32 = [count(> thr+off), count(> thr-off), xmin, ymin, xmax, ymax of (> thr), -, -] */
int sam6d_sam_mask_stats(const float* low, int N, int S, int big, int in_h, int in_w, int H, int W, float thr, float off, int* stats,
                         void* stream);
/* the selected masks at the original resolution: sel (K) i32 indices into low -> out (K,H,W) u8 = logit > thr */
int sam6d_sam_mask_binarize(const float* low, const int* sel, int K, int S, int big, int in_h, int in_w, int H, int W, float thr,
                            unsigned char* out, void* stream);
/* Sam.postprocess_masks: low (N,S,S) f32 -> out (N,H,W) f32 logits (the values sam6d_sam_mask_binarize thresholds) */
int sam6d_sam_mask_upscale(const float* low, int N, int S, int big, int in_h, int in_w, int H, int W, float* out, void* stream);
/* torchvision.ops.nms on boxes (N,4) f32 xyxy sorted by decreasing score -> keep (N) u8 */
int sam6d_sam_nms(const float* boxes, int N, float thr, unsigned char* keep, void* stream);

/* ---- fused transformer-layer tail (bf16 token stream) -------------------------------------------------------------- */

/* out = LN2(y + relu(y We^T + be) Ws^T + bs),  y = LN1(hid Wo^T + bo + x): AttentionLayer / RPEAttentionLayer tail and
 * AttentionOutput of PEM/model/transformer.py:176-197, 435-438 (and LinearAttentionLayer / LinearTransformerLayer :575-608)
 * as one persistent TMA + wgmma kernel.  hid, x, out (M,256) bf16 with row strides ld_* (multiples of 8); Wo (256,256),
 * We (512,256), Ws (256,512) bf16 row-major; bo, g1, b1, bs, g2, b2 (256) and be (512) f32; 16-byte aligned pointers. */
int sam6d_transformer_tail_bf16(const void* hid, long long ld_hid, const void* x, long long ld_x, const void* Wo, const float* bo,
                                const float* g1, const float* b1, const void* We, const float* be, const void* Ws, const float* bs,
                                const float* g2, const float* b2, void* out, long long ld_out, int M, float eps, void* stream);

/* ---- attention ---------------------------------------------------------------------------------------------------- */

/* relative-position score term of RPEMultiHeadAttention (PEM/model/transformer.py:389-394) with proj_p folded into
 * the query: E (B,S,S,256) f32 or bf16, U (B*S rows of 4x256, row stride u_ld) = W_p,h^T q_h  ->  SP (B,4,S,S) */
int sam6d_rpe_scores(const void* E, int e_is_bf16, const float* U, long long u_ld, int B, int S, float* SP, void* stream);
/* the same term on TMA + wgmma (bf16 path, the HBM-bound stream over E): E (B,S,S,256) bf16, U (B*S, 4*256) bf16
 * contiguous, S <= 200  ->  SP (B,4,S,sp_ld) f32 with padded score rows, sp_ld >= S (columns [S, sp_ld) are not written);
 * with sp_ld a multiple of 4 sam6d_attn_tc_bias_ld streams it */
int sam6d_rpe_scores_tc_ld(const void* E, const void* U, int B, int S, float* SP, int sp_ld, void* stream);
/* softmax((Q K^T + bias) * scale) V, head dim 64, Sk <= 256 (MultiHeadAttention :109-148, RPEMultiHeadAttention :369-406) */
int sam6d_mha(const float* Q, long long q_ld, long long q_bs, const float* K, long long k_ld, long long k_bs, const float* V,
              long long v_ld, long long v_bs, const float* bias, int B, int H, int Sq, int Sk, float scale, float* O,
              long long o_ld, long long o_bs, void* stream);
/* Tensor-core attention for <= 256 keys (wgmma QK^T and PV, TMA-fed, whole score row in registers; csrc/attn_tc.cu):
 * Q / K bf16 column slices of row-major matrices, Vt = V^T per (batch, head) as bf16 (B*H*D, vt_ld) rows; bias_mode 0 none,
 * 1 dense fp32 (B,H,Sq,Sk) [PEM rel-pos scores], 2 decomposed rel-pos [SAM windows; rel_h = both tables pre-packed as bf16
 * wgmma slabs, see ops.pack_rel_pos]; bv value bias (H*D) or NULL. */
int sam6d_attn_tc(const void* Q, long long q_ld, int q_col0, const void* K, long long k_ld, int k_col0, const void* Vt,
                  long long vt_ld, int B, int H, int Sq, int Sk, int head_dim, int bias_mode, const float* bias,
                  const void* rel_h, const float* rel_w, int Hs, int Ws, const float* bv, float scale, void* out,
                  int out_is_bf16, long long out_ld, void* stream);
/* sam6d_attn_tc (head dim 64) with a dense fp32 bias in padded planes (B,H,Sq,bias_ld), bias_ld >= Sk a multiple of 4 floats,
 * 16-byte aligned base: the bias is read as aligned column pairs (RPEMultiHeadAttention,
 * PEM/model/transformer.py:395-399) */
int sam6d_attn_tc_bias_ld(const void* Q, long long q_ld, int q_col0, const void* K, long long k_ld, int k_col0, const void* Vt,
                          long long vt_ld, int B, int H, int Sq, int Sk, int head_dim, const float* bias, long long bias_ld,
                          float scale, void* out, int out_is_bf16, long long out_ld, void* stream);
/* sam6d_attn_tc (no bias) over a window of keys: batch b's keys are rows [b*k_brows + k_row0, +Sk) of K and columns
 * [v_col0, +Sk) of its V^T rows; lse (B,H,Sq) f32 or NULL receives the log-sum-exp of the scaled scores */
int sam6d_attn_tc_ex(const void* Q, long long q_ld, int q_col0, const void* K, long long k_ld, int k_col0, const void* Vt,
                     long long vt_ld, int B, int H, int Sq, int Sk, int head_dim, float scale, int k_brows, int k_row0, int v_col0,
                     float* lse, void* out, int out_is_bf16, long long out_ld, void* stream);
/* folds one more key (row key_row of every batch's K rows, column key_col of its V^T rows) into the bf16 result of
 * sam6d_attn_tc_ex using its lse: the 257-token sequences of DINOv2 ViT-L/14 (ISM/model/layers/attention.py:47-69) */
int sam6d_attn_merge_key(const void* Q, long long q_ld, int q_col0, const void* K, long long k_ld, int k_col0, int k_brows,
                         int key_row, const void* Vt, long long vt_ld, int key_col, const float* lse, int B, int H, int Sq,
                         float scale, void* out, long long out_ld, void* stream);
/* V (tokens x channels, bf16 column slice at col0 of a (nB*L, ld) matrix) -> V^T (nB*C rows, N1 >= L keys), zero padded */
int sam6d_transpose_tokens_bf16(const void* src, long long ld, int col0, int C, int nB, int L, int N1, void* out, void* stream);
/* LinearAttention kv-first branch (PEM/model/transformer.py:552-559) */
int sam6d_linattn_kv(const float* Kf, long long k_ld, long long k_bs, const float* V, long long v_ld, long long v_bs, int B,
                     int H, int J, float* KV, float* KS, void* stream);
int sam6d_linattn_apply(const float* Qf, long long q_rpb, long long q_bs, long long q_ld, const float* KV, const float* KS,
                        int B, int H, float* X, long long x_bs, long long x_ld, void* stream);
/* The same branch for the dense tokens on wgmma (bf16 tokens).  linattn_kv_pack: focused keys Kf and values V ((B,J,256)
 * fp32 views) -> blob = per cloud the bf16 wgmma image of KV_h^T (4 x [64][64], 128-byte swizzle; B x 32 KB) and KS (B,4,64).
 * linattn_tc: Q = B clouds x rpb rows x 256 bf16 (row stride q_ld, cloud stride q_bs), the raw query projection; applies the focusing feature map (transformer.py:541-550),
 * X[b,i,h] = (q'_h KV_h) / (q'_h . KS_h + 1e-6), bf16. */
int sam6d_linattn_kv_pack(const float* Kf, long long k_ld, long long k_bs, const float* V, long long v_ld, long long v_bs, int B,
                          int J, void* blob, float* KS, void* stream);
int sam6d_linattn_tc(const void* Q, long long q_ld, long long q_bs, const void* blob, const float* KS,
                     const float* softplus_scale, int B, int rpb, void* X, long long x_ld, long long x_bs, void* stream);

/* ---- coarse pose (compute_coarse_Rt, PEM/utils/model_utils.py:187-246) -------------------------------------------- */
int sam6d_coarse_assign(const float* A, int B, int S, float* W, float* w1, void* stream);
int sam6d_coarse_sample(const float* W, int B, int L, const float* rand, int nr, int* idx, void* stream);
int sam6d_coarse_hypotheses(const int* idx, const float* pts1, const float* pts2, int B, int n, int n1, float* Rt,
                            float* resid, void* stream);
int sam6d_topk_smallest(const float* v, int B, int n, int k, int* out, void* stream);
int sam6d_coarse_select(const float* Rt, const int* top, int B, int n1, int n2, const float* pts1, const float* w1, int n,
                        const float* model, int nm, float* scores, float* R, float* t, void* stream);

/* ---- fine stage ---------------------------------------------------------------------------------------------------- */

/* fused QueryAndGroup + SharedMLP[6,32,64,128] (BN folded) + max-pool (PEM/model/fine_point_matching.py:101-121) */
int sam6d_pe_mlp_max(const float* pts, const int* idx, const int* cnt, int B, int N, int ns, const float* W1,
                     const float* B1, const float* W2, const float* B2, const float* W3, const float* B3, float* out,
                     int out_ld, int out_off, void* stream);
/* tensor-core version: layers 2 and 3 on wgmma (W2 (64,32), W3 (128,64) bf16), max-pool in the register epilogue */
int sam6d_pe_mlp_max_tc(const float* pts, const int* idx, int B, int N, int ns, const float* W1, const float* B1,
                        const void* W2_bf16, const float* B2, const void* W3_bf16, const float* B3, void* out, int out_is_bf16,
                        int out_ld, int out_off, void* stream);
/* compute_fine_Rt (PEM/utils/model_utils.py:250-283) in three calls.  fine_assign: A (B,S,S) fp32 scores with row stride ld,
 * ld % 4 == 0, 16-byte aligned rows, S >= 97; scratch rsum/csum (B,ld), cpart/cpi (B,ceil(S/32),ld). */
int sam6d_fine_assign(const float* A, int B, int S, int ld, float shift, const float* pts2, float* rsum, float* csum, float* cpart,
                      int* cpi, int* lab1, int* lab2, float* wts, float* pred, void* stream);
/* The same assignment without the (B,S,S) score matrix (bf16 path): every pass recomputes its score tiles on wgmma from the
 * L2-normalised bf16 tokens Fa (rows) and Fb (columns), both (B*S, 256), and reduces them in registers.
 * mode 0: out_inv (B,ld_f) = 1 / sum_j exp(alpha <a_i,b_j> - shift);  mode 1: lab (B,S) = argmax_j (e*row_f_i)*(e*col_f_j);
 * mode 2: mode 1 plus wts (B,S-1), pred (B,S-1,3) for rows >= 1 from q4 (B,ld_f) float4 (sam6d_fine_masked_points).
 * compute_fine_Rt = mode 0 on (F1,F2) and (F2,F1), mode 1 on (F2,F1) [column labels], masked points, mode 2 on (F1,F2). */
int sam6d_fine_pass_tc(const void* Fa, const void* Fb, int B, int S, float alpha, float shift, int mode, const float* row_f,
                       const float* col_f, int ld_f, const float* q4, float* out_inv, int* lab, float* wts, float* pred, void* stream);
int sam6d_fine_masked_points(const int* lab2, const float* pts2, int B, int S, int ld, float* q4, void* stream);
int sam6d_weighted_procrustes(const float* src, const float* ref, const float* wts, int B, int N, float weight_thresh,
                              float eps, float* R, float* t, void* stream);
int sam6d_pose_score(const float* pts1, const int* lab1, int B, int N, const float* R, const float* t, const float* model,
                     int nm, float dis_thres, const float* radius, float* score, float* t_scaled, void* stream);

/* ---- PEM RGB branch (SURVEY 8f, N1): pixel features at the chosen pixels without the (B,C,H,W) feature map ------------- */
/* up (B, G*G, sub*sub*C) fp32 / bf16 = ViT_AE.output_upscaling's output (PEM/model/feature_extraction.py:100-108); choose (B,K)
 * int64 pixel indices y*W + x -> out (B,K,C) fp32 = get_chosen_pixel_feats(F.interpolate(map, (H,W), bilinear), choose)
 * (PEM/utils/model_utils.py:69-81). */
int sam6d_bilinear_gather(const void* up, int up_is_bf16, const long long* choose, int B, int K, int G, int sub, int C, int H, int W,
                          float* out, void* stream);

/* ---- SAM ViT image encoder attention (ISM/segment_anything/modeling/image_encoder.py:224-240,325-361) ---------------- */
/* softmax((q*scale) k^T + q.Rh + q.Rw) v per window and head (head_dim D = 80 or 64), flash-style.  qkv: (nW*Hs*Ws, 3*nH*D)
 * rows [q|k|v], rel_h (2Hs-1,D), rel_w (2Ws-1,D), out (nW*Hs*Ws, nH*D).  Hs, Ws <= 64. */
int sam6d_attn_relpos(const float* qkv, long long tok_ld, int nW, int Hs, int Ws, int nH, int head_dim, const float* rel_h,
                      const float* rel_w, float scale, void* out, int out_is_bf16, long long out_ld, void* stream);

/* Global-attention blocks (64 x 64 token grid, 4096 keys, head_dim 80) on wgmma with an online softmax: qkv bf16
 * (B*4096, ld) rows [q|k|v]; Vt = V^T per (image, head) from sam6d_transpose_tokens_bf16 (B*H*80 rows, vt_ld >= 4096);
 * rel_blob = rel_pos_h, rel_pos_w ((127,80) each) packed as bf16 wgmma slabs of 128 rows (ops.pack_rel_pos(.., slab_rows=128));
 * out (B*4096, H*80) fp32 / bf16.  image_encoder.py:224-240 (attention), 325-361 (add_decomposed_rel_pos). */
int sam6d_attn_global_tc(const void* qkv, long long ld, const void* Vt, long long vt_ld, const void* rel_blob, int B, int H, int grid,
                         float scale, void* out, int out_is_bf16, long long out_ld, void* stream);
/* The same at head_dim 64 (SAM ViT-L: 1024 / 16, ViT-B: 768 / 12) or 80 (ViT-H): every "80" above reads head_dim; one rel-pos
 * slab per table at 64.  sam6d_attn_global_tc is this call with head_dim = 80.  Any other head_dim returns -22. */
int sam6d_attn_global_tc_ex(const void* qkv, long long ld, const void* Vt, long long vt_ld, const void* rel_blob, int B, int H, int grid,
                            int head_dim, float scale, void* out, int out_is_bf16, long long out_ld, void* stream);

/* ---- ISM template scoring (ISM/model/loss.py:21-44, ISM/model/detector.py:198-207,260-296) ------------------------ */
int sam6d_template_score(const float* Qn, const float* Rn, int P, int O, int T, int C, float* sim_out, float* obj_score,
                         int* best_obj, float* best_score, int* best_tmpl, void* stream);

/* ---- CAD template rendering (the stage SAM-6D/Render/render_{custom,bop}_templates.py runs in BlenderProc; csrc/render.cu) */

/* O meshes x T views, one pinhole K (fx, fy, cx, cy) and H x W.  verts (n_verts,3) f32 and faces (n_faces,3) i32 of all meshes
 * packed in order; faces index their own mesh's vertices.  mesh_info (O,8) i32 on the device = first vertex, vertex count,
 * first face, face count, colour mode (0 base_color (O,3) f32 in [0,1]; 1 vcol (n_verts,3) u8; 2 uv (n_verts,2) f32 sampling
 * the RGB u8 texture at tex + tex_off[o] bilinearly), texture height, texture width, 0.  poses (O,T,4,4) f32 object -> camera
 * (OpenCV axes).  Caller-owned scratch: vrec (T*n_verts,4) i32, vis (O*T*H*W) u64, big (big_cap,2) i32, counters (O+1) i32
 * (counters[1+o] = triangle-view pairs of mesh o dropped for a vertex at z <= znear or beyond the +-2^14 px guard band).
 * Outputs per (object, view, pixel): rgb u8 x3, mask u8 (255 = object), xyz f16 x3 (object coordinates, 0 off the mask),
 * tri i32 (face index within its mesh, -1 = empty), depth f32 (camera z, 0 = empty).  Shading: albedo x (ambient +
 * (1 - ambient) max(0, n.l)), point light at -1.5 t in the camera frame.  Exact visibility rules: csrc/render.cu. */
int sam6d_render_meshes(const float* verts, const int* faces, const int* mesh_info, int O, int n_verts, int n_faces,
                        const unsigned char* vcol, const float* uv, const unsigned char* tex, const long long* tex_off,
                        const float* base_color, const float* poses, int T, float fx, float fy, float cx, float cy, int H, int W,
                        float znear, float ambient, int* vrec, unsigned long long* vis, int* big, int big_cap, int* counters,
                        unsigned char* rgb, unsigned char* mask, void* xyz, int* tri, float* depth, void* stream);

/* ---- FastSAM segmentor: YOLOv8x-seg (ultralytics SegmentationModel behind ISM/model/fast_sam.py; csrc/conv_tc.cu, csrc/yolo.cu) */

/* Implicit-GEMM convolution on wgmma, NHWC bf16: x (B,Hi,Wi,ldx) channels [0,Cin) (a channel slice: offset the pointer),
 * w (Cout,k,k,Cin) bf16, k in {1,3} with padding k/2, stride 1 or 2, bias (Cout) f32 (folded BatchNorm), silu 0/1, r bf16
 * residual or NULL -> y bf16 (y_is_f32 0) or f32 (1, no residual) at
 * y[n*y_bs + ((sy*oy_pix + oy)*Wy + sx*ox_pix + ox)*ldy + c] (r addressed the same way with ldr, r_bs).  Cin % 8 == 0,
 * ldx % 8 == 0, 16-byte aligned x and w. */
int sam6d_conv2d_tc(const void* x, long long ldx, int B, int Hi, int Wi, int Cin, const void* w, int k, int stride, int Cout,
                    const float* bias, int silu, const void* r, long long ldr, long long r_bs, void* y, int y_is_f32, long long ldy,
                    long long y_bs, int Wy, int sy, int sx, int oy, int ox, void* stream);
/* stem: img (B,H,W,3) u8 letterboxed, channel-flipped and /255 on the fly; w (80,3,3,3) f32 (out,ky,kx,in), bias (80) f32 ->
 * out (B,ceil(H/2),ceil(W/2),80) bf16 = SiLU(3x3 stride-2 conv) */
int sam6d_yolo_stem(const unsigned char* img, int B, int H, int W, const float* w, const float* bias, void* out, void* stream);
/* SPPF pools: buf (B,H,W,ld) bf16, channels [0,C) -> [C,2C), [2C,3C), [3C,4C) = 5x5, 9x9, 13x13 max (-inf padding) */
int sam6d_yolo_sppf(void* buf, long long ld, int B, int H, int W, int C, void* stream);
/* nearest x2: x (B,H,W,ldx) channels [0,C) -> y (B,2H,2W,ldy) channels [0,C); C, ldx, ldy % 8 == 0 */
int sam6d_yolo_upsample2x(const void* x, long long ldx, int B, int H, int W, int C, void* y, long long ldy, void* stream);
/* Segment head decode: head (B,A,ld) f32 rows [64 DFL logits | class logit | 32 coefficients], frame stride bs, anchors of the
 * h0 x w0 (stride 8), h1 x w1 (16), h2 x w2 (32) grids -> cand (B,A,38) f32 rows (x1,y1,x2,y2,conf,cls,32 coefficients) with
 * conf > conf_thr in anchor order, count (B) i32 */
int sam6d_yolo_decode(const float* head, long long ld, long long bs, int B, int h0, int w0, int h1, int w1, int h2, int w2, float conf_thr,
                      float* cand, int* count, void* stream);
/* process_mask(upsample=True) of one frame: proto (mh,mw,32) f32, rows (N,row_ld) candidate rows, kx = mw/iw, ky = mh/ih, low
 * (N,mh,mw) f32 scratch -> out (N,ih,iw) u8 = bilinear(crop(sigmoid(coeffs . proto))) > 0.5 */
int sam6d_yolo_masks(const float* proto, int mh, int mw, const float* rows, long long row_ld, int N, int ih, int iw, float kx, float ky,
                     float* low, unsigned char* out, void* stream);

/* ---- library info ------------------------------------------------------------------------------------------------- */
/* "sam6d_b200 <version> sm_90a" */
const char* sam6d_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SAM6D_B200_H */
