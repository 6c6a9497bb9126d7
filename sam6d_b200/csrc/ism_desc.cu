// ism_desc.cu -- proposal descriptors of the Instance Segmentation Model around the DINOv2 trunk (SURVEY.md 8f row N2):
//   * crop_resize_pad : CustomDINOv2.process_rgb_proposals / process_masks_proposals (ISM/model/dinov2.py:131-147, 175-186) with
//                       CropResizePad (ISM/utils/bbox_utils.py:89-126): normalise, mask, crop the box, nearest-neighbour resize so
//                       that the longer side is 224, centre-pad to 224 x 224 -- one launch for all proposals of a frame instead of a
//                       Python loop of F.interpolate / F.pad calls per proposal
//   * masked_patch_normalize : compute_cls_and_patch_features (dinov2.py:248-258): a patch token survives when more than half of
//                       its 14 x 14 mask pixels are set (AvgPool2d > 0.5), survivors are L2-normalised, the rest are zero
//   * appearance_reduce : MaskedPatch_MatrixSimilarity.compute_straight / compute_visible_ratio (ISM/model/loss.py:52-77) on the
//                       (P, 256, 256) patch-similarity matrices the batched tensor-core GEMM produced
#include "common.cuh"
#include "crop_geom.cuh"

namespace {

// grid (T, P), block T threads: output (P, C, T, T) f32.  RGB: C = 3, value = ((img/255 - mean)/std) * mask[p]; MASK: C = 1, value = mask.
template <bool RGB>
__global__ void crop_resize_pad_kernel(const unsigned char* __restrict__ image, const float* __restrict__ masks, const int* __restrict__ boxes,
                                       int H, int W, int T, float* __restrict__ out) {
  const int p = blockIdx.y, oy = blockIdx.x, ox = threadIdx.x;
  if (ox >= T) return;
  int sy, sx;
  const bool inside = crop_resize_pad_src(boxes[p * 4], boxes[p * 4 + 1], boxes[p * 4 + 2], boxes[p * 4 + 3], T, oy, ox, sy, sx);
  const float m = inside ? masks[((size_t)p * H + sy) * W + sx] : 0.f;
  if (RGB) {
    const float mean[3] = {0.485f, 0.456f, 0.406f}, sd[3] = {0.229f, 0.224f, 0.225f};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = 0.f;
      if (inside) v = __fmul_rn(__fdiv_rn(__fsub_rn(__fdiv_rn((float)image[((size_t)sy * W + sx) * 3 + c], 255.f), mean[c]), sd[c]), m);
      out[(((size_t)p * 3 + c) * T + oy) * T + ox] = v;
    }
  } else {
    out[((size_t)p * T + oy) * T + ox] = m;
  }
}

// one warp per (proposal, patch): keep = mean of the 14 x 14 mask block > thresh; out = keep ? x / max(||x||, 1e-12) : 0
__global__ void __launch_bounds__(256) masked_patch_normalize_kernel(const float* __restrict__ tokens, long long tok_ld, long long tok_bs,
                                                                     const float* __restrict__ pmask, int P, int G, int patch, int C,
                                                                     float thresh, float* __restrict__ out_f32,
                                                                     __nv_bfloat16* __restrict__ out_bf16, unsigned char* __restrict__ valid) {
  const long long w = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= (long long)P * G * G) return;
  const int p = (int)(w / (G * G)), t = (int)(w % (G * G)), gy = t / G, gx = t % G;
  const int T = G * patch;
  float s = 0.f;
  for (int i = lane; i < patch * patch; i += 32) s += pmask[((size_t)p * T + gy * patch + i / patch) * T + gx * patch + i % patch];
  s = warp_sum(s);
  const bool keep = (s / (float)(patch * patch)) > thresh;    // AvgPool2d(kernel 14): sum / 196
  const float* x = tokens + (size_t)p * tok_bs + (size_t)t * tok_ld;
  float q = 0.f;
  if (keep)
    for (int c = lane; c < C; c += 32) q = fmaf(x[c], x[c], q);
  q = warp_sum(q);
  const float inv = keep ? 1.f / fmaxf(sqrtf(q), 1e-12f) : 0.f;
  for (int c = lane; c < C; c += 32) {
    const float v = keep ? x[c] * inv : 0.f;
    if (out_f32) out_f32[(size_t)w * C + c] = v;
    if (out_bf16) out_bf16[(size_t)w * C + c] = __float2bfloat16(v);
  }
  if (valid && lane == 0) valid[w] = keep ? 1 : 0;
}

// sim (P, N, N) f32 = query patches x reference patches of the best template.  One CTA per proposal.
//   appe[p] = clamp( sum_q max_r sim[q,r] / (count(query patch nonzero) + 1e-6), 0, 1 )                 (loss.py:52-63)
//   vis[p]  = count_r(max_q sim[q,r] > thred) / (count_r(max_q sim[q,r] != 0) + 1e-6)                    (loss.py:65-77)
__global__ void __launch_bounds__(256) appearance_reduce_kernel(const float* __restrict__ sim, long long sim_ld, long long sim_bs, int N,
                                                                const unsigned char* __restrict__ qvalid, float thred,
                                                                float* __restrict__ appe, float* __restrict__ vis) {
  __shared__ float red[8];
  __shared__ int redi[2][8];
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* S = sim + (size_t)p * sim_bs;
  // rows (queries): thread = query; columns (references): thread = reference
  float rmax = -INFINITY, cmax = -INFINITY;
  if (tid < N) {
    for (int r = 0; r < N; ++r) rmax = fmaxf(rmax, S[(size_t)tid * sim_ld + r]);
    for (int q = 0; q < N; ++q) cmax = fmaxf(cmax, S[(size_t)q * sim_ld + tid]);     // coalesced across threads
  }
  float a = tid < N ? rmax : 0.f;
  int nq = (tid < N && qvalid[(size_t)p * N + tid]) ? 1 : 0;
  int nz = (tid < N && cmax != 0.f) ? 1 : 0, hit = (tid < N && cmax > thred && cmax != 0.f) ? 1 : 0;
  a = warp_sum(a);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    nq += __shfl_xor_sync(0xffffffffu, nq, o); nz += __shfl_xor_sync(0xffffffffu, nz, o); hit += __shfl_xor_sync(0xffffffffu, hit, o);
  }
  __shared__ int redq[8];
  if (lane == 0) { red[warp] = a; redq[warp] = nq; redi[0][warp] = nz; redi[1][warp] = hit; }
  __syncthreads();
  if (tid == 0) {
    float A = 0.f; int Q = 0, Z = 0, Hh = 0;
    for (int w = 0; w < 8; ++w) { A += red[w]; Q += redq[w]; Z += redi[0][w]; Hh += redi[1][w]; }
    appe[p] = fminf(fmaxf(A / ((float)Q + 1e-6f), 0.f), 1.f);
    vis[p] = (float)Hh / ((float)Z + 1e-6f);
  }
}

}  // namespace

// image (H,W,3) u8 RGB, masks (P,H,W) f32 (0/1), boxes (P,4) i32 xyxy -> rgb (P,3,T,T) f32 normalised, masked, cropped, nearest
// resized (longer side T), centre padded; pmask (P,T,T) f32 the same treatment of the mask (either output may be NULL)
S6_API int sam6d_crop_resize_pad(const unsigned char* image, const float* masks, const int* boxes, int P, int H, int W, int T, float* rgb,
                                 float* pmask, void* stream) {
  S6_REQUIRE(masks && boxes && P >= 0 && H > 0 && W > 0 && T > 0 && T <= 1024 && (rgb == nullptr || image != nullptr));
  if (P == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  const int threads = ((T + 31) / 32) * 32;
  if (rgb) crop_resize_pad_kernel<true><<<dim3(T, P), threads, 0, st>>>(image, masks, boxes, H, W, T, rgb);
  if (pmask) crop_resize_pad_kernel<false><<<dim3(T, P), threads, 0, st>>>(image, masks, boxes, H, W, T, pmask);
  S6_LAUNCH_CHECK();
  return 0;
}

// tokens: patch token (p, t) at tokens + p*tok_bs + t*tok_ld (C floats); pmask (P, G*patch, G*patch) f32 -> out (P, G*G, C) f32
// and / or bf16 (NULL to skip), valid (P, G*G) u8 or NULL
S6_API int sam6d_masked_patch_normalize(const float* tokens, long long tok_ld, long long tok_bs, const float* pmask, int P, int G, int patch,
                                        int C, float thresh, float* out_f32, void* out_bf16, unsigned char* valid, void* stream) {
  S6_REQUIRE(tokens && pmask && P >= 0 && G > 0 && patch > 0 && C > 0 && (out_f32 || out_bf16));
  if (P == 0) return 0;
  const long long warps = (long long)P * G * G;
  masked_patch_normalize_kernel<<<s6_cdiv(warps, 8), 256, 0, s6_stream(stream)>>>(tokens, tok_ld, tok_bs, pmask, P, G, patch, C, thresh, out_f32,
                                                                                 reinterpret_cast<__nv_bfloat16*>(out_bf16), valid);
  S6_LAUNCH_CHECK();
  return 0;
}

// sim (P,N,N) f32 with row stride sim_ld and batch stride sim_bs (N <= 256), qvalid (P,N) u8 -> appe (P), vis (P)
S6_API int sam6d_appearance_reduce(const float* sim, long long sim_ld, long long sim_bs, int P, int N, const unsigned char* qvalid,
                                   float thred, float* appe, float* vis, void* stream) {
  S6_REQUIRE(sim && qvalid && appe && vis && P >= 0 && N > 0 && N <= 256);
  if (P == 0) return 0;
  appearance_reduce_kernel<<<P, 256, 0, s6_stream(stream)>>>(sim, sim_ld, sim_bs, N, qvalid, thred, appe, vis);
  S6_LAUNCH_CHECK();
  return 0;
}
