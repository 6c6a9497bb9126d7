// inputs.cu -- the PEM input builder on the GPU (SURVEY.md 8f row N3): everything PEM/run_inference_custom.py:165-253
// (get_test_data) does per detection in numpy / cv2 on one host core -- RLE decode, mask AND depth, square bounding box, masked
// compaction, depth -> camera-frame cloud, centroid + radius filter, sample gather, crop / mask / bilinear resize / normalise,
// rgb_choose -- for all detections of a frame at once.
//
// Stage A (sam6d_inputs_stage_a): decode + reduce + bbox + ordered compaction + radius filter.  The host reads back 8 ints per
//   detection (bbox, pixel count, valid count), draws the sample indices with numpy's RNG exactly like the reference
//   (np.random.choice; the reference's RNG is host state) and calls
// Stage B (sam6d_inputs_stage_b): sample gather, rgb_choose, crop / resize / normalise.
//
// Numerics follow the reference as it evaluates under numpy >= 2 (the oracle's environment): get_point_cloud_from_depth
// promotes to float64 through the float64 intrinsics (data_utils.py:92-110), the centroid and the radius test are float64, the
// outputs are rounded to float32 once (torch.FloatTensor).  cv2.resize(INTER_LINEAR) on uint8 is OpenCV's fixed-point
// algorithm (11-bit coefficients, horizontal int pass, vertical ((b*(r>>4))>>16 ... +2)>>2) and the 2x2 box average when the
// crop is exactly twice the output; reproduced bit for bit (tests/test_oracle_input.py checks the emulation against cv2).
#include "common.cuh"

namespace {

struct InCfg {
  int H, W, S;               // frame size, output crop size (224)
  double fx, fy, cx, cy;
};

// stats row per detection (ints): 0 rmin 1 rmax 2 cmin 3 cmax (raw extremes, inclusive) 4 count | 5 y1 6 y2 7 x1 8 x2 9 n_valid
constexpr int ST = 12;

// ---- 1. RLE decode (column-major runs) AND depth > 0, extremes + count ---------------------------------------------------
__global__ void __launch_bounds__(256) inp_decode_kernel(const int* __restrict__ cum, const int* __restrict__ off, const float* __restrict__ depth,
                                                         int H, int W, unsigned char* __restrict__ mask, int* __restrict__ stats) {
  const int p = blockIdx.y;
  const int i = blockIdx.x * 256 + threadIdx.x;            // row-major pixel
  const int* c = cum + off[p];
  const int n = off[p + 1] - off[p];
  bool on = false;
  int y = 0, x = 0;
  if (i < H * W) {
    y = i / W; x = i - y * W;
    const int f = x * H + y;                                 // position in the column-major run sequence
    int lo = 0, hi = n;                                      // first run whose cumulative end exceeds f
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (c[mid] <= f) lo = mid + 1; else hi = mid;
    }
    on = (lo < n) && (lo & 1) && depth[i] > 0.f;             // runs alternate 0,1,0,1,... starting with zeros (data_utils.py:73-89)
    mask[(size_t)p * H * W + i] = on ? 1 : 0;
  }
  // block-level extremes: one set of atomics per warp that has a hit
  const unsigned bal = __ballot_sync(0xffffffffu, on);
  if (bal) {
    int ymin = on ? y : 0x7fffffff, ymax = on ? y : -1, xmin = on ? x : 0x7fffffff, xmax = on ? x : -1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ymin = min(ymin, __shfl_xor_sync(0xffffffffu, ymin, o)); ymax = max(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
      xmin = min(xmin, __shfl_xor_sync(0xffffffffu, xmin, o)); xmax = max(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
    }
    if ((threadIdx.x & 31) == 0) {
      int* s = stats + p * ST;
      atomicMin(s + 0, ymin); atomicMax(s + 1, ymax); atomicMin(s + 2, xmin); atomicMax(s + 3, xmax);
      atomicAdd(s + 4, __popc(bal));
    }
  }
}

// ---- 2. get_bbox (data_utils.py:127-160) --------------------------------------------------------------------------------
__global__ void inp_bbox_kernel(int* __restrict__ stats, int P, int H, int W) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  int* s = stats + p * ST;
  if (s[4] <= 0) { s[5] = s[6] = s[7] = s[8] = 0; return; }
  int rmin = s[0], rmax = s[1] + 1, cmin = s[2], cmax = s[3] + 1;
  const int b = min(max(rmax - rmin, cmax - cmin), min(H, W));
  const int cy = (rmin + rmax) / 2, cx = (cmin + cmax) / 2, hb = b / 2;    // int(x / 2) of non-negative ints
  rmin = cy - hb; rmax = cy + hb; cmin = cx - hb; cmax = cx + hb;
  if (rmin < 0) { rmax += -rmin; rmin = 0; }
  if (cmin < 0) { cmax += -cmin; cmin = 0; }
  if (rmax > H) { rmin -= rmax - H; rmax = H; }
  if (cmax > W) { cmin -= cmax - W; cmax = W; }
  s[5] = rmin; s[6] = rmax; s[7] = cmin; s[8] = cmax;
}

__device__ __forceinline__ void cam_point(const InCfg& g, const float* depth, int y, int x, double& px, double& py, double& pz) {
  const float z = depth[y * g.W + x];
  pz = (double)z;
  px = ((double)(float)x - g.cx) * pz / g.fx;               // (xmap.astype(f32) - cx) * pt2 / fx, float64 under numpy >= 2
  py = ((double)(float)y - g.cy) * pz / g.fy;
}

// block-wide exclusive scan of one flag per thread (1024 threads); returns this thread's offset, total in *total
__device__ __forceinline__ int block_scan_flag(bool flag, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, flag);
  const int within = __popc(bal & ((1u << lane) - 1));
  if (lane == 0) warp_sums[warp] = __popc(bal);
  __syncthreads();
  if (warp == 0) {
    int v = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    warp_sums[lane] = v;                                     // inclusive
  }
  __syncthreads();
  const int base = warp ? warp_sums[warp - 1] : 0;
  *total = warp_sums[31];
  __syncthreads();
  return base + within;
}

// ---- 3. ordered compaction inside the bbox, centroid, radius filter (run_inference_custom.py:202-212) -----------------------
// one CTA of 1024 threads per detection.  thr (P) float64: each detection's float32(radius) * float32(1.2) widened
// (run_inference_custom.py:209), the radius being that of the detection's object.  choose1 / choose2: (P, cap) crop-linear pixel
// indices, cloud2: (P, cap, 3) float32.  A detection of min_count pixels or fewer is skipped (n_valid 0).
__global__ void __launch_bounds__(1024) inp_compact_kernel(InCfg g, int min_count, const double* __restrict__ thr, const unsigned char* __restrict__ mask,
                                                           const float* __restrict__ depth, int* __restrict__ stats, int cap, int* __restrict__ choose1,
                                                           int* __restrict__ choose2, float* __restrict__ cloud2) {
  __shared__ int warp_sums[32];
  __shared__ double red[3][32];
  __shared__ double center[3];
  const int p = blockIdx.x, tid = threadIdx.x;
  int* s = stats + p * ST;
  if (s[4] <= min_count) { if (tid == 0) s[9] = 0; return; }  // np.sum(mask) > 32 else continue (:199-203)
  const double th = thr[p];
  const int y1 = s[5], y2 = s[6], x1 = s[7], x2 = s[8];
  const int ch = y2 - y1, cw = x2 - x1, area = ch * cw;
  const unsigned char* m = mask + (size_t)p * g.H * g.W;
  int* c1 = choose1 + (size_t)p * cap;
  int* c2 = choose2 + (size_t)p * cap;
  float* cl = cloud2 + (size_t)p * cap * 3;
  // pass 1: choose = nonzero(mask crop, row-major); centroid of the cloud
  int n1 = 0;
  double sx = 0.0, sy = 0.0, sz = 0.0;
  for (int base = 0; base < area; base += 1024) {
    const int i = base + tid;
    bool on = false;
    int yy = 0, xx = 0;
    if (i < area) { yy = y1 + i / cw; xx = x1 + i % cw; on = m[yy * g.W + xx] != 0; }
    int tot;
    const int pos = block_scan_flag(on, warp_sums, &tot);
    if (on) {
      c1[n1 + pos] = i;
      double px, py, pz;
      cam_point(g, depth, yy, xx, px, py, pz);
      sx += px; sy += py; sz += pz;
    }
    n1 += tot;
  }
  sx = warp_sum_d(sx); sy = warp_sum_d(sy); sz = warp_sum_d(sz);
  if ((tid & 31) == 0) { red[0][tid >> 5] = sx; red[1][tid >> 5] = sy; red[2][tid >> 5] = sz; }
  __syncthreads();
  if (tid < 3) {
    double a = 0.0;
    for (int w = 0; w < 32; ++w) a += red[tid][w];
    center[tid] = a / (double)n1;                             // np.mean(cloud, axis=0)
  }
  __syncthreads();
  // pass 2: flag = ||cloud - center|| < radius * 1.2, ordered compaction of choose / cloud
  int n2 = 0;
  for (int base = 0; base < n1; base += 1024) {
    const int k = base + tid;
    bool keep = false;
    int i = 0;
    double px = 0, py = 0, pz = 0;
    if (k < n1) {
      i = c1[k];
      cam_point(g, depth, y1 + i / cw, x1 + i % cw, px, py, pz);
      const double dx = px - center[0], dy = py - center[1], dz = pz - center[2];
      keep = sqrt(dx * dx + dy * dy + dz * dz) < th;
    }
    int tot;
    const int pos = block_scan_flag(keep, warp_sums, &tot);
    if (keep) {
      c2[n2 + pos] = i;
      float* o = cl + (size_t)(n2 + pos) * 3;
      o[0] = (float)px; o[1] = (float)py; o[2] = (float)pz;
    }
    n2 += tot;
  }
  if (tid == 0) s[9] = n2;
}

// ---- 4. sample gather + rgb_choose (run_inference_custom.py:214-219,226; data_utils.py:113-124) -----------------------------
__global__ void __launch_bounds__(256) inp_gather_kernel(const int* __restrict__ stats, const int* __restrict__ keep, int cap,
                                                         const int* __restrict__ choose2, const float* __restrict__ cloud2,
                                                         const int* __restrict__ choose_idx, int ns, int S, float* __restrict__ pts,
                                                         long long* __restrict__ rgb_choose) {
  const int q = blockIdx.y, p = keep[q];
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= ns) return;
  const int* s = stats + p * ST;
  const int ci = choose_idx[(size_t)q * ns + j];
  const int c = choose2[(size_t)p * cap + ci];
  const float* src = cloud2 + ((size_t)p * cap + ci) * 3;
  float* o = pts + ((size_t)q * ns + j) * 3;
  o[0] = src[0]; o[1] = src[1]; o[2] = src[2];
  const int ch = s[6] - s[5], cw = s[8] - s[7];
  const double ratio_h = (double)S / (double)ch, ratio_w = (double)S / (double)cw;
  const int row = c / cw, col = c % cw;
  rgb_choose[(size_t)q * ns + j] = (long long)(floor((double)row * ratio_h) * (double)S + floor((double)col * ratio_w));
}

// ---- 5. crop, channel flip, mask, cv2 INTER_LINEAR (uint8 fixed point), ToTensor + Normalize -------------------------------
__device__ __forceinline__ void lin_coef(int d, int n_src, int n_dst, bool horizontal, int& i0, int& i1, int& a0, int& a1) {
  const double scale = 1.0 / ((double)n_dst / (double)n_src);
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f -= (float)s;
  if (horizontal) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= n_src - 1) { f = 0.f; s = n_src - 1; }
  }
  i0 = min(max(s, 0), n_src - 1);
  i1 = min(max(s + 1, 0), n_src - 1);
  a0 = __float2int_rn((1.f - f) * 2048.f);
  a1 = __float2int_rn(f * 2048.f);
}

// grid (S, Q); block S threads (one output pixel column each); out (Q,3,S,S) float32, also the uint8 crop (Q,S,S,3) if u8 != null.
// Item q: bbox row bbox[q_or_keep * bbox_ld .. +4) = y1,y2,x1,x2; mask plane midx = keep ? keep[q] : q; image q * image_stride.
__global__ void inp_crop_resize_kernel(const unsigned char* __restrict__ image, long long image_stride, const unsigned char* __restrict__ mask,
                                       const int* __restrict__ bbox, int bbox_ld, const int* __restrict__ keep, int H, int W, int S,
                                       int mask_flag, float* __restrict__ out, unsigned char* __restrict__ u8) {
  const int q = blockIdx.y, p = keep ? keep[q] : q, dy = blockIdx.x, dx = threadIdx.x;
  if (dx >= S) return;
  const int* s = bbox + (size_t)p * bbox_ld;
  const int y1 = s[0], x1 = s[2], n = s[1] - s[0];            // square crop
  const unsigned char* m = mask + (size_t)p * H * W;
  const unsigned char* img = image + (size_t)q * image_stride;
  auto px = [&](int yy, int xx, int c) -> int {               // crop[yy][xx][c] after [:, :, ::-1] and masking
    const int gy = y1 + yy, gx = x1 + xx;
    if (mask_flag && !m[gy * W + gx]) return 0;
    return img[((size_t)gy * W + gx) * 3 + (2 - c)];
  };
  int v[3];
  if (n == 2 * S) {                                           // OpenCV switches INTER_LINEAR to the 2x2 area average
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = (px(2 * dy, 2 * dx, c) + px(2 * dy, 2 * dx + 1, c) + px(2 * dy + 1, 2 * dx, c) + px(2 * dy + 1, 2 * dx + 1, c) + 2) >> 2;
  } else {
    int x0, x1i, xa0, xa1, y0, y1i, ya0, ya1;
    lin_coef(dx, n, S, true, x0, x1i, xa0, xa1);
    lin_coef(dy, n, S, false, y0, y1i, ya0, ya1);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int r0 = px(y0, x0, c) * xa0 + px(y0, x1i, c) * xa1;
      const int r1 = px(y1i, x0, c) * xa0 + px(y1i, x1i, c) * xa1;
      v[c] = min(max((((ya0 * (r0 >> 4)) >> 16) + ((ya1 * (r1 >> 4)) >> 16) + 2) >> 2, 0), 255);
    }
  }
  const float mean[3] = {0.485f, 0.456f, 0.406f}, sd[3] = {0.229f, 0.224f, 0.225f};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    out[(((size_t)q * 3 + c) * S + dy) * S + dx] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v[c], 255.f), mean[c]), sd[c]);
    if (u8) u8[(((size_t)q * S + dy) * S + dx) * 3 + c] = (unsigned char)v[c];
  }
}

__global__ void inp_init_stats_kernel(int* __restrict__ stats, int P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P * ST) return;
  const int f = i % ST;
  stats[i] = (f == 0 || f == 2) ? 0x7fffffff : ((f == 1 || f == 3) ? -1 : 0);
}

}  // namespace

S6_API int sam6d_inputs_stage_a_min(const int* rle_cum, const int* rle_off, int P, int H, int W, const float* depth, double fx, double fy,
                                    double cx, double cy, const double* thr, int min_count, unsigned char* mask, int* stats, int cap,
                                    int* choose1, int* choose2, float* cloud2, void* stream);

// Stage A.  rle_cum: cumulative run ends of every detection's uncompressed COCO RLE (column-major), concatenated; rle_off (P+1)
// offsets into it.  depth (H,W) f32 metres; fx, fy, cx, cy the float64 intrinsics; thr (P) f64 on the device, per detection
// float32(radius) * float32(1.2) of its object.
// mask (P,H,W) u8 out.  stats (P,12) i32 out: [0..3] raw extremes, [4] pixel count, [5..8] bbox y1,y2,x1,x2, [9] points that
// survive the radius filter.  choose1 / choose2 (P,cap) i32, cloud2 (P,cap,3) f32 scratch / out, cap >= min(H,W)^2.
S6_API int sam6d_inputs_stage_a(const int* rle_cum, const int* rle_off, int P, int H, int W, const float* depth, double fx, double fy,
                                double cx, double cy, const double* thr, unsigned char* mask, int* stats, int cap, int* choose1, int* choose2,
                                float* cloud2, void* stream) {
  return sam6d_inputs_stage_a_min(rle_cum, rle_off, P, H, W, depth, fx, fy, cx, cy, thr, 32, mask, stats, cap, choose1, choose2, cloud2,
                                  stream);
}

// Stage A with the pixel-count cut as a parameter: a detection whose mask AND depth > 0 has min_count pixels or fewer gets no
// radius filter (stats[9] = 0).  32 is run_inference_custom.py:199-203, 8 is BOPTestset.get_instance's minimum_n_point; thr is any
// float64 threshold per detection (BOP: diameter * 0.6).
S6_API int sam6d_inputs_stage_a_min(const int* rle_cum, const int* rle_off, int P, int H, int W, const float* depth, double fx, double fy,
                                    double cx, double cy, const double* thr, int min_count, unsigned char* mask, int* stats, int cap,
                                    int* choose1, int* choose2, float* cloud2, void* stream) {
  S6_REQUIRE(rle_cum && rle_off && depth && thr && mask && stats && choose1 && choose2 && cloud2 && P >= 0 && H > 0 && W > 0 &&
             cap >= min(H, W) * min(H, W) && min_count >= 0);
  if (P == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  inp_init_stats_kernel<<<s6_cdiv(P * ST, 256), 256, 0, st>>>(stats, P);
  S6_LAUNCH_CHECK();
  dim3 grid(s6_cdiv((long long)H * W, 256), P);
  inp_decode_kernel<<<grid, 256, 0, st>>>(rle_cum, rle_off, depth, H, W, mask, stats);
  S6_LAUNCH_CHECK();
  inp_bbox_kernel<<<s6_cdiv(P, 128), 128, 0, st>>>(stats, P, H, W);
  S6_LAUNCH_CHECK();
  InCfg g{H, W, 0, fx, fy, cx, cy};
  inp_compact_kernel<<<P, 1024, 0, st>>>(g, min_count, thr, mask, depth, stats, cap, choose1, choose2, cloud2);
  S6_LAUNCH_CHECK();
  return 0;
}

// Stage B for the Q kept detections keep[q] (indices into the stage-A arrays): choose_idx (Q,ns) i32 sample indices into the
// filtered point list -> pts (Q,ns,3) f32, rgb_choose (Q,ns) i64, rgb (Q,3,S,S) f32 normalised, rgb_u8 (Q,S,S,3) or NULL.
S6_API int sam6d_inputs_stage_b(const int* stats, const int* keep, int Q, int H, int W, int cap, const int* choose2, const float* cloud2,
                                const int* choose_idx, int ns, int S, const unsigned char* image, const unsigned char* mask, int mask_flag,
                                float* pts, long long* rgb_choose, float* rgb, unsigned char* rgb_u8, void* stream) {
  S6_REQUIRE(stats && keep && choose2 && cloud2 && choose_idx && image && mask && pts && rgb_choose && rgb && Q >= 0 && ns > 0 && S > 0 &&
             S <= 1024);
  if (Q == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  inp_gather_kernel<<<dim3(s6_cdiv(ns, 256), Q), 256, 0, st>>>(stats, keep, cap, choose2, cloud2, choose_idx, ns, S, pts, rgb_choose);
  S6_LAUNCH_CHECK();
  inp_crop_resize_kernel<<<dim3(S, Q), ((S + 31) / 32) * 32, 0, st>>>(image, 0, mask, stats + 5, ST, keep, H, W, S, mask_flag, rgb, rgb_u8);
  S6_LAUNCH_CHECK();
  return 0;
}

// The crop / resize / normalise step alone for Q images of their own (the 42 template renderings of _get_template,
// run_inference_custom.py:117-136): images (Q,H,W,3) u8, masks (Q,H,W) u8, bbox (Q,4) i32 = y1,y2,x1,x2 (square).
S6_API int sam6d_crop_resize_normalize(const unsigned char* images, const unsigned char* masks, const int* bbox, int Q, int H, int W, int S,
                                       int mask_flag, float* rgb, unsigned char* rgb_u8, void* stream) {
  S6_REQUIRE(images && masks && bbox && rgb && Q >= 0 && H > 0 && W > 0 && S > 0 && S <= 1024);
  if (Q == 0) return 0;
  inp_crop_resize_kernel<<<dim3(S, Q), ((S + 31) / 32) * 32, 0, s6_stream(stream)>>>(images, (long long)H * W * 3, masks, bbox, 4, nullptr,
                                                                                  H, W, S, mask_flag, rgb, rgb_u8);
  S6_LAUNCH_CHECK();
  return 0;
}
