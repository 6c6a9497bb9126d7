// mask_rle.cu -- binary masks -> uncompressed COCO RLE on the device: what ISM/model/utils.py:25-43 (mask_to_rle) does per
// proposal in numpy after copying every float mask to the host, for all proposals of a frame in three launches.
//
// A pixel is set iff value > 0 (NaN, -0.0 and negatives are unset).  Positions are column-major, k = x*H + y.  The output of
// mask m is the cumulative run ends of its RLE: every k where the pixel differs from position k-1 (position 0 counts when
// pixel (0,0) is set: mask_to_rle's leading zero-length run), then H*W.  That is the (rle_cum, rle_off) layout that
// sam6d_inputs_stage_a reads (inputs.pack_rle).
//
// Work split: a warp owns one column band (32 adjacent columns) of one mask; lane l walks column x0+l down the rows, so every
// row read is one coalesced 128-byte transaction.  Bands in order are column-major order.
//   1. count: per-column transition counts col_cnt (n,W), per-band sums (written to band_off, scanned in place by 2.)
//   2. scan (one CTA): exclusive scan of the n*nb band sums plus one terminator per mask -> band_off, rle_off (n+1)
//   3. write: lane base = band_off + shuffle scan of col_cnt over the lanes; each lane writes its column's change positions in
//      row order; lane 0 of band 0 writes the terminator H*W.
#include "common.cuh"

namespace {

constexpr int RLE_WARPS = 4;          // bands per CTA in the count / write passes
constexpr int RLE_UNROLL = 8;         // rows loaded ahead per lane

__device__ __forceinline__ bool rle_set(const float* p) { return __ldg(p) > 0.f; }

// transitions of column x (lane's column; x < W) of mask `m`: row order, calls f(k) for every change position k
template <typename F>
__device__ __forceinline__ void rle_walk_column(const float* __restrict__ m, int H, int W, int x, F&& f) {
  bool prev = x > 0 ? rle_set(m + (size_t)(H - 1) * W + (x - 1)) : false;      // position x*H - 1 (bottom of the previous column)
  const int kb = x * H;
  int y = 0;
  for (; y + RLE_UNROLL <= H; y += RLE_UNROLL) {
    bool v[RLE_UNROLL];
#pragma unroll
    for (int u = 0; u < RLE_UNROLL; ++u) v[u] = rle_set(m + (size_t)(y + u) * W + x);
#pragma unroll
    for (int u = 0; u < RLE_UNROLL; ++u) {
      if (v[u] != prev) f(kb + y + u);
      prev = v[u];
    }
  }
  for (; y < H; ++y) {
    const bool v = rle_set(m + (size_t)y * W + x);
    if (v != prev) f(kb + y);
    prev = v;
  }
}

__global__ void __launch_bounds__(RLE_WARPS * 32) rle_count_kernel(const float* __restrict__ masks, int H, int W, int nb,
                                                                   int* __restrict__ col_cnt, int* __restrict__ band_cnt) {
  const int band = blockIdx.x * RLE_WARPS + (threadIdx.x >> 5);
  if (band >= nb) return;                                        // whole warps only: the shuffles below stay full-mask
  const int mi = blockIdx.y;
  const int x = band * 32 + (threadIdx.x & 31);
  const float* m = masks + (size_t)mi * H * W;
  int c = 0;
  if (x < W) {
    rle_walk_column(m, H, W, x, [&](int) { ++c; });
    col_cnt[(size_t)mi * W + x] = c;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) band_cnt[(size_t)mi * nb + band] = c;
}

// one CTA of 1024 threads; band_off holds the band sums on entry and their exclusive offsets (plus the terminators of the
// masks before) on exit
__global__ void __launch_bounds__(1024) rle_scan_kernel(int* __restrict__ band_off, int n, int nb, int* __restrict__ rle_off) {
  __shared__ int warp_sums[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long total_n = (long long)n * nb;
  int carry = 0;
  for (long long base = 0; base < total_n; base += 1024) {
    const long long i = base + threadIdx.x;
    const int mi = i < total_n ? (int)(i / nb) : n;
    const int b = i < total_n ? (int)(i - (long long)mi * nb) : 0;
    // the terminator of mask mi - 1 precedes band 0 of mask mi: counted as one more run end on that band
    const int v = i < total_n ? band_off[i] + (b == nb - 1 ? 1 : 0) : 0;
    int s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    if (lane == 31) warp_sums[warp] = s;
    __syncthreads();
    if (warp == 0) {
      int w = warp_sums[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += t;
      }
      warp_sums[lane] = w;
    }
    __syncthreads();
    const int excl = carry + (warp ? warp_sums[warp - 1] : 0) + s - v;
    if (i < total_n) {
      band_off[i] = excl;
      if (b == 0) rle_off[mi] = excl;
    }
    carry += warp_sums[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) rle_off[n] = carry;
}

__global__ void __launch_bounds__(RLE_WARPS * 32) rle_write_kernel(const float* __restrict__ masks, int H, int W, int nb,
                                                                   const int* __restrict__ col_cnt, const int* __restrict__ band_off,
                                                                   const int* __restrict__ rle_off, int* __restrict__ rle_cum) {
  const int band = blockIdx.x * RLE_WARPS + (threadIdx.x >> 5);
  if (band >= nb) return;
  const int lane = threadIdx.x & 31;
  const int mi = blockIdx.y;
  const int x = band * 32 + lane;
  const int c = x < W ? col_cnt[(size_t)mi * W + x] : 0;
  int s = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, s, o);
    if (lane >= o) s += t;
  }
  int* out = rle_cum + band_off[(size_t)mi * nb + band] + (s - c);
  if (x < W && c > 0) rle_walk_column(masks + (size_t)mi * H * W, H, W, x, [&](int k) { *out++ = k; });
  if (band == 0 && lane == 0) rle_cum[rle_off[mi + 1] - 1] = H * W;
}

}  // namespace

S6_API int sam6d_mask_rle_count(const float* masks, int n, int H, int W, int* col_cnt, int* band_off, int* rle_off, void* stream) {
  S6_REQUIRE(n >= 0 && n <= 65535 && H > 0 && W > 0 && (long long)H * W < (1ll << 31) && rle_off);
  S6_REQUIRE(n == 0 || (masks && col_cnt && band_off));
  const int nb = s6_cdiv(W, 32);
  cudaStream_t st = s6_stream(stream);
  if (n > 0) {
    rle_count_kernel<<<dim3(s6_cdiv(nb, RLE_WARPS), n), RLE_WARPS * 32, 0, st>>>(masks, H, W, nb, col_cnt, band_off);
    S6_LAUNCH_CHECK();
  }
  rle_scan_kernel<<<1, 1024, 0, st>>>(band_off, n, nb, rle_off);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_mask_rle_write(const float* masks, int n, int H, int W, const int* col_cnt, const int* band_off, const int* rle_off,
                                int* rle_cum, void* stream) {
  S6_REQUIRE(n >= 0 && n <= 65535 && H > 0 && W > 0 && (long long)H * W < (1ll << 31));
  if (n == 0) return 0;
  S6_REQUIRE(masks && col_cnt && band_off && rle_off && rle_cum);
  const int nb = s6_cdiv(W, 32);
  rle_write_kernel<<<dim3(s6_cdiv(nb, RLE_WARPS), n), RLE_WARPS * 32, 0, s6_stream(stream)>>>(masks, H, W, nb, col_cnt, band_off,
                                                                                             rle_off, rle_cum);
  S6_LAUNCH_CHECK();
  return 0;
}
