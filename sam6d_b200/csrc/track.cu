// track.cu -- observed-point selection for tracking (not in the reference; the rule is stated in include/sam6d_b200.h at
// sam6d_track_points and restated in numpy by oracle/track_oracle.py).
//
// For O objects of one frame, a pixel is a candidate of object o when it lies in o's rendered silhouette dilated by a square
// (2m+1)^2 window, its observed depth is positive and its back-projected point lies within o's gate sphere.  Four launches:
//   1. trk_dilate_rows: the horizontal max pass of the silhouette, one CTA per (row, object), the row staged in shared memory;
//      also zeroes the row's candidate count.
//   2. trk_candidates: the vertical max pass as a running window count down each column over a TRK_ROWS-row tile, then the
//      depth and gate tests; writes the candidate mask and adds each row's count (integer atomics: order-free, so exact).
//   3. trk_scan: per object, the exclusive scan of the row counts (the rows' offsets in raster order) and the total.
//   4. trk_select: per (row, object), block scans give each candidate its raster-order rank k; the candidate writes output i
//      for every i that selects k (count >= N: floor(i count / N) = k; 0 < count < N: i = k mod count).
// Every fp32 operation that decides membership is an explicit round-to-nearest intrinsic, so nothing is contracted into an FMA
// and the oracle reproduces the candidate set exactly.
//
// sam6d_track_points_scene gives every pixel to at most one of L live tracks (the rule: include/sam6d_b200.h).  Five launches:
// trk_dilate_rows; trk_dilate_cols (the same running column window, written out as the dilated mask); trk_assign (one thread
// per pixel over the L tracks: the eligible track rendered in front, else the eligible track nearest its gate centre relative
// to its radius); trk_scan; trk_select.
#include "common.cuh"

namespace {

constexpr int TRK_THREADS = 256;
constexpr int TRK_ROWS = 32;              // rows per trk_candidates tile: each column loads TRK_ROWS + 2m mask rows for TRK_ROWS outputs

struct TrkCam {
  float depth_scale, fx, fy, cx, cy;
};

// inputs.py's depth (raw f32 * depth_scale / 1000, each in fp32) and inputs.cu's back-projection order, (x - cx) * z / fx
__device__ __forceinline__ float3 trk_point(const TrkCam& c, unsigned short raw, int y, int x) {
  const float z = __fdiv_rn(__fmul_rn((float)raw, c.depth_scale), 1000.f);
  return make_float3(__fdiv_rn(__fmul_rn(__fsub_rn((float)x, c.cx), z), c.fx), __fdiv_rn(__fmul_rn(__fsub_rn((float)y, c.cy), z), c.fy), z);
}

// (dx^2 + dy^2) + dz^2 with d = p - centre
__device__ __forceinline__ float trk_gate_d2(float3 p, const float* centre) {
  const float dx = __fsub_rn(p.x, centre[0]), dy = __fsub_rn(p.y, centre[1]), dz = __fsub_rn(p.z, centre[2]);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ bool trk_in_gate(float3 p, const float* centre, float radius) {
  return radius > 0.f && trk_gate_d2(p, centre) <= __fmul_rn(radius, radius);
}

// exclusive scan of one int per thread over a TRK_THREADS block; the block total in *total.  warp_sums: TRK_THREADS / 32 ints.
__device__ __forceinline__ int trk_block_scan(int v, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  int base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < TRK_THREADS / 32; ++w) {
    const int s = warp_sums[w];
    if (w < warp) base += s;
    tot += s;
  }
  __syncthreads();                          // warp_sums may be reused by the next call
  *total = tot;
  return base + inc - v;
}

__global__ void __launch_bounds__(TRK_THREADS) trk_dilate_rows(const float* __restrict__ rdepth, int H, int W, int m,
                                                              unsigned char* __restrict__ hmask, int* __restrict__ rows) {
  extern __shared__ unsigned char srow[];
  const int y = blockIdx.x, o = blockIdx.y;
  const size_t row = ((size_t)o * H + y) * W;
  for (int x = threadIdx.x; x < W; x += TRK_THREADS) srow[x] = rdepth[row + x] > 0.f;
  if (threadIdx.x == 0) rows[(size_t)o * H + y] = 0;
  __syncthreads();
  for (int x = threadIdx.x; x < W; x += TRK_THREADS) {
    const int x0 = max(x - m, 0), x1 = min(x + m, W - 1);
    unsigned char v = 0;
    for (int xx = x0; xx <= x1 && !v; ++xx) v = srow[xx];
    hmask[row + x] = v;
  }
}

__global__ void __launch_bounds__(TRK_THREADS) trk_candidates(const unsigned char* __restrict__ hmask, const unsigned short* __restrict__ depth,
                                                             TrkCam cam, const float* __restrict__ centre, const float* __restrict__ radius,
                                                             int H, int W, int m, unsigned char* __restrict__ cand, int* __restrict__ rows) {
  __shared__ int srows[TRK_ROWS];
  const int x = blockIdx.x * TRK_THREADS + threadIdx.x, y0 = blockIdx.y * TRK_ROWS, o = blockIdx.z;
  const int y1 = min(y0 + TRK_ROWS, H);
  if (threadIdx.x < TRK_ROWS) srows[threadIdx.x] = 0;
  __syncthreads();
  const float c[3] = {centre[o * 3], centre[o * 3 + 1], centre[o * 3 + 2]};
  const float r = radius[o];
  const unsigned char* hm = hmask + (size_t)o * H * W;
  const bool col = x < W;
  int win = 0;                              // silhouette rows of this column within [y - m, y + m]
  if (col)
    for (int yy = max(y0 - m, 0); yy < min(y0 + m, H); ++yy) win += hm[(size_t)yy * W + x];
  for (int y = y0; y < y1; ++y) {
    bool on = false;
    if (col) {
      if (y + m < H) win += hm[(size_t)(y + m) * W + x];
      if (win > 0) {
        const unsigned short raw = depth[(size_t)y * W + x];
        const float3 p = trk_point(cam, raw, y, x);
        on = p.z > 0.f && trk_in_gate(p, c, r);
      }
      cand[((size_t)o * H + y) * W + x] = on;
      if (y - m >= 0) win -= hm[(size_t)(y - m) * W + x];
    }
    const unsigned bal = __ballot_sync(0xffffffffu, on);
    if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&srows[y - y0], __popc(bal));
  }
  __syncthreads();
  if (threadIdx.x < y1 - y0 && srows[threadIdx.x]) atomicAdd(&rows[(size_t)o * H + y0 + threadIdx.x], srows[threadIdx.x]);
}

// sam6d_track_points_scene's vertical pass: the (2m+1)-row window of hmask down each column, as trk_candidates counts it
__global__ void __launch_bounds__(TRK_THREADS) trk_dilate_cols(const unsigned char* __restrict__ hmask, int H, int W, int m,
                                                              unsigned char* __restrict__ dmask) {
  const int x = blockIdx.x * TRK_THREADS + threadIdx.x, y0 = blockIdx.y * TRK_ROWS, j = blockIdx.z;
  if (x >= W) return;
  const int y1 = min(y0 + TRK_ROWS, H);
  const unsigned char* hm = hmask + (size_t)j * H * W;
  unsigned char* dm = dmask + (size_t)j * H * W;
  int win = 0;
  for (int yy = max(y0 - m, 0); yy < min(y0 + m, H); ++yy) win += hm[(size_t)yy * W + x];
  for (int y = y0; y < y1; ++y) {
    if (y + m < H) win += hm[(size_t)(y + m) * W + x];
    dm[(size_t)y * W + x] = win > 0;
    if (y - m >= 0) win -= hm[(size_t)(y - m) * W + x];
  }
}

// sam6d_track_points_scene's assignment: one thread per pixel walks the L tracks in order, keeps the eligible track with the
// least rendered depth and the eligible track with the least d2 / r^2 (strict <: exact ties stay with the lower j), writes
// every track's candidate byte and adds one to the winner's row count (warp-aggregated integer atomics: exact)
__global__ void __launch_bounds__(TRK_THREADS) trk_assign(const float* __restrict__ rdepth, const unsigned char* __restrict__ dmask,
                                                         const unsigned short* __restrict__ depth, TrkCam cam,
                                                         const float* __restrict__ centre, const float* __restrict__ radius, int L,
                                                         int H, int W, unsigned char* __restrict__ cand, int* __restrict__ rows) {
  const int x = blockIdx.x * TRK_THREADS + threadIdx.x, y = blockIdx.y;
  const bool col = x < W;
  int win = -1;
  if (col) {
    const size_t px = (size_t)y * W + x, plane = (size_t)H * W;
    const float3 p = trk_point(cam, depth[px], y, x);
    int front = -1, band = -1;
    float front_z = 0.f, band_q = 0.f;
    if (p.z > 0.f)
      for (int j = 0; j < L; ++j) {
        if (!dmask[j * plane + px]) continue;
        const float r = radius[j];
        if (!(r > 0.f)) continue;
        const float d2 = trk_gate_d2(p, centre + 3 * j), r2 = __fmul_rn(r, r);
        if (!(d2 <= r2)) continue;
        const float rz = rdepth[j * plane + px];
        if (rz > 0.f) {
          if (front < 0 || rz < front_z) front = j, front_z = rz;
        } else if (front < 0) {
          const float q = __fdiv_rn(d2, r2);
          if (band < 0 || q < band_q) band = j, band_q = q;
        }
      }
    win = front >= 0 ? front : band;
    for (int j = 0; j < L; ++j) cand[j * plane + px] = j == win;
  }
  const unsigned same = __match_any_sync(0xffffffffu, win);
  if (win >= 0 && (threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(&rows[(size_t)win * H + y], __popc(same));
}

// rows (O,H): counts in, exclusive offsets out; count (O) the totals.  An object with no candidate gets zeros (and index -1).
__global__ void __launch_bounds__(TRK_THREADS) trk_scan(int* __restrict__ rows, int H, int N, int* __restrict__ count,
                                                       float* __restrict__ pts, int* __restrict__ index) {
  __shared__ int warp_sums[TRK_THREADS / 32];
  const int o = blockIdx.x;
  int* r = rows + (size_t)o * H;
  int base = 0;
  for (int y0 = 0; y0 < H; y0 += TRK_THREADS) {
    const int y = y0 + threadIdx.x;
    const int v = y < H ? r[y] : 0;
    int tot;
    const int off = trk_block_scan(v, warp_sums, &tot);
    if (y < H) r[y] = base + off;
    base += tot;
  }
  if (threadIdx.x == 0) count[o] = base;
  if (base == 0)
    for (int i = threadIdx.x; i < N; i += TRK_THREADS) {
      pts[((size_t)o * N + i) * 3] = 0.f;
      pts[((size_t)o * N + i) * 3 + 1] = 0.f;
      pts[((size_t)o * N + i) * 3 + 2] = 0.f;
      if (index) index[(size_t)o * N + i] = -1;
    }
}

__global__ void __launch_bounds__(TRK_THREADS) trk_select(const unsigned char* __restrict__ cand, const unsigned short* __restrict__ depth,
                                                         TrkCam cam, const int* __restrict__ rows, const int* __restrict__ count, int H, int W,
                                                         int N, float* __restrict__ pts, int* __restrict__ index) {
  __shared__ int warp_sums[TRK_THREADS / 32];
  const int y = blockIdx.x, o = blockIdx.y;
  const long long cnt = count[o];
  if (cnt == 0) return;
  int base = rows[(size_t)o * H + y];
  const unsigned char* cr = cand + ((size_t)o * H + y) * W;
  for (int x0 = 0; x0 < W; x0 += TRK_THREADS) {
    const int x = x0 + threadIdx.x;
    const bool on = x < W && cr[x];
    int tot;
    const long long k = base + trk_block_scan(on, warp_sums, &tot);
    base += tot;
    if (!on) continue;
    const float3 p = trk_point(cam, depth[(size_t)y * W + x], y, x);
    const auto put = [&](long long i) {
      float* q = pts + ((size_t)o * N + i) * 3;
      q[0] = p.x; q[1] = p.y; q[2] = p.z;
      if (index) index[(size_t)o * N + i] = y * W + x;
    };
    if (cnt >= N) {
      const long long i = (k * N + cnt - 1) / cnt;            // the least i with i cnt / N >= k; it selects k iff floor(i cnt / N) == k
      if (i < N && i * cnt / N == k) put(i);
    } else {
      for (long long i = k; i < N; i += cnt) put(i);
    }
  }
}

}  // namespace

S6_API int sam6d_track_points(const float* rdepth, const unsigned short* depth, int O, int H, int W, float depth_scale, float fx,
                              float fy, float cx, float cy, const float* centre, const float* radius, int margin, int N,
                              unsigned char* hmask, unsigned char* cand, int* rows, float* pts, int* count, int* index, void* stream) {
  S6_REQUIRE(O >= 0 && H >= 1 && W >= 1 && margin >= 0 && N >= 1 && (long long)H * W <= 0x7fffffffLL);
  if (O == 0) return 0;
  S6_REQUIRE(rdepth && depth && centre && radius && hmask && cand && rows && pts && count);
  S6_REQUIRE(W <= 48 * 1024 && O <= 65535 && H <= 65535);             // one row in static-limit shared memory; grid y / z limits
  cudaStream_t st = s6_stream(stream);
  const TrkCam cam{depth_scale, fx, fy, cx, cy};
  const int m = margin < (H > W ? H : W) ? margin : (H > W ? H : W);
  trk_dilate_rows<<<dim3(H, O), TRK_THREADS, W, st>>>(rdepth, H, W, m, hmask, rows);
  S6_LAUNCH_CHECK();
  trk_candidates<<<dim3(s6_cdiv(W, TRK_THREADS), s6_cdiv(H, TRK_ROWS), O), TRK_THREADS, 0, st>>>(hmask, depth, cam, centre, radius, H, W,
                                                                                                 m, cand, rows);
  S6_LAUNCH_CHECK();
  trk_scan<<<O, TRK_THREADS, 0, st>>>(rows, H, N, count, pts, index);
  S6_LAUNCH_CHECK();
  trk_select<<<dim3(H, O), TRK_THREADS, 0, st>>>(cand, depth, cam, rows, count, H, W, N, pts, index);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_track_points_scene(const float* rdepth, const unsigned short* depth, int L, int H, int W, float depth_scale, float fx,
                                    float fy, float cx, float cy, const float* centre, const float* radius, int margin, int N,
                                    unsigned char* hmask, unsigned char* dmask, unsigned char* cand, int* rows, float* pts, int* count,
                                    int* index, void* stream) {
  S6_REQUIRE(L >= 0 && H >= 1 && W >= 1 && margin >= 0 && N >= 1 && (long long)H * W <= 0x7fffffffLL);
  if (L == 0) return 0;
  S6_REQUIRE(rdepth && depth && centre && radius && hmask && dmask && cand && rows && pts && count);
  S6_REQUIRE(W <= 48 * 1024 && L <= 65535 && H <= 65535);
  cudaStream_t st = s6_stream(stream);
  const TrkCam cam{depth_scale, fx, fy, cx, cy};
  const int m = margin < (H > W ? H : W) ? margin : (H > W ? H : W);
  trk_dilate_rows<<<dim3(H, L), TRK_THREADS, W, st>>>(rdepth, H, W, m, hmask, rows);
  S6_LAUNCH_CHECK();
  trk_dilate_cols<<<dim3(s6_cdiv(W, TRK_THREADS), s6_cdiv(H, TRK_ROWS), L), TRK_THREADS, 0, st>>>(hmask, H, W, m, dmask);
  S6_LAUNCH_CHECK();
  trk_assign<<<dim3(s6_cdiv(W, TRK_THREADS), H), TRK_THREADS, 0, st>>>(rdepth, dmask, depth, cam, centre, radius, L, H, W, cand, rows);
  S6_LAUNCH_CHECK();
  trk_scan<<<L, TRK_THREADS, 0, st>>>(rows, H, N, count, pts, index);
  S6_LAUNCH_CHECK();
  trk_select<<<dim3(H, L), TRK_THREADS, 0, st>>>(cand, depth, cam, rows, count, H, W, N, pts, index);
  S6_LAUNCH_CHECK();
  return 0;
}
