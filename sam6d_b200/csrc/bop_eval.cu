// bop_eval.cu -- pose errors of the BOP19 pose task (sam6d_b200/bop_eval.py, oracle/bop_eval_oracle.py).
//
// MSSD / MSPD (Hodan et al., BOP Challenge 2020, sec. 2.2): for each (estimate, GT) pair and each symmetry S of the object,
// the maximum over the model vertices x of the 3D distance |(R_e x + t_e) - (R_g (S x) + t_g)| (MSSD) and of the distance of
// the two projections through K (MSPD), then the minimum over S.  The 3D residual is formed as A x + b with A = R_e - R_g R_s
// and b = t_e - R_g t_s - t_g (one 3x4 per thread and symmetry), so it does not cancel two large camera-frame points; the
// GT point for MSPD is p_e - (A x + b).  Maxima and minima are order-free, so the result is deterministic.
//
// VSD (same paper; Hodan et al., ECCV 2016 workshop): per pair, integer counts over the pixels of |U|, |I| and, per tau,
// #{p in I : |dist_g - dist_e| / diameter >= tau}, from the rendered depths of the estimate and the GT and the test depth;
// the host forms e(tau) = (cost + |U| - |I|) / |U|.  No distance or visibility image is written.
//
// COCO mask IoU of the BOP detection / segmentation task (sam6d_b200/bop_eval_coco.py, oracle/bop_coco_oracle.py): masks are
// bit-packed in COCO's RLE order (column-major, bit k = x H + y, LSB first in 32-bit words), from run ends or from decoded PNG
// masks, and |A & B| of a pair is the popcount of the AND of their words.  Every result is an exact integer.
#include "common.cuh"

namespace {

constexpr int BE_THREADS = 256;
constexpr int BE_WARPS = BE_THREADS / 32;
constexpr int BE_SYM_TILE = 32;              // symmetries per CTA of the MSSD / MSPD kernel
constexpr int BE_VTILE = 1024;               // vertices per shared-memory tile (16 KB as float4)
constexpr int BE_NTAU = 10;
constexpr int BE_VSD_PIX = 4096;             // pixels per CTA of the VSD kernel

// grid (P, max symmetry tiles).  A warp's 32 lanes are SL symmetries x VL vertex lanes (SL = the tile's symmetry count rounded
// up to a power of two, VL = 32 / SL), so an object without symmetries still uses every lane.  Each thread keeps the maxima of
// its symmetry over its vertices; lanes and warps of the same symmetry combine by a max, the tile's symmetries by a min, and
// the CTAs of a pair by an atomicMin on the float bits (non-negative floats order as their bit patterns).
__global__ void __launch_bounds__(BE_THREADS) bop_mssd_mspd_kernel(const float* __restrict__ est, const float* __restrict__ gt,
                                                                   const int* __restrict__ pair_obj, const float* __restrict__ Kp,
                                                                   const float* __restrict__ verts, const int* __restrict__ vert_off,
                                                                   const float* __restrict__ syms, const int* __restrict__ sym_off,
                                                                   unsigned* __restrict__ out) {
  __shared__ float4 sv[BE_VTILE];
  __shared__ float red[BE_WARPS][BE_SYM_TILE][2];
  const int p = blockIdx.x, o = pair_obj[p];
  const int s_begin = sym_off[o], n_sym = sym_off[o + 1] - s_begin;
  const int s0 = blockIdx.y * BE_SYM_TILE;
  if (s0 >= n_sym) return;
  const int ns = min(BE_SYM_TILE, n_sym - s0);
  int SL = 1;
  while (SL < ns) SL <<= 1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sl = lane & (SL - 1), vl = lane / SL, VL = 32 / SL;
  const bool active = sl < ns;

  const float* Re = est + (long long)p * 12;      // R row-major (9), t (3)
  const float* Rg = gt + (long long)p * 12;
  const float* S = syms + (long long)(s_begin + s0 + (active ? sl : 0)) * 12;
  float A[9], b[3], Rv[9], te[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      A[r * 3 + c] = Re[r * 3 + c] - (Rg[r * 3] * S[c] + Rg[r * 3 + 1] * S[3 + c] + Rg[r * 3 + 2] * S[6 + c]);
      Rv[r * 3 + c] = Re[r * 3 + c];
    }
    te[r] = Re[9 + r];
    b[r] = Re[9 + r] - (Rg[r * 3] * S[9] + Rg[r * 3 + 1] * S[10] + Rg[r * 3 + 2] * S[11]) - Rg[9 + r];
  }
  const float fx = Kp[p * 4], fy = Kp[p * 4 + 1];

  float m3 = 0.f, m2 = 0.f;                       // squared maxima: 3D distance, projected distance
  const int v_begin = vert_off[o], nv = vert_off[o + 1] - v_begin;
  for (int t0 = 0; t0 < nv; t0 += BE_VTILE) {
    const int nt = min(BE_VTILE, nv - t0);
    __syncthreads();
    for (int i = threadIdx.x; i < nt; i += BE_THREADS) {
      const float* v = verts + (long long)(v_begin + t0 + i) * 3;
      sv[i] = make_float4(v[0], v[1], v[2], 0.f);
    }
    __syncthreads();
    if (!active) continue;
    for (int i = warp * VL + vl; i < nt; i += BE_WARPS * VL) {
      const float4 x = sv[i];
      float d[3], pe[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        d[r] = A[r * 3] * x.x + A[r * 3 + 1] * x.y + A[r * 3 + 2] * x.z + b[r];
        pe[r] = Rv[r * 3] * x.x + Rv[r * 3 + 1] * x.y + Rv[r * 3 + 2] * x.z + te[r];
      }
      m3 = fmaxf(m3, d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
      const float gx = pe[0] - d[0], gy = pe[1] - d[1], gz = pe[2] - d[2];
      const float du = fx * (pe[0] / pe[2] - gx / gz), dv = fy * (pe[1] / pe[2] - gy / gz);
      m2 = fmaxf(m2, du * du + dv * dv);
    }
  }
  // lanes of one symmetry differ in the bits above log2(SL)
  for (int off = 16; off >= SL; off >>= 1) {
    m3 = fmaxf(m3, __shfl_xor_sync(0xffffffffu, m3, off));
    m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, off));
  }
  if (lane < SL) { red[warp][lane][0] = m3; red[warp][lane][1] = m2; }
  __syncthreads();
  if (warp == 0) {
    float a = INFINITY, c = INFINITY;
    if (lane < ns) {
      a = red[0][lane][0]; c = red[0][lane][1];
#pragma unroll
      for (int w = 1; w < BE_WARPS; ++w) { a = fmaxf(a, red[w][lane][0]); c = fmaxf(c, red[w][lane][1]); }
    }
    for (int off = 16; off > 0; off >>= 1) {
      a = fminf(a, __shfl_xor_sync(0xffffffffu, a, off));
      c = fminf(c, __shfl_xor_sync(0xffffffffu, c, off));
    }
    if (lane == 0) {
      atomicMin(out + p * 2, __float_as_uint(sqrtf(a)));
      atomicMin(out + p * 2 + 1, __float_as_uint(sqrtf(c)));
    }
  }
}

__device__ __forceinline__ int be_block_sum(int v, int* sh) {
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) atomicAdd(sh, v);
  return v;
}

// grid (ceil(H*W / BE_VSD_PIX), P).  dist = depth * sqrt(((u - cx) / fx)^2 + ((v - cy) / fy)^2 + 1) at integer (u, v);
// V_g = d_g > 0 and (d_g - d_t <= delta or d_t = 0); V_e the same on d_e, or (V_g and d_e > 0).
__global__ void __launch_bounds__(BE_THREADS) bop_vsd_kernel(const float* __restrict__ dep_e, const float* __restrict__ dep_g,
                                                             const float* __restrict__ dep_t, const int* __restrict__ pair_img, int H,
                                                             int W, float fx, float fy, float cx, float cy, float delta, float diameter,
                                                             const float* __restrict__ taus, int* __restrict__ out) {
  __shared__ int cnt[2 + BE_NTAU];
  __shared__ float tau[BE_NTAU];
  if (threadIdx.x < 2 + BE_NTAU) cnt[threadIdx.x] = 0;
  if (threadIdx.x < BE_NTAU) tau[threadIdx.x] = taus[threadIdx.x];
  __syncthreads();
  const int p = blockIdx.y;
  const long long hw = (long long)H * W;
  const float* de = dep_e + p * hw;
  const float* dg = dep_g + p * hw;
  const float* dt = dep_t + pair_img[p] * hw;
  int nu = 0, ni = 0, nc[BE_NTAU];
#pragma unroll
  for (int k = 0; k < BE_NTAU; ++k) nc[k] = 0;
  const long long end = min(hw, (long long)(blockIdx.x + 1) * BE_VSD_PIX);
  for (long long i = (long long)blockIdx.x * BE_VSD_PIX + threadIdx.x; i < end; i += BE_THREADS) {
    const float ze = de[i], zg = dg[i], zt = dt[i];
    if (ze <= 0.f && zg <= 0.f) continue;         // in neither V_g nor V_e
    const int v = (int)(i / W), u = (int)(i - (long long)v * W);
    const float a = (u - cx) / fx, c = (v - cy) / fy;
    const float f = sqrtf(a * a + c * c + 1.f);
    const float e = ze * f, g = zg * f, t = zt * f;
    const bool vg = zg > 0.f && (g - t <= delta || zt == 0.f);
    const bool ve = (ze > 0.f && (e - t <= delta || zt == 0.f)) || (vg && ze > 0.f);
    nu += vg || ve;
    if (vg && ve) {
      ++ni;
      const float r = fabsf(g - e) / diameter;
#pragma unroll
      for (int k = 0; k < BE_NTAU; ++k) nc[k] += r >= tau[k];
    }
  }
  be_block_sum(nu, cnt);
  be_block_sum(ni, cnt + 1);
#pragma unroll
  for (int k = 0; k < BE_NTAU; ++k) be_block_sum(nc[k], cnt + 2 + k);
  __syncthreads();
  if (threadIdx.x < 2 + BE_NTAU && cnt[threadIdx.x]) atomicAdd(out + p * (2 + BE_NTAU) + threadIdx.x, cnt[threadIdx.x]);
}

// ---- COCO masks ----------------------------------------------------------------------------------------------------------------
constexpr int BM_THREADS = 256;
constexpr int BM_WARPS = BM_THREADS / 32;

// grid (n masks).  Each thread builds whole words: the run holding the word's first pixel by a binary search over the mask's run
// ends (the first end > that pixel), then the runs up to the word's last pixel; odd runs are foreground.  Zero-length runs are
// skipped by the search and add no bits.  Every word of the mask is written, so no clearing pass is needed.
__global__ void __launch_bounds__(BM_THREADS) bop_pack_rle_kernel(const int* __restrict__ rle_cum, const int* __restrict__ rle_off,
                                                                  const int* __restrict__ hw, const int* __restrict__ word_off,
                                                                  unsigned* __restrict__ bits) {
  const int i = blockIdx.x;
  const int* cum = rle_cum + rle_off[i];
  const int nr = rle_off[i + 1] - rle_off[i];
  const long long npix = (long long)hw[2 * i] * hw[2 * i + 1];
  const int nw = (int)((npix + 31) >> 5);
  unsigned* out = bits + word_off[i];
  for (int w = threadIdx.x; w < nw; w += BM_THREADS) {
    const long long p0 = (long long)w << 5, p1 = p0 + 32;
    int lo = 0, hi = nr;
    while (lo < hi) {                                // first k with cum[k] > p0
      const int mid = (lo + hi) >> 1;
      if (cum[mid] > p0) hi = mid; else lo = mid + 1;
    }
    unsigned word = 0u;
    for (int k = lo; k < nr; ++k) {
      const long long a = k ? cum[k - 1] : 0, b = cum[k];
      if (a >= p1) break;
      if ((k & 1) && b > a) {
        const int s = (int)max(a - p0, 0LL), e = (int)min(b - p0, 32LL);      // bits [s, e) of this word
        word |= (e - s == 32) ? 0xffffffffu : (((1u << (e - s)) - 1u) << s);
      }
    }
    out[w] = word;
  }
}

__device__ __forceinline__ int bm_block_reduce(int v, bool is_max, int* sh) {
  // warp then block min / max; sh holds BM_WARPS ints; every thread gets the result
  for (int o = 16; o > 0; o >>= 1) {
    const int u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? max(v, u) : min(v, u);
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  v = sh[0];
#pragma unroll
  for (int w = 1; w < BM_WARPS; ++w) v = is_max ? max(v, sh[w]) : min(v, sh[w]);
  return v;
}

// grid (n masks).  Warp-per-word: lane j tests pixel 32 w + j (x = p / H, y = p % H, read from the row-major mask) and a ballot
// forms the word.  The 32 rows a warp reads share their cache sectors with the next 31 columns' reads, which follow within the
// same CTA.  Area by popcount of the words, the tight box by block min / max; bits may be NULL (area and box only).
__global__ void __launch_bounds__(BM_THREADS) bop_pack_u8_kernel(const unsigned char* __restrict__ masks, int H, int W,
                                                                 const int* __restrict__ word_off, unsigned* __restrict__ bits,
                                                                 int* __restrict__ area, int* __restrict__ box) {
  __shared__ int sh[BM_WARPS];
  __shared__ int sh_area[BM_WARPS];
  const int i = blockIdx.x;
  const long long npix = (long long)H * W;
  const unsigned char* m = masks + (long long)i * npix;
  const int nw = (int)((npix + 31) >> 5);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int cnt = 0, x0 = INT_MAX, y0 = INT_MAX, x1 = -1, y1 = -1;
  for (int w = warp; w < nw; w += BM_WARPS) {
    const long long p = ((long long)w << 5) + lane;
    bool on = false;
    int x = 0, y = 0;
    if (p < npix) {
      x = (int)(p / H);
      y = (int)(p - (long long)x * H);
      on = m[(long long)y * W + x] != 0;
    }
    const unsigned word = __ballot_sync(0xffffffffu, on);
    if (lane == 0) {
      if (bits) bits[word_off[i] + w] = word;
      cnt += __popc(word);
    }
    if (on) { x0 = min(x0, x); x1 = max(x1, x); y0 = min(y0, y); y1 = max(y1, y); }
  }
  if (lane == 0) sh_area[warp] = cnt;
  x0 = bm_block_reduce(x0, false, sh);
  y0 = bm_block_reduce(y0, false, sh);
  x1 = bm_block_reduce(x1, true, sh);
  y1 = bm_block_reduce(y1, true, sh);
  if (threadIdx.x == 0) {
    int a = 0;
#pragma unroll
    for (int w = 0; w < BM_WARPS; ++w) a += sh_area[w];
    area[i] = a;
    const bool empty = a == 0;
    box[4 * i] = empty ? -1 : x0;
    box[4 * i + 1] = empty ? -1 : y0;
    box[4 * i + 2] = empty ? -1 : x1;
    box[4 * i + 3] = empty ? -1 : y1;
  }
}

// grid (ceil(P / BM_WARPS)), one warp per pair: 16-byte loads of both masks' words (offsets and lengths are multiples of 4
// words), popcount of the AND, a warp sum.  Order-free integer sums, so deterministic.
__global__ void __launch_bounds__(BM_THREADS) bop_pair_counts_kernel(const unsigned* __restrict__ bits, const int* __restrict__ word_off,
                                                                     const int* __restrict__ pair_a, const int* __restrict__ pair_b, int P,
                                                                     int* __restrict__ out) {
  const int p = blockIdx.x * BM_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= P) return;
  const int a = pair_a[p], b = pair_b[p];
  const int nq = min(word_off[a + 1] - word_off[a], word_off[b + 1] - word_off[b]) >> 2;
  const uint4* A = reinterpret_cast<const uint4*>(bits + word_off[a]);
  const uint4* B = reinterpret_cast<const uint4*>(bits + word_off[b]);
  int c = 0;
#pragma unroll 4
  for (int j = lane; j < nq; j += 32) {
    const uint4 u = __ldg(A + j), v = __ldg(B + j);
    c += __popc(u.x & v.x) + __popc(u.y & v.y) + __popc(u.z & v.z) + __popc(u.w & v.w);
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if (lane == 0) out[p] = c;
}

}  // namespace

S6_API int sam6d_bop_mssd_mspd(const float* est, const float* gt, const int* pair_obj, const float* K, int P, const float* verts,
                               const int* vert_off, const float* syms, const int* sym_off, int O, int max_sym, float* out,
                               void* stream) {
  S6_REQUIRE(est && gt && pair_obj && K && verts && vert_off && syms && sym_off && out);
  S6_REQUIRE(P >= 0 && O > 0 && max_sym > 0 && s6_cdiv(max_sym, BE_SYM_TILE) <= 65535);
  cudaStream_t st = s6_stream(stream);
  if (P == 0) return 0;
  // 0x7f7f7f7f = 3.4e38: every pair has at least one symmetry tile, which lowers it
  S6_CHECK(cudaMemsetAsync(out, 0x7f, (size_t)P * 2 * sizeof(float), st));
  dim3 grid(P, s6_cdiv(max_sym, BE_SYM_TILE));
  bop_mssd_mspd_kernel<<<grid, BE_THREADS, 0, st>>>(est, gt, pair_obj, K, verts, vert_off, syms, sym_off,
                                                    reinterpret_cast<unsigned*>(out));
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_bop_vsd_counts(const float* depth_est, const float* depth_gt, const float* depth_test, const int* pair_img, int P,
                                int H, int W, float fx, float fy, float cx, float cy, float delta, float diameter, const float* taus,
                                int* out, void* stream) {
  S6_REQUIRE(depth_est && depth_gt && depth_test && pair_img && taus && out);
  S6_REQUIRE(P >= 0 && H > 0 && W > 0 && P <= 65535 && diameter > 0.f && fx != 0.f && fy != 0.f);
  cudaStream_t st = s6_stream(stream);
  if (P == 0) return 0;
  S6_CHECK(cudaMemsetAsync(out, 0, (size_t)P * (2 + BE_NTAU) * sizeof(int), st));
  dim3 grid(s6_cdiv((long long)H * W, BE_VSD_PIX), P);
  bop_vsd_kernel<<<grid, BE_THREADS, 0, st>>>(depth_est, depth_gt, depth_test, pair_img, H, W, fx, fy, cx, cy, delta, diameter, taus, out);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_bop_pack_rle(const int* rle_cum, const int* rle_off, const int* hw, const int* word_off, int n, unsigned* bits,
                              void* stream) {
  S6_REQUIRE(rle_off && hw && word_off && bits && n >= 0);
  cudaStream_t st = s6_stream(stream);
  if (n == 0) return 0;
  S6_REQUIRE(rle_cum);
  bop_pack_rle_kernel<<<n, BM_THREADS, 0, st>>>(rle_cum, rle_off, hw, word_off, bits);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_bop_pack_u8(const unsigned char* masks, int n, int H, int W, const int* word_off, unsigned* bits, int* area, int* box,
                             void* stream) {
  S6_REQUIRE(masks && area && box && n >= 0 && H > 0 && W > 0 && (long long)H * W < (1LL << 31));
  S6_REQUIRE(!bits || word_off);
  cudaStream_t st = s6_stream(stream);
  if (n == 0) return 0;
  bop_pack_u8_kernel<<<n, BM_THREADS, 0, st>>>(masks, H, W, word_off, bits, area, box);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_bop_mask_pair_counts(const unsigned* bits, const int* word_off, const int* pair_a, const int* pair_b, int P, int* out,
                                      void* stream) {
  S6_REQUIRE(bits && word_off && pair_a && pair_b && out && P >= 0);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(bits) & 15) == 0);
  cudaStream_t st = s6_stream(stream);
  if (P == 0) return 0;
  bop_pair_counts_kernel<<<s6_cdiv(P, BM_WARPS), BM_THREADS, 0, st>>>(bits, word_off, pair_a, pair_b, P, out);
  S6_LAUNCH_CHECK();
  return 0;
}
