// geo_lut.cu -- GeometricStructureEmbedding (PEM/model/transformer.py:334-349) by table interpolation (bf16 token stream).
//
//   E[p,:] = g_d(d_p) + max_{k<3} g_a(a_{p,k}),     g_a(x) = W_a emb(x),   g_d(x) = W_d emb(x) + (b_a + b_d),   p = (cloud, n, m)
//
// emb(x) is the 256-entry sinusoidal embedding of ONE scalar, so g_a and g_d are smooth vector-valued functions of a scalar:
// frequencies <= 1 rad per index unit, angle indices in [0, 12] (angles in [0, pi] / sigma_a), distance indices of points in
// normalised clouds below 12 (the table spans [0, 32): 6.4 object radii).  The reference evaluates them with 4 x 256 sin/cos and two 256 x 256 products PER PAIR (651 GFLOP
// per cloud batch; the tensor-core version of this repo, geo_tc.cu, still runs those products, bound by MUFU, MMA issue and
// its epilogue together).  Here both functions are tabulated once per weight set on a grid of step 1/8 (host side, float64,
// from the fp32 weights: 97 + 257 rows of 256 bf16 = 181 KB) and a pair costs four linear interpolations out of shared memory:
// no sin/cos, no MMA, E written exactly once.  Interpolation error at step 1/8 is < 1e-4 of |E| -- below the bf16 rounding of
// the table and of E itself (tools/geo_lut_error.py compares it with the float64 embedding).
//
// Kernel: persistent, 16 warps per CTA (two pairs in flight per warp), both tables resident in shared memory.  A warp takes 32 consecutive pairs: lane l loads
// the indices of pair l (one coalesced 512-byte read), then for each pair the four indices are broadcast by shuffles and lane l
// interpolates channels [8l, 8l+8) in fp32 (interpolation, maximum and sum; ONE rounding to bf16 at the store), one 16-byte store
// per lane = one 512-byte row of E per warp instruction.
// Bounds per 64-cloud call: E write 1.27 GB (HBM), 4 KB of table reads per pair (shared-memory bandwidth), ~70 warp
// instructions per pair.
//
// Distance indices outside the table (>= 32): pairs of row 0 / column 0 -- the background point of SAM-6D sits at (100,100,100),
// ~870 index units from everything -- read g_d from `far` (clouds, 2, S, 256), computed exactly (tensor-core distance pass of
// geo_tc.cu) from the 2 S distances of that row and column; any other out-of-range pair takes a slow exact path (sin/cos + a
// 256 x 256 product per pair on CUDA cores, ~5000 warp instructions against ~100 for a table pair: the bench's synthetic clouds,
// whose 20 % gaussian outliers put 3 % of the pairs beyond index 16, would spend most of the time there with a [0, 16) table --
// hence the [0, 32) span), so the kernel is correct for any input and fast for the clouds the model produces.
#include <cuda_bf16.h>

#include "common.cuh"

namespace {

__device__ __forceinline__ uint32_t bf2_pack(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// table position of an index value: row offset (in uint4 units, lane-relative) and interpolation weight.  Computed ONCE per pair by
// the lane that loaded the pair's indices and broadcast by shuffles (per lane and lookup it cost 8 of the ~25 instructions)
__device__ __forceinline__ void lut_pos(float x, float inv_h, int nent, int& row, float& t) {
  const float u = x * inv_h;
  int i = (int)u;
  i = max(0, min(i, nent - 2));
  t = u - (float)i;
  row = i * 32;
}
// linear interpolation between table rows `row` and `row + 1` in fp32 (table entries unpacked, no intermediate rounding): lane's
// 8 channels of g(x)
__device__ __forceinline__ void lut_lerp_f32(const uint4* __restrict__ tab, int row, float t, float v[8]) {
  const uint4 lo = tab[row], hi = tab[row + 32];
  const uint32_t l[4] = {lo.x, lo.y, lo.z, lo.w}, h[4] = {hi.x, hi.y, hi.z, hi.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float l0 = __uint_as_float(l[k] << 16), l1 = __uint_as_float(l[k] & 0xffff0000u);
    const float h0 = __uint_as_float(h[k] << 16), h1 = __uint_as_float(h[k] & 0xffff0000u);
    v[2 * k] = fmaf(t, h0 - l0, l0);
    v[2 * k + 1] = fmaf(t, h1 - l1, l1);
  }
}
__device__ __forceinline__ void unpack8(const uint4& a, float v[8]) {
  const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) { v[2 * k] = __uint_as_float(w[k] << 16); v[2 * k + 1] = __uint_as_float(w[k] & 0xffff0000u); }
}

// exact g_d(x) for one pair, warp-cooperative (rare path): lane l evaluates frequencies 4l .. 4l+3, every lane accumulates its 8
// output channels over the 256 embedding entries (weights: W_d^T (in, out) bf16 from global / L2)
__device__ __noinline__ uint4 slow_distance(float x, const float* __restrict__ div_term, const uint4* __restrict__ WdT,
                                            const float* __restrict__ bias, int lane) {
  float e[8];
#pragma unroll
  for (int q = 0; q < 4; ++q) sincosf(x * div_term[lane * 4 + q], &e[2 * q], &e[2 * q + 1]);
  float acc[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c] = bias[lane * 8 + c];
  for (int s = 0; s < 32; ++s) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float v = __shfl_sync(0xffffffffu, e[q], s);
      const uint4 w = WdT[(size_t)(s * 8 + q) * 32 + lane];
      const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc[2 * i] = fmaf(v, __uint_as_float(ww[i] << 16), acc[2 * i]);
        acc[2 * i + 1] = fmaf(v, __uint_as_float(ww[i] & 0xffff0000u), acc[2 * i + 1]);
      }
    }
  }
  return make_uint4(bf2_pack(acc[0], acc[1]), bf2_pack(acc[2], acc[3]), bf2_pack(acc[4], acc[5]), bf2_pack(acc[6], acc[7]));
}

// fp32 arithmetic was chosen over a packed bf16x2 form of the same kernel, which had rms error 1.6e-3 against 1.2e-3 (emulated in
// torch at step 1/8) at about half the instructions per pair.  LUT_THREADS / UNROLL: warps per CTA against pairs in flight per warp (the kernel is bound by the
// shared-memory pipe, warps waiting on their LDS results); 16 x 2 was chosen by measurement over 32 x 1 and 24 x 2.
constexpr int LUT_THREADS = 512, UNROLL = 2;
__global__ void __launch_bounds__(LUT_THREADS, 1) geo_embed_lut_kernel(const float4* __restrict__ T, long long npairs, int S,
                                                                      const uint4* __restrict__ tabA_g, int na, float inv_ha,
                                                                      const uint4* __restrict__ tabD_g, int nd, float inv_hd,
                                                                      const uint4* __restrict__ far, const float* __restrict__ div_term,
                                                                      const uint4* __restrict__ WdT, const float* __restrict__ bias,
                                                                      uint4* __restrict__ E) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint4* tabA = reinterpret_cast<uint4*>(smem_raw);
  uint4* tabD = tabA + na * 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int u = tid; u < na * 32; u += LUT_THREADS) tabA[u] = tabA_g[u];
  for (int u = tid; u < nd * 32; u += LUT_THREADS) tabD[u] = tabD_g[u];
  __syncthreads();
  const float d_limit = (float)(nd - 1) / inv_hd;          // distance indices below this are inside the table
  const long long nblocks = (npairs + 31) / 32;
  const long long SS = (long long)S * S;
  for (long long blk = (long long)blockIdx.x * (LUT_THREADS / 32) + warp; blk < nblocks; blk += (long long)gridDim.x * (LUT_THREADS / 32)) {
    const long long base = blk * 32;
    const int cnt = (int)min(32LL, npairs - base);
    float4 tv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane < cnt) tv = T[base + lane];
    // this lane's pair: table rows and weights of its four indices (a distance outside the table is flagged by row -1)
    int r0, r1, r2, r3;
    float t0, t1, t2, t3;
    lut_pos(tv.x, inv_ha, na, r0, t0);
    lut_pos(tv.y, inv_ha, na, r1, t1);
    lut_pos(tv.z, inv_ha, na, r2, t2);
    lut_pos(tv.w, inv_hd, nd, r3, t3);
    if (!(tv.w < d_limit)) r3 = -1;
    const uint4* tabA_l = tabA + lane;
    const uint4* tabD_l = tabD + lane;
#pragma unroll UNROLL
    for (int j = 0; j < cnt; ++j) {
      const int q0 = __shfl_sync(0xffffffffu, r0, j), q1 = __shfl_sync(0xffffffffu, r1, j);
      const int q2 = __shfl_sync(0xffffffffu, r2, j), q3 = __shfl_sync(0xffffffffu, r3, j);
      const float w0 = __shfl_sync(0xffffffffu, t0, j), w1 = __shfl_sync(0xffffffffu, t1, j);
      const float w2 = __shfl_sync(0xffffffffu, t2, j), w3 = __shfl_sync(0xffffffffu, t3, j);
      uint4 dv;
      const bool in_table = q3 >= 0;                       // warp-uniform: a broadcast value
      if (!in_table) {
        const long long p = base + j;
        const long long c = p / SS;
        const int rem = (int)(p - c * SS), n = rem / S, m = rem - n * S;
        if (n == 0) dv = far[((c * 2 + 0) * S + m) * 32 + lane];
        else if (m == 0) dv = far[((c * 2 + 1) * S + n) * 32 + lane];
        else dv = slow_distance(__shfl_sync(0xffffffffu, tv.w, j), div_term, WdT, bias, lane);
      }
      float f0[8], f1[8], f2[8], fd[8];
      lut_lerp_f32(tabA_l, q0, w0, f0);
      lut_lerp_f32(tabA_l, q1, w1, f1);
      lut_lerp_f32(tabA_l, q2, w2, f2);
      if (in_table) lut_lerp_f32(tabD_l, q3, w3, fd);
      else unpack8(dv, fd);
#pragma unroll
      for (int k = 0; k < 8; ++k) fd[k] += fmaxf(fmaxf(f0[k], f1[k]), f2[k]);
      const uint4 o = make_uint4(bf2_pack(fd[0], fd[1]), bf2_pack(fd[2], fd[3]), bf2_pack(fd[4], fd[5]), bf2_pack(fd[6], fd[7]));
      E[(base + j) * 32 + lane] = o;
    }
  }
}

}  // namespace

// T (clouds*S*S, 4) f32 = (a0, a1, a2, d) indices of every pair; tabA (na, 256) bf16 = W_a emb(i / inv_ha), tabD (nd, 256) bf16 =
// W_d emb(i / inv_hd) + bias; far (clouds, 2, S, 256) bf16 = exact g_d of row 0 ([:,0]) and column 0 ([:,1]) of every cloud;
// div_term (128) f32, WdT (256 in, 256 out) bf16 and bias (256) f32 for the exact fallback of other out-of-table distances
// -> E (clouds*S*S, 256) bf16
S6_API int sam6d_geo_embed_lut(const float* T, long long clouds, int S, const void* tabA, int na, float inv_ha, const void* tabD, int nd,
                               float inv_hd, const void* far, const float* div_term, const void* WdT_bf16, const float* bias, void* E,
                               void* stream) {
  S6_REQUIRE(T && tabA && tabD && far && div_term && WdT_bf16 && bias && E && clouds >= 0 && S > 0 && na >= 2 && nd >= 2);
  S6_REQUIRE(inv_ha > 0.f && inv_hd > 0.f && (long long)(na + nd) * 512 <= 200 * 1024);
  S6_REQUIRE(((reinterpret_cast<uintptr_t>(T) | reinterpret_cast<uintptr_t>(tabA) | reinterpret_cast<uintptr_t>(tabD) | reinterpret_cast<uintptr_t>(far) |
               reinterpret_cast<uintptr_t>(WdT_bf16) | reinterpret_cast<uintptr_t>(E)) & 15) == 0);
  const long long npairs = clouds * S * S;
  S6_REQUIRE(npairs < (1LL << 40));
  if (npairs == 0) return 0;
  const long long nblocks = (npairs + 31) / 32, want = (nblocks + LUT_THREADS / 32 - 1) / (LUT_THREADS / 32);
  int grid;
  S6_CHECK(s6_persistent_grid(want, 1, &grid));
  const int smem = (na + nd) * 512;
  S6_CHECK(cudaFuncSetAttribute(geo_embed_lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  geo_embed_lut_kernel<<<grid, LUT_THREADS, smem, s6_stream(stream)>>>(
      reinterpret_cast<const float4*>(T), npairs, S, reinterpret_cast<const uint4*>(tabA), na, inv_ha, reinterpret_cast<const uint4*>(tabD),
      nd, inv_hd, reinterpret_cast<const uint4*>(far), div_term, reinterpret_cast<const uint4*>(WdT_bf16), bias, reinterpret_cast<uint4*>(E));
  S6_LAUNCH_CHECK();
  return 0;
}
