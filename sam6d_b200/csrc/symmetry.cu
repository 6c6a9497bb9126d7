// symmetry.cu -- object symmetry search (not in the reference; sam6d_b200/symmetry.py, oracle/symmetry_oracle.py)
//   1. symmetry_agreement : per candidate transform (R, t), the query samples whose nearest target sample lies within geo_tol
//                           (and within color_tol in colour) -> count, sum of squared nearest-neighbour distances
//   2. point_diameter     : the largest distance between two of V points (models_info's diameter)
// Both are brute force over shared-memory tiles of the second point set; each thread carries SYM_Q (DIA_Q) points of the first
// so that one broadcast shared-memory load feeds that many independent distance chains.
#include "common.cuh"

namespace {

constexpr int SYM_THREADS = 256, SYM_Q = 4, SYM_CHUNK = SYM_THREADS * SYM_Q, SYM_TILE = 2048;
constexpr int DIA_THREADS = 256, DIA_Q = 4, DIA_CHUNK = DIA_THREADS * DIA_Q;

// grid (query chunk, candidate): SYM_CHUNK queries of one candidate per CTA -> that chunk's agreeing count and sum of squared
// distances in part_cnt / part_ss [candidate][chunk]
__global__ void __launch_bounds__(SYM_THREADS) symmetry_agreement_kernel(const float* __restrict__ Rt, const float* __restrict__ q,
                                                                        const float* __restrict__ qc, int Nq, const float* __restrict__ tg,
                                                                        const float* __restrict__ tc, int M, float tol2, float ctol,
                                                                        int* __restrict__ part_cnt, float* __restrict__ part_ss) {
  __shared__ float4 st[SYM_TILE];
  __shared__ int wc[SYM_THREADS / 32];
  __shared__ float ws[SYM_THREADS / 32];
  const int c = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  const float* T = Rt + (size_t)c * 12;
  float y[SYM_Q][3], best[SYM_Q];
  int bi[SYM_Q];
#pragma unroll
  for (int k = 0; k < SYM_Q; ++k) {
    const int i = min(chunk * SYM_CHUNK + k * SYM_THREADS + tid, Nq - 1);
    const float x0 = q[(size_t)i * 3], x1 = q[(size_t)i * 3 + 1], x2 = q[(size_t)i * 3 + 2];
#pragma unroll
    for (int r = 0; r < 3; ++r) y[k][r] = fmaf(T[r * 3], x0, fmaf(T[r * 3 + 1], x1, fmaf(T[r * 3 + 2], x2, T[9 + r])));
    best[k] = INFINITY;
    bi[k] = 0;
  }
  for (int j0 = 0; j0 < M; j0 += SYM_TILE) {
    const int n = min(SYM_TILE, M - j0);
    __syncthreads();
    for (int j = tid; j < n; j += SYM_THREADS) {
      const float* p = tg + (size_t)(j0 + j) * 3;
      st[j] = make_float4(p[0], p[1], p[2], 0.f);
    }
    __syncthreads();
    for (int j = 0; j < n; ++j) {
      const float4 p = st[j];
#pragma unroll
      for (int k = 0; k < SYM_Q; ++k) {
        const float dx = p.x - y[k][0], dy = p.y - y[k][1], dz = p.z - y[k][2];
        const float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
        if (d2 < best[k]) { best[k] = d2; bi[k] = j0 + j; }   // strict: the first index wins a tie
      }
    }
  }
  int cnt = 0;
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < SYM_Q; ++k) {
    const int i = chunk * SYM_CHUNK + k * SYM_THREADS + tid;
    if (i >= Nq) continue;
    bool ok = best[k] <= tol2;
    if (ok && qc && tc) {
      const float* a = qc + (size_t)i * 3;
      const float* b = tc + (size_t)bi[k] * 3;
      ok = fmaxf(fabsf(a[0] - b[0]), fmaxf(fabsf(a[1] - b[1]), fabsf(a[2] - b[2]))) <= ctol;
    }
    cnt += ok;
    ss += best[k];
  }
  // fixed reduction order: the result does not depend on scheduling
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  if ((tid & 31) == 0) { wc[tid >> 5] = cnt; ws[tid >> 5] = ss; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < SYM_THREADS / 32; ++w) { cnt += wc[w]; ss += ws[w]; }
    part_cnt[(size_t)c * gridDim.x + chunk] = cnt;
    part_ss[(size_t)c * gridDim.x + chunk] = ss;
  }
}

// one thread per candidate: the chunks' partial results in chunk order
__global__ void symmetry_reduce_kernel(const int* __restrict__ part_cnt, const float* __restrict__ part_ss, int C, int nchunk,
                                       int* __restrict__ count, float* __restrict__ sumsq) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  int n = 0;
  float s = 0.f;
  for (int k = 0; k < nchunk; ++k) { n += part_cnt[(size_t)c * nchunk + k]; s += part_ss[(size_t)c * nchunk + k]; }
  count[c] = n;
  sumsq[c] = s;
}

// grid (i tile, j tile), tiles of DIA_CHUNK points; only the CTAs with j tile >= i tile work.  Squared distances in fp32, rounded
// to nearest without fused multiply-add; the largest one of the CTA goes to d2 through an integer atomicMax on its bits (every
// value is >= 0, where float order and bit order agree), so the result does not depend on scheduling.
__global__ void __launch_bounds__(DIA_THREADS) point_diameter_kernel(const float* __restrict__ pts, int V, float* __restrict__ d2) {
  const int ti = blockIdx.x, tj = blockIdx.y, tid = threadIdx.x;
  if (tj < ti) return;
  __shared__ float4 sp[DIA_CHUNK];
  __shared__ float wm[DIA_THREADS / 32];
  float x[DIA_Q][3];
#pragma unroll
  for (int k = 0; k < DIA_Q; ++k) {
    const int i = min(ti * DIA_CHUNK + k * DIA_THREADS + tid, V - 1);   // a repeated point adds no new distance
#pragma unroll
    for (int r = 0; r < 3; ++r) x[k][r] = pts[(size_t)i * 3 + r];
  }
  const int j0 = tj * DIA_CHUNK, n = min(DIA_CHUNK, V - j0);
  for (int j = tid; j < n; j += DIA_THREADS) {
    const float* p = pts + (size_t)(j0 + j) * 3;
    sp[j] = make_float4(p[0], p[1], p[2], 0.f);
  }
  __syncthreads();
  float m = 0.f;
  for (int j = 0; j < n; ++j) {
    const float4 p = sp[j];
#pragma unroll
    for (int k = 0; k < DIA_Q; ++k) {
      const float dx = __fsub_rn(p.x, x[k][0]), dy = __fsub_rn(p.y, x[k][1]), dz = __fsub_rn(p.z, x[k][2]);
      m = fmaxf(m, __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    }
  }
  m = warp_max(m);
  if ((tid & 31) == 0) wm[tid >> 5] = m;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < DIA_THREADS / 32; ++w) m = fmaxf(m, wm[w]);
    atomicMax(reinterpret_cast<unsigned int*>(d2), __float_as_uint(m));
  }
}

}  // namespace

S6_API int sam6d_symmetry_agreement(const float* Rt, int C, const float* q, const float* qc, int Nq, const float* tg, const float* tc,
                                    int M, float geo_tol, float color_tol, int* count, float* sumsq, void* work, void* stream) {
  S6_REQUIRE(C >= 0 && Nq >= 1 && M >= 1 && C <= 65535);
  S6_REQUIRE(isfinite(geo_tol) && geo_tol >= 0.f && isfinite(color_tol) && color_tol >= 0.f);
  S6_REQUIRE((qc == nullptr) == (tc == nullptr));
  S6_REQUIRE(Rt && q && tg && count && sumsq && work);
  if (C == 0) return 0;
  const int nchunk = s6_cdiv(Nq, SYM_CHUNK);
  int* part_cnt = static_cast<int*>(work);
  float* part_ss = reinterpret_cast<float*>(part_cnt + (size_t)C * nchunk);
  cudaStream_t st = s6_stream(stream);
  symmetry_agreement_kernel<<<dim3(nchunk, C), SYM_THREADS, 0, st>>>(Rt, q, qc, Nq, tg, tc, M, geo_tol * geo_tol, color_tol,
                                                                   part_cnt, part_ss);
  S6_LAUNCH_CHECK();
  symmetry_reduce_kernel<<<s6_cdiv(C, 128), 128, 0, st>>>(part_cnt, part_ss, C, nchunk, count, sumsq);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_point_diameter(const float* pts, int V, float* d2, void* stream) {
  S6_REQUIRE(V >= 1 && (long long)V <= 65535LL * DIA_CHUNK);
  S6_REQUIRE(pts && d2);
  cudaStream_t st = s6_stream(stream);
  S6_CHECK(cudaMemsetAsync(d2, 0, sizeof(float), st));
  const int nt = s6_cdiv(V, DIA_CHUNK);
  point_diameter_kernel<<<dim3(nt, nt), DIA_THREADS, 0, st>>>(pts, V, d2);
  S6_LAUNCH_CHECK();
  return 0;
}
