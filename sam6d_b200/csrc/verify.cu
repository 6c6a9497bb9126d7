// verify.cu -- depth agreement of rendered pose hypotheses (not in the reference; the rule is stated in include/sam6d_b200.h
// at sam6d_pose_verify and restated in float64 by oracle/verify_oracle.py).
//
// One pass over the P rendered depths, grid (pixel tiles, hypotheses).  A thread classifies four adjacent pixels per step
// (a float4 of the rendered depth, a float4 of the observed depth, a uchar4 of the hypothesis's mask row) when the frame allows
// aligned vector loads, else one pixel.  The six counts are summed per warp (__reduce_add_sync), per CTA in shared memory,
// and added to counts with one integer atomic per CTA and counter: order-free, so exact and deterministic.
// The mask rows and tolerances are host arrays: the entry point validates them before anything is launched and passes them
// in the launch parameters, up to VF_BATCH hypotheses per launch.
#include "common.cuh"

namespace {

constexpr int VF_THREADS = 256;
constexpr int VF_PIX = 16384;              // pixels per CTA: 16 vector steps per thread
constexpr int VF_BATCH = 448;              // hypotheses per launch: their rows and tolerances fill 3.5 KB of the 4 KB parameter space
constexpr int VF_NC = 6;

struct VfBatch {
  int mrow[VF_BATCH];
  float tau[VF_BATCH];
};

struct VfCount {
  int sil = 0, occ = 0, fit = 0, viol = 0, mask = 0, mfit = 0;
};

// dr = rdepth * rscale, e = do - dr, both rounded to nearest (no FMA contraction)
__device__ __forceinline__ void vf_pixel(float rd, float dob, unsigned char m, float rscale, float tau, VfCount& c) {
  const float dr = __fmul_rn(rd, rscale);
  const float e = __fsub_rn(dob, dr);
  const bool sil = dr > 0.f;
  const bool seen = sil && dob > 0.f;
  const bool fit = seen && fabsf(e) <= tau;
  c.sil += sil;
  c.occ += seen && e < -tau;
  c.fit += fit;
  c.viol += seen && e > tau;
  c.mask += m != 0;
  c.mfit += (m != 0) && fit;
}

template <bool VEC>
__global__ void __launch_bounds__(VF_THREADS) vf_count_kernel(const float* __restrict__ rdepth, const float* __restrict__ depth,
                                                              const unsigned char* __restrict__ mask, long long hw, float rscale,
                                                              const __grid_constant__ VfBatch b, int* __restrict__ counts) {
  __shared__ int sh[VF_NC];
  if (threadIdx.x < VF_NC) sh[threadIdx.x] = 0;
  __syncthreads();
  const int q = blockIdx.y;
  const float* rd = rdepth + (long long)q * hw;
  const unsigned char* mk = mask + (long long)b.mrow[q] * hw;
  const float tau = b.tau[q];
  VfCount c;
  const long long i0 = (long long)blockIdx.x * VF_PIX;
  const long long i1 = min(hw, i0 + VF_PIX);
  if (VEC) {                                   // hw % 4 == 0 and aligned rows: i0, i1 and every row offset are multiples of 4
    for (long long i = i0 + 4 * threadIdx.x; i < i1; i += 4 * VF_THREADS) {
      const float4 r = __ldcs(reinterpret_cast<const float4*>(rd + i));        // read once: evict first
      const float4 d = __ldg(reinterpret_cast<const float4*>(depth + i));      // shared by every hypothesis
      const uchar4 m = __ldg(reinterpret_cast<const uchar4*>(mk + i));
      vf_pixel(r.x, d.x, m.x, rscale, tau, c);
      vf_pixel(r.y, d.y, m.y, rscale, tau, c);
      vf_pixel(r.z, d.z, m.z, rscale, tau, c);
      vf_pixel(r.w, d.w, m.w, rscale, tau, c);
    }
  } else {
    for (long long i = i0 + threadIdx.x; i < i1; i += VF_THREADS) vf_pixel(__ldcs(rd + i), __ldg(depth + i), __ldg(mk + i), rscale, tau, c);
  }
  const int v[VF_NC] = {c.sil, c.occ, c.fit, c.viol, c.mask, c.mfit};
#pragma unroll
  for (int k = 0; k < VF_NC; ++k) {
    const int s = __reduce_add_sync(0xffffffffu, v[k]);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(sh + k, s);
  }
  __syncthreads();
  if (threadIdx.x < VF_NC && sh[threadIdx.x]) atomicAdd(counts + (long long)q * VF_NC + threadIdx.x, sh[threadIdx.x]);
}

}  // namespace

S6_API int sam6d_pose_verify(const float* rdepth, const float* depth, const unsigned char* mask, const int* mrow, const float* tau,
                             int P, int M, int H, int W, float rscale, int* counts, void* stream) {
  S6_REQUIRE(P >= 0 && H >= 1 && W >= 1);
  if (P == 0) return 0;
  S6_REQUIRE(rdepth && depth && mask && mrow && tau && counts);
  S6_REQUIRE(M >= 1 && isfinite(rscale) && rscale > 0.f);
  for (int p = 0; p < P; ++p) S6_REQUIRE(mrow[p] >= 0 && mrow[p] < M && isfinite(tau[p]) && tau[p] > 0.f);
  cudaStream_t st = s6_stream(stream);
  const long long hw = (long long)H * W;
  const bool vec = hw % 4 == 0 && reinterpret_cast<uintptr_t>(rdepth) % 16 == 0 && reinterpret_cast<uintptr_t>(depth) % 16 == 0 &&
                   reinterpret_cast<uintptr_t>(mask) % 4 == 0;
  S6_CHECK(cudaMemsetAsync(counts, 0, (size_t)P * VF_NC * sizeof(int), st));
  VfBatch b{};
  for (int p0 = 0; p0 < P; p0 += VF_BATCH) {
    const int n = P - p0 < VF_BATCH ? P - p0 : VF_BATCH;
    for (int j = 0; j < n; ++j) {
      b.mrow[j] = mrow[p0 + j];
      b.tau[j] = tau[p0 + j];
    }
    const dim3 grid(s6_cdiv(hw, VF_PIX), n);
    if (vec)
      vf_count_kernel<true><<<grid, VF_THREADS, 0, st>>>(rdepth + p0 * hw, depth, mask, hw, rscale, b, counts + (long long)p0 * VF_NC);
    else
      vf_count_kernel<false><<<grid, VF_THREADS, 0, st>>>(rdepth + p0 * hw, depth, mask, hw, rscale, b, counts + (long long)p0 * VF_NC);
    S6_LAUNCH_CHECK();
  }
  return 0;
}
