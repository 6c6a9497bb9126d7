// icp.cu -- batched point-to-plane ICP refinement of PEM poses against the observed points (not in the reference; the
// algorithm is stated in include/sam6d_b200.h at sam6d_icp_refine and restated in float64 by oracle/icp_oracle.py).
//
// One thread-block cluster of ICP_CS CTAs per instance.  Each CTA stages the instance's object samples and normals in shared
// memory (float4 each) and owns a contiguous slice of the observed points.  Per iteration every thread transforms its points
// with the fp32-rounded pose, scans all M samples (broadcast shared-memory reads; strict '<' keeps the lowest index on an
// exact tie), and accumulates the 29 fp64 sums of the normal equations over its inliers in point order.  The sums are reduced
// in a fixed order (xor butterfly within a warp, warps in order, CTAs in rank order through distributed shared memory into
// rank 0), so the result is bit-reproducible.  One thread of rank 0 solves the damped 6 x 6 system by Cholesky and updates
// the fp64 pose; after a cluster barrier every CTA reads the new pose from rank 0's shared memory.  All K iterations run in
// one launch with no global-memory scratch.
#include "common.cuh"

namespace {

constexpr int ICP_CS = 4;                 // CTAs per instance: B = 32 fills 128 of the H100's 132 SMs
constexpr int ICP_THREADS = 256;
constexpr int ICP_PPT = 2;                // points per thread per pass: each broadcast sample load serves two distance evaluations
constexpr int ICP_NW = ICP_THREADS / 32;
constexpr int ICP_NS = 29;                // A (21 upper-triangle terms), b (6), inlier count, sum of e^2
constexpr int ICP_MIN_INLIERS = 32;
constexpr double ICP_STEP_TOL = 1e-7;
constexpr double ICP_DAMPING = 1e-4;

// inlier radius of iteration k as a fraction of the object radius.  The PEM's pose is typically within a few percent of the
// object radius, so 0.3 r at k = 0 keeps the true correspondences while cutting background points far off the surface; the
// radius halves each iteration as the pose converges and stops at 0.05 r, which still admits depth noise and the spacing of
// the M samples.  Not tuned on BOP data.
__device__ __forceinline__ double icp_tau_fraction(int k) { return fmax(0.3 * ldexp(1.0, -k), 0.05); }

__device__ __forceinline__ unsigned cluster_rank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned dsmem_addr(const void* local_smem, unsigned cta) {
  unsigned la = (unsigned)__cvta_generic_to_shared(local_smem), ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(cta));
  return ra;
}
__device__ __forceinline__ void st_dsmem_f64(unsigned addr, double v) {
  asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(addr), "d"(v) : "memory");
}
__device__ __forceinline__ double ld_dsmem_f64(unsigned addr) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(addr) : "memory");
  return v;
}

// R <- R Exp(w) (Rodrigues) with R row-major
__device__ void icp_right_update(double* R, const double* w) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  double a, b;                            // Exp(w) = I + a [w]x + b [w]x^2
  if (th < 1e-4) { a = 1.0 - th2 / 6.0 + th2 * th2 / 120.0; b = 0.5 - th2 / 24.0 + th2 * th2 / 720.0; }
  else { a = sin(th) / th; b = (1.0 - cos(th)) / th2; }
  const double K[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
  double E[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double k2 = K[r * 3 + 0] * K[0 * 3 + c] + K[r * 3 + 1] * K[1 * 3 + c] + K[r * 3 + 2] * K[2 * 3 + c];
      E[r * 3 + c] = (r == c ? 1.0 : 0.0) + a * K[r * 3 + c] + b * k2;
    }
  double out[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) out[r * 3 + c] = R[r * 3 + 0] * E[0 * 3 + c] + R[r * 3 + 1] * E[1 * 3 + c] + R[r * 3 + 2] * E[2 * 3 + c];
  for (int i = 0; i < 9; ++i) R[i] = out[i];
}

// (A + lambda I) x = b, A symmetric positive semi-definite from its 21 upper-triangle terms (row-major); false if not positive
__device__ bool icp_solve6(const double* s, double* x) {
  double L[6][6];
  int q = 0;
  double tr = 0.0;
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) { L[r][c] = L[c][r] = s[q++]; }
  for (int r = 0; r < 6; ++r) tr += L[r][r];
  const double lam = ICP_DAMPING * tr / 6.0;
  for (int r = 0; r < 6; ++r) L[r][r] += lam;
  for (int j = 0; j < 6; ++j) {
    double d = L[j][j];
    for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
    if (!(d > 0.0)) return false;
    d = sqrt(d);
    L[j][j] = d;
    for (int i = j + 1; i < 6; ++i) {
      double v = L[i][j];
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      L[i][j] = v / d;
    }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double v = s[21 + i];
    for (int k = 0; k < i; ++k) v -= L[i][k] * y[k];
    y[i] = v / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double v = y[i];
    for (int k = i + 1; k < 6; ++k) v -= L[k][i] * x[k];
    x[i] = v / L[i][i];
  }
  return true;
}

// pose block in rank 0's shared memory: R (9) and t (3) fp64, then the stop flag
constexpr int ICP_POSE = 13;

__global__ void __cluster_dims__(ICP_CS, 1, 1) __launch_bounds__(ICP_THREADS, 1)
icp_refine_kernel(const float* __restrict__ R_in, const float* __restrict__ t_in, const float* __restrict__ pts, int N,
                  const float* __restrict__ samples, const float* __restrict__ normals, int O, int M, const int* __restrict__ obj,
                  const float* __restrict__ radius, int iters, float* __restrict__ R_out, float* __restrict__ t_out,
                  int* __restrict__ inliers_out, float* __restrict__ rms_out, int* __restrict__ iters_out, int* __restrict__ corr,
                  double* __restrict__ sums) {
  extern __shared__ float4 sm4[];
  __shared__ double warp_part[ICP_NW][ICP_NS];
  __shared__ double cta_part[ICP_CS][ICP_NS];       // rank 0's: written by every CTA of the cluster through DSMEM
  __shared__ double pose[ICP_POSE];                 // rank 0's is the instance's pose; the others hold a copy
  __shared__ float posef[12];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned rank = cluster_rank();
  const int b = blockIdx.x / ICP_CS;
  const int o = obj[b];
  const float r_f = radius[b];
  const bool valid = o >= 0 && o < O && r_f > 0.f && isfinite(r_f);
  float4* sq = sm4;
  float4* sn = sm4 + M;

  if (valid) {
    const float* qs = samples + (size_t)o * M * 3;
    const float* ns = normals + (size_t)o * M * 3;
    for (int j = tid; j < M; j += ICP_THREADS) {
      sq[j] = make_float4(qs[j * 3], qs[j * 3 + 1], qs[j * 3 + 2], 0.f);
      sn[j] = make_float4(ns[j * 3], ns[j * 3 + 1], ns[j * 3 + 2], 0.f);
    }
  }
  if (rank == 0 && tid < 12) pose[tid] = tid < 9 ? (double)R_in[(size_t)b * 9 + tid] : (double)t_in[(size_t)b * 3 + tid - 9];
  if (rank == 0 && tid == 12) pose[12] = valid && iters > 0 ? 0.0 : 1.0;
  const int chunk = (N + ICP_CS - 1) / ICP_CS;
  const int p0 = (int)rank * chunk, cnt = max(0, min(chunk, N - p0));
  const float* P = pts + ((size_t)b * N + p0) * 3;
  const double r = (double)r_f, inv_r = 1.0 / r;
  const unsigned pose0 = dsmem_addr(pose, 0u);
  const unsigned part0 = dsmem_addr(&cta_part[rank][0], 0u);
  int last_inl = 0, done_iters = 0;
  double last_rms = 0.0;
  __syncthreads();
  cluster_sync();                                   // every CTA's shared memory exists and rank 0's pose is set

  for (int k = 0; k < iters; ++k) {
    if (tid < ICP_POSE) pose[tid] = ld_dsmem_f64(pose0 + tid * 8u);
    __syncthreads();
    if (pose[12] != 0.0) break;                     // uniform across the cluster: every CTA read the same flag
    if (tid < 12) posef[tid] = (float)pose[tid];
    __syncthreads();
    const float R00 = posef[0], R01 = posef[1], R02 = posef[2], R10 = posef[3], R11 = posef[4], R12 = posef[5];
    const float R20 = posef[6], R21 = posef[7], R22 = posef[8], tx = posef[9], ty = posef[10], tz = posef[11];
    const double tau = r * icp_tau_fraction(k);
    const float tau2 = (float)(tau * tau);

    double acc[ICP_NS];
#pragma unroll
    for (int s = 0; s < ICP_NS; ++s) acc[s] = 0.0;
    for (int i0 = tid; i0 < cnt; i0 += ICP_THREADS * ICP_PPT) {
      float yx[ICP_PPT], yy[ICP_PPT], yz[ICP_PPT], best[ICP_PPT];
      int bj[ICP_PPT];
#pragma unroll
      for (int u = 0; u < ICP_PPT; ++u) {
        const int i = min(i0 + u * ICP_THREADS, cnt - 1);
        const float dx = P[i * 3] - tx, dy = P[i * 3 + 1] - ty, dz = P[i * 3 + 2] - tz;
        yx[u] = R00 * dx + R10 * dy + R20 * dz;    // y = R^T (p - t)
        yy[u] = R01 * dx + R11 * dy + R21 * dz;
        yz[u] = R02 * dx + R12 * dy + R22 * dz;
        best[u] = INFINITY;
        bj[u] = 0;
      }
#pragma unroll 4
      for (int j = 0; j < M; ++j) {
        const float4 q = sq[j];
#pragma unroll
        for (int u = 0; u < ICP_PPT; ++u) {
          const float ex = yx[u] - q.x, ey = yy[u] - q.y, ez = yz[u] - q.z;
          const float d = ex * ex + ey * ey + ez * ez;
          if (d < best[u]) { best[u] = d; bj[u] = j; }
        }
      }
#pragma unroll
      for (int u = 0; u < ICP_PPT; ++u) {
        if (corr != nullptr && i0 + u * ICP_THREADS < cnt)
          corr[(size_t)b * N + p0 + i0 + u * ICP_THREADS] = best[u] < tau2 ? bj[u] : -1 - bj[u];
        if (i0 + u * ICP_THREADS < cnt && best[u] < tau2) {
          const float4 q = sq[bj[u]], n = sn[bj[u]];
          const double y0 = yx[u] * inv_r, y1 = yy[u] * inv_r, y2 = yz[u] * inv_r;
          const double n0 = n.x, n1 = n.y, n2 = n.z;
          const double e = n0 * (y0 - q.x * inv_r) + n1 * (y1 - q.y * inv_r) + n2 * (y2 - q.z * inv_r);
          const double J[6] = {y1 * n2 - y2 * n1, y2 * n0 - y0 * n2, y0 * n1 - y1 * n0, n0, n1, n2};
          int s = 0;
#pragma unroll
          for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int c = a; c < 6; ++c) acc[s++] += J[a] * J[c];
#pragma unroll
          for (int a = 0; a < 6; ++a) acc[21 + a] += J[a] * e;
          acc[27] += 1.0;
          acc[28] += e * e;
        }
      }
    }
#pragma unroll
    for (int s = 0; s < ICP_NS; ++s) {
      const double v = warp_sum_d(acc[s]);
      if (lane == 0) warp_part[warp][s] = v;
    }
    __syncthreads();
    if (tid < ICP_NS) {
      double v = warp_part[0][tid];
#pragma unroll
      for (int w = 1; w < ICP_NW; ++w) v += warp_part[w][tid];
      st_dsmem_f64(part0 + tid * 8u, v);
    }
    cluster_sync();                                 // rank 0 holds every CTA's sums
    if (rank == 0 && tid == 0) {
      double s[ICP_NS];
      for (int q = 0; q < ICP_NS; ++q) {
        double v = cta_part[0][q];
        for (int c = 1; c < ICP_CS; ++c) v += cta_part[c][q];
        s[q] = v;
      }
      if (sums != nullptr)
        for (int q = 0; q < ICP_NS; ++q) sums[(size_t)b * ICP_NS + q] = s[q];
      last_inl = (int)s[27];
      last_rms = last_inl > 0 ? r * sqrt(s[28] / s[27]) : 0.0;
      double x[6];
      if (last_inl < ICP_MIN_INLIERS || !icp_solve6(s, x)) {
        pose[12] = 1.0;                             // the pose stays as it was before this iteration
      } else {
        const double v0 = r * x[3], v1 = r * x[4], v2 = r * x[5];
        const double t0 = pose[0] * v0 + pose[1] * v1 + pose[2] * v2;
        const double t1 = pose[3] * v0 + pose[4] * v1 + pose[5] * v2;
        const double t2 = pose[6] * v0 + pose[7] * v1 + pose[8] * v2;
        pose[9] += t0; pose[10] += t1; pose[11] += t2;
        icp_right_update(pose, x);
        ++done_iters;
        const double wn = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]), vn = sqrt(x[3] * x[3] + x[4] * x[4] + x[5] * x[5]);
        if (wn < ICP_STEP_TOL && vn < ICP_STEP_TOL) pose[12] = 1.0;
      }
    }
    cluster_sync();                                 // the new pose is visible to every CTA
  }
  if (rank == 0 && tid == 0) {
    for (int i = 0; i < 9; ++i) R_out[(size_t)b * 9 + i] = (float)pose[i];
    for (int i = 0; i < 3; ++i) t_out[(size_t)b * 3 + i] = (float)pose[9 + i];
    inliers_out[b] = valid ? last_inl : -1;
    rms_out[b] = (float)last_rms;
    iters_out[b] = done_iters;
  }
  cluster_sync();                                   // no CTA exits while a peer may still read its shared memory
}

int icp_smem_optin(int* optin) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return (int)e;
}

int icp_max_samples(int* m_max) {
  int optin = 0;
  int e = icp_smem_optin(&optin);
  if (e) return e;
  cudaFuncAttributes fa;
  cudaError_t ce = cudaFuncGetAttributes(&fa, icp_refine_kernel);
  if (ce != cudaSuccess) return (int)ce;
  *m_max = (int)((optin - (long long)fa.sharedSizeBytes) / (2 * (long long)sizeof(float4)));
  return 0;
}

}  // namespace

S6_API int sam6d_icp_max_samples(void) {
  int m = 0;
  int e = icp_max_samples(&m);
  return e ? -e : m;
}

S6_API int sam6d_icp_refine(const float* R, const float* t, const float* pts, int B, int N, const float* samples,
                            const float* normals, int O, int M, const int* obj, const float* radius, int iters, float* R_out,
                            float* t_out, int* inliers, float* rms, int* iters_run, int* corr, double* sums, void* stream) {
  S6_REQUIRE(B >= 0 && N >= 1 && O >= 1 && M >= 1 && iters >= 0);
  if (B == 0) return 0;
  S6_REQUIRE(R && t && pts && samples && normals && obj && radius && R_out && t_out && inliers && rms && iters_run);
  S6_REQUIRE((long long)B * ICP_CS <= 0x7fffffffLL);
  int m_max = 0;
  S6_CHECK((cudaError_t)icp_max_samples(&m_max));
  S6_REQUIRE(M <= m_max);
  const size_t smem = (size_t)M * 2 * sizeof(float4);
  S6_CHECK(cudaFuncSetAttribute(icp_refine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  icp_refine_kernel<<<B * ICP_CS, ICP_THREADS, smem, s6_stream(stream)>>>(R, t, pts, N, samples, normals, O, M, obj, radius, iters,
                                                                           R_out, t_out, inliers, rms, iters_run, corr, sums);
  S6_LAUNCH_CHECK();
  return 0;
}
