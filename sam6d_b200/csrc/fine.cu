// fine.cu -- soft assignment on the dense (N+1)x(M+1) score matrix and the final weighted-SVD pose
// (compute_fine_Rt, PEM/utils/model_utils.py:250-283).
//
// A = F1 F2^T / temp with L2-normalised features, so |A| <= 1/temp and softmax can use the fixed shift
// `shift` = 1/temp instead of a per-row/column maximum: e_ij = exp(A_ij - shift),
//   P_ij = (e_ij / sum_j e_ij) * (e_ij / sum_i e_ij).
// Three streaming passes over A (row/col sums; column argmax of P; row argmax + masked weighted sums), then a per-proposal
// weighted Procrustes and the inlier score against the CAD samples.
#include "common.cuh"
#include "svd3.cuh"

namespace {

constexpr int RT = 32;  // rows per tile in the column-reducing passes

// All three passes stream A with 16-byte loads (row stride ld % 4 == 0, the padded layout compute_feature_similarity writes):
// a thread owns 4 adjacent columns, keeps its partial sums / maxima in registers and has up to 32 independent loads in
// flight; reciprocals of the row and column sums are stored once (rinv, cinv) so the later passes multiply.
__device__ __forceinline__ float4 exp4(const float4 v, float shift, int j, int S) {
  float4 e;
  e.x = (j + 0 < S) ? __expf(v.x - shift) : 0.f;   // padding columns hold arbitrary bits: select, never multiply
  e.y = (j + 1 < S) ? __expf(v.y - shift) : 0.f;
  e.z = (j + 2 < S) ? __expf(v.z - shift) : 0.f;
  e.w = (j + 3 < S) ? __expf(v.w - shift) : 0.f;
  return e;
}

// pass 1: rinv (B,ld) = 1 / row sums; column partial sums cpart (B,tiles,ld)
__global__ void __launch_bounds__(256) fine_sums_kernel(const float* __restrict__ A, int S, int ld, float shift, float* __restrict__ rinv,
                                                        float* __restrict__ cpart) {
  __shared__ float red[8][RT];
  const int tile = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int i0 = tile * RT, rmax = min(RT, S - i0);
  const float* Ab = A + (size_t)b * S * ld + (size_t)i0 * ld;
  float racc[RT];
#pragma unroll
  for (int r = 0; r < RT; ++r) racc[r] = 0.f;
  // S = 2049: the last 16-byte column group would be a third sweep with one active thread whose 32 serial loads the whole
  // block then waits for.  Such a short tail (<= 4 columns past a multiple of 1024) is handled row-parallel instead.
  const int tail = S & 1023, S_main = (tail != 0 && tail <= 4) ? S - tail : S;
  for (int j = tid * 4; j < S_main; j += 1024) {
    float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < RT; ++r) {
      if (r < rmax) {
        const float4 e = exp4(__ldcs(reinterpret_cast<const float4*>(Ab + (size_t)r * ld + j)), shift, j, S);
        c.x += e.x; c.y += e.y; c.z += e.z; c.w += e.w;
        racc[r] += (e.x + e.y) + (e.z + e.w);
      }
    }
    *reinterpret_cast<float4*>(cpart + ((size_t)b * gridDim.x + tile) * ld + j) = c;
  }
  float tail_row = 0.f;                                   // thread r < 32: row r of the tail columns
  if (S_main < S && warp == 0) {
    float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane < rmax) e = exp4(__ldcs(reinterpret_cast<const float4*>(Ab + (size_t)lane * ld + S_main)), shift, S_main, S);
    tail_row = (e.x + e.y) + (e.z + e.w);
    const float4 c = make_float4(warp_sum(e.x), warp_sum(e.y), warp_sum(e.z), warp_sum(e.w));
    if (lane == 0) *reinterpret_cast<float4*>(cpart + ((size_t)b * gridDim.x + tile) * ld + S_main) = c;
  }
#pragma unroll
  for (int r = 0; r < RT; ++r) {
    const float v = warp_sum(racc[r]);
    if (lane == 0) red[warp][r] = v;
  }
  __syncthreads();
  if (tid < rmax) {
    float s = tail_row;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][tid];
    rinv[(size_t)b * ld + i0 + tid] = 1.f / s;
  }
}

__global__ void colsum_reduce_kernel(const float* __restrict__ cpart, int tiles, int S, int ld, float* __restrict__ cinv) {
  const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ld) return;
  float s = 0.f;
  for (int t = 0; t < tiles; ++t) s += cpart[((size_t)b * tiles + t) * ld + j];
  cinv[(size_t)b * ld + j] = (j < S) ? 1.f / s : 0.f;
}

// pass 2: column labels lab2[b,j] = argmax_i P_ij (first max) as per-tile partials; the full product is evaluated like the
// reference does.
__global__ void __launch_bounds__(256) fine_collabels_kernel(const float* __restrict__ A, int S, int ld, float shift, const float* __restrict__ rinv,
                                                             const float* __restrict__ cinv, float* __restrict__ cpv,
                                                             int* __restrict__ cpi) {
  __shared__ float ri[RT];
  const int tile = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int i0 = tile * RT, rmax = min(RT, S - i0);
  if (tid < RT) ri[tid] = (tid < rmax) ? rinv[(size_t)b * ld + i0 + tid] : 0.f;
  __syncthreads();
  const float* Ab = A + (size_t)b * S * ld + (size_t)i0 * ld;
  const int tail = S & 1023, S_main = (tail != 0 && tail <= 4) ? S - tail : S;    // see fine_sums_kernel
  for (int j = tid * 4; j < S_main; j += 1024) {
    const float4 ci = *reinterpret_cast<const float4*>(cinv + (size_t)b * ld + j);
    float4 bv = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    int4 bi = make_int4(0, 0, 0, 0);
#pragma unroll
    for (int r = 0; r < RT; ++r) {
      if (r < rmax) {
        const float4 e = exp4(__ldcs(reinterpret_cast<const float4*>(Ab + (size_t)r * ld + j)), shift, j, S);
        const float rr = ri[r];
        const float p0 = (e.x * rr) * (e.x * ci.x), p1 = (e.y * rr) * (e.y * ci.y), p2 = (e.z * rr) * (e.z * ci.z), p3 = (e.w * rr) * (e.w * ci.w);
        if (p0 > bv.x) { bv.x = p0; bi.x = i0 + r; }              // ascending i: first max wins
        if (p1 > bv.y) { bv.y = p1; bi.y = i0 + r; }
        if (p2 > bv.z) { bv.z = p2; bi.z = i0 + r; }
        if (p3 > bv.w) { bv.w = p3; bi.w = i0 + r; }
      }
    }
    *reinterpret_cast<float4*>(cpv + ((size_t)b * gridDim.x + tile) * ld + j) = bv;
    *reinterpret_cast<int4*>(cpi + ((size_t)b * gridDim.x + tile) * ld + j) = bi;
  }
  if (S_main < S && tid < 32) {                            // tail columns: lane = row, warp argmax (smallest row on ties)
    const int lane = tid;
    const float4 ci = *reinterpret_cast<const float4*>(cinv + (size_t)b * ld + S_main);
    float pv[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    if (lane < rmax) {
      const float4 e = exp4(__ldcs(reinterpret_cast<const float4*>(Ab + (size_t)lane * ld + S_main)), shift, S_main, S);
      const float rr = ri[lane];
      pv[0] = (e.x * rr) * (e.x * ci.x); pv[1] = (e.y * rr) * (e.y * ci.y); pv[2] = (e.z * rr) * (e.z * ci.z); pv[3] = (e.w * rr) * (e.w * ci.w);
    }
    float ov[4]; int oi[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float v = pv[k]; int i = (lane < rmax) ? i0 + lane : 0x7fffffff;
      warp_argmax_first(v, i);
      ov[k] = v; oi[k] = (i == 0x7fffffff) ? 0 : i;
    }
    if (lane == 0) {
      *reinterpret_cast<float4*>(cpv + ((size_t)b * gridDim.x + tile) * ld + S_main) = make_float4(ov[0], ov[1], ov[2], ov[3]);
      *reinterpret_cast<int4*>(cpi + ((size_t)b * gridDim.x + tile) * ld + S_main) = make_int4(oi[0], oi[1], oi[2], oi[3]);
    }
  }
}

__global__ void collab_reduce_kernel(const float* __restrict__ cpv, const int* __restrict__ cpi, int tiles, int S, int ld,
                                     int* __restrict__ lab2) {
  const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= S) return;
  float bv = -INFINITY; int bi = 0;
  for (int t = 0; t < tiles; ++t) {
    float v = cpv[((size_t)b * tiles + t) * ld + j];
    if (v > bv) { bv = v; bi = cpi[((size_t)b * tiles + t) * ld + j]; }
  }
  lab2[(size_t)b * S + j] = bi;
}

// the masked template points of pass 3: q4[b,j] = (pts2[b,j-1], 1) if column j >= 1 is matched to a non-background row
// (lab2 > 0), else 0.  Written over the (now consumed) partials.
__global__ void masked_points_kernel(const int* __restrict__ lab2, const float* __restrict__ pts2, int S, int ld,
                                     float4* __restrict__ q4) {
  const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ld) return;
  float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
  if (j >= 1 && j < S && lab2[(size_t)b * S + j] > 0) {
    const float* p = pts2 + ((size_t)b * (S - 1) + (j - 1)) * 3;
    q = make_float4(p[0], p[1], p[2], 1.f);
  }
  q4[(size_t)b * ld + j] = q;
}

// pass 3, one warp per row i >= 1: lab1_i = argmax_j P_ij (first max); if it is not the background column,
//   w_i = sum_{j>=1, lab2_j>0} P_ij,  pred_i = sum_j P_ij pts2_j / (w_i + 1e-6)      (second sweep hits L1/L2)
__global__ void __launch_bounds__(256) fine_weighted_kernel(const float* __restrict__ A, int S, int ld, float shift, const float* __restrict__ rinv,
                                                            const float* __restrict__ cinv, int* __restrict__ lab1,
                                                            const float4* __restrict__ q4, float* __restrict__ wts, float* __restrict__ pred) {
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);   // dense index 0..N-1
  const int N = S - 1;
  if (i >= N) return;
  const float* row = A + ((size_t)b * S + i + 1) * ld;
  const float ri = rinv[(size_t)b * ld + i + 1];
  const float* ci = cinv + (size_t)b * ld;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
#pragma unroll 4
  for (int j = lane * 4; j < S; j += 128) {
    const float4 e = exp4(*reinterpret_cast<const float4*>(row + j), shift, j, S);
    const float4 c = *reinterpret_cast<const float4*>(ci + j);
    const float p0 = (e.x * ri) * (e.x * c.x), p1 = (e.y * ri) * (e.y * c.y), p2 = (e.z * ri) * (e.z * c.z), p3 = (e.w * ri) * (e.w * c.w);
    if (p0 > bv) { bv = p0; bi = j; }                       // padding columns give p = 0 (cinv = 0, e = 0): never a strict max
    if (p1 > bv) { bv = p1; bi = j + 1; }
    if (p2 > bv) { bv = p2; bi = j + 2; }
    if (p3 > bv) { bv = p3; bi = j + 3; }
  }
  warp_argmax_first(bv, bi);
  if (lane == 0) lab1[(size_t)b * S + i + 1] = bi;
  float w = 0.f, px = 0.f, py = 0.f, pz = 0.f;
  if (bi > 0) {
    const float4* qb = q4 + (size_t)b * ld;
#pragma unroll 2
    for (int j = lane * 4; j < S; j += 128) {
      const float4 e = exp4(*reinterpret_cast<const float4*>(row + j), shift, j, S);
      const float4 c = *reinterpret_cast<const float4*>(ci + j);
      const float pk[4] = {(e.x * ri) * (e.x * c.x), (e.y * ri) * (e.y * c.y), (e.z * ri) * (e.z * c.z), (e.w * ri) * (e.w * c.w)};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float4 q = qb[j + k];
        const float p = pk[k] * q.w;
        w += p; px = fmaf(p, q.x, px); py = fmaf(p, q.y, py); pz = fmaf(p, q.z, pz);
      }
    }
    w = warp_sum(w); px = warp_sum(px); py = warp_sum(py); pz = warp_sum(pz);
  }
  if (lane == 0) {
    wts[(size_t)b * N + i] = w;
    float d = w + 1e-6f;
    float* o = pred + ((size_t)b * N + i) * 3;
    o[0] = px / d; o[1] = py / d; o[2] = pz / d;
  }
}

// weighted Procrustes (model_utils.py:287-363, weight_thresh 0, eps 1e-5): ref ~= R src + t
__device__ __forceinline__ double block_sum_d(double v, double* sh) {
  v = warp_sum_d(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += sh[w];
  return s;
}

__global__ void __launch_bounds__(256) weighted_procrustes_kernel(const float* __restrict__ src, const float* __restrict__ ref,
                                                                  const float* __restrict__ wts, int N, float thresh, float eps,
                                                                  float* __restrict__ R, float* __restrict__ t) {
  __shared__ double sh[8];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* s = src + (size_t)b * N * 3;
  const float* r = ref + (size_t)b * N * 3;
  const float* w = wts + (size_t)b * N;
  double ws = 0.0;
  for (int i = tid; i < N; i += 256) { float wi = w[i]; ws += (wi < thresh) ? 0.0 : (double)wi; }
  const float wsum = (float)block_sum_d(ws, sh) + eps;
  double c[6] = {0, 0, 0, 0, 0, 0};
  for (int i = tid; i < N; i += 256) {
    float wi = w[i];
    wi = (wi < thresh) ? 0.f : wi;
    float wn = wi / wsum;
    for (int d = 0; d < 3; ++d) { c[d] += (double)(s[i * 3 + d] * wn); c[3 + d] += (double)(r[i * 3 + d] * wn); }
  }
  float cen[6];
  for (int d = 0; d < 6; ++d) cen[d] = (float)block_sum_d(c[d], sh);
  double h[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = tid; i < N; i += 256) {
    float wi = w[i];
    wi = (wi < thresh) ? 0.f : wi;
    float wn = wi / wsum;
    float sc[3] = {s[i * 3] - cen[0], s[i * 3 + 1] - cen[1], s[i * 3 + 2] - cen[2]};
    float rc[3] = {wn * (r[i * 3] - cen[3]), wn * (r[i * 3 + 1] - cen[4]), wn * (r[i * 3 + 2] - cen[5])};
    for (int a = 0; a < 3; ++a)
      for (int d = 0; d < 3; ++d) h[a * 3 + d] += (double)sc[a] * (double)rc[d];
  }
  double H[3][3];
  for (int a = 0; a < 9; ++a) H[a / 3][a % 3] = block_sum_d(h[a], sh);
  if (tid == 0) {
    double Rd[3][3];
    procrustes_rotation(H, Rd);
    for (int a = 0; a < 3; ++a) {
      float Ra[3] = {(float)Rd[a][0], (float)Rd[a][1], (float)Rd[a][2]};
      for (int d = 0; d < 3; ++d) R[(size_t)b * 9 + a * 3 + d] = Ra[d];
      t[(size_t)b * 3 + a] = cen[3 + a] - (Ra[0] * cen[0] + Ra[1] * cen[1] + Ra[2] * cen[2]);
    }
  }
}

// pose score (model_utils.py:275-281) and rescaled translation (fine_point_matching.py:80).
// One thread-block CLUSTER of PS_CS CTAs per proposal (one CTA per proposal leaves 100 of the 132 SMs idle at 32 proposals for the longest
// kernel of the tail): each CTA scores a slice of the points against the CAD samples in its shared memory and publishes its
// two counts (hits, valid points -- integers, so any summation order gives the same result) into CTA 0's distributed
// shared memory; one cluster barrier later CTA 0 writes the score.
constexpr int PS_CS = 8, PS_THREADS = 256;
__device__ __forceinline__ unsigned ps_cluster_ctarank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__global__ void __launch_bounds__(PS_THREADS) pose_score_kernel(const float* __restrict__ pts1, const int* __restrict__ lab1, int S,
                                                                const float* __restrict__ R, const float* __restrict__ t,
                                                                const float* __restrict__ model, int nm, float dis_thres,
                                                                const float* __restrict__ radius, float* __restrict__ score,
                                                                float* __restrict__ t_scaled) {
  extern __shared__ float4 smq4[];          // (x, y, z, |m|^2) per CAD sample
  __shared__ int sh[2][PS_THREADS / 32];
  __shared__ int slot[PS_CS][2];            // CTA 0's copy is written by every CTA of the cluster
  const unsigned rank = ps_cluster_ctarank();
  const int b = blockIdx.x / PS_CS, tid = threadIdx.x, N = S - 1;
  for (int i = tid; i < nm; i += PS_THREADS) {
    const float* q = model + ((size_t)b * nm + i) * 3;
    const float x = q[0], y = q[1], z = q[2];
    smq4[i] = make_float4(x, y, z, x * x + y * y + z * z);
  }
  float Rb[9], tb[3];
  for (int a = 0; a < 9; ++a) Rb[a] = R[(size_t)b * 9 + a];
  for (int a = 0; a < 3; ++a) tb[a] = t[(size_t)b * 3 + a];
  __syncthreads();
  int hits = 0, msum = 0;
  for (int i = rank * PS_THREADS + tid; i < N; i += PS_CS * PS_THREADS) {
    const float* p = pts1 + ((size_t)b * N + i) * 3;
    float x = p[0] - tb[0], y = p[1] - tb[1], z = p[2] - tb[2];
    float tx = x * Rb[0] + y * Rb[3] + z * Rb[6];
    float ty = x * Rb[1] + y * Rb[4] + z * Rb[7];
    float tz = x * Rb[2] + y * Rb[5] + z * Rb[8];
    float x2 = tx * tx + ty * ty + tz * tz;
    float best = INFINITY;
#pragma unroll 4
    for (int m = 0; m < nm; ++m) {
      const float4 q = smq4[m];
      float xy = tx * q.x + ty * q.y + tz * q.z;
      best = fminf(best, fmaxf(x2 - 2.f * xy + q.w, 0.f));
    }
    const int mk = lab1[(size_t)b * S + i + 1] > 0 ? 1 : 0;
    if (sqrtf(best) < dis_thres) hits += mk;
    msum += mk;
  }
  hits = __reduce_add_sync(0xffffffffu, hits);
  msum = __reduce_add_sync(0xffffffffu, msum);
  if ((tid & 31) == 0) { sh[0][tid >> 5] = hits; sh[1][tid >> 5] = msum; }
  __syncthreads();
  if (tid < 2) {
    int v = 0;
    for (int w = 0; w < PS_THREADS / 32; ++w) v += sh[tid][w];
    unsigned la = (unsigned)__cvta_generic_to_shared(&slot[rank][tid]), ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(0u));
    asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(ra), "r"(v) : "memory");
  }
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
  if (rank == 0 && tid == 0) {
    int hsum = 0, ms_i = 0;
    for (int c = 0; c < PS_CS; ++c) { hsum += slot[c][0]; ms_i += slot[c][1]; }
    const float h = (float)hsum, ms = (float)ms_i;
    score[b] = (h / (ms + 1e-8f)) * (ms / (float)N);
    float rad = radius[b] + 1e-6f;
    for (int a = 0; a < 3; ++a) t_scaled[(size_t)b * 3 + a] = tb[a] * rad;
  }
}

}  // namespace

// A (B,S,S) f32 score matrix with row stride ld >= S, ld % 4 == 0, 16-byte aligned (row/col 0 = background), pts2 (B,S-1,3).
// Outputs: lab1 (B,S) i32 (row argmax of P; entry 0 unused), lab2 (B,S) i32, wts (B,S-1), pred (B,S-1,3).
// Scratch: rsum (B,ld), csum (B,ld) [hold the reciprocal sums], cpart (B,tiles,ld) f32, cpi (B,tiles,ld) i32, tiles = ceil(S/32).
S6_API int sam6d_fine_assign(const float* A, int B, int S, int ld, float shift, const float* pts2, float* rsum, float* csum,
                             float* cpart, int* cpi, int* lab1, int* lab2, float* wts, float* pred, void* stream) {
  S6_REQUIRE(A && pts2 && rsum && csum && cpart && cpi && lab1 && lab2 && wts && pred && B >= 0 && S >= 2 && ld >= S);
  S6_REQUIRE((ld % 4) == 0 && ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(rsum) | reinterpret_cast<uintptr_t>(csum) |
                               reinterpret_cast<uintptr_t>(cpart) | reinterpret_cast<uintptr_t>(cpi)) & 15) == 0);
  if (B == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  const int tiles = s6_cdiv(S, RT);
  S6_REQUIRE(tiles >= 4);                                  // the masked points (B,ld) float4 live in cpart after pass 2
  dim3 gt(tiles, B), gc(s6_cdiv(ld, 256), B);
  fine_sums_kernel<<<gt, 256, 0, st>>>(A, S, ld, shift, rsum, cpart);
  S6_LAUNCH_CHECK();
  colsum_reduce_kernel<<<gc, 256, 0, st>>>(cpart, tiles, S, ld, csum);
  S6_LAUNCH_CHECK();
  fine_collabels_kernel<<<gt, 256, 0, st>>>(A, S, ld, shift, rsum, csum, cpart, cpi);
  S6_LAUNCH_CHECK();
  collab_reduce_kernel<<<gc, 256, 0, st>>>(cpart, cpi, tiles, S, ld, lab2);
  S6_LAUNCH_CHECK();
  float4* q4 = reinterpret_cast<float4*>(cpart);
  masked_points_kernel<<<gc, 256, 0, st>>>(lab2, pts2, S, ld, q4);
  S6_LAUNCH_CHECK();
  dim3 gw(s6_cdiv(S - 1, 8), B);
  fine_weighted_kernel<<<gw, 256, 0, st>>>(A, S, ld, shift, rsum, csum, lab1, q4, wts, pred);
  S6_LAUNCH_CHECK();
  return 0;
}

// src, ref (B,N,3), wts (B,N) -> R (B,3,3), t (B,3) with ref ~= R src + t
S6_API int sam6d_weighted_procrustes(const float* src, const float* ref, const float* wts, int B, int N, float weight_thresh,
                                     float eps, float* R, float* t, void* stream) {
  S6_REQUIRE(src && ref && wts && R && t && B >= 0 && N > 0);
  if (B == 0) return 0;
  weighted_procrustes_kernel<<<B, 256, 0, s6_stream(stream)>>>(src, ref, wts, N, weight_thresh, eps, R, t);
  S6_LAUNCH_CHECK();
  return 0;
}

// pts1 (B,N,3), lab1 (B,N+1) from sam6d_fine_assign, R,t, model (B,nm,3), radius (B) -> score (B), t_scaled (B,3)
S6_API int sam6d_pose_score(const float* pts1, const int* lab1, int B, int N, const float* R, const float* t, const float* model,
                            int nm, float dis_thres, const float* radius, float* score, float* t_scaled, void* stream) {
  S6_REQUIRE(pts1 && lab1 && R && t && model && radius && score && t_scaled && B >= 0 && N > 0 && nm > 0);
  if (B == 0) return 0;
  size_t smem = (size_t)nm * 4 * sizeof(float);
  S6_REQUIRE(smem <= 200 * 1024);
  S6_CHECK(cudaFuncSetAttribute(pose_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(B * PS_CS); cfg.blockDim = dim3(PS_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s6_stream(stream);
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = PS_CS; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  S6_CHECK(cudaLaunchKernelEx(&cfg, pose_score_kernel, pts1, (const int*)lab1, N + 1, R, t, model, nm, dis_thres, radius, score, t_scaled));
  return 0;
}
