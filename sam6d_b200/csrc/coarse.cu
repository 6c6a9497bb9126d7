// coarse.cu -- soft assignment and the hypothesis-and-verify pose initialisation of the coarse stage
// (compute_coarse_Rt, PEM/utils/model_utils.py:187-246).
//
// Pipeline per proposal b (N1 = N2 = n sparse points, the score matrix is (n+1) x (n+1) with row/col 0 = background):
//   1. coarse_assign  : P = softmax_row(A) * softmax_col(A); labels; masked inner block ^1.5      -> W (b, n*n), w1 (b,n)
//   2. coarse_sample  : cdf = cumsum(W) / (sum + 1e-8) (double accumulation like the CPU reference);
//                       idx = searchsorted(cdf, rand)                                              -> (b, 3*n1) pairs
//   3. coarse_hypotheses : 3-point Procrustes per hypothesis + mean residual                      -> Rt (b,n1,12), resid
//   4. coarse_topk    : the n2 smallest residuals (value, then index)                              -> top (b,n2)
//   5. coarse_select  : score = sum(w1) / (sum_i w1_i min_m ||(p_i - t) R - model_m|| + 1e-8); argmax -> init_R, init_t
//   6. coarse_pick_distinct (opt-in, not in the reference): K mutually distinct hypotheses of the n2 scored ones
//   7. coarse_pick_distinct_sym (opt-in, not in the reference): the same, distinct up to the object's symmetries
#include "common.cuh"
#include "svd3.cuh"

namespace {

// ---- 1. soft assignment -------------------------------------------------------------------------------------
// 1024 threads: one CTA per proposal, so the block is the only parallelism there is (every reduction keeps its order: rows are
// reduced by one warp each, columns by one thread each, whatever the block size)
constexpr int ASSIGN_THREADS = 1024;
__global__ void __launch_bounds__(ASSIGN_THREADS) coarse_assign_kernel(const float* __restrict__ A, int S, float* __restrict__ W,
                                                            float* __restrict__ w1out) {
  extern __shared__ float sm[];
  float* a = sm;                 // S*S
  float* rmax = a + S * S;       // S
  float* rsum = rmax + S;
  float* cmax = rsum + S;
  float* csum = cmax + S;
  int* lab1 = (int*)(csum + S);  // S (row labels, index i in 1..S-1)
  int* lab2 = lab1 + S;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* Ab = A + (size_t)b * S * S;
  for (int e = tid; e < S * S; e += ASSIGN_THREADS) a[e] = Ab[e];
  __syncthreads();
  // row stats (warp per row) and column stats (thread per column)
  for (int i = warp; i < S; i += ASSIGN_THREADS / 32) {
    float m = -INFINITY;
    for (int j = lane; j < S; j += 32) m = fmaxf(m, a[i * S + j]);
    m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < S; j += 32) s += expf(a[i * S + j] - m);
    s = warp_sum(s);
    if (lane == 0) { rmax[i] = m; rsum[i] = s; }
  }
  for (int j = tid; j < S; j += ASSIGN_THREADS) {
    float m = -INFINITY;
    for (int i = 0; i < S; ++i) m = fmaxf(m, a[i * S + j]);
    float s = 0.f;
    for (int i = 0; i < S; ++i) s += expf(a[i * S + j] - m);
    cmax[j] = m; csum[j] = s;
  }
  __syncthreads();
  // P in place
  for (int e = tid; e < S * S; e += ASSIGN_THREADS) {
    int i = e / S, j = e - i * S;
    float v = a[e];
    a[e] = (expf(v - rmax[i]) / rsum[i]) * (expf(v - cmax[j]) / csum[j]);
  }
  __syncthreads();
  // labels: first maximal index (torch.max)
  for (int i = warp; i < S; i += ASSIGN_THREADS / 32) {
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int j = lane; j < S; j += 32) argmax_first(bv, bi, a[i * S + j], j);
    warp_argmax_first(bv, bi);
    if (lane == 0) lab1[i] = bi;
  }
  for (int j = tid; j < S; j += ASSIGN_THREADS) {
    float bv = -INFINITY; int bi = 0;
    for (int i = 0; i < S; ++i) { float v = a[i * S + j]; if (v > bv) { bv = v; bi = i; } }
    lab2[j] = bi;
  }
  __syncthreads();
  const int n = S - 1;
  float* Wb = W + (size_t)b * n * n;
  for (int e = tid; e < n * n; e += ASSIGN_THREADS) {
    int i = e / n, j = e - i * n;
    float v = a[(i + 1) * S + (j + 1)];
    v = v * (lab1[i + 1] > 0 ? 1.f : 0.f) * (lab2[j + 1] > 0 ? 1.f : 0.f);
    Wb[e] = v * sqrtf(v);   // ** 1.5
  }
  for (int i = tid; i < n; i += ASSIGN_THREADS) w1out[(size_t)b * n + i] = lab1[i + 1] > 0 ? 1.f : 0.f;
}

// ---- 2. cdf + searchsorted ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) coarse_sample_kernel(const float* __restrict__ W, int L, const float* __restrict__ rand,
                                                             int nr, int* __restrict__ idx_out) {
  extern __shared__ float cdf[];  // L floats
  __shared__ double part[1024];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* Wb = W + (size_t)b * L;
  const int per = (L + 1023) / 1024;
  const int beg = min(tid * per, L), end = min(beg + per, L);
  double s = 0.0;
  for (int i = beg; i < end; ++i) s += (double)Wb[i];
  part[tid] = s;
  __syncthreads();
  // exclusive scan of the 1024 partials (Hillis-Steele in double)
  for (int o = 1; o < 1024; o <<= 1) {
    double v = (tid >= o) ? part[tid - o] : 0.0;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  double run = (tid == 0) ? 0.0 : part[tid - 1];
  for (int i = beg; i < end; ++i) { run += (double)Wb[i]; cdf[i] = (float)run; }
  __syncthreads();
  const float denom = cdf[L - 1] + 1e-8f;
  __syncthreads();
  for (int i = tid; i < L; i += 1024) cdf[i] = cdf[i] / denom;
  __syncthreads();
  // searchsorted(right=False): first i with cdf[i] >= v; L if none
  for (int r = tid; r < nr; r += 1024) {
    float v = rand[(size_t)b * nr + r];
    int lo = 0, hi = L;
    while (lo < hi) {
      int mid = (lo + hi) >> 1;
      if (cdf[mid] < v) lo = mid + 1; else hi = mid;
    }
    idx_out[(size_t)b * nr + r] = lo;
  }
}

// ---- 3. hypotheses --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) coarse_hyp_kernel(const int* __restrict__ idx, const float* __restrict__ pts1,
                                                         const float* __restrict__ pts2, int n, int n1, float* __restrict__ Rt,
                                                         float* __restrict__ resid) {
  const int b = blockIdx.y;
  const int hpt = blockIdx.x * blockDim.x + threadIdx.x;
  if (hpt >= n1) return;
  const int* id = idx + ((size_t)b * n1 + hpt) * 3;
  float p1[3][3], p2[3][3];
  int i1s[3], i2s[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int v = id[k];
    int i1 = min(v / n, n - 1), i2 = min(v % n, n - 1);
    i1s[k] = i1; i2s[k] = i2;
    const float* a = pts1 + ((size_t)b * n + i1) * 3;
    const float* c = pts2 + ((size_t)b * n + i2) * 3;
#pragma unroll
    for (int d = 0; d < 3; ++d) { p1[k][d] = a[d]; p2[k][d] = c[d]; }
  }
  // The triplet is drawn with replacement (model_utils.py:218-226).  A repeated point in either cloud leaves collinear
  // centred points, i.e. a rank-1 cross-covariance (rank 0 when one cloud contributes a single point): svd3.cuh.
  const int eq1 = (i1s[0] == i1s[1]) + (i1s[0] == i1s[2]) + (i1s[1] == i1s[2]);
  const int eq2 = (i2s[0] == i2s[1]) + (i2s[0] == i2s[2]) + (i2s[1] == i2s[2]);
  const bool rank0 = (eq1 == 3) || (eq2 == 3);
  const bool rank1 = !rank0 && (eq1 + eq2 > 0);
  // weighted_procrustes(src = p2, ref = p1, weights = 1, thresh 0.5, eps 1e-5): w = 1 / (3 + 1e-5)
  const float w = 1.f / (3.f + 1e-5f);
  float cs[3], cr[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    cs[d] = p2[0][d] * w + p2[1][d] * w + p2[2][d] * w;
    cr[d] = p1[0][d] * w + p1[1][d] * w + p1[2][d] * w;
  }
  double H[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) s += (double)(p2[k][i] - cs[i]) * (double)(w * (p1[k][j] - cr[j]));
      H[i][j] = s;
    }
  double Rd[3][3];
  if (rank0) {   // H is zero up to the 1e-5 of the weight normalisation: the reference's svd(0) gives U = V = I
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) Rd[i][j] = (i == j) ? 1.0 : 0.0;
  } else {
    procrustes_rotation(H, Rd, rank1);
  }
  float R[3][3], t[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) R[i][j] = (float)Rd[i][j];
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = cr[i] - (R[i][0] * cs[0] + R[i][1] * cs[1] + R[i][2] * cs[2]);
  // residual: mean_k || (p1_k - t) R - p2_k ||
  float rs = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float x = p1[k][0] - t[0], y = p1[k][1] - t[1], z = p1[k][2] - t[2];
    float ex = x * R[0][0] + y * R[1][0] + z * R[2][0] - p2[k][0];
    float ey = x * R[0][1] + y * R[1][1] + z * R[2][1] - p2[k][1];
    float ez = x * R[0][2] + y * R[1][2] + z * R[2][2] - p2[k][2];
    rs += sqrtf(ex * ex + ey * ey + ez * ez);
  }
  float* o = Rt + ((size_t)b * n1 + hpt) * 12;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) o[i * 3 + j] = R[i][j];
  o[9] = t[0]; o[10] = t[1]; o[11] = t[2];
  resid[(size_t)b * n1 + hpt] = rs / 3.f;
}

// ---- 4. top-k smallest (bitonic sort of (value, index) keys in shared memory) ---------------------------------
__global__ void __launch_bounds__(1024) topk_smallest_kernel(const float* __restrict__ v, int n, int npow2, int k,
                                                             int* __restrict__ out) {
  extern __shared__ unsigned long long keys[];  // npow2
  const int b = blockIdx.x, tid = threadIdx.x;
  for (int i = tid; i < npow2; i += 1024) {
    unsigned long long key = ~0ull;
    if (i < n) {
      float f = v[(size_t)b * n + i];
      unsigned u = __float_as_uint(f);
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // order-preserving map of the bit pattern (see sam6d_topk_smallest)
      key = ((unsigned long long)u << 32) | (unsigned)i;
    }
    keys[i] = key;
  }
  __syncthreads();
  for (int size = 2; size <= npow2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < npow2 / 2; i += 1024) {
        int lo = 2 * i - (i & (stride - 1));
        int hi = lo + stride;
        bool asc = ((lo & size) == 0);
        unsigned long long a = keys[lo], c = keys[hi];
        if ((a > c) == asc) { keys[lo] = c; keys[hi] = a; }
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < k; i += 1024) out[(size_t)b * k + i] = (int)(keys[i] & 0xffffffffu);
}

// ---- 5. pose selection ----------------------------------------------------------------------------------------
// grid = (ceil(n2 / SEL_PP), B); a thread owns one point of pts1 under SEL_PP hypotheses; the CAD samples sit in shared memory as
// (x, y, z, |m|^2) quadruples, so the inner loop is one 16-byte broadcast load and 4 instructions per (hypothesis, point, sample):
// min_m (|x|^2 - 2 x.m + |m|^2) = |x|^2 + min_m (|m|^2 - 2 x.m), the clamp at 0 commutes with the minimum
// (pairwise_distance, model_utils.py:98-111).
// (Alternatives that lose: a packed-fp32 FFMA2 variant -- FFMA2 issues at half rate; a uniform 8^3 grid over the CAD samples walked
// shell by shell per thread -- the walks of a warp's 32 points diverge, and at 1024 samples the regular scan below is only ~110 warp
// instructions per point.)
constexpr int SEL_PP = 4, SEL_THREADS = 224;
__device__ __forceinline__ float min3f(float a, float b, float c) { return fminf(fminf(a, b), c); }
__global__ void __launch_bounds__(SEL_THREADS) coarse_select_kernel(const float* __restrict__ Rt, const int* __restrict__ top, int n1,
                                                                    int n2, const float* __restrict__ pts1, const float* __restrict__ w1,
                                                                    int n, const float* __restrict__ model, int nm,
                                                                    float* __restrict__ scores) {
  extern __shared__ float4 smq[];   // nm quadruples
  __shared__ float red[2 * SEL_PP][SEL_THREADS / 32];
  __shared__ float rts[SEL_PP][12];
  const int pose0 = blockIdx.x * SEL_PP, b = blockIdx.y, tid = threadIdx.x;
  for (int i = tid; i < nm; i += SEL_THREADS) {
    const float* q = model + ((size_t)b * nm + i) * 3;
    const float x = q[0], y = q[1], z = q[2];
    smq[i] = make_float4(x, y, z, x * x + y * y + z * z);
  }
  if (tid < SEL_PP * 12) {
    const int pp = tid / 12, e = tid - pp * 12;
    const int pose = min(pose0 + pp, n2 - 1);
    rts[pp][e] = Rt[((size_t)b * n1 + top[(size_t)b * n2 + pose]) * 12 + e];
  }
  __syncthreads();
  float num = 0.f, den[SEL_PP];
#pragma unroll
  for (int pp = 0; pp < SEL_PP; ++pp) den[pp] = 0.f;
  for (int i = tid; i < n; i += SEL_THREADS) {
    const float* p = pts1 + ((size_t)b * n + i) * 3;
    const float px = p[0], py = p[1], pz = p[2];
    float ax[SEL_PP], ay[SEL_PP], az[SEL_PP], x2[SEL_PP], best[SEL_PP];
#pragma unroll
    for (int pp = 0; pp < SEL_PP; ++pp) {
      const float* R = rts[pp];
      const float x = px - R[9], y = py - R[10], z = pz - R[11];
      const float tx = x * R[0] + y * R[3] + z * R[6];
      const float ty = x * R[1] + y * R[4] + z * R[7];
      const float tz = x * R[2] + y * R[5] + z * R[8];
      x2[pp] = tx * tx + ty * ty + tz * tz;
      ax[pp] = -2.f * tx; ay[pp] = -2.f * ty; az[pp] = -2.f * tz;
      best[pp] = INFINITY;
    }
    // two CAD samples per step and a three-input minimum (FMNMX3): 3.5 instead of 4 issue slots per (hypothesis, point, sample);
    // a minimum is exact, so the grouping does not change the result
    int m = 0;
#pragma unroll 2
    for (; m + 1 < nm; m += 2) {
      const float4 q = smq[m], q2 = smq[m + 1];
#pragma unroll
      for (int pp = 0; pp < SEL_PP; ++pp)
        best[pp] = min3f(best[pp], fmaf(ax[pp], q.x, fmaf(ay[pp], q.y, fmaf(az[pp], q.z, q.w))),
                         fmaf(ax[pp], q2.x, fmaf(ay[pp], q2.y, fmaf(az[pp], q2.z, q2.w))));
    }
    if (m < nm) {
      const float4 q = smq[m];
#pragma unroll
      for (int pp = 0; pp < SEL_PP; ++pp) best[pp] = fminf(best[pp], fmaf(ax[pp], q.x, fmaf(ay[pp], q.y, fmaf(az[pp], q.z, q.w))));
    }
    const float wi = w1[(size_t)b * n + i];
    num += wi;
#pragma unroll
    for (int pp = 0; pp < SEL_PP; ++pp) den[pp] += sqrtf(fmaxf(x2[pp] + best[pp], 0.f)) * wi;
  }
  num = warp_sum(num);
#pragma unroll
  for (int pp = 0; pp < SEL_PP; ++pp) den[pp] = warp_sum(den[pp]);
  if ((tid & 31) == 0) {
#pragma unroll
    for (int pp = 0; pp < SEL_PP; ++pp) { red[pp][tid >> 5] = num; red[SEL_PP + pp][tid >> 5] = den[pp]; }
  }
  __syncthreads();
  if (tid < SEL_PP && pose0 + tid < n2) {
    float a = 0.f, c = 0.f;
    for (int w = 0; w < SEL_THREADS / 32; ++w) { a += red[tid][w]; c += red[SEL_PP + tid][w]; }
    scores[(size_t)b * n2 + pose0 + tid] = a / (c + 1e-8f);
  }
}

__global__ void coarse_pick_kernel(const float* __restrict__ scores, const int* __restrict__ top, const float* __restrict__ Rt,
                                   int n1, int n2, float* __restrict__ R, float* __restrict__ t) {
  const int b = blockIdx.x, lane = threadIdx.x;
  float bv = -INFINITY; int bi = 0x7fffffff;
  for (int i = lane; i < n2; i += 32) argmax_first(bv, bi, scores[(size_t)b * n2 + i], i);
  warp_argmax_first(bv, bi);
  if (bi == 0x7fffffff) bi = 0;   // all-NaN row: keep the first hypothesis
  const float* rt = Rt + ((size_t)b * n1 + top[(size_t)b * n2 + bi]) * 12;
  if (lane < 9) R[(size_t)b * 9 + lane] = rt[lane];
  if (lane < 3) t[(size_t)b * 3 + lane] = rt[9 + lane];
}

// ---- 6. K mutually distinct hypotheses (not in the reference) ---------------------------------------------------
// one CTA per proposal; the n2 retained hypotheses sit in shared memory as R (9), t (3), score and a live flag.  K greedy rounds:
// block argmax of the live scores (coarse_pick_kernel's rule), write the pick, drop every live hypothesis that is not distinct
// from it (the rule and its fp32 order: include/sam6d_b200.h, sam6d_coarse_pick_distinct)
constexpr int PICK_THREADS = 256, PICK_MAX_N2 = 2048;
__global__ void __launch_bounds__(PICK_THREADS) coarse_pick_distinct_kernel(const float* __restrict__ Rt, const int* __restrict__ top,
                                                                            const float* __restrict__ scores, int n1, int n2, int K,
                                                                            float cos_thr, float d2_min, float* __restrict__ R_out,
                                                                            float* __restrict__ t_out, float* __restrict__ score_out,
                                                                            unsigned char* __restrict__ valid, int* __restrict__ count) {
  extern __shared__ float hs[];
  float* hr = hs;                    // n2 x 12: R row-major, t
  float* sc = hr + (size_t)n2 * 12;  // n2
  unsigned char* live = reinterpret_cast<unsigned char*>(sc + n2);
  __shared__ float rv[PICK_THREADS / 32];
  __shared__ int ri[PICK_THREADS / 32];
  __shared__ int pick;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int e = tid; e < n2 * 12; e += PICK_THREADS) {
    const int j = e / 12, c = e - j * 12;
    hr[e] = Rt[((size_t)b * n1 + top[(size_t)b * n2 + j]) * 12 + c];
  }
  for (int j = tid; j < n2; j += PICK_THREADS) { sc[j] = scores[(size_t)b * n2 + j]; live[j] = 1; }
  __syncthreads();
  int found = 0;
  for (int r = 0; r < K; ++r) {
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int j = tid; j < n2; j += PICK_THREADS)
      if (live[j]) argmax_first(bv, bi, sc[j], j);
    warp_argmax_first(bv, bi);
    if (lane == 0) { rv[warp] = bv; ri[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < PICK_THREADS / 32; ++w) argmax_first(bv, bi, rv[w], ri[w]);
      if (bi == 0x7fffffff && r == 0) bi = 0;   // all-NaN row: keep the first hypothesis, as coarse_pick_kernel
      pick = bi;
    }
    __syncthreads();
    const int i = pick;
    if (i == 0x7fffffff) break;                 // no live hypothesis left (or only NaN scores)
    const float* hi = hr + (size_t)i * 12;
    if (tid < 9) R_out[((size_t)b * K + r) * 9 + tid] = hi[tid];
    if (tid < 3) t_out[((size_t)b * K + r) * 3 + tid] = hi[9 + tid];
    if (tid == 0) { score_out[(size_t)b * K + r] = sc[i]; valid[(size_t)b * K + r] = 1; }
    for (int j = tid; j < n2; j += PICK_THREADS) {
      if (!live[j]) continue;
      const float* hj = hr + (size_t)j * 12;
      float tr = __fmul_rn(hi[0], hj[0]);
#pragma unroll
      for (int e = 1; e < 9; ++e) tr = __fadd_rn(tr, __fmul_rn(hi[e], hj[e]));
      const float dx = __fsub_rn(hi[9], hj[9]), dy = __fsub_rn(hi[10], hj[10]), dz = __fsub_rn(hi[11], hj[11]);
      const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      if (j == i || !(tr < cos_thr || d2 >= d2_min)) live[j] = 0;
    }
    found = r + 1;
    __syncthreads();
  }
  // slots past the last pick: copies of slot 0, not valid
  for (int e = tid; e < (K - found) * 14; e += PICK_THREADS) {
    const int r = found + e / 14, c = e - (e / 14) * 14;
    const size_t s0 = (size_t)b * K, s = s0 + r;
    if (c < 9) R_out[s * 9 + c] = R_out[s0 * 9 + c];
    else if (c < 12) t_out[s * 3 + c - 9] = t_out[s0 * 3 + c - 9];
    else if (c == 12) score_out[s] = score_out[s0];
    else valid[s] = 0;
  }
  if (tid == 0) count[b] = found;
}

// ---- 7. K hypotheses distinct up to the object's symmetries (not in the reference) -----------------------------------------
// coarse_pick_distinct_kernel with one more shared-memory stage: after each pick i, the cnt transforms of i's symmetric copies,
// A_s = R_i R_s and w_s = R_i t_s / radius + t_i, then j is dropped when it is near any copy (the rule and its fp32 order:
// include/sam6d_b200.h, sam6d_coarse_pick_distinct_sym)
constexpr int PICK_MAX_SYM = 2048;
__global__ void __launch_bounds__(PICK_THREADS) coarse_pick_distinct_sym_kernel(
    const float* __restrict__ Rt, const int* __restrict__ top, const float* __restrict__ scores, int n1, int n2, int K, float cos_thr,
    float d2_min, const float* __restrict__ symR, const float* __restrict__ symt, int S, const int* __restrict__ sym_range, int max_count,
    const float* __restrict__ radius, float* __restrict__ R_out, float* __restrict__ t_out, float* __restrict__ score_out,
    unsigned char* __restrict__ valid, int* __restrict__ count) {
  extern __shared__ float hs[];
  float* hr = hs;                            // n2 x 12: R row-major, t
  float* sc = hr + (size_t)n2 * 12;          // n2
  float* cp = sc + n2;                       // max_count x 12: A_s row-major, w_s
  unsigned char* live = reinterpret_cast<unsigned char*>(cp + (size_t)max_count * 12);
  __shared__ float rv[PICK_THREADS / 32];
  __shared__ int ri[PICK_THREADS / 32];
  __shared__ int pick;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int off = sym_range[(size_t)b * 2], cnt0 = sym_range[(size_t)b * 2 + 1];
  // a range outside the set: only the pick itself is dropped
  const int cnt = (off < 0 || cnt0 < 1 || cnt0 > max_count || off > S - cnt0) ? 0 : cnt0;
  const float rad = radius[b];
  for (int e = tid; e < n2 * 12; e += PICK_THREADS) {
    const int j = e / 12, c = e - j * 12;
    hr[e] = Rt[((size_t)b * n1 + top[(size_t)b * n2 + j]) * 12 + c];
  }
  for (int j = tid; j < n2; j += PICK_THREADS) { sc[j] = scores[(size_t)b * n2 + j]; live[j] = 1; }
  __syncthreads();
  int found = 0;
  for (int r = 0; r < K; ++r) {
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int j = tid; j < n2; j += PICK_THREADS)
      if (live[j]) argmax_first(bv, bi, sc[j], j);
    warp_argmax_first(bv, bi);
    if (lane == 0) { rv[warp] = bv; ri[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < PICK_THREADS / 32; ++w) argmax_first(bv, bi, rv[w], ri[w]);
      if (bi == 0x7fffffff && r == 0) bi = 0;   // all-NaN row: keep the first hypothesis, as coarse_pick_kernel
      pick = bi;
    }
    __syncthreads();
    const int i = pick;
    if (i == 0x7fffffff) break;                 // no live hypothesis left (or only NaN scores)
    const float* hi = hr + (size_t)i * 12;
    if (tid < 9) R_out[((size_t)b * K + r) * 9 + tid] = hi[tid];
    if (tid < 3) t_out[((size_t)b * K + r) * 3 + tid] = hi[9 + tid];
    if (tid == 0) { score_out[(size_t)b * K + r] = sc[i]; valid[(size_t)b * K + r] = 1; }
    for (int s = tid; s < cnt; s += PICK_THREADS) {
      const float* Rs = symR + (size_t)(off + s) * 9;
      const float* ts = symt + (size_t)(off + s) * 3;
      float* o = cp + (size_t)s * 12;
#pragma unroll
      for (int y = 0; y < 3; ++y) {
#pragma unroll
        for (int x = 0; x < 3; ++x)
          o[y * 3 + x] = __fadd_rn(__fadd_rn(__fmul_rn(hi[y * 3], Rs[x]), __fmul_rn(hi[y * 3 + 1], Rs[3 + x])), __fmul_rn(hi[y * 3 + 2], Rs[6 + x]));
        const float u = __fadd_rn(__fadd_rn(__fmul_rn(hi[y * 3], ts[0]), __fmul_rn(hi[y * 3 + 1], ts[1])), __fmul_rn(hi[y * 3 + 2], ts[2]));
        o[9 + y] = __fadd_rn(__fdiv_rn(u, rad), hi[9 + y]);
      }
    }
    __syncthreads();
    for (int j = tid; j < n2; j += PICK_THREADS) {
      if (!live[j]) continue;
      const float* hj = hr + (size_t)j * 12;
      bool drop = j == i;
      for (int s = 0; s < cnt && !drop; ++s) {
        const float* a = cp + (size_t)s * 12;
        float tr = __fmul_rn(a[0], hj[0]);
#pragma unroll
        for (int e = 1; e < 9; ++e) tr = __fadd_rn(tr, __fmul_rn(a[e], hj[e]));
        const float dx = __fsub_rn(a[9], hj[9]), dy = __fsub_rn(a[10], hj[10]), dz = __fsub_rn(a[11], hj[11]);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        drop = !(tr < cos_thr || d2 >= d2_min);
      }
      if (drop) live[j] = 0;
    }
    found = r + 1;
    __syncthreads();
  }
  for (int e = tid; e < (K - found) * 14; e += PICK_THREADS) {
    const int r = found + e / 14, c = e - (e / 14) * 14;
    const size_t s0 = (size_t)b * K, s = s0 + r;
    if (c < 9) R_out[s * 9 + c] = R_out[s0 * 9 + c];
    else if (c < 12) t_out[s * 3 + c - 9] = t_out[s0 * 3 + c - 9];
    else if (c == 12) score_out[s] = score_out[s0];
    else valid[s] = 0;
  }
  if (tid == 0) count[b] = found;
}

}  // namespace

// A (B,S,S) f32 -> W (B,(S-1)^2) masked soft assignment ^1.5, w1 (B,S-1)      (model_utils.py:206-216)
S6_API int sam6d_coarse_assign(const float* A, int B, int S, float* W, float* w1, void* stream) {
  S6_REQUIRE(A && W && w1 && B >= 0 && S >= 2);
  if (B == 0) return 0;
  size_t smem = ((size_t)S * S + 6 * S) * sizeof(float);
  S6_REQUIRE(smem <= 220 * 1024);
  S6_CHECK(cudaFuncSetAttribute(coarse_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  coarse_assign_kernel<<<B, ASSIGN_THREADS, smem, s6_stream(stream)>>>(A, S, W, w1);
  S6_LAUNCH_CHECK();
  return 0;
}

// W (B,L) f32, rand (B,nr) f32 in [0,1) -> idx (B,nr) i32 in [0,L]             (model_utils.py:218-220)
S6_API int sam6d_coarse_sample(const float* W, int B, int L, const float* rand, int nr, int* idx, void* stream) {
  S6_REQUIRE(W && rand && idx && B >= 0 && L > 0 && nr >= 0);
  if (B == 0 || nr == 0) return 0;
  size_t smem = (size_t)L * sizeof(float);
  S6_REQUIRE(smem <= 200 * 1024);
  S6_CHECK(cudaFuncSetAttribute(coarse_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  coarse_sample_kernel<<<B, 1024, smem, s6_stream(stream)>>>(W, L, rand, nr, idx);
  S6_LAUNCH_CHECK();
  return 0;
}

// idx (B,n1,3) flat pair indices -> Rt (B,n1,12) = [R row-major, t], resid (B,n1)   (model_utils.py:221-234)
S6_API int sam6d_coarse_hypotheses(const int* idx, const float* pts1, const float* pts2, int B, int n, int n1, float* Rt,
                                   float* resid, void* stream) {
  S6_REQUIRE(idx && pts1 && pts2 && Rt && resid && B >= 0 && n > 0 && n1 >= 0);
  if (B == 0 || n1 == 0) return 0;
  dim3 grid(s6_cdiv(n1, 128), B);
  coarse_hyp_kernel<<<grid, 128, 0, s6_stream(stream)>>>(idx, pts1, pts2, n, n1, Rt, resid);
  S6_LAUNCH_CHECK();
  return 0;
}

// v (B,n) -> out (B,k): indices of the k smallest values, ascending by (value, index)   (model_utils.py:235).
// The order is that of the fp32 bit patterns: -0.0 sorts before +0.0 whatever their indices, a NaN with the sign bit set
// before every value and any other NaN after +inf.  The residuals this ranks are norms, never -0 or NaN from finite points.
S6_API int sam6d_topk_smallest(const float* v, int B, int n, int k, int* out, void* stream) {
  S6_REQUIRE(v && out && B >= 0 && n > 0 && k > 0 && k <= n);
  if (B == 0) return 0;
  int npow2 = 2;
  while (npow2 < n) npow2 <<= 1;
  size_t smem = (size_t)npow2 * sizeof(unsigned long long);
  S6_REQUIRE(smem <= 200 * 1024);
  S6_CHECK(cudaFuncSetAttribute(topk_smallest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  topk_smallest_kernel<<<B, 1024, smem, s6_stream(stream)>>>(v, n, npow2, k, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// scores the n2 retained hypotheses against the CAD samples and returns the best (model_utils.py:239-246)
// scratch: scores (B,n2) f32
S6_API int sam6d_coarse_select(const float* Rt, const int* top, int B, int n1, int n2, const float* pts1, const float* w1, int n,
                               const float* model, int nm, float* scores, float* R, float* t, void* stream) {
  S6_REQUIRE(Rt && top && pts1 && w1 && model && scores && R && t && B >= 0 && n > 0 && nm > 0 && n2 > 0);
  if (B == 0) return 0;
  size_t smem = (size_t)nm * 4 * sizeof(float);
  S6_REQUIRE(smem <= 200 * 1024);
  S6_CHECK(cudaFuncSetAttribute(coarse_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(s6_cdiv(n2, SEL_PP), B);
  coarse_select_kernel<<<grid, SEL_THREADS, smem, s6_stream(stream)>>>(Rt, top, n1, n2, pts1, w1, n, model, nm, scores);
  S6_LAUNCH_CHECK();
  coarse_pick_kernel<<<B, 32, 0, s6_stream(stream)>>>(scores, top, Rt, n1, n2, R, t);
  S6_LAUNCH_CHECK();
  return 0;
}

// K mutually distinct hypotheses of the n2 that sam6d_coarse_select scored (the rule: include/sam6d_b200.h)
S6_API int sam6d_coarse_pick_distinct(const float* Rt, const int* top, const float* scores, int B, int n1, int n2, int K, float cos_thr,
                                      float d2_min, float* R_out, float* t_out, float* score_out, unsigned char* valid, int* count,
                                      void* stream) {
  S6_REQUIRE(B >= 0 && n1 > 0 && n2 > 0 && n2 <= PICK_MAX_N2 && K >= 1 && K <= n2);
  S6_REQUIRE(isfinite(cos_thr) && isfinite(d2_min));
  S6_REQUIRE(Rt && top && scores && R_out && t_out && score_out && valid && count);
  if (B == 0) return 0;
  const size_t smem = (size_t)n2 * 13 * sizeof(float) + n2;
  S6_CHECK(cudaFuncSetAttribute(coarse_pick_distinct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  coarse_pick_distinct_kernel<<<B, PICK_THREADS, smem, s6_stream(stream)>>>(Rt, top, scores, n1, n2, K, cos_thr, d2_min, R_out, t_out,
                                                                          score_out, valid, count);
  S6_LAUNCH_CHECK();
  return 0;
}

// sam6d_coarse_pick_distinct with "distinct" read up to each proposal's symmetry set (the rule: include/sam6d_b200.h)
S6_API int sam6d_coarse_pick_distinct_sym(const float* Rt, const int* top, const float* scores, int B, int n1, int n2, int K,
                                          float cos_thr, float d2_min, const float* symR, const float* symt, int S, const int* sym_range,
                                          int max_count, const float* radius, float* R_out, float* t_out, float* score_out,
                                          unsigned char* valid, int* count, void* stream) {
  S6_REQUIRE(B >= 0 && n1 > 0 && n2 > 0 && n2 <= PICK_MAX_N2 && K >= 1 && K <= n2);
  S6_REQUIRE(S >= 1 && max_count >= 1 && max_count <= PICK_MAX_SYM);
  S6_REQUIRE(isfinite(cos_thr) && isfinite(d2_min));
  S6_REQUIRE(Rt && top && scores && symR && symt && sym_range && radius && R_out && t_out && score_out && valid && count);
  if (B == 0) return 0;
  const size_t smem = ((size_t)n2 * 13 + (size_t)max_count * 12) * sizeof(float) + n2;
  S6_CHECK(cudaFuncSetAttribute(coarse_pick_distinct_sym_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  coarse_pick_distinct_sym_kernel<<<B, PICK_THREADS, smem, s6_stream(stream)>>>(Rt, top, scores, n1, n2, K, cos_thr, d2_min, symR, symt, S,
                                                                              sym_range, max_count, radius, R_out, t_out, score_out,
                                                                              valid, count);
  S6_LAUNCH_CHECK();
  return 0;
}
