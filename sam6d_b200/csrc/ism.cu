// ism.cu -- per-proposal template scoring of the Instance Segmentation Model
// (PairwiseSimilarity, ISM/model/loss.py:21-44; compute_semantic_score + best_template_pose,
//  ISM/model/detector.py:198-207,260-296).
//
//   s[p,o,t]  = clamp(cos(q_p, r_{o,t}), 0, 1)            on L2-normalised descriptors
//   S[p,o]    = agg_t s[p,o,:]    agg = mean (sum / T), median (lower: sorted[(T-1)/2]), max, or
//                                 avg_5 (mean of the 5 largest, all T when T < 5)
//   o*[p]     = argmax_o S[p,o]   (first max),  score[p] = S[p,o*]
//   t*[p]     = argmax_t s[p,o*,:] (first max)
// template_score_kernel: one CTA per (tile of kPT proposals, object).  The tile's normalised queries stay in shared memory and
// the object's T reference rows stream once per tile (coalesced float4 reads, two rows per warp so that each shared-memory
// query read feeds two rows), so reference traffic is ceil(P / kPT) x O x T x C x 4 bytes instead of P x O x T x C x 4.  Every
// (p, row) dot product is the same lane-strided float4 FMA chain and warp_sum as the one-CTA-per-proposal kernel this replaced,
// so similarities and avg_5 scores are bit-identical to it.  The tile's T similarities per
// proposal sit in shared memory; warp p aggregates proposal p and finds its best template.  template_pick_kernel then takes
// the first-max object of every proposal.  The reference's P-fold replication of the reference descriptors never exists.
#include "common.cuh"

namespace {

constexpr int kPT = 8;                 // proposals per CTA = warps per CTA: warp w aggregates proposal w of the tile
constexpr int kThreads = 32 * kPT;
enum { kAggMean = 0, kAggMedian = 1, kAggMax = 2, kAggAvg5 = 3 };

__device__ __forceinline__ float pick_lane(const float (&v)[kPT], int lane) {
  float r = v[0];
#pragma unroll
  for (int i = 1; i < kPT; ++i)
    if (lane == i) r = v[i];
  return r;
}

// shared memory: q (kPT, C) normalised queries | sim (kPT, ld) similarities (ld = T, or T rounded up to a power of two for
// the median's bitonic sort) | red (kThreads / 32)
__global__ void __launch_bounds__(kThreads) template_score_kernel(const float* __restrict__ Qn, const float* __restrict__ Rn, int P,
                                                                  int O, int T, int C, int ld, int agg, float* __restrict__ sim_out,
                                                                  float* __restrict__ obj_score, int* __restrict__ obj_tmpl) {
  extern __shared__ float sm[];
  float* q = sm;
  float* sim = q + (size_t)kPT * C;
  float* red = sim + (size_t)kPT * ld;
  const int p0 = blockIdx.x * kPT, o = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float eps = 1e-8f;
  // F.cosine_similarity re-normalises its (already unit) inputs: x / max(||x||, 1e-8); one proposal at a time over the whole
  // CTA, the summation order of the one-CTA-per-proposal kernel
  for (int pl = 0; pl < kPT; ++pl) {
    float* qp = q + (size_t)pl * C;
    if (p0 + pl >= P) {
      for (int c = tid; c < C; c += kThreads) qp[c] = 0.f;
      continue;
    }
    const float* src = Qn + (size_t)(p0 + pl) * C;
    float ss = 0.f;
    for (int c = tid; c < C; c += kThreads) { float v = src[c]; qp[c] = v; ss += v * v; }
    ss = warp_sum(ss);
    if (lane == 0) red[warp] = ss;
    __syncthreads();
    float qn = 0.f;
    for (int w = 0; w < kThreads / 32; ++w) qn += red[w];
    qn = fmaxf(sqrtf(qn), eps);
    __syncthreads();
    for (int c = tid; c < C; c += kThreads) qp[c] = qp[c] / qn;
  }
  __syncthreads();

  // similarities: warp w takes rows (t, t + 1), t = 2w, 2w + 16, ...; lane pl stores proposal pl's values
  for (int t = 2 * warp; t < T; t += 2 * kThreads / 32) {
    const bool two = t + 1 < T;
    const float* r0 = Rn + ((size_t)o * T + t) * C;
    const float* r1 = two ? r0 + C : r0;
    float d0[kPT], d1[kPT], rr0 = 0.f, rr1 = 0.f;
#pragma unroll
    for (int i = 0; i < kPT; ++i) { d0[i] = 0.f; d1[i] = 0.f; }
#pragma unroll 4
    for (int c = lane * 4; c < C; c += 128) {                    // unrolled so that several loads are in flight per warp
      const float4 v = __ldg(reinterpret_cast<const float4*>(r0 + c));
      const float4 w = __ldg(reinterpret_cast<const float4*>(r1 + c));
#pragma unroll
      for (int i = 0; i < kPT; ++i) {
        const float4 u = *reinterpret_cast<const float4*>(q + (size_t)i * C + c);
        d0[i] = fmaf(u.x, v.x, d0[i]); d0[i] = fmaf(u.y, v.y, d0[i]); d0[i] = fmaf(u.z, v.z, d0[i]); d0[i] = fmaf(u.w, v.w, d0[i]);
        d1[i] = fmaf(u.x, w.x, d1[i]); d1[i] = fmaf(u.y, w.y, d1[i]); d1[i] = fmaf(u.z, w.z, d1[i]); d1[i] = fmaf(u.w, w.w, d1[i]);
      }
      rr0 = fmaf(v.x, v.x, rr0); rr0 = fmaf(v.y, v.y, rr0); rr0 = fmaf(v.z, v.z, rr0); rr0 = fmaf(v.w, v.w, rr0);
      rr1 = fmaf(w.x, w.x, rr1); rr1 = fmaf(w.y, w.y, rr1); rr1 = fmaf(w.z, w.z, rr1); rr1 = fmaf(w.w, w.w, rr1);
    }
    rr0 = warp_sum(rr0); rr1 = warp_sum(rr1);
#pragma unroll
    for (int i = 0; i < kPT; ++i) { d0[i] = warp_sum(d0[i]); d1[i] = warp_sum(d1[i]); }
    const int pl = lane, p = p0 + lane;
    if (lane < kPT && p < P) {
      float s0 = pick_lane(d0, lane) / fmaxf(sqrtf(rr0), eps);
      s0 = fminf(fmaxf(s0, 0.f), 1.f);
      sim[(size_t)pl * ld + t] = s0;
      if (sim_out) sim_out[((size_t)p * O + o) * T + t] = s0;
      if (two) {
        float s1 = pick_lane(d1, lane) / fmaxf(sqrtf(rr1), eps);
        s1 = fminf(fmaxf(s1, 0.f), 1.f);
        sim[(size_t)pl * ld + t + 1] = s1;
        if (sim_out) sim_out[((size_t)p * O + o) * T + t + 1] = s1;
      }
    }
  }
  __syncthreads();

  // aggregation: warp pl over proposal p0 + pl
  const int p = p0 + warp;
  if (p >= P) return;
  float* row = sim + (size_t)warp * ld;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int t = lane; t < T; t += 32) argmax_first(bv, bi, row[t], t);
  warp_argmax_first(bv, bi);
  if (bi == 0x7fffffff) bi = 0;
  float score;
  if (agg == kAggMax) {
    score = bv;
  } else if (agg == kAggMean) {
    float s = 0.f;
    for (int t = lane; t < T; t += 32) s += row[t];
    score = warp_sum(s) / (float)T;
  } else if (agg == kAggAvg5) {
    // each lane's 5 largest, merged largest first; summed in descending order like topk -> mean
    float top[5] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (int t = lane; t < T; t += 32) {
      float v = row[t];
      if (v > top[4]) {
        int k = 4;
        while (k > 0 && v > top[k - 1]) { top[k] = top[k - 1]; --k; }
        top[k] = v;
      }
    }
    const int kk = min(T, 5);
    float s = 0.f;
    for (int k = 0; k < kk; ++k) {
      const float m = warp_max(top[0]);
      const unsigned owner = __ballot_sync(0xffffffffu, top[0] == m);
      if (lane == __ffs(owner) - 1) { top[0] = top[1]; top[1] = top[2]; top[2] = top[3]; top[3] = top[4]; top[4] = -INFINITY; }
      s += m;
    }
    score = s / (float)kk;
  } else {
    // lower median: bitonic sort of the row, padded with +inf to ld = 2^k, ascending
    for (int t = T + lane; t < ld; t += 32) row[t] = INFINITY;
    __syncwarp();
    for (int k = 2; k <= ld; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = lane; i < ld; i += 32) {
          const int ij = i ^ j;
          if (ij > i) {
            const float a = row[i], b = row[ij];
            if ((a > b) == ((i & k) == 0)) { row[i] = b; row[ij] = a; }
          }
        }
        __syncwarp();
      }
    }
    score = row[(T - 1) / 2];
  }
  if (lane == 0) {
    obj_score[(size_t)p * O + o] = score;
    obj_tmpl[(size_t)p * O + o] = bi;
  }
}

// one warp per proposal: first-max object over obj_score (P,O), its score and its best template
__global__ void __launch_bounds__(256) template_pick_kernel(const float* __restrict__ obj_score, const int* __restrict__ obj_tmpl, int P,
                                                            int O, int* __restrict__ best_obj, float* __restrict__ best_score,
                                                            int* __restrict__ best_tmpl) {
  const int p = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= P) return;
  const float* so = obj_score + (size_t)p * O;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int o = lane; o < O; o += 32) argmax_first(bv, bi, so[o], o);
  warp_argmax_first(bv, bi);
  if (bi == 0x7fffffff) bi = 0;
  if (lane == 0) {
    best_obj[p] = bi;
    best_score[p] = so[bi];
    best_tmpl[p] = obj_tmpl[(size_t)p * O + bi];
  }
}

}  // namespace

// Qn (P,C) and Rn (O,T,C): descriptors already passed through F.normalize (sam6d_l2norm_rows).  C % 4 == 0.
// aggregation 0 mean, 1 median, 2 max, 3 avg_5.  sim_out (P,O,T) is optional (may be null); obj_score (P,O) f32 and
// obj_tmpl (P,O) i32 are required: per (proposal, object) score and first-max template.
S6_API int sam6d_template_score_agg(const float* Qn, const float* Rn, int P, int O, int T, int C, int aggregation, float* sim_out,
                                    float* obj_score, int* obj_tmpl, int* best_obj, float* best_score, int* best_tmpl, void* stream) {
  S6_REQUIRE(P >= 0 && O > 0 && T > 0 && C > 0 && C % 4 == 0 && aggregation >= kAggMean && aggregation <= kAggAvg5);
  S6_REQUIRE(O <= 65535);                                                        // grid.y
  if (P == 0) return 0;                                                          // no proposal: the (empty) outputs may be null
  S6_REQUIRE(Qn && Rn && obj_score && obj_tmpl && best_obj && best_score && best_tmpl);
  int ld = T;
  if (aggregation == kAggMedian) {
    S6_REQUIRE(T <= (1 << 20));
    ld = 1;
    while (ld < T) ld <<= 1;
  }
  const size_t smem = ((size_t)kPT * C + (size_t)kPT * ld + kThreads / 32) * sizeof(float);
  int dev = 0, optin = 0;
  S6_CHECK(cudaGetDevice(&dev));
  S6_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  S6_REQUIRE(smem <= (size_t)optin);
  cudaStream_t st = s6_stream(stream);
  S6_CHECK(cudaFuncSetAttribute(template_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((P + kPT - 1) / kPT, O);
  template_score_kernel<<<grid, kThreads, smem, st>>>(Qn, Rn, P, O, T, C, ld, aggregation, sim_out, obj_score, obj_tmpl);
  S6_LAUNCH_CHECK();
  template_pick_kernel<<<(P + 7) / 8, 256, 0, st>>>(obj_score, obj_tmpl, P, O, best_obj, best_score, best_tmpl);
  S6_LAUNCH_CHECK();
  return 0;
}

// avg_5 with the per-object scratch allocated on the stream (obj_score may be null here)
S6_API int sam6d_template_score(const float* Qn, const float* Rn, int P, int O, int T, int C, float* sim_out, float* obj_score,
                                int* best_obj, float* best_score, int* best_tmpl, void* stream) {
  S6_REQUIRE(Qn && Rn && best_obj && best_score && best_tmpl && P >= 0 && O > 0 && T > 0 && C > 0 && C % 4 == 0);
  if (P == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  const size_t n = (size_t)P * O;
  void* ws = nullptr;
  S6_CHECK(cudaMallocAsync(&ws, n * (obj_score ? 1 : 2) * sizeof(float), st));
  int* tmpl = static_cast<int*>(ws);
  float* score = obj_score ? obj_score : reinterpret_cast<float*>(tmpl + n);
  const int rc = sam6d_template_score_agg(Qn, Rn, P, O, T, C, kAggAvg5, sim_out, score, tmpl, best_obj, best_score, best_tmpl, stream);
  const cudaError_t fe = cudaFreeAsync(ws, st);
  return rc != 0 ? rc : (int)fe;
}
