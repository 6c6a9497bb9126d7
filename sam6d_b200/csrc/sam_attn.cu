// sam_attn.cu -- SAM ViT attention with decomposed relative-position bias
// (Attention.forward + add_decomposed_rel_pos, ISM/segment_anything/modeling/image_encoder.py:224-240, 325-361).
//
//   attn[n, m] = (q_n * scale) . k_m + q_n . Rh[h(n) - h(m) + Hs - 1] + q_n . Rw[w(n) - w(m) + Ws - 1]     (unscaled q in the bias)
//   out_n = softmax_m(attn[n, :]) v
// for every window (nW = B*25 windows of 14x14 tokens, or B "windows" of 64x64 for the global blocks) and head (dim D = 80 for
// ViT-H, 64 for ViT-L / ViT-B).
// Flash-style: the (HW x HW) score tensor of the reference (1.07 GB per global layer) never exists.  Keys / values stream
// through shared memory in 64-key tiles with an online softmax; a warp owns 4 queries, a lane 2 keys per tile (QK^T) and
// 3 output channels at D = 80 / 2 at D = 64 (PV), so each K/V word read from shared memory feeds 4 FMAs.  The two bias tables of a query (Hs + Ws
// dot products instead of Hs*Ws) are built once per query in shared memory.  fp32 CUDA-core version.
#include "common.cuh"

namespace {

constexpr int KT = 64, QT = 32, MAXS = 64;

// K rows padded by 4 floats (DP) to spread the QK^T row reads over the banks; a K / V tile is LOADS float4 per thread
template <int D>
struct RelposCfg {
  static constexpr int DP = D + 4, LOADS = KT * D / 4 / 256;
  static constexpr size_t SMEM = ((size_t)KT * DP + KT * D + 8 * D * 4 + 8 * KT * 4 + 2 * 8 * MAXS * 4) * sizeof(float);
  static_assert((KT * D / 4) % 256 == 0 && D > 32 && D <= 96, "head dim: whole float4 loads per thread, 2 or 3 channels per lane");
};

__device__ __forceinline__ void st_o(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_o(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }

template <int D, typename OT>
__global__ void __launch_bounds__(256) sam_attn_kernel(const float* __restrict__ qkv, long long tok_ld, int Hs, int Ws, int nH,
                                                       const float* __restrict__ rel_h, const float* __restrict__ rel_w,
                                                       float scale, OT* __restrict__ out, long long out_ld) {
  constexpr int DP = RelposCfg<D>::DP, LOADS = RelposCfg<D>::LOADS, C4 = D / 4;
  extern __shared__ __align__(16) float sm[];
  float* ks = sm;                         // KT * DP
  float* vs = ks + KT * DP;               // KT * D
  float* qs = vs + KT * D;                // 8 warps * [D][4]
  float* ps = qs + 8 * D * 4;             // 8 warps * [KT][4]
  float* bh = ps + 8 * KT * 4;            // 8 warps * [MAXS][4]
  float* bw = bh + 8 * MAXS * 4;          // 8 warps * [MAXS][4]
  const int L = Hs * Ws, C = nH * D;
  const int win = blockIdx.z, head = blockIdx.y, q0 = blockIdx.x * QT;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* base = qkv + (size_t)win * L * tok_ld;
  const float* Qb = base + head * D;
  const float* Kb = base + C + head * D;
  const float* Vb = base + 2 * C + head * D;
  float* qw = qs + warp * D * 4;
  float* pw = ps + warp * KT * 4;
  float* bhw = bh + warp * MAXS * 4;
  float* bww = bw + warp * MAXS * 4;
  const int n0 = q0 + warp * 4;
  // queries of this warp, 4 interleaved per channel
  for (int e = lane; e < D * 4; e += 32) {
    const int c = e >> 2, qi = e & 3, n = min(n0 + qi, L - 1);
    qw[e] = Qb[(size_t)n * tok_ld + c];
  }
  __syncwarp();
  // decomposed relative-position bias tables: bhw[kh][qi] = q . Rh[qh - kh + Hs - 1], bww[kw][qi] = q . Rw[qw - kw + Ws - 1]
  for (int e = lane; e < Hs * 4; e += 32) {
    const int kh = e >> 2, qi = e & 3, n = min(n0 + qi, L - 1);
    const float* r = rel_h + (size_t)(n / Ws - kh + Hs - 1) * D;
    float a = 0.f;
    for (int c = 0; c < D; ++c) a = fmaf(qw[c * 4 + qi], r[c], a);
    bhw[e] = a;
  }
  for (int e = lane; e < Ws * 4; e += 32) {
    const int kw = e >> 2, qi = e & 3, n = min(n0 + qi, L - 1);
    const float* r = rel_w + (size_t)(n % Ws - kw + Ws - 1) * D;
    float a = 0.f;
    for (int c = 0; c < D; ++c) a = fmaf(qw[c * 4 + qi], r[c], a);
    bww[e] = a;
  }
  float mrun[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY}, lrun[4] = {0.f, 0.f, 0.f, 0.f};
  float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f}, o2[4] = {0.f, 0.f, 0.f, 0.f};
  const int c2 = 64 + (lane & 15);                         // D = 80: the lane's third channel
  for (int kt0 = 0; kt0 < L; kt0 += KT) {
    __syncthreads();
    {  // stage the K / V tile: 64 keys x D/4 float4 each; all loads issued before the stores
      float4 kreg[LOADS], vreg[LOADS];
#pragma unroll
      for (int i = 0; i < LOADS; ++i) {
        const int u = i * 256 + tid, m = u / C4, c4 = (u - m * C4) * 4;
        const int key = min(kt0 + m, L - 1);
        kreg[i] = *reinterpret_cast<const float4*>(Kb + (size_t)key * tok_ld + c4);
        vreg[i] = *reinterpret_cast<const float4*>(Vb + (size_t)key * tok_ld + c4);
      }
#pragma unroll
      for (int i = 0; i < LOADS; ++i) {
        const int u = i * 256 + tid, m = u / C4, c4 = (u - m * C4) * 4;
        *reinterpret_cast<float4*>(ks + m * DP + c4) = kreg[i];
        *reinterpret_cast<float4*>(vs + m * D + c4) = vreg[i];
      }
    }
    __syncthreads();
    float s[2][4];
    float tmax[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int m = lane + 32 * t, key = kt0 + m;
      float a[4] = {0.f, 0.f, 0.f, 0.f};
      const float* kr = ks + m * DP;
#pragma unroll (D / 16)
      for (int c = 0; c < D; c += 4) {
        const float4 kv = *reinterpret_cast<const float4*>(kr + c);
        const float4 qa = *reinterpret_cast<const float4*>(qw + (c + 0) * 4);
        const float4 qb = *reinterpret_cast<const float4*>(qw + (c + 1) * 4);
        const float4 qc = *reinterpret_cast<const float4*>(qw + (c + 2) * 4);
        const float4 qd = *reinterpret_cast<const float4*>(qw + (c + 3) * 4);
        a[0] = fmaf(kv.x, qa.x, a[0]); a[1] = fmaf(kv.x, qa.y, a[1]); a[2] = fmaf(kv.x, qa.z, a[2]); a[3] = fmaf(kv.x, qa.w, a[3]);
        a[0] = fmaf(kv.y, qb.x, a[0]); a[1] = fmaf(kv.y, qb.y, a[1]); a[2] = fmaf(kv.y, qb.z, a[2]); a[3] = fmaf(kv.y, qb.w, a[3]);
        a[0] = fmaf(kv.z, qc.x, a[0]); a[1] = fmaf(kv.z, qc.y, a[1]); a[2] = fmaf(kv.z, qc.z, a[2]); a[3] = fmaf(kv.z, qc.w, a[3]);
        a[0] = fmaf(kv.w, qd.x, a[0]); a[1] = fmaf(kv.w, qd.y, a[1]); a[2] = fmaf(kv.w, qd.z, a[2]); a[3] = fmaf(kv.w, qd.w, a[3]);
      }
      if (key < L) {
        const float4 h4 = *reinterpret_cast<const float4*>(bhw + (key / Ws) * 4);
        const float4 w4 = *reinterpret_cast<const float4*>(bww + (key % Ws) * 4);
        a[0] = fmaf(a[0], scale, h4.x + w4.x); a[1] = fmaf(a[1], scale, h4.y + w4.y);
        a[2] = fmaf(a[2], scale, h4.z + w4.z); a[3] = fmaf(a[3], scale, h4.w + w4.w);
      } else {
        a[0] = a[1] = a[2] = a[3] = -INFINITY;
      }
#pragma unroll
      for (int qi = 0; qi < 4; ++qi) { s[t][qi] = a[qi]; tmax[qi] = fmaxf(tmax[qi], a[qi]); }
    }
    float corr[4];
#pragma unroll
    for (int qi = 0; qi < 4; ++qi) {
      const float mnew = fmaxf(mrun[qi], warp_max(tmax[qi]));
      corr[qi] = __expf(mrun[qi] - mnew);          // 0 on the first tile (mrun = -inf)
      mrun[qi] = mnew;
      lrun[qi] *= corr[qi];
      o0[qi] *= corr[qi]; o1[qi] *= corr[qi];
      if constexpr (D > 64) o2[qi] *= corr[qi];
    }
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      float p[4];
#pragma unroll
      for (int qi = 0; qi < 4; ++qi) { p[qi] = __expf(s[t][qi] - mrun[qi]); lrun[qi] += p[qi]; }
      *reinterpret_cast<float4*>(pw + (lane + 32 * t) * 4) = make_float4(p[0], p[1], p[2], p[3]);
    }
    __syncwarp();
#pragma unroll 4
    for (int m = 0; m < KT; ++m) {
      const float4 p = *reinterpret_cast<const float4*>(pw + m * 4);
      const float v0 = vs[m * D + lane], v1 = vs[m * D + lane + 32];
      o0[0] = fmaf(p.x, v0, o0[0]); o0[1] = fmaf(p.y, v0, o0[1]); o0[2] = fmaf(p.z, v0, o0[2]); o0[3] = fmaf(p.w, v0, o0[3]);
      o1[0] = fmaf(p.x, v1, o1[0]); o1[1] = fmaf(p.y, v1, o1[1]); o1[2] = fmaf(p.z, v1, o1[2]); o1[3] = fmaf(p.w, v1, o1[3]);
      if constexpr (D > 64) {
        const float v2 = vs[m * D + c2];
        o2[0] = fmaf(p.x, v2, o2[0]); o2[1] = fmaf(p.y, v2, o2[1]); o2[2] = fmaf(p.z, v2, o2[2]); o2[3] = fmaf(p.w, v2, o2[3]);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int qi = 0; qi < 4; ++qi) {
    const int n = n0 + qi;
    const float inv = 1.f / warp_sum(lrun[qi]);
    if (n < L) {
      OT* op = out + ((size_t)win * L + n) * out_ld + head * D;
      st_o(op + lane, o0[qi] * inv);
      st_o(op + lane + 32, o1[qi] * inv);
      if (D > 64 && lane < D - 64) st_o(op + 64 + lane, o2[qi] * inv);
    }
  }
}

template <int D, typename OT>
int launch_relpos(const float* qkv, long long tok_ld, int nW, int Hs, int Ws, int nH, const float* rel_h, const float* rel_w,
                  float scale, void* out, long long out_ld, cudaStream_t st) {
  constexpr size_t smem = RelposCfg<D>::SMEM;
  dim3 grid(s6_cdiv(Hs * Ws, QT), nH, nW);
  S6_CHECK(cudaFuncSetAttribute(sam_attn_kernel<D, OT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sam_attn_kernel<D, OT><<<grid, 256, smem, st>>>(qkv, tok_ld, Hs, Ws, nH, rel_h, rel_w, scale, reinterpret_cast<OT*>(out), out_ld);
  S6_LAUNCH_CHECK();
  return 0;
}

}  // namespace

// qkv: (nW * Hs*Ws tokens, 3 * nH * D) fp32 rows [q | k | v] with head-major channels (the output layout of the qkv Linear),
// row stride tok_ld; rel_h (2*Hs-1, D), rel_w (2*Ws-1, D); out (nW * Hs*Ws, nH*D) with row stride out_ld.  Hs, Ws <= 64;
// head_dim D = 80 (ViT-H) or 64 (ViT-L, ViT-B).
S6_API int sam6d_attn_relpos(const float* qkv, long long tok_ld, int nW, int Hs, int Ws, int nH, int head_dim, const float* rel_h,
                             const float* rel_w, float scale, void* out, int out_is_bf16, long long out_ld, void* stream) {
  S6_REQUIRE(qkv && rel_h && rel_w && out && nW >= 0 && Hs > 0 && Ws > 0 && Hs <= MAXS && Ws <= MAXS && nH > 0);
  S6_REQUIRE((head_dim == 64 || head_dim == 80) && (tok_ld % 4) == 0);
  if (nW == 0) return 0;
  S6_REQUIRE(nW <= 65535 && nH <= 65535);
  cudaStream_t st = s6_stream(stream);
  if (head_dim == 64)
    return out_is_bf16 ? launch_relpos<64, __nv_bfloat16>(qkv, tok_ld, nW, Hs, Ws, nH, rel_h, rel_w, scale, out, out_ld, st)
                       : launch_relpos<64, float>(qkv, tok_ld, nW, Hs, Ws, nH, rel_h, rel_w, scale, out, out_ld, st);
  return out_is_bf16 ? launch_relpos<80, __nv_bfloat16>(qkv, tok_ld, nW, Hs, Ws, nH, rel_h, rel_w, scale, out, out_ld, st)
                     : launch_relpos<80, float>(qkv, tok_ld, nW, Hs, Ws, nH, rel_h, rel_w, scale, out, out_ld, st);
}
