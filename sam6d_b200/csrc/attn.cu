// attn.cu -- attention kernels of the geometric transformer and the dense linear-attention layer.
//
//  * rpe_scores : the relative-position term of RPEMultiHeadAttention (PEM/model/transformer.py:369-399),
//      s_p[b,h,n,m] = q_h[b,n,:] . proj_p(E[b,n,m,:])_h
//    evaluated as (W_p,h^T q_h) . E[b,n,m,:]  (the q.b_p term is constant along m and cancels in the softmax),
//    so proj_p(E) -- 163 GFLOP and 2.5 GB per call in the reference -- is never formed and the kernel is one
//    streaming pass over E: the HBM-bound "PEM attention" kernel of the roofline report.
//  * mha        : softmax((q k^T + s_p) / sqrt(d)) v for <= 256 keys per cloud (self and cross attention).
//  * linattn_*  : focused linear attention, kv-first branch (transformer.py:552-559).
#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------
// rpe_scores.  grid = B*S rows (b,n); 8 warps; warp w handles keys m = w*MB .. in chunks of MB = 4.
// lane l holds channels [8l, 8l+8) of the four per-head query vectors u_h (32 registers).
// ------------------------------------------------------------------------------------------
template <typename ET>
__device__ __forceinline__ void load8(const ET* p, float v[8]);
template <>
__device__ __forceinline__ void load8<float>(const float* p, float v[8]) {
  float4 a = __ldcs(reinterpret_cast<const float4*>(p));
  float4 b = __ldcs(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <>
__device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float v[8]) {
  uint4 a = __ldcs(reinterpret_cast<const uint4*>(p));
  const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[2 * i] = __uint_as_float(w[i] << 16);
    v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}

template <typename ET>
__global__ void __launch_bounds__(256) rpe_scores_kernel(const ET* __restrict__ E, const float* __restrict__ U, long long u_ld, int S,
                                                         float* __restrict__ SP) {
  // E: (B,S,S,256); U: (B*S rows, 4*256) with row stride u_ld; SP: (B,4,S,S)
  const int row = blockIdx.x;  // b*S + n
  const int b = row / S, n = row - b * S;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  s6_pdl_trigger();
  s6_pdl_wait();                 // U comes from the GEMM before us
  float u[4][8];
  const float* up = U + (size_t)row * u_ld + lane * 8;
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    float4 a = *reinterpret_cast<const float4*>(up + h * 256);
    float4 c = *reinterpret_cast<const float4*>(up + h * 256 + 4);
    u[h][0] = a.x; u[h][1] = a.y; u[h][2] = a.z; u[h][3] = a.w;
    u[h][4] = c.x; u[h][5] = c.y; u[h][6] = c.z; u[h][7] = c.w;
  }
  const ET* Erow = E + (size_t)row * S * 256 + lane * 8;
  float* out = SP + ((size_t)b * 4 * S + n) * S;  // + h*S*S + m
  for (int m0 = warp * 4; m0 < S; m0 += 32) {
    float e[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int m = min(m0 + i, S - 1);
      load8<ET>(Erow + (size_t)m * 256, e[i]);
    }
    float acc[16];  // index i*4 + h
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) s = fmaf(u[h][c], e[i][c], s);
        acc[i * 4 + h] = s;
      }
    // transpose-reduce 16 values over 32 lanes: after the 4 halving steps lane l holds value (l >> 1) & 15
    // summed over half the lanes; one more xor-1 step completes it.
#pragma unroll
    for (int step = 0; step < 4; ++step) {
      const int o = 16 >> step;             // lane distance 16, 8, 4, 2
      const int half = 8 >> step;           // values kept: 8, 4, 2, 1
      const bool upper = (lane & o) != 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (i < half) {
          float send = upper ? acc[i] : acc[i + half];
          float keep = upper ? acc[i + half] : acc[i];
          acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
      }
    }
    float tot = acc[0] + __shfl_xor_sync(0xffffffffu, acc[0], 1);
    // value index held by this lane: bit3 = lane&16, bit2 = lane&8, bit1 = lane&4, bit0 = lane&2
    const int vi = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
    const int i = vi >> 2, h = vi & 3, m = m0 + i;
    if ((lane & 1) == 0 && m < S) out[(size_t)h * S * S + m] = tot;
  }
}

// ------------------------------------------------------------------------------------------
// mha.  grid = (ceil(Sq/32), B*H); K_h, V_h of the cloud staged once per 32 queries in shared memory.
// Each warp owns 4 queries at a time: a lane holds one key (QK^T) / two output channels (PV) for all four, so every K / V
// word read from shared memory feeds 4 FMAs and the query / probability operands arrive as one broadcast LDS.128.
// ------------------------------------------------------------------------------------------
constexpr int MHA_QT = 32;    // queries per CTA (4 per warp)
constexpr int MHA_MAXK = 256; // keys per cloud supported by the register tile (8 per lane)
constexpr int MHA_KP = 68;    // padded K row (floats): 16-byte aligned, conflict-free for LDS.128 across lanes

__global__ void __launch_bounds__(256) mha_kernel(const float* __restrict__ Q, long long q_ld, long long q_bs,
                                                  const float* __restrict__ K, long long k_ld, long long k_bs,
                                                  const float* __restrict__ V, long long v_ld, long long v_bs,
                                                  const float* __restrict__ bias,  // (B,H,Sq,Sk) or null
                                                  int H, int Sq, int Sk, float scale, float* __restrict__ O, long long o_ld,
                                                  long long o_bs) {
  extern __shared__ __align__(16) float sm[];
  constexpr int D = 64;
  float* ks = sm;                       // Sk * MHA_KP
  float* vs = ks + Sk * MHA_KP;         // Sk * D
  float* qs = vs + Sk * D;              // 8 warps * [D][4]   (4 queries interleaved per channel)
  float* ps = qs + 8 * D * 4;           // 8 warps * [MHA_MAXK][4]
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int q0 = blockIdx.x * MHA_QT;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* Kb = K + (size_t)b * k_bs + h * D;
  const float* Vb = V + (size_t)b * v_bs + h * D;
  for (int e = tid; e < Sk * (D / 4); e += 256) {
    int m = e / (D / 4), c4 = (e - m * (D / 4)) * 4;
    *reinterpret_cast<float4*>(ks + m * MHA_KP + c4) = *reinterpret_cast<const float4*>(Kb + (size_t)m * k_ld + c4);
    *reinterpret_cast<float4*>(vs + m * D + c4) = *reinterpret_cast<const float4*>(Vb + (size_t)m * v_ld + c4);
  }
  float* qw = qs + warp * D * 4;
  float* pw = ps + warp * MHA_MAXK * 4;
  const int n0 = q0 + warp * 4;
  for (int e = lane; e < D * 4; e += 32) {
    int c = e >> 2, qi = e & 3;
    int n = n0 + qi;
    qw[e] = (n < Sq) ? Q[(size_t)b * q_bs + (size_t)n * q_ld + h * D + c] : 0.f;
  }
  __syncthreads();
  if (n0 >= Sq) return;
  float s[MHA_MAXK / 32][4];
  float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
#pragma unroll
  for (int t = 0; t < MHA_MAXK / 32; ++t) {
    const int m = lane + 32 * t;
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    if (m < Sk) {
      const float* kr = ks + m * MHA_KP;
#pragma unroll 4
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
#pragma unroll
      for (int qi = 0; qi < 4; ++qi) {
        const int n = min(n0 + qi, Sq - 1);
        if (bias) a[qi] += bias[(((size_t)b * H + h) * Sq + n) * Sk + m];
        a[qi] *= scale;
      }
    } else {
#pragma unroll
      for (int qi = 0; qi < 4; ++qi) a[qi] = -INFINITY;
    }
#pragma unroll
    for (int qi = 0; qi < 4; ++qi) { s[t][qi] = a[qi]; mx[qi] = fmaxf(mx[qi], a[qi]); }
  }
  float sum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int qi = 0; qi < 4; ++qi) mx[qi] = warp_max(mx[qi]);
#pragma unroll
  for (int t = 0; t < MHA_MAXK / 32; ++t) {
    const int m = lane + 32 * t;
#pragma unroll
    for (int qi = 0; qi < 4; ++qi) {
      float e = (m < Sk) ? __expf(s[t][qi] - mx[qi]) : 0.f;
      s[t][qi] = e;
      sum[qi] += e;
    }
  }
#pragma unroll
  for (int qi = 0; qi < 4; ++qi) sum[qi] = 1.f / warp_sum(sum[qi]);
#pragma unroll
  for (int t = 0; t < MHA_MAXK / 32; ++t) {
    const int m = lane + 32 * t;
    if (m < Sk) *reinterpret_cast<float4*>(pw + m * 4) = make_float4(s[t][0] * sum[0], s[t][1] * sum[1], s[t][2] * sum[2], s[t][3] * sum[3]);
  }
  __syncwarp();
  float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
  for (int m = 0; m < Sk; ++m) {
    const float4 p = *reinterpret_cast<const float4*>(pw + m * 4);
    const float v0 = vs[m * D + lane], v1 = vs[m * D + lane + 32];
    o0[0] = fmaf(p.x, v0, o0[0]); o0[1] = fmaf(p.y, v0, o0[1]); o0[2] = fmaf(p.z, v0, o0[2]); o0[3] = fmaf(p.w, v0, o0[3]);
    o1[0] = fmaf(p.x, v1, o1[0]); o1[1] = fmaf(p.y, v1, o1[1]); o1[2] = fmaf(p.z, v1, o1[2]); o1[3] = fmaf(p.w, v1, o1[3]);
  }
#pragma unroll
  for (int qi = 0; qi < 4; ++qi) {
    const int n = n0 + qi;
    if (n < Sq) {
      float* op = O + (size_t)b * o_bs + (size_t)n * o_ld + h * D;
      op[lane] = o0[qi];
      op[lane + 32] = o1[qi];
    }
  }
}

// ------------------------------------------------------------------------------------------
// focused linear attention, kv-first branch (transformer.py:552-559):
//   z = 1 / (q . sum_j k_j + 1e-6);  kv = sum_j k_j v_j^T (per head, d x d);  x = (q kv) z
// linattn_kv : grid = B*H, builds KV (B,H,64,64) and KS (B,H,64) from the <= few-hundred sparse tokens.
// linattn_apply : one warp per dense token.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) linattn_kv_kernel(const float* __restrict__ Kf, long long k_ld, long long k_bs,
                                                         const float* __restrict__ V, long long v_ld, long long v_bs, int H, int J,
                                                         float* __restrict__ KV, float* __restrict__ KS) {
  constexpr int D = 64;
  extern __shared__ float sm[];
  float* ks = sm;           // J * D
  float* vs = ks + J * D;   // J * D
  const int bh = blockIdx.x, b = bh / H, h = bh - b * H, tid = threadIdx.x;
  for (int e = tid; e < J * D; e += 256) {
    int j = e / D, c = e - j * D;
    ks[e] = Kf[(size_t)b * k_bs + (size_t)j * k_ld + h * D + c];
    vs[e] = V[(size_t)b * v_bs + (size_t)j * v_ld + h * D + c];
  }
  __syncthreads();
  // thread -> (c, d-block of 16): 64 x 4 = 256 threads
  const int c = tid >> 2, d0 = (tid & 3) * 16;
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  float ksum = 0.f;
  for (int j = 0; j < J; ++j) {
    float kc = ks[j * D + c];
    ksum += kc;
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = fmaf(kc, vs[j * D + d0 + i], acc[i]);
  }
  float* o = KV + ((size_t)bh * D + c) * D + d0;
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i] = acc[i];
  if ((tid & 3) == 0) KS[(size_t)bh * D + c] = ksum;
}

__global__ void __launch_bounds__(256) linattn_apply_kernel(const float* __restrict__ Qf, long long q_rpb, long long q_bs, long long q_ld,
                                                            const float* __restrict__ KV, const float* __restrict__ KS, int H,
                                                            long long rows, float* __restrict__ X, long long x_rpb,
                                                            long long x_bs, long long x_ld) {
  constexpr int D = 64;
  extern __shared__ float sm[];  // KV of this cloud: H*D*D, then KS: H*D
  const int b = blockIdx.y;
  float* kv = sm;
  float* ksm = kv + H * D * D;
  for (int e = threadIdx.x; e < H * D * D; e += 256) kv[e] = KV[(size_t)b * H * D * D + e];
  for (int e = threadIdx.x; e < H * D; e += 256) ksm[e] = KS[(size_t)b * H * D + e];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long i = (long long)blockIdx.x * 8 + warp; i < q_rpb; i += (long long)gridDim.x * 8) {
    const float* q = Qf + (size_t)b * q_bs + (size_t)i * q_ld;
    float* x = X + (size_t)b * x_bs + (size_t)i * x_ld;
    for (int h = 0; h < H; ++h) {
      float q0 = q[h * D + lane], q1 = q[h * D + lane + 32];
      float zden = warp_sum(q0 * ksm[h * D + lane] + q1 * ksm[h * D + lane + 32]);
      float z = 1.f / (zden + 1e-6f);
      float o0 = 0.f, o1 = 0.f;
      const float* kvh = kv + h * D * D;
#pragma unroll 8
      for (int c = 0; c < D; ++c) {
        float qc = __shfl_sync(0xffffffffu, (c < 32) ? q0 : q1, c & 31);
        o0 = fmaf(qc, kvh[c * D + lane], o0);
        o1 = fmaf(qc, kvh[c * D + lane + 32], o1);
      }
      x[h * D + lane] = o0 * z;
      x[h * D + lane + 32] = o1 * z;
    }
  }
}

}  // namespace

// E (B,S,S,256) [f32 or bf16], U (B,S,4,256) f32 -> SP (B,4,S,S) f32
S6_API int sam6d_rpe_scores(const void* E, int e_is_bf16, const float* U, long long u_ld, int B, int S, float* SP, void* stream) {
  S6_REQUIRE(E && U && SP && B >= 0 && S > 0 && u_ld >= 1024 && (u_ld % 4) == 0);
  // U and E rows are read with 16-byte loads
  S6_REQUIRE(((reinterpret_cast<uintptr_t>(U) | reinterpret_cast<uintptr_t>(E)) & 15) == 0);
  if (B == 0) return 0;
  if (e_is_bf16)
    S6_CHECK(s6_launch_pdl(rpe_scores_kernel<__nv_bfloat16>, dim3(B * S), dim3(256), 0, s6_stream(stream), (const __nv_bfloat16*)E, U,
                           u_ld, S, SP));
  else
    S6_CHECK(s6_launch_pdl(rpe_scores_kernel<float>, dim3(B * S), dim3(256), 0, s6_stream(stream), (const float*)E, U, u_ld, S, SP));
  S6_LAUNCH_CHECK();
  return 0;
}

// O[b,n,h*64:(h+1)*64] = softmax_m((Q_h[b,n] . K_h[b,m] + bias[b,h,n,m]) * scale) V_h[b,m];  head dim 64.
S6_API int sam6d_mha(const float* Q, long long q_ld, long long q_bs, const float* K, long long k_ld, long long k_bs,
                     const float* V, long long v_ld, long long v_bs, const float* bias, int B, int H, int Sq, int Sk,
                     float scale, float* O, long long o_ld, long long o_bs, void* stream) {
  S6_REQUIRE(Q && K && V && O && B >= 0 && H > 0 && Sq > 0 && Sk > 0 && Sk <= MHA_MAXK);
  S6_REQUIRE((k_ld % 4 == 0) && (v_ld % 4 == 0) && (k_bs % 4 == 0) && (v_bs % 4 == 0));
  // K and V are staged with 16-byte loads; B*H is grid.y
  S6_REQUIRE(((reinterpret_cast<uintptr_t>(K) | reinterpret_cast<uintptr_t>(V)) & 15) == 0);
  S6_REQUIRE((long long)B * H <= 65535);
  if (B == 0) return 0;
  size_t smem = ((size_t)Sk * (MHA_KP + 64) + 8 * 64 * 4 + 8 * MHA_MAXK * 4) * sizeof(float);
  S6_CHECK(cudaFuncSetAttribute(mha_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(s6_cdiv(Sq, MHA_QT), B * H);
  mha_kernel<<<grid, 256, smem, s6_stream(stream)>>>(Q, q_ld, q_bs, K, k_ld, k_bs, V, v_ld, v_bs, bias, H, Sq, Sk, scale, O,
                                                     o_ld, o_bs);
  S6_LAUNCH_CHECK();
  return 0;
}

// Kf, V: (B,J,H*64) views -> KV (B,H,64,64), KS (B,H,64)
S6_API int sam6d_linattn_kv(const float* Kf, long long k_ld, long long k_bs, const float* V, long long v_ld, long long v_bs,
                            int B, int H, int J, float* KV, float* KS, void* stream) {
  S6_REQUIRE(Kf && V && KV && KS && B >= 0 && H > 0 && J > 0);
  if (B == 0) return 0;
  size_t smem = (size_t)2 * J * 64 * sizeof(float);
  S6_REQUIRE(smem <= 200 * 1024);
  S6_CHECK(cudaFuncSetAttribute(linattn_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  linattn_kv_kernel<<<B * H, 256, smem, s6_stream(stream)>>>(Kf, k_ld, k_bs, V, v_ld, v_bs, H, J, KV, KS);
  S6_LAUNCH_CHECK();
  return 0;
}

// Qf: B clouds x q_rpb tokens (batch stride q_bs, row stride q_ld) -> X same addressing scheme
S6_API int sam6d_linattn_apply(const float* Qf, long long q_rpb, long long q_bs, long long q_ld, const float* KV, const float* KS,
                               int B, int H, float* X, long long x_bs, long long x_ld, void* stream) {
  S6_REQUIRE(Qf && KV && KS && X && B >= 0 && H > 0 && q_rpb >= 0);
  if (B == 0 || q_rpb == 0) return 0;
  size_t smem = ((size_t)H * 64 * 64 + H * 64) * sizeof(float);
  S6_CHECK(cudaFuncSetAttribute(linattn_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(min(64, s6_cdiv(q_rpb, 8)), B);
  linattn_apply_kernel<<<grid, 256, smem, s6_stream(stream)>>>(Qf, q_rpb, q_bs, q_ld, KV, KS, H, (long long)B * q_rpb, X, q_rpb,
                                                              x_bs, x_ld);
  S6_LAUNCH_CHECK();
  return 0;
}
