// attn_tc.cu -- multi-head attention on the tensor cores (wgmma) for up to 256 keys per (batch, head):
//     O = softmax((Q K^T + bias) * scale) V (+ b_v)
// covering PEM's geometric-transformer self / cross attention (197 tokens, head dim 64, dense relative-position bias from
// rpe_scores; PEM/model/transformer.py:109-148, 369-406) and SAM's windowed attention (196 tokens, head dim 80, decomposed
// rel-pos bias; ISM/segment_anything/modeling/image_encoder.py:224-240, 325-361).
//
// One CTA per (128-query tile, head, batch); one thread of warpgroup 2 issues the TMA loads, warpgroup g (warps 4g..4g+3) owns queries
// [64 g, 64 g + 64) of the tile:
//   TMA      : Q tile, K tile (boxes of 64 channels x rows, SWIZZLE_128B) and V^T tiles (64 keys x D channels) land in
//              K-major slabs; V^T (channels x keys) is produced by a GEMM upstream so that P V is a K-major MMA
//   MMA 1    : S = Q K^T          wgmma m64n256k16 x D/16 into 128 registers per thread (columns past the keys are ignored)
//   softmax  : the whole score row sits in the registers of one quad (<= 256 keys), so it is a plain two-pass softmax (no online
//              rescaling): x = (s + bias) * scale, row max and sum by quad shuffles, P written as bf16 into the A-operand slabs
//              (they alias Q / K, dead once both warpgroups are past MMA 1)
//   MMA 2    : O = P V            wgmma m64nDk16 x keys/16
//   epilogue : O / rowsum (+ b_v; rows of P sum to 1, so the value bias moves out of the MMA), stored from the registers
// Rows of a tile that run past the batch (197 is not a multiple of 128) are computed on whatever the TMA box fetched (the
// next batch's finite rows or zero fill) and never stored; keys past Sk are masked to probability 0.
#include "epilogue.cuh"
#include "tc.cuh"

namespace {

constexpr int QT = 128, MAXK = 256;
constexpr int CONSUMERS = 256, NUM_THREADS = CONSUMERS + 128;   // warps 0-7 two MMA warpgroups, warp 8 TMA
constexpr int REL_SLAB = 32 * 128;                              // BIAS_MODE 2: [32 rows][64 ch] bf16 slab of a rel-pos table
constexpr int SCR_LD = 64;                                      // BIAS_MODE 2: per query row, Q rel_h^T (0..31) and Q rel_w^T (32..63)

struct AttnArgs {
  const float* bias;     // BIAS_MODE 1: (B,H,Sq,Sk) fp32
  const void* rel_blob;  // BIAS_MODE 2: rel_h, rel_w pre-packed on the host as bf16 wgmma slabs (2 x DS x [32][64], SWIZZLE_128B)
  const float* rel_unused;
  const void* q_rows;    // BIAS_MODE 2: the bf16 matrix Q is a column slice of (for the unscaled-q bias tables)
  long long q_ld;
  int q_col0;            // column of Q inside q_rows
  const float* bv;       // (H*D) value bias added to the output, or null
  void* out;             // (B*Sq, H*D) fp32 or bf16
  long long out_ld;
  int H, Sq, Sk, N1;     // N1 = Sk rounded up to 16
  int Hs, Ws;            // BIAS_MODE 2 window grid
  int k_col0;            // column of K inside its matrix (per head: + h*D)
  float scale;
  // extended form (sam6d_attn_tc_ex): the keys of batch b are rows [b*k_brows + k_row0, +Sk) of the K matrix and columns
  // [v_col0, v_col0 + Sk) of its V^T rows; lse (B,H,Sq) receives max + log(sum) of the scaled scores (natural log), so that a
  // caller can merge further keys (the 257th token of a DINOv2 sequence) into the result
  int k_brows, k_row0, v_col0;
  float* lse;
  long long bias_ld;     // BIAS_MODE 4: row stride of the bias planes (B,H,Sq,bias_ld), a multiple of 4 floats, >= Sk
};

// shared memory: [Q][K] (P aliases them once the score MMAs are done) [V^T: 4 slabs] (BIAS_MODE 2: [rel tables][T scratch])
template <int D>
__host__ __device__ constexpr int qkp_bytes(int N1) {
  return ((((D + 63) / 64) * (QT + N1) * 128 > 4 * QT * 128 ? ((D + 63) / 64) * (QT + N1) * 128 : 4 * QT * 128) + 1023) & ~1023;
}

template <int D, int BIAS_MODE, typename OT>
__global__ void __launch_bounds__(NUM_THREADS, 1) attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                                                const __grid_constant__ CUtensorMap tmVt, AttnArgs a) {
  constexpr int DS = (D + 63) / 64;                 // 64-channel slabs of Q / K
  constexpr int Q_SLAB = QT * 128, V_SLAB = D * 128, P_SLAB = QT * 128;
  const int K_SLAB = a.N1 * 128;                    // N1 is a multiple of 16 -> multiple of 2048 bytes: slabs stay 1024-aligned
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* q_s = smem;
  uint8_t* k_s = q_s + DS * Q_SLAB;
  uint8_t* p_s = smem;                              // 4 slabs [128 rows][64 keys]
  uint8_t* v_s = smem + qkp_bytes<D>(a.N1);         // 4 slabs [D rows][64 keys]
  uint8_t* rel_s = v_s + 4 * V_SLAB;                // BIAS_MODE 2: 2 tables x DS slabs [32 rows][64 ch]
  float* scr = reinterpret_cast<float*>(rel_s + 2 * DS * REL_SLAB);   // BIAS_MODE 2: [128][SCR_LD]
  __shared__ __align__(8) uint64_t load_bar;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.x * QT, h = blockIdx.y, b = blockIdx.z;
  const int nslab = (a.N1 + 63) / 64;

  if (tid == 0) {
    tc::mbar_init(&load_bar, 1);
    tc::mbar_fence_init();
  }
  s6_pdl_trigger();
  __syncthreads();
  s6_pdl_wait();                                   // Q / K / V^T / bias come from the kernels before us

  if (warp >= CONSUMERS / 32) {
    tc::producer_regs();
    if (tid == CONSUMERS) {
      // ---------------------------------------------------------------- TMA loads (one transaction barrier)
      uint32_t bytes = (uint32_t)(DS * (QT * 128) + DS * (a.N1 * 128) + nslab * V_SLAB);
      if (BIAS_MODE == 2) bytes += 2 * DS * REL_SLAB;
      tc::mbar_arrive_expect_tx(&load_bar, bytes);
      if (BIAS_MODE == 2) tc::bulk_load_1d(rel_s, a.rel_blob, 2 * DS * REL_SLAB, &load_bar);
#pragma unroll
      for (int s = 0; s < DS; ++s) {
        tc::tma_load_2d(&tmQ, &load_bar, q_s + s * Q_SLAB, a.q_col0 + h * D + s * 64, b * a.Sq + n0);
        tc::tma_load_2d(&tmK, &load_bar, k_s + s * K_SLAB, a.k_col0 + h * D + s * 64, b * a.k_brows + a.k_row0);
      }
      for (int s = 0; s < nslab; ++s) tc::tma_load_2d(&tmVt, &load_bar, v_s + s * V_SLAB, a.v_col0 + s * 64, (b * a.H + h) * D);
    }
    return;
  }
  // ------------------------------------------------------------------ warpgroup wg <-> queries [64 wg, 64 wg + 64) of the tile
  tc::consumer_regs();
  const int wg = warp >> 2, w = warp & 3;
  const int Sk = a.Sk;
  tc::mbar_wait(&load_bar, 0);
  // ---------------------------------------------------------------- S = Q K^T (columns >= N1 read past the K slab: ignored)
  float sacc[MAXK / 2];
  {
    const uint32_t q_addr = tc::smem_u32(q_s) + wg * (64 * 128), k_addr = tc::smem_u32(k_s);
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k) {
      const int sl = k >> 2, kk = k & 3;
      tc::wgmma_bf16<MAXK>(sacc, tc::wg_desc(q_addr + sl * Q_SLAB + kk * 32), tc::wg_desc(k_addr + sl * K_SLAB + kk * 32), k ? 1u : 0u);
    }
    tc::wg_commit();
    if (BIAS_MODE == 2) {
      // decomposed rel-pos: T_h = Q rel_h^T, T_w = Q rel_w^T (64 x 32 each per warpgroup) -> scr[row][0..31], [32..63]
      float tacc[2][16];
#pragma unroll
      for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int k = 0; k < D / 16; ++k) {
          const int sl = k >> 2, kk = k & 3;
          tc::wgmma_bf16<32>(tacc[t], tc::wg_desc(q_addr + sl * Q_SLAB + kk * 32),
                             tc::wg_desc(tc::smem_u32(rel_s + (t * DS + sl) * REL_SLAB) + kk * 32), k ? 1u : 0u);
        }
      tc::wg_commit();
      tc::wg_wait<0>();
#pragma unroll
      for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int e = 0; e < 16; ++e) scr[(wg * 64 + tc::frag_row(e, w, lane)) * SCR_LD + t * 32 + tc::frag_col(e, lane)] = tacc[t][e];
      tc::named_bar(1 + wg, 128);
    } else {
      tc::wg_wait<0>();
    }
  }
  // ---------------------------------------------------------------- softmax over the thread's two rows
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int r = wg * 64 + tc::frag_row(2 * hr, w, lane), n = n0 + r, nq = min(n, a.Sq - 1);
    const float* brow = nullptr;
    if (BIAS_MODE == 1) brow = a.bias + (((size_t)b * a.H + h) * a.Sq + nq) * Sk;
    if (BIAS_MODE == 4) brow = a.bias + (((size_t)b * a.H + h) * a.Sq + nq) * a.bias_ld;
    const float* trow = (BIAS_MODE == 2) ? scr + r * SCR_LD : nullptr;
    const int qh = (BIAS_MODE == 2) ? nq / a.Ws : 0, qw = (BIAS_MODE == 2) ? nq % a.Ws : 0;
#pragma unroll
    for (int j = 0; j < MAXK / 8; ++j) {
      const int col = tc::frag_col(4 * j, lane);
      float bb[2] = {0.f, 0.f};
      if (BIAS_MODE == 4 && col < Sk) { const float2 t = __ldg(reinterpret_cast<const float2*>(brow + col)); bb[0] = t.x; bb[1] = t.y; }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = col + e;
        float x = -INFINITY;
        if (c < Sk) {
          x = sacc[4 * j + 2 * hr + e];
          if (BIAS_MODE == 1) x += __ldg(brow + c);
          if (BIAS_MODE == 4) x += bb[e];
          x *= a.scale;
          if (BIAS_MODE == 2) { const int kh = c / a.Ws, kw = c - kh * a.Ws; x += trow[qh - kh + a.Hs - 1] + trow[32 + qw - kw + a.Ws - 1]; }
          mx[hr] = fmaxf(mx[hr], x);
        }
        sacc[4 * j + 2 * hr + e] = x;
      }
    }
    mx[hr] = tc::quad_max(mx[hr]);
  }
  tc::named_bar(3, CONSUMERS);                     // both warpgroups are past MMA 1: Q / K may be overwritten by P (ids 1, 2: per warpgroup)
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < MAXK / 8; ++j) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int r = wg * 64 + tc::frag_row(2 * hr, w, lane), col = tc::frag_col(4 * j, lane);
      const float p0 = (col < Sk) ? __expf(sacc[4 * j + 2 * hr] - mx[hr]) : 0.f;
      const float p1 = (col + 1 < Sk) ? __expf(sacc[4 * j + 2 * hr + 1] - mx[hr]) : 0.f;
      sum[hr] += p0 + p1;
      *reinterpret_cast<uint32_t*>(p_s + (col >> 6) * P_SLAB + tc::sw128_offset(r, col & 63)) = tc::pack_bf16(p0, p1);
    }
  }
  tc::fence_proxy_async_smem();
  tc::named_bar(1 + wg, 128);                      // this warpgroup's P rows are complete
  // ---------------------------------------------------------------- O = P V
  float oacc[D / 2];
  {
    const uint32_t p_addr = tc::smem_u32(p_s) + wg * (64 * 128), v_addr = tc::smem_u32(v_s);
    tc::wg_fence();
    const int ksteps = a.N1 / 16;
    for (int k = 0; k < ksteps; ++k) {
      const int sl = k >> 2, kk = k & 3;
      tc::wgmma_bf16<D>(oacc, tc::wg_desc(p_addr + sl * P_SLAB + kk * 32), tc::wg_desc(v_addr + sl * V_SLAB + kk * 32), k ? 1u : 0u);
    }
    tc::wg_commit();
    tc::wg_wait<0>();
  }
  // ---------------------------------------------------------------- epilogue
  const int m_lim = b * a.Sq + a.Sq;                                   // rows of the next batch are not ours
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const float t = tc::quad_sum(sum[hr]), inv = 1.f / t;
    const int n = n0 + wg * 64 + tc::frag_row(2 * hr, w, lane), row = b * a.Sq + n;
    if (a.lse && n < a.Sq && (lane & 3) == 0) a.lse[((size_t)b * a.H + h) * a.Sq + n] = mx[hr] + __logf(t);
    if (row >= m_lim) continue;
    OT* orow = reinterpret_cast<OT*>(a.out) + (size_t)row * a.out_ld + h * D;
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      const int col = tc::frag_col(4 * j, lane);
      float o0 = oacc[4 * j + 2 * hr] * inv, o1 = oacc[4 * j + 2 * hr + 1] * inv;
      if (a.bv) { o0 += __ldg(a.bv + h * D + col); o1 += __ldg(a.bv + h * D + col + 1); }
      epi::st2(orow + col, o0, o1);
    }
  }
}

template <int D, int BM, typename OT>
int launch(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnArgs& a, int B, cudaStream_t st) {
  constexpr int DS = (D + 63) / 64;
  size_t smem = (size_t)qkp_bytes<D>(a.N1) + (size_t)4 * D * 128 + 1024;
  if (BM == 2) smem += (size_t)2 * DS * REL_SLAB + (size_t)QT * SCR_LD * sizeof(float);
  if (smem > 227 * 1024) return S6_EINVAL;
  auto kern = attn_tc_kernel<D, BM, OT>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  dim3 grid(s6_cdiv(a.Sq, QT), a.H, B);
  cudaError_t le = s6_launch_pdl(kern, grid, dim3(NUM_THREADS), smem, st, tq, tk, tv, a);
  if (le != cudaSuccess) return (int)le;
  return (int)cudaGetLastError();
}

// out[(w*C + c), l] = src[(w*L + l), col0 + c] for l < L, 0 for L <= l < N1: V (tokens x channels) -> V^T (channels x keys)
__global__ void __launch_bounds__(256) transpose_tokens_kernel(const __nv_bfloat16* __restrict__ src, long long ld, int col0, int C,
                                                               int L, int N1, __nv_bfloat16* __restrict__ out) {
  __shared__ __nv_bfloat16 tile[64][66];
  const int w = blockIdx.z, c0 = blockIdx.y * 64, l0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  s6_pdl_trigger();
  s6_pdl_wait();
  for (int i = ty; i < 64; i += 4) {
    const int l = l0 + i, c = c0 + tx;
    tile[i][tx] = (l < L && c < C) ? src[((size_t)w * L + l) * ld + col0 + c] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int i = ty; i < 64; i += 4) {
    const int c = c0 + i, l = l0 + tx;
    if (c < C && l < N1) out[((size_t)w * C + c) * N1 + l] = tile[tx][i];
  }
}

}  // namespace

S6_API int sam6d_transpose_tokens_bf16(const void* src, long long ld, int col0, int C, int nB, int L, int N1, void* out, void* stream) {
  S6_REQUIRE(src && out && nB >= 0 && C > 0 && L > 0 && N1 >= L);
  if (nB == 0) return 0;
  S6_REQUIRE(nB <= 65535);
  dim3 grid(s6_cdiv(N1, 64), s6_cdiv(C, 64), nB);
  S6_CHECK(s6_launch_pdl(transpose_tokens_kernel, grid, dim3(256), 0, s6_stream(stream), reinterpret_cast<const __nv_bfloat16*>(src), ld,
                         col0, C, L, N1, reinterpret_cast<__nv_bfloat16*>(out)));
  S6_LAUNCH_CHECK();
  return 0;
}

namespace {
}  // namespace (the API below uses the helpers above)

// Q: bf16 matrix (B*Sq rows, q_ld) with head h at columns [q_col0 + h*D, +D); K likewise in (B*Sk rows, k_ld) at k_col0;
// Vt: bf16 (B*H*D rows, vt_ld >= N1) = V^T per (batch, head): row (b*H + h)*D + c holds channel c over the keys;
// bias_mode 0 none | 1 dense fp32 (B,H,Sq,Sk) | 2 decomposed rel-pos, Sq = Sk = Hs*Ws, rel_h = the two tables pre-packed as
// bf16 wgmma slabs (sam6d_b200.ops.pack_rel_pos: 2 x ceil(D/64) x [32 rows][64 ch], 128-byte swizzle), rel_w unused;
// bv (H*D) fp32 or NULL; out (B*Sq, H*D) fp32 or bf16 with row stride out_ld.  head_dim 64 or 80, Sk <= 256.
namespace {
int attn_tc_launch(const void* Q, long long q_ld, int q_col0, const void* K, long long k_ld, int k_col0, const void* Vt,
                   long long vt_ld, int B, int H, int Sq, int Sk, int head_dim, int bias_mode, const float* bias,
                   const void* rel_h, const float* rel_w, int Hs, int Ws, const float* bv, float scale, void* out,
                   int out_is_bf16, long long out_ld, int k_brows, int k_row0, int v_col0, float* lse, void* stream,
                   long long bias_ld = 0) {
  S6_REQUIRE(Q && K && Vt && out && B >= 0 && H > 0 && Sq > 0 && Sk > 0 && Sk <= MAXK);
  S6_REQUIRE((head_dim == 64 || head_dim == 80) && bias_mode >= 0 && bias_mode <= 4 && bias_mode != 3);
  if (bias_mode == 4)
    S6_REQUIRE(bias && head_dim == 64 && bias_ld >= Sk && (bias_ld % 4) == 0 && (reinterpret_cast<uintptr_t>(bias) & 15) == 0);
  S6_REQUIRE((q_ld % 8) == 0 && (k_ld % 8) == 0 && (vt_ld % 8) == 0 && (q_col0 % 8) == 0 && (k_col0 % 8) == 0);
  S6_REQUIRE(k_brows >= k_row0 + Sk && k_row0 >= 0 && v_col0 >= 0 && (v_col0 % 8) == 0);   // TMA boxes start on 16-byte boundaries
  if (bias_mode == 1) S6_REQUIRE(bias != nullptr);
  if (bias_mode == 2) S6_REQUIRE(rel_h && Hs > 0 && Ws > 0 && Hs <= 16 && Ws <= 16 && Hs * Ws == Sk && Sq == Sk && (reinterpret_cast<uintptr_t>(rel_h) & 15) == 0);
  if (B == 0) return 0;
  S6_REQUIRE(B <= 65535 && H <= 65535);
  const int N1 = (Sk + 15) & ~15;
  S6_REQUIRE(vt_ld >= v_col0 + N1);
  CUtensorMap tq, tk, tv;
  int rc = tc::make_map_2d(&tq, Q, (long long)B * Sq, q_ld, q_ld, 64, QT);
  if (rc) return rc;
  rc = tc::make_map_2d(&tk, K, (long long)B * k_brows, k_ld, k_ld, 64, N1);
  if (rc) return rc;
  rc = tc::make_map_2d(&tv, Vt, (long long)B * H * head_dim, vt_ld, vt_ld, 64, head_dim);
  if (rc) return rc;
  AttnArgs a{bias, rel_h, rel_w, Q, q_ld, q_col0, bv, out, out_ld, H, Sq, Sk, N1, Hs, Ws, k_col0, scale, k_brows, k_row0, v_col0, lse, bias_ld};   // mode 2: rel_h = packed blob
  cudaStream_t st = s6_stream(stream);
#define ATT_LAUNCH(DD, MM) (out_is_bf16 ? launch<DD, MM, __nv_bfloat16>(tq, tk, tv, a, B, st) : launch<DD, MM, float>(tq, tk, tv, a, B, st))
  if (head_dim == 64) {
    if (bias_mode == 0) return ATT_LAUNCH(64, 0);
    if (bias_mode == 1) return ATT_LAUNCH(64, 1);
    if (bias_mode == 4) return ATT_LAUNCH(64, 4);
    return ATT_LAUNCH(64, 2);
  }
  if (bias_mode == 0) return ATT_LAUNCH(80, 0);
  if (bias_mode == 1) return ATT_LAUNCH(80, 1);
  return ATT_LAUNCH(80, 2);
#undef ATT_LAUNCH
}

// out[b,n,h,:] <- (w_p out[b,n,h,:] + w_c v_c) / (w_p + w_c), w_p = exp(lse - m), w_c = exp(s_c - m), s_c = scale q.k_c: one more
// key (row key_row of every batch, V^T column key_col) folded into an attention result that came with its log-sum-exp.
// one warp per (b, n, h), head dim 64: lane l owns channels 2l, 2l+1.
__global__ void __launch_bounds__(256) attn_merge_key_kernel(const __nv_bfloat16* __restrict__ Q, long long q_ld, int q_col0,
                                                             const __nv_bfloat16* __restrict__ K, long long k_ld, int k_col0, int k_brows,
                                                             int key_row, const __nv_bfloat16* __restrict__ Vt, long long vt_ld, int key_col,
                                                             const float* __restrict__ lse, int B, int H, int Sq, float scale,
                                                             __nv_bfloat16* __restrict__ out, long long out_ld) {
  const long long w = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  s6_pdl_trigger();
  s6_pdl_wait();
  if (w >= (long long)B * Sq * H) return;
  const int h = (int)(w % H);
  const long long bn = w / H;
  const int n = (int)(bn % Sq), b = (int)(bn / Sq);
  const __nv_bfloat162 q2 = *reinterpret_cast<const __nv_bfloat162*>(Q + (size_t)bn * q_ld + q_col0 + h * 64 + lane * 2);
  const __nv_bfloat162 k2 = *reinterpret_cast<const __nv_bfloat162*>(K + ((size_t)b * k_brows + key_row) * k_ld + k_col0 + h * 64 + lane * 2);
  float s = __bfloat162float(q2.x) * __bfloat162float(k2.x) + __bfloat162float(q2.y) * __bfloat162float(k2.y);
  s = warp_sum(s) * scale;
  const float l = lse[((size_t)b * H + h) * Sq + n];
  const float m = fmaxf(l, s), wp = __expf(l - m), wc = __expf(s - m), inv = 1.f / (wp + wc);
  const __nv_bfloat16* vrow = Vt + ((size_t)(b * H + h) * 64 + lane * 2) * vt_ld + key_col;
  const float v0 = __bfloat162float(vrow[0]), v1 = __bfloat162float(vrow[vt_ld]);
  __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(out + (size_t)bn * out_ld + h * 64 + lane * 2);
  const __nv_bfloat162 o2 = *o;
  *o = __floats2bfloat162_rn((wp * __bfloat162float(o2.x) + wc * v0) * inv, (wp * __bfloat162float(o2.y) + wc * v1) * inv);
}
}  // namespace

S6_API int sam6d_attn_tc(const void* Q, long long q_ld, int q_col0, const void* K, long long k_ld, int k_col0, const void* Vt,
                         long long vt_ld, int B, int H, int Sq, int Sk, int head_dim, int bias_mode, const float* bias,
                         const void* rel_h, const float* rel_w, int Hs, int Ws, const float* bv, float scale, void* out,
                         int out_is_bf16, long long out_ld, void* stream) {
  return attn_tc_launch(Q, q_ld, q_col0, K, k_ld, k_col0, Vt, vt_ld, B, H, Sq, Sk, head_dim, bias_mode, bias, rel_h, rel_w, Hs, Ws, bv,
                        scale, out, out_is_bf16, out_ld, Sk, 0, 0, nullptr, stream);
}

// sam6d_attn_tc with a dense fp32 bias whose planes are PADDED: (B,H,Sq,bias_ld), bias_ld >= Sk a multiple of 4 floats, base
// 16-byte aligned (what sam6d_rpe_scores_tc_ld writes).  Head dim 64.  The bias is then read as aligned column pairs.
S6_API int sam6d_attn_tc_bias_ld(const void* Q, long long q_ld, int q_col0, const void* K, long long k_ld, int k_col0, const void* Vt,
                                 long long vt_ld, int B, int H, int Sq, int Sk, int head_dim, const float* bias, long long bias_ld,
                                 float scale, void* out, int out_is_bf16, long long out_ld, void* stream) {
  return attn_tc_launch(Q, q_ld, q_col0, K, k_ld, k_col0, Vt, vt_ld, B, H, Sq, Sk, head_dim, 4, bias, nullptr, nullptr, 0, 0, nullptr,
                        scale, out, out_is_bf16, out_ld, Sk, 0, 0, nullptr, stream, bias_ld);
}

// sam6d_attn_tc without bias over a WINDOW of keys: batch b's keys are rows [b*k_brows + k_row0, +Sk) of K and columns
// [v_col0, +Sk) of its V^T rows; lse (B,H,Sq) f32 (or NULL) receives the log-sum-exp of the scaled scores.
S6_API int sam6d_attn_tc_ex(const void* Q, long long q_ld, int q_col0, const void* K, long long k_ld, int k_col0, const void* Vt,
                            long long vt_ld, int B, int H, int Sq, int Sk, int head_dim, float scale, int k_brows, int k_row0, int v_col0,
                            float* lse, void* out, int out_is_bf16, long long out_ld, void* stream) {
  return attn_tc_launch(Q, q_ld, q_col0, K, k_ld, k_col0, Vt, vt_ld, B, H, Sq, Sk, head_dim, 0, nullptr, nullptr, nullptr, 0, 0, nullptr,
                        scale, out, out_is_bf16, out_ld, k_brows, k_row0, v_col0, lse, stream);
}

// folds ONE more key (row key_row of every batch's K rows, column key_col of its V^T rows) into a bf16 attention result `out`
// (B*Sq, H*64) produced by sam6d_attn_tc_ex with its lse: the 257-token sequences of DINOv2 ViT-L/14 (256 patch keys on the
// tensor cores + the class token here).  head dim 64.
S6_API int sam6d_attn_merge_key(const void* Q, long long q_ld, int q_col0, const void* K, long long k_ld, int k_col0, int k_brows,
                                int key_row, const void* Vt, long long vt_ld, int key_col, const float* lse, int B, int H, int Sq,
                                float scale, void* out, long long out_ld, void* stream) {
  S6_REQUIRE(Q && K && Vt && lse && out && B >= 0 && H > 0 && Sq > 0 && (q_ld % 2) == 0 && (k_ld % 2) == 0 && (out_ld % 2) == 0 &&
             (q_col0 % 2) == 0 && (k_col0 % 2) == 0);
  if (B == 0) return 0;
  const long long warps = (long long)B * Sq * H;
  S6_CHECK(s6_launch_pdl(attn_merge_key_kernel, dim3(s6_cdiv(warps, 8)), dim3(256), 0, s6_stream(stream),
                         reinterpret_cast<const __nv_bfloat16*>(Q), q_ld, q_col0, reinterpret_cast<const __nv_bfloat16*>(K), k_ld, k_col0,
                         k_brows, key_row, reinterpret_cast<const __nv_bfloat16*>(Vt), vt_ld, key_col, lse, B, H, Sq, scale,
                         reinterpret_cast<__nv_bfloat16*>(out), out_ld));
  S6_LAUNCH_CHECK();
  return 0;
}
