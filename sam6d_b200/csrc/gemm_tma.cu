// gemm_tma.cu -- persistent, TMA-fed bf16 GEMM on wgmma:   C = act(A W^T + bias) (+ R),   A (M,K) bf16, W (N,K) bf16.
//
// One CTA per SM loops over 128 x 256 output tiles (m fastest, so CTAs running together share the same W tile in L2):
//   warp 8      TMA producer : (one thread; its warpgroup hands its registers to the two below) cp.async.bulk.tensor 2-D boxes {64 k, 128 rows} of A and {64 k, 256 rows} of W, SWIZZLE_128B,
//                              straight into the K-major slabs of a 4-stage ring (48 KB per stage); out-of-range rows /
//                              columns are zero-filled by the TMA unit
//   warps 0..7  two consumer warpgroups: warpgroup g owns rows [64 g, 64 g + 64) of the tile, 4 x wgmma m64n256k16 per stage
//                              into 128 fp32 registers per thread; one wgmma group stays in flight while the stage before it is
//                              released; then alpha, bias, activation, residual -> fp32 or bf16 straight from the registers
//                              (epilogue.cuh) while the producer already fills the ring with the next tile
#include "epilogue.cuh"
#include "tc.cuh"

namespace {

constexpr int BM = 128, BN = 256, BK = 64, STAGES = 4;
constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int CONSUMERS = 256, THREADS = CONSUMERS + 128;
constexpr int SMEM = STAGES * STAGE_BYTES + 1024;

struct Args {
  const float* bias; const void* R; void* C;   // R has the element type of C
  int M, N, K;
  long long ldc, ldr;
  float alpha;
  int act;
  int batch;                 // independent problems stacked along the rows of A and W (score matrices: one per proposal)
  long long a_rpb, w_rpb;    // rows of A / W per problem (a tile may run into the next problem's rows: masked on store)
  long long c_bs, r_bs;      // element strides of C / R between problems
  // VT kernels: output columns >= vt_col0 are V of an attention layer and are written transposed, as the K-major B operand of
  // the P V MMA: vt[(cloud * vt_C + c) * vt_N1 + token], cloud = row / vt_S (saves the transpose pass over V)
  void* vt; int vt_col0, vt_S, vt_N1, vt_C;
  // ... and columns >= vt_col1 = vt_col0 + vt_C go to a SECOND row-major output c2 (ldc2), column j at c2[row * ldc2 + j - vt_col1]
  // (the folded rel-pos queries of an RPE layer: one launch projects q | k, V^T and u)
  int vt_col1; void* c2; long long ldc2;
};

template <typename OT, int ACT, bool HAS_BIAS, bool HAS_RES, bool VT = false>
__global__ void __launch_bounds__(THREADS, 1) gemm_tma_kernel(const __grid_constant__ CUtensorMap tmA,
                                                              const __grid_constant__ CUtensorMap tmW, Args g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m_tiles = (g.M + BM - 1) / BM, n_tiles = (g.N + BN - 1) / BN;
  const long long tpb = (long long)m_tiles * n_tiles, ntiles = tpb * g.batch;
  const int nkb = (g.K + BK - 1) / BK;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], CONSUMERS / 32); }
    tc::mbar_fence_init();
    tc::tma_prefetch_desc(&tmA);
    tc::tma_prefetch_desc(&tmW);
  }
  s6_pdl_trigger();
  __syncthreads();
  s6_pdl_wait();                                   // operands / residual may come from the kernel before us

  if (warp >= CONSUMERS / 32) {
    // ------------------------------------------------------------------ TMA producer (one thread of the third warpgroup)
    tc::producer_regs();
    if (tid == CONSUMERS) {
      long long gk = 0;
      for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long bz = tile / tpb, t = tile - bz * tpb;
        const int m0 = (int)(t % m_tiles) * BM, n0 = (int)(t / m_tiles) * BN;
        const int a_row = (int)(bz * g.a_rpb) + m0, w_row = (int)(bz * g.w_rpb) + n0;
        for (int kb = 0; kb < nkb; ++kb, ++gk) {
          const int s = (int)(gk % STAGES);
          tc::mbar_wait(&empty_bar[s], (uint32_t)(((gk / STAGES) & 1) ^ 1));
          tc::mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
          uint8_t* a_slab = smem + s * STAGE_BYTES;
          tc::tma_load_2d(&tmA, &full_bar[s], a_slab, kb * BK, a_row);
          tc::tma_load_2d(&tmW, &full_bar[s], a_slab + A_BYTES, kb * BK, w_row);
        }
      }
    }
    return;
  }
  // ------------------------------------------------------------------ consumers: warpgroup wg <-> rows [64 wg, 64 wg + 64)
  tc::consumer_regs();
  const int wg = warp >> 2, w = warp & 3;
  float acc[BN / 2];
  long long gk = 0;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long bz = tile / tpb, t = tile - bz * tpb;
    const int m0 = (int)(t % m_tiles) * BM, n0 = (int)(t / m_tiles) * BN;
    int prev = -1;
    for (int kb = 0; kb < nkb; ++kb, ++gk) {
      const int s = (int)(gk % STAGES);
      tc::mbar_wait(&full_bar[s], (uint32_t)((gk / STAGES) & 1));
      const uint32_t a_addr = tc::smem_u32(smem + s * STAGE_BYTES) + wg * (64 * 128), b_addr = tc::smem_u32(smem + s * STAGE_BYTES) + A_BYTES;
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) tc::wgmma_bf16<BN>(acc, tc::wg_desc(a_addr + k * 32), tc::wg_desc(b_addr + k * 32), (kb | k) ? 1u : 0u);
      tc::wg_commit();
      if (prev >= 0) {
        tc::wg_wait<1>();                          // the previous stage's MMAs are complete: hand it back to the producer
        if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);
      }
      prev = s;
    }
    tc::wg_wait<0>();
    if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);

    const int row0 = m0 + wg * 64;
    OT* Cb = reinterpret_cast<OT*>(g.C) + bz * g.c_bs;
    const OT* Rb = reinterpret_cast<const OT*>(g.R) + bz * g.r_bs;
    if constexpr (VT) {
      // 8-column groups below vt_col0 -> C, [vt_col0, vt_col1) -> V^T (transposed per cloud), from vt_col1 -> c2; the group
      // boundaries are multiples of 32 columns, so no group straddles two outputs
      const int jv = min(max((g.vt_col0 - n0) / 8, 0), BN / 8), ju = min(max((g.vt_col1 - n0) / 8, 0), BN / 8);
      epi::store_frag<OT, ACT, HAS_BIAS, false, OT, BN>(acc, w, lane, row0, g.M, n0, g.N, g.alpha, g.bias, nullptr, 0, Cb, g.ldc, 0, jv);
      epi::store_frag<OT, ACT, HAS_BIAS, false, OT, BN>(acc, w, lane, row0, g.M, n0 - g.vt_col1, g.N - g.vt_col1, g.alpha,
                                                        g.bias ? g.bias + g.vt_col1 : nullptr, nullptr, 0, reinterpret_cast<OT*>(g.c2),
                                                        g.ldc2, ju, BN / 8);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if (j < jv || j >= ju) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + tc::frag_row(2 * h, w, lane);
          if (row >= g.M) continue;
          const int cloud = row / g.vt_S, tok = row - cloud * g.vt_S;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = n0 + tc::frag_col(4 * j + e, lane);
            float x = acc[4 * j + 2 * h + e] * g.alpha;
            if constexpr (HAS_BIAS) x += __ldg(g.bias + col);
            reinterpret_cast<__nv_bfloat16*>(g.vt)[((size_t)cloud * g.vt_C + (col - g.vt_col0)) * g.vt_N1 + tok] =
                __float2bfloat16(epi::act_fn<ACT>(x));
          }
        }
      }
    } else if constexpr (ACT == 3) {
      // SwiGLU: N tile t holds the gate and up rows of hidden units [128 t, 128 t + 128) -> output columns n0 / 2 + [0, 128)
      epi::store_frag_swiglu(acc, w, lane, row0, g.M, n0, n0 / 2, g.alpha, g.bias, Cb, g.ldc);
    } else {
      epi::store_frag<OT, ACT, HAS_BIAS, HAS_RES, OT, BN>(acc, w, lane, row0, g.M, n0, g.N, g.alpha, g.bias, Rb, g.ldr, Cb, g.ldc);
    }
  }
}

int launch_gemm_tma(const void* A, const void* W, const float* bias, const void* R, void* C, int c_dtype, int M, int N, int K,
                    long long lda, long long ldw, long long ldc, long long ldr, int batch, long long a_rpb, long long w_rpb,
                    long long c_bs, long long r_bs, float alpha, int act, void* stream, void* vt = nullptr, int vt_col0 = 0, int vt_S = 1,
                    int vt_N1 = 0, int vt_col1 = -1, void* c2 = nullptr, long long ldc2 = 0) {
  S6_REQUIRE(A && W && C && M >= 0 && N > 0 && K > 0 && (K % 8) == 0 && (lda % 8) == 0 && (ldw % 8) == 0 && act >= 0 && act <= 3);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0 && batch >= 0);
  S6_REQUIRE(a_rpb * (long long)batch < 2000000000LL && w_rpb * (long long)batch < 2000000000LL);
  if (M == 0 || batch == 0) return 0;
  CUtensorMap tmA, tmW;
  const long long a_rows = batch > 1 ? a_rpb * (batch - 1) + M : M, w_rows = batch > 1 ? w_rpb * (batch - 1) + N : N;
  int rc = tc::make_map_2d(&tmA, A, a_rows, K, lda, 64, BM);
  if (rc) return rc;
  rc = tc::make_map_2d(&tmW, W, w_rows, K, ldw, 64, BN);
  if (rc) return rc;
  const long long ntiles = (long long)s6_cdiv(M, BM) * s6_cdiv(N, BN) * batch;
  int grid;
  S6_CHECK(s6_persistent_grid(ntiles, 1, &grid));
  if (vt_col1 < 0) vt_col1 = N;
  Args g{bias, R, C, M, N, K, ldc, ldr, alpha, act, batch, a_rpb, w_rpb, c_bs, r_bs, vt, vt_col0, vt_S, vt_N1, vt_col1 - vt_col0,
         vt_col1, c2, ldc2};
  cudaStream_t st = s6_stream(stream);
#define LAUNCH_ONE(OT, ACT, HB, HR, VTK)                                                                               \
  do {                                                                                                                 \
    auto k = gemm_tma_kernel<OT, ACT, HB, HR, VTK>;                                                                    \
    S6_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));                              \
    S6_CHECK(s6_launch_pdl(k, dim3(grid), dim3(THREADS), SMEM, st, tmA, tmW, g));                                      \
  } while (0)
#define LAUNCH_TMA(ACT, HB, HR)                                                                                        \
  do {                                                                                                                 \
    if (c_dtype) LAUNCH_ONE(__nv_bfloat16, ACT, HB, HR, false); else LAUNCH_ONE(float, ACT, HB, HR, false);           \
  } while (0)
  if (vt) {
    // V^T epilogue: bf16 output, bias, no activation / residual (the QKV and KV projections)
    S6_REQUIRE(c_dtype == 1 && bias && !R && act == 0 && batch == 1 && vt_col0 > 0 && vt_col0 < N && (vt_col0 % 32) == 0 && vt_S > 0 &&
               vt_N1 >= vt_S);
    S6_REQUIRE(vt_col1 > vt_col0 && vt_col1 <= N && (vt_col1 % 32) == 0 &&
               (vt_col1 == N || (c2 && (ldc2 % 8) == 0 && ldc2 >= N - vt_col1 && (reinterpret_cast<uintptr_t>(c2) & 15) == 0)));
    LAUNCH_ONE(__nv_bfloat16, 0, true, false, true);
    S6_LAUNCH_CHECK();
    return 0;
  }
  if (act == 3) {
    // SwiGLU: bf16 output of N / 2 columns, bias, no residual; every N tile holds 128 gate rows then their 128 up rows
    S6_REQUIRE(c_dtype == 1 && bias && !R && (N % BN) == 0 && (ldc % 2) == 0 && ldc >= N / 2);
    LAUNCH_ONE(__nv_bfloat16, 3, true, false, false);
    S6_LAUNCH_CHECK();
    return 0;
  }
  EPI_DISPATCH(act, bias, R, LAUNCH_TMA);
#undef LAUNCH_TMA
#undef LAUNCH_ONE
  S6_LAUNCH_CHECK();
  return 0;
}

}  // namespace

// A (M,K) bf16 lda, W (N,K) bf16 ldw, C (M,N) fp32 (c_dtype 0) or bf16 (1), bias (N) fp32 or NULL, R (M,N) or NULL: the
// residual has the element type of C (fp32 stream with fp32 output, bf16 stream with bf16 output).
// K % 8 == 0, lda % 8 == 0, ldw % 8 == 0, 16-byte aligned bases.  act: 0 none, 1 ReLU, 2 GELU(erf), 3 SwiGLU.
// act 3: W is a SwiGLU w12 with its rows interleaved in blocks of 128 (gate rows of hidden units [128t, 128t + 128), then their
// up rows), bias packed the same way; C (M, N/2) bf16 = silu(gate) * up with row stride ldc; N % 256 == 0, bias required,
// no residual, bf16 output only (-22 otherwise).
S6_API int sam6d_gemm_tma(const void* A, const void* W, const float* bias, const void* R, void* C, int c_dtype, int M, int N, int K,
                          long long lda, long long ldw, long long ldc, long long ldr, float alpha, int act, void* stream) {
  return launch_gemm_tma(A, W, bias, R, C, c_dtype, M, N, K, lda, ldw, ldc, ldr, 1, 0, 0, 0, 0, alpha, act, stream);
}

// `batch` independent problems C_z = act(alpha A_z W_z^T + bias) (+ R_z): problem z reads rows [z*a_rpb, z*a_rpb + M) of A and
// [z*w_rpb, z*w_rpb + N) of W (w_rpb = 0: shared W) (both matrices are the problems stacked along the rows) and writes C + z*c_bs (elements).
// The cosine score matrices of the matching stages: A = normalised scene tokens, W = normalised template tokens per proposal.
S6_API int sam6d_gemm_tma_batched(const void* A, const void* W, const float* bias, const void* R, void* C, int c_dtype, int M, int N,
                                  int K, long long lda, long long ldw, long long ldc, long long ldr, int batch, long long a_rpb,
                                  long long w_rpb, long long c_bs, long long r_bs, float alpha, int act, void* stream) {
  S6_REQUIRE(a_rpb >= M && (w_rpb >= N || w_rpb == 0));       // w_rpb = 0: one weight matrix shared by every problem
  return launch_gemm_tma(A, W, bias, R, C, c_dtype, M, N, K, lda, ldw, ldc, ldr, batch, a_rpb, w_rpb, c_bs, r_bs, alpha, act, stream);
}

// sam6d_gemm_tma for a fused QKV / KV projection (bf16 output, bias): columns [vt_col0, N) are the values of an attention layer
// and go to Vt instead of C, transposed per cloud of vt_S token rows: Vt[(cloud * (N - vt_col0) + c) * vt_N1 + token] -- the
// layout sam6d_transpose_tokens_bf16 produces and sam6d_attn_tc / sam6d_attn_global_tc consume.  The key-padding columns
// [vt_S, vt_N1) of Vt are not written (the caller keeps them finite, e.g. zeroed once).
S6_API int sam6d_gemm_tma_vt(const void* A, const void* W, const float* bias, void* C, int M, int N, int K, long long lda, long long ldw,
                             long long ldc, void* Vt, int vt_col0, int vt_S, int vt_N1, void* stream) {
  S6_REQUIRE(Vt != nullptr);
  return launch_gemm_tma(A, W, bias, nullptr, C, 1, M, N, K, lda, ldw, ldc, 0, 1, 0, 0, 0, 0, 1.f, 0, stream, Vt, vt_col0, vt_S, vt_N1);
}

// sam6d_gemm_tma_vt with a third column range: [0, vt_col0) -> C, [vt_col0, vt_col1) -> Vt (transposed per cloud), [vt_col1, N) ->
// C2 (M, N - vt_col1) bf16 with row stride ldc2.  One launch for the q | k | v | u projections of an RPE self-attention layer
// (PEM/model/transformer.py:369-394 with proj_p folded into the query).
S6_API int sam6d_gemm_tma_vt2(const void* A, const void* W, const float* bias, void* C, int M, int N, int K, long long lda, long long ldw,
                              long long ldc, void* Vt, int vt_col0, int vt_col1, int vt_S, int vt_N1, void* C2, long long ldc2,
                              void* stream) {
  S6_REQUIRE(Vt != nullptr && C2 != nullptr);
  return launch_gemm_tma(A, W, bias, nullptr, C, 1, M, N, K, lda, ldw, ldc, 0, 1, 0, 0, 0, 0, 1.f, 0, stream, Vt, vt_col0, vt_S, vt_N1, vt_col1,
                         C2, ldc2);
}
