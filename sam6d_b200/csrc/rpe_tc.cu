// rpe_tc.cu -- the relative-position score term of RPEMultiHeadAttention on TMA + wgmma (bf16 path).
//
//   s_p[b,h,n,m] = q_h[b,n,:] . proj_p(E[b,n,m,:])_h = u_h[b,n,:] . E[b,n,m,:],   u_h = W_p,h^T q_h      (PEM/model/transformer.py:369-399)
//
// E (clouds, S, S, 256) bf16 is the 1.27 GB pair embedding: this kernel is the one streaming pass over it per self-attention
// layer, bound by HBM bandwidth.  The CUDA-core version (attn.cu: rpe_scores_kernel) spends one LDG.128 + 4 unpack + 32 FMA +
// a 16-value shuffle transpose per 8 channels.  Here no CUDA core touches E:
//   * a query row (b, n) owns the contiguous S x 256 bf16 block E[b, n, :, :] (100 KB).  The TMA unit drops it into shared
//     memory as four K-major SWIZZLE_128B slabs [keys][64 channels] -- exactly the A operand of a wgmma with M = keys;
//   * the four per-head folded queries u_h[b,n,:] (4 x 256 bf16 = 2 KB, contiguous in the projection GEMM's output) arrive by TMA
//     as rows 0..3 of a 16-row B operand whose other rows stay zero;
//   * D^T[m, h] = sum_c E[n,m,c] u_h[c]: per 64-key block 16 x wgmma m64n16k16 into 8 registers per thread; lane = key, so the
//     threads holding a head's column write adjacent keys of s_p[b, h, n, :].
// Persistent: one CTA per SM walks a contiguous range of the clouds*S query rows (rows are independent); warp 4 feeds a 2-stage
// TMA ring, warps 0-3 (one warpgroup) run the MMAs and the stores.
#include "tc.cuh"

namespace {

constexpr int C = 256, KSLABS = C / 64;
constexpr int SLAB_ROWS = 200;                        // keys per slab (S <= 200), 25 swizzle atoms
constexpr int SLAB_BYTES = SLAB_ROWS * 128;           // 25600
constexpr int E_BYTES = KSLABS * SLAB_BYTES;          // 102400
constexpr int NB = 16;                                // MMA N: 4 heads + 12 zero rows
constexpr int U_SLAB = NB * 128, U_BYTES = KSLABS * U_SLAB;   // 8192
constexpr int STAGE_BYTES = E_BYTES + U_BYTES;        // 110592
constexpr int STAGES = 2;
constexpr int THREADS = 128 + 32;
constexpr int SMEM = STAGES * STAGE_BYTES + 1024;

__global__ void __launch_bounds__(THREADS, 1) rpe_scores_tc_kernel(const __grid_constant__ CUtensorMap tmE,
                                                                   const __grid_constant__ CUtensorMap tmU, int S, int total_rows,
                                                                   float* __restrict__ SP, int sp_ld) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // contiguous, balanced row range of this CTA
  const int per = total_rows / gridDim.x, rem = total_rows % gridDim.x;
  const int r0 = blockIdx.x * per + min((int)blockIdx.x, rem), nrows = per + ((int)blockIdx.x < rem ? 1 : 0);
  const int nblk = (S + 63) >> 6;                     // 64-key blocks (M of the MMA)

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], 4); }
    tc::mbar_fence_init();
    tc::tma_prefetch_desc(&tmE);
    tc::tma_prefetch_desc(&tmU);
  }
  s6_pdl_trigger();
  // rows 4..15 of every B slab are zero for the lifetime of the kernel (the TMA boxes only ever write rows 0..3)
  for (int i = tid; i < STAGES * U_BYTES / 16; i += THREADS) {
    const int s = i / (U_BYTES / 16), o = i - s * (U_BYTES / 16);
    *reinterpret_cast<uint4*>(smem + s * STAGE_BYTES + E_BYTES + o * 16) = make_uint4(0, 0, 0, 0);
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  s6_pdl_wait();                                      // u comes from the projection GEMM right before us

  if (warp == 4) {
    // ------------------------------------------------------------------ TMA producer: one query row per stage
    if (lane == 0) {
      const uint32_t tx = (uint32_t)(KSLABS * S * 128 + KSLABS * 4 * 128);
      for (int i = 0; i < nrows; ++i) {
        const int s = i % STAGES, row = r0 + i;
        tc::mbar_wait(&empty_bar[s], (uint32_t)(((i / STAGES) & 1) ^ 1));
        tc::mbar_arrive_expect_tx(&full_bar[s], tx);
        uint8_t* st = smem + s * STAGE_BYTES;
#pragma unroll
        for (int kb = 0; kb < KSLABS; ++kb) tc::tma_load_2d(&tmE, &full_bar[s], st + kb * SLAB_BYTES, kb * 64, row * S);
#pragma unroll
        for (int kb = 0; kb < KSLABS; ++kb) tc::tma_load_2d(&tmU, &full_bar[s], st + E_BYTES + kb * U_SLAB, kb * 64, row * 4);
      }
    }
    return;
  }
  // ------------------------------------------------------------------ warpgroup: MMAs and stores
  const size_t SS = (size_t)S * sp_ld;
  const int w = warp;
  for (int i = 0; i < nrows; ++i) {
    const int s = i % STAGES, row = r0 + i;
    tc::mbar_wait(&full_bar[s], (uint32_t)((i / STAGES) & 1));
    const uint32_t e_addr = tc::smem_u32(smem + s * STAGE_BYTES), u_addr = e_addr + E_BYTES;
    float acc[4][NB / 2];
    tc::wg_fence();
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (t < nblk) {
#pragma unroll
        for (int kb = 0; kb < KSLABS; ++kb)
#pragma unroll
          for (int k = 0; k < 4; ++k)
            tc::wgmma_bf16<NB>(acc[t], tc::wg_desc(e_addr + kb * SLAB_BYTES + t * (64 * 128) + k * 32), tc::wg_desc(u_addr + kb * U_SLAB + k * 32),
                               (kb | k) ? 1u : 0u);
      }
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    if (lane == 0) tc::mbar_arrive(&empty_bar[s]);  // values are in registers: the producer may refill the stage
    // heads 0..3 are columns 0..3 of the fragment: elements 0..3 of the lanes with (lane & 3) < 2
    if ((lane & 3) < 2) {
      const int b = row / S, n = row - b * S;
      float* o = SP + ((size_t)b * 4 * S + n) * sp_ld;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int m = t * 64 + tc::frag_row(e, w, lane), h = tc::frag_col(e, lane);
          if (t < nblk && m < S) o[h * SS + m] = acc[t][e];
        }
      }
    }
  }
}

}  // namespace

// E (B,S,S,256) bf16 contiguous, U (B*S, 4*256) bf16 contiguous (row = the four folded per-head queries of a token)
// -> SP (B,4,S,sp_ld) fp32, sp_ld >= S (columns [S, sp_ld) are left untouched).  S <= 200.  The wgmma / TMA form of
// sam6d_rpe_scores (PEM/model/transformer.py:369-399); with sp_ld a multiple of 4 the attention kernel can stream the planes
// with 16-byte copies (sam6d_attn_tc_bias_ld)
S6_API int sam6d_rpe_scores_tc_ld(const void* E, const void* U, int B, int S, float* SP, int sp_ld, void* stream) {
  S6_REQUIRE(E && U && SP && B >= 0 && S > 0 && S <= SLAB_ROWS && sp_ld >= S);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(E) & 15) == 0 && (reinterpret_cast<uintptr_t>(U) & 15) == 0);
  S6_REQUIRE((long long)B * S * S < 2000000000LL);
  if (B == 0) return 0;
  CUtensorMap tmE, tmU;
  int rc = tc::make_map_2d(&tmE, E, (long long)B * S * S, C, C, 64, S);
  if (rc) return rc;
  rc = tc::make_map_2d(&tmU, U, (long long)B * S * 4, C, C, 64, 4);
  if (rc) return rc;
  const int total = B * S;
  int grid;
  S6_CHECK(s6_persistent_grid(total, 1, &grid));
  S6_CHECK(cudaFuncSetAttribute(rpe_scores_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  S6_CHECK(s6_launch_pdl(rpe_scores_tc_kernel, dim3(grid), dim3(THREADS), SMEM, s6_stream(stream), tmE, tmU, S, total, SP, sp_ld));
  S6_LAUNCH_CHECK();
  return 0;
}
