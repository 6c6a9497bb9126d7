// fine_tc.cu -- the dual-softmax assignment of compute_fine_Rt (PEM/utils/model_utils.py:250-283) without the score matrix.
//
// The reference forms A = F1 F2^T / temp ((B, 2049, 2049) fp32, 538 MB at B = 32) and walks it about a dozen times.  Here the
// normalised bf16 tokens are the only inputs and every pass recomputes its score tile on the tensor cores (69 GFLOP per pass)
// and reduces it while it is still in registers; nothing of size S x S ever reaches HBM.
//
//   pass ROWSUM (mode 0)   inv[b,i] = 1 / sum_j e_ij,  e_ij = exp(alpha * <a_i, b_j> - shift)     (shift = 1/temp >= any score)
//   pass ARGMAX (mode 1)   lab[b,i] = argmax_j P_ij (first maximum),  P_ij = (e_ij * rowf_i) * (e_ij * colf_j)
//   pass ASSIGN (mode 2)   ARGMAX plus  w_i = sum_j P_ij q4_j.w,  pred_i = sum_j P_ij q4_j.xyz / (w_i + 1e-6)   for rows i >= 1
//
// Column sums and column labels are the same passes with the two token matrices swapped (the score matrix of the swapped pair
// is the transpose), so compute_fine_Rt is: ROWSUM(F1,F2), ROWSUM(F2,F1), ARGMAX(F2,F1), masked points, ASSIGN(F1,F2).
//
// One persistent CTA per SM walks work items (cloud b, 128-row tile); the row tile (4 k-blocks of A, 64 KB) stays in shared
// memory while the 256-column tiles of B stream through a 4-stage TMA ring fed by one thread of warpgroup 2.  Warpgroup g (warps 4g..4g+3) owns
// rows [64 g, 64 g + 64) of the item: wgmma m64n256k16 into 128 registers per thread, reduced in place; a thread keeps the state
// of its two rows across the column tiles, and the four threads of a row merge theirs with quad shuffles at the end of the item.
#include "common.cuh"
#include "tc.cuh"

namespace {

constexpr int BM = 128, BN = 256, BK = 64, KB = 4, STAGES = 4;       // K = 256 channels
constexpr int A_KB = BM * BK * 2, B_KB = BN * BK * 2;
constexpr int CONSUMERS = 256, NUM_THREADS = CONSUMERS + 128;
constexpr int SMEM_BYTES = KB * A_KB + STAGES * B_KB + 1024;
constexpr float LOG2E = 1.4426950408889634f;

struct FArgs {
  int B, S, mode, ld_f;
  float a2, s2;                 // alpha * log2(e), shift * log2(e)
  const float* row_f;           // (B, ld_f) factor of the rows    (modes 1, 2)
  const float* col_f;           // (B, ld_f) factor of the columns (modes 1, 2)
  const float4* q4;             // (B, ld_f) masked template points (mode 2)
  float* out_inv;               // mode 0: (B, ld_f)
  int* lab;                     // modes 1, 2: (B, S)
  float* wts; float* pred;      // mode 2: (B, S-1), (B, S-1, 3)
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1) fine_pass_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, FArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_res = smem;                       // 4 k-block slabs [128][64] of the row tile
  uint8_t* ring = smem + KB * A_KB;            // stages of [256][64]
  __shared__ __align__(8) uint64_t a_full, a_empty, full_bar[STAGES], empty_bar[STAGES];
  __shared__ float sc[2][BN];                  // column factors of the current / next column tile (modes 1, 2)
  __shared__ __align__(16) float4 sq[2][BN];   // masked template points of the tile (mode 2)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m_tiles = (g.S + BM - 1) / BM, n_tiles = (g.S + BN - 1) / BN;
  const int items = g.B * m_tiles;

  if (tid == 0) {
    tc::mbar_init(&a_full, 1); tc::mbar_init(&a_empty, CONSUMERS / 32);
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], CONSUMERS / 32); }
    tc::mbar_fence_init();
    tc::tma_prefetch_desc(&tmA);
    tc::tma_prefetch_desc(&tmB);
  }
  __syncthreads();

  if (warp >= CONSUMERS / 32) {
    // ------------------------------------------------------------------ TMA producer (one thread of the third warpgroup)
    tc::producer_regs();
    if (tid == CONSUMERS) {
      long long gk = 0;
      int it = 0;
      for (int item = blockIdx.x; item < items; item += gridDim.x, ++it) {
        const int b = item / m_tiles, mt = item - b * m_tiles;
        tc::mbar_wait(&a_empty, (uint32_t)((it & 1) ^ 1));           // the previous item's MMAs no longer read the row tile
        tc::mbar_arrive_expect_tx(&a_full, KB * A_KB);
        for (int kb = 0; kb < KB; ++kb) tc::tma_load_2d(&tmA, &a_full, a_res + kb * A_KB, kb * BK, b * g.S + mt * BM);
        for (int nt = 0; nt < n_tiles; ++nt)
          for (int kb = 0; kb < KB; ++kb, ++gk) {
            const int s = (int)(gk % STAGES);
            tc::mbar_wait(&empty_bar[s], (uint32_t)(((gk / STAGES) & 1) ^ 1));
            tc::mbar_arrive_expect_tx(&full_bar[s], B_KB);
            tc::tma_load_2d(&tmB, &full_bar[s], ring + s * B_KB, kb * BK, b * g.S + nt * BN);
          }
      }
    }
    return;
  }
  // ------------------------------------------------------------------ consumers: thread = (two rows of the item, column pairs)
  tc::consumer_regs();
  const int wg = warp >> 2, w = warp & 3;
  const uint32_t a_addr = tc::smem_u32(a_res) + wg * (64 * 128);
  long long gk = 0, tcount = 0;
  int it = 0;
  for (int item = blockIdx.x; item < items; item += gridDim.x, ++it) {
    const int b = item / m_tiles, mt = item - b * m_tiles;
    float rf[2] = {0.f, 0.f};
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int i = mt * BM + wg * 64 + tc::frag_row(2 * hr, w, lane);      // row index inside the cloud
      if (MODE != 0 && i < g.S) rf[hr] = g.row_f[(size_t)b * g.ld_f + i];
    }
    const float* cf = (MODE != 0) ? g.col_f + (size_t)b * g.ld_f : nullptr;
    const float4* q4 = (MODE == 2) ? g.q4 + (size_t)b * g.ld_f : nullptr;
    float sum[2] = {0.f, 0.f}, bv[2] = {-INFINITY, -INFINITY}, ws[2] = {0.f, 0.f}, px[2] = {0.f, 0.f}, py[2] = {0.f, 0.f}, pz[2] = {0.f, 0.f};
    int bi[2] = {0x7fffffff, 0x7fffffff};
    tc::mbar_wait(&a_full, (uint32_t)(it & 1));
    for (int nt = 0; nt < n_tiles; ++nt, ++tcount) {
      const int buf = (int)(tcount & 1);
      if (MODE != 0) {
        // stage the tile's 256 column factors (and masked points) once per CTA; the element loop then reads them as
        // shared-memory broadcasts instead of two dependent global loads per element
        const int j = nt * BN + tid;
        sc[buf][tid] = (j < g.S) ? cf[j] : 0.f;
        if (MODE == 2) sq[buf][tid] = (j < g.S) ? q4[j] : make_float4(0.f, 0.f, 0.f, 0.f);
        tc::named_bar(1, CONSUMERS);
      }
      float acc[BN / 2];
      int prev = -1;
      for (int kb = 0; kb < KB; ++kb, ++gk) {
        const int s = (int)(gk % STAGES);
        tc::mbar_wait(&full_bar[s], (uint32_t)((gk / STAGES) & 1));
        const uint32_t b_addr = tc::smem_u32(ring + s * B_KB);
        tc::wg_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          tc::wgmma_bf16<BN>(acc, tc::wg_desc(a_addr + kb * A_KB + k * 32), tc::wg_desc(b_addr + k * 32), (kb | k) ? 1u : 0u);
        tc::wg_commit();
        if (prev >= 0) {
          tc::wg_wait<1>();
          if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);
        }
        prev = s;
      }
      tc::wg_wait<0>();
      if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);
      if (nt == n_tiles - 1 && lane == 0) tc::mbar_arrive(&a_empty);   // the row tile is no longer read
#pragma unroll
      for (int e = 0; e < BN / 2; ++e) {
        const int hr = (e >> 1) & 1, cl = tc::frag_col(e, lane), j = nt * BN + cl;
        const float ev = (j < g.S) ? ex2(fmaf(acc[e], g.a2, -g.s2)) : 0.f;
        if (MODE == 0) {
          sum[hr] += ev;
        } else {
          const float p = (ev * rf[hr]) * (ev * sc[buf][cl]);         // column factor 0 past the last column
          if (p > bv[hr]) { bv[hr] = p; bi[hr] = j; }                 // ascending j inside this thread: first maximum
          if (MODE == 2) {
            const float4 q = sq[buf][cl];
            const float pm = p * q.w;
            ws[hr] += pm; px[hr] = fmaf(pm, q.x, px[hr]); py[hr] = fmaf(pm, q.y, py[hr]); pz[hr] = fmaf(pm, q.z, pz[hr]);
          }
        }
      }
    }
    // ---- merge the four threads of every row (they hold interleaved columns: compare indices so that the first maximum wins)
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int i = mt * BM + wg * 64 + tc::frag_row(2 * hr, w, lane);
      if (MODE == 0) {
        const float t = tc::quad_sum(sum[hr]);
        if ((lane & 3) == 0 && i < g.S) g.out_inv[(size_t)b * g.ld_f + i] = 1.f / t;
      } else {
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv[hr], o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi[hr], o);
          if (ov > bv[hr] || (ov == bv[hr] && oi < bi[hr])) { bv[hr] = ov; bi[hr] = oi; }
        }
        float ww = 0.f, qx = 0.f, qy = 0.f, qz = 0.f;
        if (MODE == 2) { ww = tc::quad_sum(ws[hr]); qx = tc::quad_sum(px[hr]); qy = tc::quad_sum(py[hr]); qz = tc::quad_sum(pz[hr]); }
        if ((lane & 3) == 0 && i < g.S) {
          int lb = bi[hr];
          if (lb == 0x7fffffff) lb = 0;
          g.lab[(size_t)b * g.S + i] = lb;
          if (MODE == 2 && i >= 1) {
            if (lb == 0) { ww = 0.f; qx = 0.f; qy = 0.f; qz = 0.f; }    // background label: the row carries no weight
            const size_t o = (size_t)b * (g.S - 1) + (i - 1);
            const float d = ww + 1e-6f;
            g.wts[o] = ww;
            g.pred[o * 3 + 0] = qx / d; g.pred[o * 3 + 1] = qy / d; g.pred[o * 3 + 2] = qz / d;
          }
        }
      }
    }
  }
}

// masked template points for the ASSIGN pass: q4[b,j] = (pts2[b,j-1], 1) if column j >= 1 carries a non-background label
__global__ void fine_masked_points_kernel(const int* __restrict__ lab2, const float* __restrict__ pts2, int S, int ld, float4* __restrict__ q4) {
  const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ld) return;
  float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
  if (j >= 1 && j < S && lab2[(size_t)b * S + j] > 0) {
    const float* p = pts2 + ((size_t)b * (S - 1) + (j - 1)) * 3;
    q = make_float4(p[0], p[1], p[2], 1.f);
  }
  q4[(size_t)b * ld + j] = q;
}

}  // namespace

// One pass over the (never materialised) score matrix of Fa (rows) against Fb (columns): both (B*S, 256) bf16, L2-normalised.
// mode 0: out_inv (B,ld_f) = 1 / row sums of exp(alpha <a,b> - shift).
// mode 1: lab (B,S) = row arg-max of P = (e * row_f_i) * (e * col_f_j).
// mode 2: mode 1 plus wts (B,S-1), pred (B,S-1,3) for rows >= 1 from the masked points q4 (B,ld_f) float4.
S6_API int sam6d_fine_pass_tc(const void* Fa, const void* Fb, int B, int S, float alpha, float shift, int mode, const float* row_f,
                              const float* col_f, int ld_f, const float* q4, float* out_inv, int* lab, float* wts, float* pred,
                              void* stream) {
  S6_REQUIRE(Fa && Fb && B >= 0 && S >= 2 && mode >= 0 && mode <= 2 && ld_f >= S);
  S6_REQUIRE(((reinterpret_cast<uintptr_t>(Fa) | reinterpret_cast<uintptr_t>(Fb)) & 15) == 0 && (long long)B * S < 2000000000LL);
  if (mode == 0) S6_REQUIRE(out_inv != nullptr);
  if (mode >= 1) S6_REQUIRE(row_f && col_f && lab);
  if (mode == 2) S6_REQUIRE(q4 && wts && pred && (reinterpret_cast<uintptr_t>(q4) & 15) == 0);
  if (B == 0) return 0;
  CUtensorMap tmA, tmB;
  int rc = tc::make_map_2d(&tmA, Fa, (long long)B * S, 256, 256, 64, BM);
  if (rc) return rc;
  rc = tc::make_map_2d(&tmB, Fb, (long long)B * S, 256, 256, 64, BN);
  if (rc) return rc;
  int grid;
  S6_CHECK(s6_persistent_grid(B * s6_cdiv(S, BM), 1, &grid));
  FArgs g{B, S, mode, ld_f, alpha * LOG2E, shift * LOG2E, row_f, col_f, reinterpret_cast<const float4*>(q4), out_inv, lab, wts, pred};
  cudaStream_t st = s6_stream(stream);
#define FINE_LAUNCH(M)                                                                                              \
  do {                                                                                                              \
    S6_CHECK(cudaFuncSetAttribute(fine_pass_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));   \
    fine_pass_kernel<M><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(tmA, tmB, g);                                        \
  } while (0)
  if (mode == 0) FINE_LAUNCH(0); else if (mode == 1) FINE_LAUNCH(1); else FINE_LAUNCH(2);
#undef FINE_LAUNCH
  S6_LAUNCH_CHECK();
  return 0;
}

// lab2 (B,S) i32, pts2 (B,S-1,3) -> q4 (B,ld) float4 for sam6d_fine_pass_tc mode 2
S6_API int sam6d_fine_masked_points(const int* lab2, const float* pts2, int B, int S, int ld, float* q4, void* stream) {
  S6_REQUIRE(lab2 && pts2 && q4 && B >= 0 && S >= 2 && ld >= S && (reinterpret_cast<uintptr_t>(q4) & 15) == 0);
  if (B == 0) return 0;
  dim3 grid(s6_cdiv(ld, 256), B);
  fine_masked_points_kernel<<<grid, 256, 0, s6_stream(stream)>>>(lab2, pts2, S, ld, reinterpret_cast<float4*>(q4));
  S6_LAUNCH_CHECK();
  return 0;
}
