// attn_global_tc.cu -- SAM ViT global attention (64 x 64 = 4096 tokens per image, head dim D = 80 for ViT-H, 64 for ViT-L / ViT-B,
// decomposed relative-position bias) on wgmma with an online softmax (ISM/segment_anything/modeling/image_encoder.py:224-240, 325-361).
//
//     O = softmax(scale * Q K^T + Rh[q, kh] + Rw[q, kw]) V,     Rh[q, kh] = q . rel_h[qh - kh + 63], Rw likewise (unscaled q)
//
// One CTA per (128-query tile = two rows of the token grid, head, image); it walks the 32 key tiles of 128 keys:
//   warp 8     TMA      : (one thread of warpgroup 2) Q and the rel tables once; then K tiles and V^T tiles into two independent 2-deep rings (the rel
//                         tables occupy the K ring and the bias scratch the V ring / P slabs until the bias tables are built)
//   warps 0-7  two warpgroups, warpgroup g owns queries [64 g, 64 g + 64) (one row of the token grid):
//                G_w = Q rel_w^T, G_h = Q rel_h^T (once) -> the row's 32 Rw values of its key columns in registers, Rh in
//                shared memory; per key tile: S_j = Q K_j^T (wgmma m64n128k16, 64 registers), row max / exp2 in registers
//                (rows live in quads), o = o * alpha in registers, P_j as bf16 into the swizzled A slabs, o += P_j V_j
//                (wgmma m64nDk16, D/2 registers)
// Q, K and each rel table are DS = ceil(D/64) slabs of 64 channels (two at D = 80, the second one 16 channels deep; one at D = 64);
// a V^T tile is two [D rows][64 keys] slabs.  Both head dims share the code; only the slab counts and the k-step counts differ.
// The reference materialises a (16 x 4096 x 4096) fp32 score tensor per image and block; here scores never leave registers.
#include "epilogue.cuh"
#include "tc.cuh"

namespace {

constexpr int QT = 128, KT = 128, GRID = 64;
constexpr int CONSUMERS = 256, NUM_THREADS = CONSUMERS + 128;
constexpr int Q_SLAB = QT * 128, K_SLAB = KT * 128, P_SLAB = QT * 128, REL_SLAB = 128 * 128;
constexpr int TABH_LD = 64, SCR_LD = 128;

// shared-memory plan of the head-dim-D kernel: [Q: DS slabs][K ring: 2 x DS slabs][V ring: 2 x 2 slabs][P: 2 slabs][tab_h]
template <int D>
struct Cfg {
  static constexpr int DS = (D + 63) / 64, V_SLAB = D * 128;
  static constexpr int OFF_Q = 0, OFF_K0 = OFF_Q + DS * Q_SLAB, OFF_K1 = OFF_K0 + DS * K_SLAB, OFF_V0 = OFF_K1 + DS * K_SLAB,
                       OFF_V1 = OFF_V0 + 2 * V_SLAB, OFF_P = OFF_V1 + 2 * V_SLAB, OFF_TABH = OFF_P + 2 * P_SLAB;
  static constexpr int SMEM_BYTES = OFF_TABH + QT * TABH_LD * 4 + 1024;
  static_assert(D % 16 == 0 && D <= 128, "head dim: whole k-steps, at most two 64-channel slabs");
  static_assert(OFF_K0 % 1024 == 0 && OFF_K1 % 1024 == 0 && OFF_V0 % 1024 == 0 && OFF_V1 % 1024 == 0 && OFF_P % 1024 == 0,
                "slabs must be 1024-byte aligned");
  static_assert(OFF_K1 + DS * K_SLAB - OFF_K0 >= 2 * DS * REL_SLAB, "the rel tables occupy the K ring");
  static_assert(OFF_TABH - OFF_V0 >= QT * SCR_LD * 4, "the bias scratch occupies the V ring and the P slabs");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one CTA");
};
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct GArgs {
  const void* rel_blob;   // rel_h, rel_w as bf16 wgmma B slabs: 2 tables x DS slabs x [128 rows][64 ch], SWIZZLE_128B
  void* out; long long out_ld;
  int H;
  float scale;
};

template <int D, typename OT>
__global__ void __launch_bounds__(NUM_THREADS, 1) attn_global_tc_kernel(const __grid_constant__ CUtensorMap tmQK, const __grid_constant__ CUtensorMap tmVt,
                                                       GArgs a) {
  using CF = Cfg<D>;
  constexpr int DS = CF::DS, V_SLAB = CF::V_SLAB, OFF_Q = CF::OFF_Q, OFF_K0 = CF::OFF_K0, OFF_K1 = CF::OFF_K1, OFF_V0 = CF::OFF_V0,
                OFF_V1 = CF::OFF_V1, OFF_P = CF::OFF_P, OFF_TABH = CF::OFF_TABH;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* q_s = smem + OFF_Q;
  uint8_t* p_s = smem + OFF_P;
  uint8_t* rel_s = smem + OFF_K0;                                   // before the key loop: rel tables in the K ring
  float* scratch = reinterpret_cast<float*>(smem + OFF_V0);         // ... and the G_w / G_h rows over the V ring and P
  float* tab_h = reinterpret_cast<float*>(smem + OFF_TABH);
  __shared__ __align__(8) uint64_t q_bar, tab_done, k_full[2], k_empty[2], v_full[2], v_empty[2];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tq = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  constexpr int L = GRID * GRID, NT = L / KT;
  const int C = a.H * D;

  if (tid == 0) {
    tc::mbar_init(&q_bar, 1); tc::mbar_init(&tab_done, CONSUMERS / 32);
    for (int s = 0; s < 2; ++s) {
      tc::mbar_init(&k_full[s], 1); tc::mbar_init(&k_empty[s], CONSUMERS / 32);
      tc::mbar_init(&v_full[s], 1); tc::mbar_init(&v_empty[s], CONSUMERS / 32);
    }
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (warp >= CONSUMERS / 32) {
    // -------------------------------------------------------------------------------------------------- TMA producer
    tc::producer_regs();
    if (tid == CONSUMERS) {
      tc::mbar_arrive_expect_tx(&q_bar, DS * Q_SLAB + 2 * DS * REL_SLAB);
      tc::bulk_load_1d(rel_s, a.rel_blob, 2 * DS * REL_SLAB, &q_bar);
      for (int s = 0; s < DS; ++s) tc::tma_load_2d(&tmQK, &q_bar, q_s + s * Q_SLAB, h * D + s * 64, b * L + tq * QT);
      tc::mbar_wait(&tab_done, 0);                                  // the rings hold the rel tables / bias scratch until then
      for (int j = 0; j < NT; ++j) {
        const int st = j & 1, use = j >> 1;
        uint8_t* k_s = smem + (st ? OFF_K1 : OFF_K0);
        uint8_t* v_s = smem + (st ? OFF_V1 : OFF_V0);
        tc::mbar_wait(&k_empty[st], (uint32_t)((use & 1) ^ 1));
        tc::mbar_arrive_expect_tx(&k_full[st], DS * K_SLAB);
        for (int s = 0; s < DS; ++s) tc::tma_load_2d(&tmQK, &k_full[st], k_s + s * K_SLAB, C + h * D + s * 64, b * L + j * KT);
        tc::mbar_wait(&v_empty[st], (uint32_t)((use & 1) ^ 1));
        tc::mbar_arrive_expect_tx(&v_full[st], 2 * V_SLAB);
        for (int s = 0; s < 2; ++s) tc::tma_load_2d(&tmVt, &v_full[st], v_s + s * V_SLAB, j * KT + s * 64, (b * a.H + h) * D);
      }
    }
    return;
  }
  // -------------------------------------------------------------------------------------------------- warpgroups
  tc::consumer_regs();
  const int wg = warp >> 2, w = warp & 3;
  const uint32_t q_addr = tc::smem_u32(q_s) + wg * (64 * 128), p_addr = tc::smem_u32(p_s) + wg * (64 * 128);
  const int qh = 2 * tq + wg;                                       // this warpgroup's row of the token grid
  float tw[2][32];                                                  // Rw * log2(e) of the thread's 32 key columns (kw), per row half
  tc::mbar_wait(&q_bar, 0);
  // G_w (blob table 1) -> tw,  G_h (blob table 0) -> tab_h, through this warpgroup's rows of the scratch
#pragma unroll 1
  for (int t = 0; t < 2; ++t) {
    float g[KT / 2];
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k)
      tc::wgmma_bf16<KT>(g, tc::wg_desc(q_addr + (k >> 2) * Q_SLAB + (k & 3) * 32),
                         tc::wg_desc(tc::smem_u32(rel_s) + ((1 - t) * DS + (k >> 2)) * REL_SLAB + (k & 3) * 32), k ? 1u : 0u);
    tc::wg_commit();
    tc::wg_wait<0>();
#pragma unroll
    for (int e = 0; e < KT / 2; ++e) scratch[(wg * 64 + tc::frag_row(e, w, lane)) * SCR_LD + tc::frag_col(e, lane)] = g[e] * LOG2E;
    tc::named_bar(1 + wg, 128);
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int rl = tc::frag_row(2 * hr, w, lane), r = wg * 64 + rl;   // query column qw = rl
      const float* srow = scratch + r * SCR_LD;
      if (t == 0) {
#pragma unroll
        for (int i = 0; i < 32; ++i) tw[hr][i] = srow[rl + (GRID - 1) - tc::frag_col(4 * (i >> 1) + (i & 1), lane)];
      } else if ((lane & 3) == 0) {
        for (int kh = 0; kh < GRID; ++kh) tab_h[r * TABH_LD + kh] = srow[qh + (GRID - 1) - kh];
      }
    }
    tc::named_bar(1 + wg, 128);                                     // the scratch rows are read before they are rewritten
  }
  if (lane == 0) tc::mbar_arrive(&tab_done);                        // rel tables and scratch are dead: the rings may fill
  tc::mbar_wait(&tab_done, 0);                                      // ... and P (over the other warpgroup's scratch rows) be written

  const float sl2 = a.scale * LOG2E;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
#pragma unroll 1
  for (int j = 0; j < NT; ++j) {
    const int st = j & 1;
    float sacc[KT / 2];
    tc::mbar_wait(&k_full[st], (uint32_t)((j >> 1) & 1));
    const uint32_t k_addr = tc::smem_u32(smem + (st ? OFF_K1 : OFF_K0));
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k)
      tc::wgmma_bf16<KT>(sacc, tc::wg_desc(q_addr + (k >> 2) * Q_SLAB + (k & 3) * 32), tc::wg_desc(k_addr + (k >> 2) * K_SLAB + (k & 3) * 32),
                         k ? 1u : 0u);
    tc::wg_commit();
    tc::wg_wait<0>();
    if (lane == 0) tc::mbar_arrive(&k_empty[st]);
    float alpha[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int r = wg * 64 + tc::frag_row(2 * hr, w, lane);
      const float th0 = tab_h[r * TABH_LD + 2 * j], th1 = tab_h[r * TABH_LD + 2 * j + 1];   // key rows 2j, 2j+1 of the grid
      float mt = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < KT / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 4 * jj + 2 * hr + e;
          const float x = fmaf(sacc[i], sl2, (jj < 8 ? th0 : th1) + tw[hr][2 * (jj & 7) + e]);
          sacc[i] = x;
          mt = fmaxf(mt, x);
        }
      const float m_new = fmaxf(m[hr], tc::quad_max(mt));
      alpha[hr] = ex2(m[hr] - m_new);
      m[hr] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < KT / 8; ++jj) {
        const int i = 4 * jj + 2 * hr;
        const float p0 = ex2(sacc[i] - m_new), p1 = ex2(sacc[i + 1] - m_new);
        sum += p0 + p1;
        sacc[i] = p0; sacc[i + 1] = p1;
      }
      l[hr] = fmaf(l[hr], alpha[hr], sum);
    }
    if (j > 0) tc::named_bar(1 + wg, 128);                          // every warp's P_{j-1} V_{j-1} has completed: P may be rewritten
#pragma unroll
    for (int i = 0; i < KT / 2; i += 2) {
      const int r = wg * 64 + tc::frag_row(i, w, lane), col = tc::frag_col(i, lane);
      *reinterpret_cast<uint32_t*>(p_s + (col >> 6) * P_SLAB + tc::sw128_offset(r, col & 63)) = tc::pack_bf16(sacc[i], sacc[i + 1]);
    }
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    tc::fence_proxy_async_smem();
    tc::named_bar(1 + wg, 128);                                     // this warpgroup's P_j rows are complete
    tc::mbar_wait(&v_full[st], (uint32_t)((j >> 1) & 1));
    const uint32_t v_addr = tc::smem_u32(smem + (st ? OFF_V1 : OFF_V0));
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < KT / 16; ++k)
      tc::wgmma_bf16<D>(o, tc::wg_desc(p_addr + (k >> 2) * P_SLAB + (k & 3) * 32), tc::wg_desc(v_addr + (k >> 2) * V_SLAB + (k & 3) * 32), 1u);
    tc::wg_commit();
    tc::wg_wait<0>();
    if (lane == 0) tc::mbar_arrive(&v_empty[st]);
  }
  OT* outp = reinterpret_cast<OT*>(a.out);
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const float inv = 1.f / tc::quad_sum(l[hr]);
    const int row = b * L + tq * QT + wg * 64 + tc::frag_row(2 * hr, w, lane);
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj) {
      const int i = 4 * jj + 2 * hr;
      epi::st2(outp + (size_t)row * a.out_ld + h * D + tc::frag_col(i, lane), o[i] * inv, o[i + 1] * inv);
    }
  }
}

template <int D, typename OT>
int launch_global(const CUtensorMap& tqk, const CUtensorMap& tv, const GArgs& a, int B, cudaStream_t st) {
  constexpr int SMEM = Cfg<D>::SMEM_BYTES;
  auto k = attn_global_tc_kernel<D, OT>;
  S6_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  k<<<dim3(GRID * GRID / QT, a.H, B), NUM_THREADS, SMEM, st>>>(tqk, tv, a);
  S6_LAUNCH_CHECK();
  return 0;
}

}  // namespace

// qkv: bf16 (B*4096 rows, ld >= 2*H*D) rows [q | k (| v)], head h at columns h*D of q and H*D + h*D of k; Vt: bf16 (B*H*D rows,
// vt_ld >= 4096) = V^T per (image, head) (sam6d_transpose_tokens_bf16); rel_blob: rel_pos_h / rel_pos_w ((127, D) each) packed as
// bf16 wgmma slabs with 128-row slabs (ops.pack_rel_pos(..., slab_rows=128)); out (B*4096, H*D) fp32 or bf16.  64 x 64 token grid
// only; head_dim D = 80 (ViT-H) or 64 (ViT-L, ViT-B).
S6_API int sam6d_attn_global_tc_ex(const void* qkv, long long ld, const void* Vt, long long vt_ld, const void* rel_blob, int B, int H,
                                   int grid, int head_dim, float scale, void* out, int out_is_bf16, long long out_ld, void* stream) {
  S6_REQUIRE(head_dim == 64 || head_dim == 80);
  S6_REQUIRE(qkv && Vt && rel_blob && out && B >= 0 && H > 0 && grid == GRID);
  S6_REQUIRE((ld % 8) == 0 && ld >= 2LL * H * head_dim && (vt_ld % 8) == 0 && vt_ld >= GRID * GRID &&
             (out_ld % (out_is_bf16 ? 8 : 4)) == 0);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(rel_blob) & 15) == 0 && (reinterpret_cast<uintptr_t>(qkv) & 15) == 0 &&
             (reinterpret_cast<uintptr_t>(Vt) & 15) == 0);
  if (B == 0) return 0;
  S6_REQUIRE(B <= 65535 && H <= 65535);
  constexpr int L = GRID * GRID;
  CUtensorMap tqk, tv;
  int rc = tc::make_map_2d(&tqk, qkv, (long long)B * L, ld, ld, 64, QT);
  if (rc) return rc;
  rc = tc::make_map_2d(&tv, Vt, (long long)B * H * head_dim, vt_ld, vt_ld, 64, head_dim);
  if (rc) return rc;
  GArgs a{rel_blob, out, out_ld, H, scale};
  cudaStream_t st = s6_stream(stream);
  if (head_dim == 64)
    return out_is_bf16 ? launch_global<64, __nv_bfloat16>(tqk, tv, a, B, st) : launch_global<64, float>(tqk, tv, a, B, st);
  return out_is_bf16 ? launch_global<80, __nv_bfloat16>(tqk, tv, a, B, st) : launch_global<80, float>(tqk, tv, a, B, st);
}

// sam6d_attn_global_tc_ex at head_dim 80 (SAM ViT-H)
S6_API int sam6d_attn_global_tc(const void* qkv, long long ld, const void* Vt, long long vt_ld, const void* rel_blob, int B, int H,
                                int grid, float scale, void* out, int out_is_bf16, long long out_ld, void* stream) {
  return sam6d_attn_global_tc_ex(qkv, ld, Vt, vt_ld, rel_blob, B, H, grid, 80, scale, out, out_is_bf16, out_ld, stream);
}
