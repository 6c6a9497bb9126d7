// geo_tc.cu -- GeometricStructureEmbedding projections on the tensor cores (wgmma; PEM/model/transformer.py:334-349).
//
//   E[p,:] = proj_d(sin_emb(d_p)) + max_{k<3} proj_a(sin_emb(a_{p,k})) + (b_a + b_d)           p = (b,i,j) pair
//
// The reference materialises sin_emb for 4 scalars per pair (3.8 GB at B=32) and runs two 256x256 Linears over them
// (651 GFLOP per cloud).  Here one persistent, warp-specialised kernel per projection keeps the 256x256 bf16 weight
// resident in shared memory (128 KB, K-major SWIZZLE_128B slabs) and never materialises the embeddings:
//   producers (warps 8-11): a thread owns one 16-byte chunk column (4 frequencies, kept in registers) of 6-8 token rows:
//                           x*omega_f -> __sincosf -> bf16 (sin,cos) pairs written straight into the swizzled A slab of a
//                           4-deep k-block ring (16 KB per 128x64 slab).  The angle pass skips the unused 4th row of every
//                           pair (it repeats the 3rd).
//   consumers (warps 0-7) : warpgroup g owns rows [64 g, 64 g + 64) of the tile: 4 x wgmma m64n256k16 per k-block into 128
//                           registers per thread; pass ANGLE: rows are (pair, k) quadruples, the max over k is two shuffles
//                           (the four rows of a pair sit in lanes 4 apart) and each of the four lanes adds a quarter of the
//                           columns into E; pass DIST (runs first): rows are pairs, E = acc + bias.
// E is fp32 or bf16.  Accuracy: operands rounded to bf16 (sin/cos via MUFU), fp32 accumulation.
#include "epilogue.cuh"
#include "tc.cuh"

namespace {

constexpr int BM = 128, BN = 256, BK = 64, KBLOCKS = 4;
constexpr int A_SLAB = BM * BK * 2;          // 16 KB
constexpr int W_SLAB = BN * BK * 2;          // 32 KB
constexpr int CONSUMERS = 256;                      // warps 0-7
constexpr int NUM_PRODUCERS = 128;                  // warps 8-11
constexpr int NUM_THREADS = CONSUMERS + NUM_PRODUCERS;
constexpr int ASTAGES = 4;
constexpr int SMEM = KBLOCKS * W_SLAB + ASTAGES * A_SLAB + 1024;

__device__ __forceinline__ uint32_t bf16x2_add(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}

// MODE 0: angle pass (rows = pair*4 + k), MODE 1: distance pass (rows = pairs)
template <int MODE, typename ET>
__global__ void __launch_bounds__(NUM_THREADS, 1) geo_embed_tc_kernel(const float* __restrict__ T, long long npairs,
                                                                      const float* __restrict__ div_term,
                                                                      const __nv_bfloat16* __restrict__ Wb,   // (256 out, 256 in) bf16
                                                                      const float* __restrict__ bias, ET* __restrict__ E) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* w_smem = smem;                              // 4 slabs [256][64] bf16
  uint8_t* a_smem = smem + KBLOCKS * W_SLAB;           // ring of [128][64] bf16
  __shared__ __align__(8) uint64_t full_bar[ASTAGES], empty_bar[ASTAGES];
  __shared__ float omega[128];
  __shared__ __align__(16) float sbias[256];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int PAIRS_PER_TILE = (MODE == 0) ? 32 : 128;
  const long long ntiles = (npairs + PAIRS_PER_TILE - 1) / PAIRS_PER_TILE;

  if (tid == 0) {
    for (int s = 0; s < ASTAGES; ++s) { tc::mbar_init(&full_bar[s], NUM_PRODUCERS / 32); tc::mbar_init(&empty_bar[s], CONSUMERS / 32); }
    tc::mbar_fence_init();
  }
  if (tid < 128) omega[tid] = div_term[tid];
  if (tid < 256) sbias[tid] = bias[tid];
  // resident weight: W (n, k) row-major bf16 -> slab kb holds columns [64 kb, 64 kb + 64) of every row, swizzled
  for (int u = tid; u < 256 * 32; u += NUM_THREADS) {      // 16-byte units: 256 rows x 32 units
    const int n = u >> 5, c = (u & 31) << 3;
    const uint4 v = *reinterpret_cast<const uint4*>(Wb + (size_t)n * 256 + c);
    *reinterpret_cast<uint4*>(w_smem + (c >> 6) * W_SLAB + tc::sw128_offset(n, c & 63)) = v;
  }
  for (int u = tid; u < ASTAGES * A_SLAB / 16; u += NUM_THREADS)   // rows the angle pass never writes must be finite
    reinterpret_cast<uint4*>(a_smem)[u] = make_uint4(0u, 0u, 0u, 0u);
  tc::fence_proxy_async_smem();
  __syncthreads();

  if (tid >= CONSUMERS) {
    // ------------------------------------------------------------------ producers: thread <-> (chunk column, NT token rows)
    const int pt = tid - CONSUMERS;
    const int c = pt & 7;                               // 16-byte chunk of the 128-byte slab row: frequencies 32 kb + 4c .. + 3
    constexpr int NT = (MODE == 0) ? 96 * 8 / NUM_PRODUCERS : 128 * 8 / NUM_PRODUCERS;   // tasks per thread per k-block
    int row[NT];
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const int u = (j * NUM_PRODUCERS + pt) >> 3;      // MODE 0: useful row index 0..95 -> row (u/3)*4 + u%3
      row[j] = (MODE == 0) ? (u / 3) * 4 + (u % 3) : u;
    }
    float om[KBLOCKS][4];
#pragma unroll
    for (int kb = 0; kb < KBLOCKS; ++kb)
#pragma unroll
      for (int q = 0; q < 4; ++q) om[kb][q] = omega[kb * 32 + c * 4 + q];
    const uint32_t a_base = tc::smem_u32(a_smem);
    long long g = 0;
    // the indices of the NEXT tile are fetched before this tile's k-blocks are produced (the load latency would otherwise
    // sit in front of every tile: the ring holds exactly one tile, so the producers cannot run further ahead than that)
    auto fetch = [&](long long tile, float (&xx)[NT]) {
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        if (MODE == 0) {
          const long long pair = tile * 32 + (row[j] >> 2);
          xx[j] = (pair < npairs) ? __ldg(T + pair * 4 + (row[j] & 3)) : 0.f;
        } else {
          const long long pair = tile * 128 + row[j];
          xx[j] = (pair < npairs) ? __ldg(T + pair * 4 + 3) : 0.f;
        }
      }
    };
    float xn[NT];
    fetch(blockIdx.x, xn);
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      float x[NT];
#pragma unroll
      for (int j = 0; j < NT; ++j) x[j] = xn[j];
#pragma unroll
      for (int kb = 0; kb < KBLOCKS; ++kb, ++g) {
        const int s = (int)(g % ASTAGES);
        tc::mbar_wait(&empty_bar[s], (uint32_t)(((g / ASTAGES) & 1) ^ 1));
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          uint32_t w[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float sv, cv;
            __sincosf(x[j] * om[kb][q], &sv, &cv);
            w[q] = tc::pack_bf16(sv, cv);
          }
          const uint32_t addr = a_base + s * A_SLAB + row[j] * 128 + ((c ^ (row[j] & 7)) << 4);
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
          if (MODE == 0 && (row[j] & 3) == 2) {
            // the pair's 4th (padding) row repeats its 3rd neighbour: a maximum ignores duplicates, so the epilogue needs no mask
            const uint32_t addr2 = a_base + s * A_SLAB + (row[j] + 1) * 128 + ((c ^ ((row[j] + 1) & 7)) << 4);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr2), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
          }
        }
        tc::fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&full_bar[s]);
        // next tile's indices: issued behind the first fence (a fence waits for the thread's outstanding loads, so a prefetch
        // issued before it would stall the first k-block by the full load latency); k-block 1 covers the latency
        if (kb == 0) fetch(tile + gridDim.x, xn);
      }
    }
    return;
  }
  // ------------------------------------------------------------------ consumers: warpgroup wg <-> rows [64 wg, 64 wg + 64)
  const int wg = warp >> 2, w = warp & 3;
  const uint32_t w_addr = tc::smem_u32(w_smem), a_addr0 = tc::smem_u32(a_smem) + wg * (64 * 128);
  long long g = 0;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    float acc[BN / 2];
    int prev = -1;
    for (int kb = 0; kb < KBLOCKS; ++kb, ++g) {
      const int s = (int)(g % ASTAGES);
      tc::mbar_wait(&full_bar[s], (uint32_t)((g / ASTAGES) & 1));
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        tc::wgmma_bf16<BN>(acc, tc::wg_desc(a_addr0 + s * A_SLAB + k * 32), tc::wg_desc(w_addr + kb * W_SLAB + k * 32), (kb | k) ? 1u : 0u);
      tc::wg_commit();
      if (prev >= 0) {
        tc::wg_wait<1>();
        if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);
      }
      prev = s;
    }
    tc::wg_wait<0>();
    if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);
    if (MODE == 0) {
      // rows 4p .. 4p+3 of a pair are held by lanes l, l^4, l^8, l^12: max over them, then lane quarter q = (l >> 2) & 3
      // adds the 8-column groups j with j % 4 == q into E (E already holds proj_d(...) + biases from the distance pass)
      const int q = (lane >> 2) & 3;
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const long long pair = tile * 32 + (wg * 64 + 16 * w + 8 * hr + (lane >> 2)) / 4;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          float m0 = acc[4 * j + 2 * hr], m1 = acc[4 * j + 2 * hr + 1];
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 4)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 4));
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 8)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 8));
          if ((j & 3) == q && pair < npairs) {
            ET* e = E + pair * 256 + tc::frag_col(4 * j, lane);
            if constexpr (sizeof(ET) == 2) {
              // rounding to bf16 is monotone, so bf16(max) = max of the bf16 values; the sum is a packed bf16 add
              uint32_t* e2 = reinterpret_cast<uint32_t*>(e);
              *e2 = bf16x2_add(*e2, tc::pack_bf16(m0, m1));
            } else {
              float2* e2 = reinterpret_cast<float2*>(e);
              const float2 v = *e2;
              *e2 = make_float2(v.x + m0, v.y + m1);
            }
          }
        }
      }
    } else {
      // rows = pairs: E = acc + (b_a + b_d)
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const long long pair = tile * 128 + wg * 64 + tc::frag_row(2 * hr, w, lane);
        if (pair >= npairs) continue;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = tc::frag_col(4 * j, lane);
          epi::st2(E + pair * 256 + col, acc[4 * j + 2 * hr] + sbias[col], acc[4 * j + 2 * hr + 1] + sbias[col + 1]);
        }
      }
    }
  }
}

template <int MODE, typename ET>
int launch_pass(const float* T, long long npairs, const float* div_term, const __nv_bfloat16* W, const float* bias, ET* E,
                cudaStream_t st) {
  const long long per = (MODE == 0) ? 32 : 128;
  int grid;
  S6_CHECK(s6_persistent_grid((npairs + per - 1) / per, 1, &grid));
  auto kern = geo_embed_tc_kernel<MODE, ET>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
  if (e != cudaSuccess) return (int)e;
  kern<<<grid, NUM_THREADS, SMEM, st>>>(T, npairs, div_term, W, bias, E);
  return (int)cudaGetLastError();
}

}  // namespace

// T (npairs,4) fp32 -> E (npairs,256) fp32 (e_is_bf16 = 0) or bf16 (1).  Wa, Wd: proj_a / proj_d weights (out,in) in bf16;
// bias = proj_a.bias + proj_d.bias (fp32); div_term: the module buffer (128 frequencies).  Two persistent launches.
S6_API int sam6d_geo_embed_tc(const float* T, long long npairs, const float* div_term, const void* Wa_bf16, const void* Wd_bf16,
                              const float* bias, void* E, int e_is_bf16, void* stream) {
  S6_REQUIRE(T && div_term && Wa_bf16 && Wd_bf16 && bias && E && npairs >= 0 && npairs < 2000000000LL);
  if (npairs == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  const __nv_bfloat16* Wa = reinterpret_cast<const __nv_bfloat16*>(Wa_bf16);
  const __nv_bfloat16* Wd = reinterpret_cast<const __nv_bfloat16*>(Wd_bf16);
  int rc;
  if (e_is_bf16) {
    rc = launch_pass<1, __nv_bfloat16>(T, npairs, div_term, Wd, bias, reinterpret_cast<__nv_bfloat16*>(E), st);
    if (rc) return rc;
    rc = launch_pass<0, __nv_bfloat16>(T, npairs, div_term, Wa, bias, reinterpret_cast<__nv_bfloat16*>(E), st);
  } else {
    rc = launch_pass<1, float>(T, npairs, div_term, Wd, bias, reinterpret_cast<float*>(E), st);
    if (rc) return rc;
    rc = launch_pass<0, float>(T, npairs, div_term, Wa, bias, reinterpret_cast<float*>(E), st);
  }
  return rc;
}

// the distance projection alone: T (npairs,4) fp32 (index 3 = distance index) -> E (npairs,256) bf16 = proj_d(emb(d)) + bias.
// Used by the table-interpolation kernel (geo_lut.cu) for the few distances outside its table (row / column of the background point)
S6_API int sam6d_geo_embed_dist_tc(const float* T, long long npairs, const float* div_term, const void* Wd_bf16, const float* bias, void* E,
                                   void* stream) {
  S6_REQUIRE(T && div_term && Wd_bf16 && bias && E && npairs >= 0 && npairs < 2000000000LL);
  if (npairs == 0) return 0;
  return launch_pass<1, __nv_bfloat16>(T, npairs, div_term, reinterpret_cast<const __nv_bfloat16*>(Wd_bf16), bias,
                                       reinterpret_cast<__nv_bfloat16*>(E), s6_stream(stream));
}
