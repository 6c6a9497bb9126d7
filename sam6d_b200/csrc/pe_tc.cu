// pe_tc.cu -- PositionalEncoding shared MLP on the tensor cores (PEM/model/fine_point_matching.py:101-121).
//
// Rows are (point, sample) pairs of the ball-query groups, 128 rows per tile (4 points at nsample 32, 2 at nsample 64).
// Per tile, in one CTA of one warpgroup (layer 1: thread <-> row):
//   layer 1 (6 -> 32)   CUDA cores, fp32: x = [p_j - p_i, p_j]; h1 = relu(W1 x + b1) -> bf16 row of the A1 slab
//   layer 2 (32 -> 64)  2 x (2 x wgmma m64n64k16), one per 64-row half; + b2, ReLU, bf16 -> A2 slab straight from the registers
//   layer 3 (64 -> 128) wgmma with the operands swapped: D^T = W3 A2^T (M = output channel, N = the tile's 128 rows; both slabs are
//                       K-major, either can be the A operand), one 64-channel half at a time
//   max-pool            the samples of a point are 32 / 64 adjacent columns: a register max over the thread's columns, then over
//                       the quad; + b3, ReLU (monotone, commutes with max)
// BatchNorm is folded into the 1x1 convs on the host.  The (B,6,N,ns) grouped tensor and the (B,128,N,ns) activations of the
// reference are never materialised; padded duplicate samples are simply recomputed (they cannot change a max).
// Four CTAs share an SM (49 KB smem each), so one tile's serial chain hides behind the others'.
#include "tc.cuh"

namespace {

constexpr int ROWS = 128;
constexpr int SLAB = ROWS * 128;            // [128 rows][64 bf16]
constexpr int W2_SLAB = 64 * 128;           // [64 out][64 k] (k >= 32 unused)
constexpr int W3_SLAB = 128 * 128;          // [128 out][64 k]
// W2 (64 x 32) lives in the UNUSED K columns 32..63 of the first 64 rows of the A1 slab (layer 1 has 32 channels, so A1 fills only
// K 0..31 of its 128-byte rows): with a slab of its own a CTA takes 57 KB + static and only three fit an SM.
constexpr int SMEM_BYTES = 2 * SLAB + W3_SLAB + 1024;
constexpr int NUM_THREADS = 128;

__device__ __forceinline__ void worker_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

__device__ __forceinline__ void st_feat(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_feat(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }

template <int NS, typename OT>
__global__ void __launch_bounds__(NUM_THREADS, 4) pe_tc_kernel(const float* __restrict__ pts, const int* __restrict__ idx, int N,
                                                               long long total_points,
                                                               const float* __restrict__ W1, const float* __restrict__ B1,
                                                               const __nv_bfloat16* __restrict__ W2, const float* __restrict__ B2,
                                                               const __nv_bfloat16* __restrict__ W3, const float* __restrict__ B3,
                                                               OT* __restrict__ out, int out_ld, int out_off) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a1 = smem;
  uint8_t* a2 = a1 + SLAB;
  uint8_t* w3s = a2 + SLAB;
  __shared__ __align__(16) float w1s[32 * 8];
  __shared__ __align__(16) float b1s[32], b2s[64], b3s[128];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int PPT = ROWS / NS;                                  // points per tile
  const long long ntiles = (total_points + PPT - 1) / PPT;

  for (int e = tid; e < 32 * 8; e += NUM_THREADS) { int r = e >> 3, c = e & 7; w1s[e] = (c < 6) ? W1[r * 6 + c] : 0.f; }
  if (tid < 32) b1s[tid] = B1[tid];
  if (tid < 64) b2s[tid] = B2[tid];
  if (tid < 128) b3s[tid] = B3[tid];
  // W2 (64 x 32) and W3 (128 x 64) bf16 -> K-major swizzled slabs
  for (int u = tid; u < 64 * 4; u += NUM_THREADS) {
    const int n = u >> 2, c = (u & 3) << 3;
    *reinterpret_cast<uint4*>(a1 + tc::sw128_offset(n, 32 + c)) = *reinterpret_cast<const uint4*>(W2 + n * 32 + c);
  }
  for (int u = tid; u < 128 * 8; u += NUM_THREADS) {
    const int n = u >> 3, c = (u & 7) << 3;
    *reinterpret_cast<uint4*>(w3s + tc::sw128_offset(n, c)) = *reinterpret_cast<const uint4*>(W3 + n * 64 + c);
  }
  tc::fence_proxy_async_smem();
  __syncthreads();

  {
    // ------------------------------------------------------------------ workers: thread <-> row of the tile
    const int r = tid;
    const uint32_t a1_addr = tc::smem_u32(a1), a2_addr = tc::smem_u32(a2), w2_addr = tc::smem_u32(a1) + 64, w3_addr = tc::smem_u32(w3s);
    // gather pipeline: the neighbour index of tile t+2 and the coordinates of tile t+1 are in flight while tile t is computed.
    // They are issued behind the tile's LAST fence.proxy.async (a fence waits for the thread's outstanding loads).
    auto load_idx = [&](long long tile) -> int {
      const long long gp = tile * PPT + r / NS;
      return (tile < ntiles && gp < total_points) ? __ldg(idx + gp * NS + (r % NS)) : -1;
    };
    auto load_x = [&](long long tile, int j, float (&xx)[6]) {
      const long long gp = tile * PPT + r / NS;
      if (j >= 0) {
        const long long b = gp / N;
        const float* pi = pts + gp * 3;
        const float* pj = pts + (b * N + j) * 3;
        const float jx = __ldg(pj), jy = __ldg(pj + 1), jz = __ldg(pj + 2);
        xx[0] = jx - __ldg(pi); xx[1] = jy - __ldg(pi + 1); xx[2] = jz - __ldg(pi + 2); xx[3] = jx; xx[4] = jy; xx[5] = jz;
      } else {
#pragma unroll
        for (int e = 0; e < 6; ++e) xx[e] = 0.f;
      }
    };
    float xn[6];
    load_x(blockIdx.x, load_idx(blockIdx.x), xn);
    int jn = load_idx((long long)blockIdx.x + gridDim.x);
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      // ---- layer 1
      {
        float x[6];
#pragma unroll
        for (int e = 0; e < 6; ++e) x[e] = xn[e];
        uint8_t* row_ptr = a1 + r * 128;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          uint32_t w[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float h[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int o = c * 8 + q * 2 + e;
              const float4 wa = *reinterpret_cast<const float4*>(&w1s[o * 8]);
              const float2 wb = *reinterpret_cast<const float2*>(&w1s[o * 8 + 4]);
              float a = b1s[o];
              a = fmaf(wa.x, x[0], a); a = fmaf(wa.y, x[1], a); a = fmaf(wa.z, x[2], a);
              a = fmaf(wa.w, x[3], a); a = fmaf(wb.x, x[4], a); a = fmaf(wb.y, x[5], a);
              h[e] = fmaxf(a, 0.f);
            }
            w[q] = tc::pack_bf16(h[0], h[1]);
          }
          *reinterpret_cast<uint4*>(row_ptr + ((c ^ (r & 7)) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
        }
        tc::fence_proxy_async_smem();
        worker_bar();
      }
      // ---- layer 2 -> A2
#pragma unroll
      for (int blk = 0; blk < 2; ++blk) {
        float acc[32];
        tc::wg_fence();
#pragma unroll
        for (int k = 0; k < 2; ++k)
          tc::wgmma_bf16<64>(acc, tc::wg_desc(a1_addr + blk * (64 * 128) + k * 32), tc::wg_desc(w2_addr + k * 32), k ? 1u : 0u);
        tc::wg_commit();
        tc::wg_wait<0>();
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int row = blk * 64 + tc::frag_row(i, warp, lane), col = tc::frag_col(i, lane);
          *reinterpret_cast<uint32_t*>(a2 + tc::sw128_offset(row, col)) =
              tc::pack_bf16(fmaxf(acc[i] + b2s[col], 0.f), fmaxf(acc[i + 1] + b2s[col + 1], 0.f));
        }
      }
      tc::fence_proxy_async_smem();
      worker_bar();                                         // A2 complete; every thread is past its layer-2 reads of A1
      load_x(tile + gridDim.x, jn, xn);
      jn = load_idx(tile + 2LL * gridDim.x);
      // ---- layer 3: rows of the accumulator are output channels, columns the tile's rows
#pragma unroll
      for (int blk = 0; blk < 2; ++blk) {
        float acc[64];
        tc::wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          tc::wgmma_bf16<128>(acc, tc::wg_desc(w3_addr + blk * (64 * 128) + k * 32), tc::wg_desc(a2_addr + k * 32), k ? 1u : 0u);
        tc::wg_commit();
        tc::wg_wait<0>();
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int ch = blk * 64 + tc::frag_row(2 * hr, warp, lane);
          const float bias = b3s[ch];
#pragma unroll
          for (int p = 0; p < PPT; ++p) {
            constexpr int JG = NS / 8;                        // 8-column groups per point
            float m = -INFINITY;
#pragma unroll
            for (int j = p * JG; j < (p + 1) * JG; ++j) m = fmaxf(m, fmaxf(acc[4 * j + 2 * hr], acc[4 * j + 2 * hr + 1]));
            m = tc::quad_max(m);
            const long long p_out = tile * PPT + p;
            if ((lane & 3) == 0 && p_out < total_points) st_feat(out + p_out * out_ld + out_off + ch, fmaxf(m + bias, 0.f));
          }
        }
      }
    }
  }
}

}  // namespace

// Same contract as sam6d_pe_mlp_max, with W2 (64,32) and W3 (128,64) in bf16 (W1 / biases fp32); cnt is not needed.
// out: fp32 (out_is_bf16 = 0) or bf16 rows of out_ld elements.
S6_API int sam6d_pe_mlp_max_tc(const float* pts, const int* idx, int B, int N, int ns, const float* W1, const float* B1,
                               const void* W2_bf16, const float* B2, const void* W3_bf16, const float* B3, void* out, int out_is_bf16,
                               int out_ld, int out_off, void* stream) {
  S6_REQUIRE(pts && idx && W1 && B1 && W2_bf16 && B2 && W3_bf16 && B3 && out && B >= 0 && N > 0);
  S6_REQUIRE(ns == 32 || ns == 64);
  if (B == 0) return 0;
  const long long total = (long long)B * N;
  const long long ntiles = (total + (128 / ns) - 1) / (128 / ns);
  // four CTAs per SM: 4 x (49 KB + static) shared memory, 4 x 128 x 128 registers.  (The occupancy API is not used: with the
  // default carve-out it answers fewer and the grid shrinks.)
  int grid;
  S6_CHECK(s6_persistent_grid(ntiles, 4, &grid));
  cudaStream_t st = s6_stream(stream);
  const __nv_bfloat16* W2 = reinterpret_cast<const __nv_bfloat16*>(W2_bf16);
  const __nv_bfloat16* W3 = reinterpret_cast<const __nv_bfloat16*>(W3_bf16);
#define PE_LAUNCH(NSV, OT)                                                                                                          \
  do {                                                                                                                              \
    S6_CHECK(cudaFuncSetAttribute(pe_tc_kernel<NSV, OT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));                 \
    /* ask for the largest shared-memory carve-out: with the default the driver sizes it for fewer resident CTAs */                   \
    S6_CHECK(cudaFuncSetAttribute(pe_tc_kernel<NSV, OT>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));                     \
    pe_tc_kernel<NSV, OT><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(pts, idx, N, total, W1, B1, W2, B2, W3, B3,                         \
                                                                 reinterpret_cast<OT*>(out), out_ld, out_off);                      \
  } while (0)
  if (ns == 32) { if (out_is_bf16) PE_LAUNCH(32, __nv_bfloat16); else PE_LAUNCH(32, float); }
  else { if (out_is_bf16) PE_LAUNCH(64, __nv_bfloat16); else PE_LAUNCH(64, float); }
#undef PE_LAUNCH
  S6_LAUNCH_CHECK();
  return 0;
}
