// tail_tc.cu -- the tail of every transformer layer of the PEM path as ONE persistent kernel (bf16 token stream):
//
//     y   = LayerNorm1(hid W_o^T + b_o + x)                      AttentionLayer / RPEAttentionLayer (transformer.py:176-180, 435-438)
//     out = LayerNorm2(y + relu(y W_e^T + b_e) W_s^T + b_s)      AttentionOutput                    (transformer.py:191-197)
//
// hid, x, out: (M, 256) bf16;  W_o (256,256), W_e (512,256), W_s (256,512) bf16;  fp32 biases and LayerNorm parameters.
// The five launches this replaces (GEMM+residual, LayerNorm, GEMM+ReLU, GEMM+residual, LayerNorm) moved each 128-row tile through
// HBM/L2 nine times; here the tile stays on chip from the attention output to the layer output:
//   warp 8      TMA (one thread; its warpgroup hands its registers to warps 0-7): hid tile and x tile (SWIZZLE_128B slabs), then the 20 weight k-blocks {64 k, 256 rows} of the tile through a
//               3-stage ring (weights come from L2: 640 KB per tile)
//   warps 0-7   two warpgroups; warpgroup g owns rows [64 g, 64 g + 64) of the tile and runs, with one m64n256 fp32 accumulator
//               in registers (128 per thread):
//                 G1 : hid W_o^T        E1 : + b_o + x -> LayerNorm1 -> y: bf16 over the hid rows (next A operand) and into the
//                                            tile's rows of out, where the same thread reads it back as the residual of E3
//                 G2a: y W_e[0:256]^T   E2a: relu(+ b_e) -> h[:, 0:256] over the x rows
//                 G2b: y W_e[256:512]^T E2b: relu(+ b_e) -> h[:, 256:512] over the y rows
//                 G3 : h W_s^T (8 k-blocks from both buffers)   E3 : + b_s + y -> LayerNorm2 -> bf16 rows of out
//               A row lives in the four threads of a quad: the LayerNorm statistics are two shuffles.  The warpgroups share the
//               weight stream and nothing else.
// Shared memory: 64 KB (hid -> y -> h half 1) + 64 KB (x -> h half 0) + 96 KB weight ring.
#include "tc.cuh"

namespace {

constexpr int BM = 128, C = 256, HID = 512, BK = 64;
constexpr int T_SLAB = BM * 128;                 // 16 KB: [128 rows][64 ch] bf16
constexpr int T_BYTES = 4 * T_SLAB;              // 64 KB token tile
constexpr int W_STAGE = 256 * 128;               // 32 KB: [256 rows][64 k] bf16
constexpr int W_STAGES = 3;
constexpr int W_PER_TILE = 20;                   // weight k-blocks per tile: 4 (W_o) + 8 (W_e) + 8 (W_s)
constexpr int CONSUMERS = 256, THREADS = CONSUMERS + 128;
constexpr int SMEM = 2 * T_BYTES + W_STAGES * W_STAGE + 1024;

struct TailArgs {
  const float* bo; const float* g1; const float* b1;
  const float* be; const float* bs; const float* g2; const float* b2;
  int M;
  float eps;
};

// bf16 pair (row r, columns col, col + 1; col even) of a token tile stored as 4 SWIZZLE_128B slabs
__device__ __forceinline__ uint32_t* tile_pair(uint8_t* tile, int r, int col) {
  return reinterpret_cast<uint32_t*>(tile + (col >> 6) * T_SLAB + r * 128 + ((((col & 63) >> 3) ^ (r & 7)) << 4) + (col & 7) * 2);
}
__device__ __forceinline__ float2 unpack2(uint32_t w) { return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u)); }

__global__ void __launch_bounds__(THREADS, 1) tail_tc_kernel(const __grid_constant__ CUtensorMap tmHid, const __grid_constant__ CUtensorMap tmX,
                                                const __grid_constant__ CUtensorMap tmWo, const __grid_constant__ CUtensorMap tmWe,
                                                const __grid_constant__ CUtensorMap tmWs, TailArgs a, __nv_bfloat16* __restrict__ out,
                                                long long ld_out) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_buf = smem;                      // hid -> y -> h half 1
  uint8_t* x_buf = smem + T_BYTES;            // x -> h half 0
  uint8_t* w_ring = smem + 2 * T_BYTES;
  __shared__ __align__(8) uint64_t in_full, in_empty, w_full[W_STAGES], w_empty[W_STAGES];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntiles = (a.M + BM - 1) / BM;

  if (tid == 0) {
    tc::mbar_init(&in_full, 1); tc::mbar_init(&in_empty, CONSUMERS / 32);
    for (int s = 0; s < W_STAGES; ++s) { tc::mbar_init(&w_full[s], 1); tc::mbar_init(&w_empty[s], CONSUMERS / 32); }
    tc::mbar_fence_init();
    tc::tma_prefetch_desc(&tmHid); tc::tma_prefetch_desc(&tmX); tc::tma_prefetch_desc(&tmWo);
    tc::tma_prefetch_desc(&tmWe); tc::tma_prefetch_desc(&tmWs);
  }
  s6_pdl_trigger();
  if (tid < CONSUMERS) {
    // the 2048 bias / LayerNorm parameters (8 KB) do not depend on the previous kernel: pull them into L1 in front of the
    // dependency wait instead of paying an L2 round trip inside the first epilogue
    for (int i = tid; i < 512; i += CONSUMERS) {
      const float* p = i < 64 ? a.bo + i * 4 : i < 128 ? a.g1 + (i - 64) * 4 : i < 192 ? a.b1 + (i - 128) * 4 : i < 320 ? a.be + (i - 192) * 4
                     : i < 384 ? a.bs + (i - 320) * 4 : i < 448 ? a.g2 + (i - 384) * 4 : a.b2 + (i - 448) * 4;
      asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
    }
  }
  __syncthreads();
  s6_pdl_wait();                                     // hid / x come from the kernels before us

  if (warp >= CONSUMERS / 32) {
    // ------------------------------------------------------------------ TMA producer (one thread of the third warpgroup)
    tc::producer_regs();
    if (tid == CONSUMERS) {
      long long gw = 0;
      int it = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const int m0 = tile * BM;
        auto load_w = [&](int j) {
          const int s = (int)(gw % W_STAGES);
          tc::mbar_wait(&w_empty[s], (uint32_t)(((gw / W_STAGES) & 1) ^ 1));
          tc::mbar_arrive_expect_tx(&w_full[s], W_STAGE);
          uint8_t* dst = w_ring + s * W_STAGE;
          if (j < 4) tc::tma_load_2d(&tmWo, &w_full[s], dst, j * BK, 0);                              // G1
          else if (j < 12) tc::tma_load_2d(&tmWe, &w_full[s], dst, ((j - 4) & 3) * BK, ((j - 4) >> 2) * 256);   // G2a, G2b
          else tc::tma_load_2d(&tmWs, &w_full[s], dst, (j - 12) * BK, 0);                             // G3: k-blocks 0..7
          ++gw;
        };
        int j = 0;
        for (; j < W_STAGES; ++j) load_w(j);         // the ring refills while the previous tile is still in its last GEMM
        tc::mbar_wait(&in_empty, (uint32_t)((it & 1) ^ 1));   // previous tile: its G3 no longer reads the h halves
        tc::mbar_arrive_expect_tx(&in_full, 2 * T_BYTES);
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
          tc::tma_load_2d(&tmHid, &in_full, a_buf + kb * T_SLAB, kb * BK, m0);
          tc::tma_load_2d(&tmX, &in_full, x_buf + kb * T_SLAB, kb * BK, m0);
        }
        for (; j < W_PER_TILE; ++j) load_w(j);
      }
    }
    return;
  }
  // ------------------------------------------------------------------ warpgroups
  tc::consumer_regs();
  const int wg = warp >> 2, w = warp & 3;
  const uint32_t a_addr = tc::smem_u32(a_buf) + wg * (64 * 128), x_addr = tc::smem_u32(x_buf) + wg * (64 * 128), w_addr0 = tc::smem_u32(w_ring);
  long long gw = 0;
  float acc[C / 2];
  // nkb weight k-blocks against the slabs of an operand tile (k-block kb reads slab kb & 3 of op_addr, or of op_addr2 from kb 4 on)
  auto gemm = [&](uint32_t op_addr, uint32_t op_addr2, int nkb) {
    int prev = -1;
    for (int kb = 0; kb < nkb; ++kb, ++gw) {
      const int s = (int)(gw % W_STAGES);
      tc::mbar_wait(&w_full[s], (uint32_t)((gw / W_STAGES) & 1));
      const uint32_t op = (kb < 4 ? op_addr : op_addr2) + (kb & 3) * T_SLAB;
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        tc::wgmma_bf16<C>(acc, tc::wg_desc(op + k * 32), tc::wg_desc(w_addr0 + s * W_STAGE + k * 32), (kb | k) ? 1u : 0u);
      tc::wg_commit();
      if (prev >= 0) {
        tc::wg_wait<1>();
        if (lane == 0) tc::mbar_arrive(&w_empty[prev]);
      }
      prev = s;
    }
    tc::wg_wait<0>();
    if (lane == 0) tc::mbar_arrive(&w_empty[prev]);
  };
  // acc <- LayerNorm(acc + bias + residual) * g + b, the residual given per element pair
  auto layernorm = [&](const float* __restrict__ bias, const float* __restrict__ g, const float* __restrict__ b, auto&& residual) {
    float s[2] = {0.f, 0.f}, q[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < C / 2; e += 2) {
      const int hr = (e >> 1) & 1, col = tc::frag_col(e, lane);
      const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col)), rr = residual(e, hr, col);
      acc[e] += bb.x + rr.x; acc[e + 1] += bb.y + rr.y;
      s[hr] += acc[e] + acc[e + 1];
      q[hr] = fmaf(acc[e], acc[e], fmaf(acc[e + 1], acc[e + 1], q[hr]));
    }
    float mean[2], rstd[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      mean[hr] = tc::quad_sum(s[hr]) * (1.f / C);
      rstd[hr] = rsqrtf(fmaxf(tc::quad_sum(q[hr]) * (1.f / C) - mean[hr] * mean[hr], 0.f) + a.eps);
    }
#pragma unroll
    for (int e = 0; e < C / 2; e += 2) {
      const int hr = (e >> 1) & 1, col = tc::frag_col(e, lane);
      const float2 gg = __ldg(reinterpret_cast<const float2*>(g + col)), bb = __ldg(reinterpret_cast<const float2*>(b + col));
      acc[e] = fmaf((acc[e] - mean[hr]) * rstd[hr], gg.x, bb.x);
      acc[e + 1] = fmaf((acc[e + 1] - mean[hr]) * rstd[hr], gg.y, bb.y);
    }
  };
  // h half = relu(acc + b_e[...]) -> dst rows of this warpgroup
  auto relu_store = [&](const float* __restrict__ bias, uint8_t* dst) {
#pragma unroll
    for (int e = 0; e < C / 2; e += 2) {
      const int col = tc::frag_col(e, lane), r = wg * 64 + tc::frag_row(e, w, lane);
      const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col));
      *tile_pair(dst, r, col) = tc::pack_bf16(fmaxf(acc[e] + bb.x, 0.f), fmaxf(acc[e + 1] + bb.y, 0.f));
    }
  };
  auto publish = [&]() {                             // generic-proxy tile writes -> the warpgroup's next wgmma
    tc::fence_proxy_async_smem();
    tc::named_bar(1 + wg, 128);
  };
  int it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    tc::mbar_wait(&in_full, (uint32_t)(it & 1));
    gemm(a_addr, a_addr, 4);                         // G1
    layernorm(a.bo, a.g1, a.b1, [&](int e, int hr, int col) {
      return unpack2(*tile_pair(x_buf, wg * 64 + tc::frag_row(e, w, lane), col));
    });
#pragma unroll
    for (int e = 0; e < C / 2; e += 2) {             // E1: y -> over the hid rows (G1 has completed) and into out
      const int r = wg * 64 + tc::frag_row(e, w, lane), col = tc::frag_col(e, lane), row = tile * BM + r;
      const uint32_t y2 = tc::pack_bf16(acc[e], acc[e + 1]);
      *tile_pair(a_buf, r, col) = y2;
      if (row < a.M) *reinterpret_cast<uint32_t*>(out + (size_t)row * ld_out + col) = y2;
    }
    publish();                                       // also: every thread has read its x before h half 0 goes there
    gemm(a_addr, a_addr, 4);                         // G2a
    relu_store(a.be, x_buf);
    gemm(a_addr, a_addr, 4);                         // G2b
    tc::named_bar(1 + wg, 128);                      // all of G2b has read y before h half 1 overwrites it
    relu_store(a.be + 256, a_buf);
    publish();
    gemm(x_addr, a_addr, 8);                         // G3
    if (lane == 0) tc::mbar_arrive(&in_empty);       // the tile buffers are free for the next tile's hid / x
    layernorm(a.bs, a.g2, a.b2, [&](int e, int, int col) {
      const int row = tile * BM + wg * 64 + tc::frag_row(e, w, lane);
      return row < a.M ? unpack2(*reinterpret_cast<const uint32_t*>(out + (size_t)row * ld_out + col)) : make_float2(0.f, 0.f);
    });
#pragma unroll
    for (int e = 0; e < C / 2; e += 2) {
      const int row = tile * BM + wg * 64 + tc::frag_row(e, w, lane);
      if (row < a.M) *reinterpret_cast<uint32_t*>(out + (size_t)row * ld_out + tc::frag_col(e, lane)) = tc::pack_bf16(acc[e], acc[e + 1]);
    }
  }
}

}  // namespace

// out = LN2(y + relu(y We^T + be) Ws^T + bs),  y = LN1(hid Wo^T + bo + x)   (PEM/model/transformer.py:176-197, 435-438)
// hid, x, out: (M,256) bf16 with row strides ld_* (multiples of 8 elements); Wo (256,256), We (512,256), Ws (256,512) bf16
// row-major contiguous; fp32 vectors bo, g1, b1 (256), be (512), bs, g2, b2 (256).  out may not overlap hid or x of other rows
// (it is the scratch of the intermediate y of its own rows).
S6_API int sam6d_transformer_tail_bf16(const void* hid, long long ld_hid, const void* x, long long ld_x, const void* Wo, const float* bo,
                                       const float* g1, const float* b1, const void* We, const float* be, const void* Ws, const float* bs,
                                       const float* g2, const float* b2, void* out, long long ld_out, int M, float eps, void* stream) {
  S6_REQUIRE(hid && x && Wo && bo && g1 && b1 && We && be && Ws && bs && g2 && b2 && out && M >= 0);
  S6_REQUIRE((ld_hid % 8) == 0 && (ld_x % 8) == 0 && (ld_out % 8) == 0 && ld_hid >= C && ld_x >= C && ld_out >= C);
  S6_REQUIRE(((reinterpret_cast<uintptr_t>(hid) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(Wo) |
               reinterpret_cast<uintptr_t>(We) | reinterpret_cast<uintptr_t>(Ws) | reinterpret_cast<uintptr_t>(bo) | reinterpret_cast<uintptr_t>(be) |
               reinterpret_cast<uintptr_t>(bs) | reinterpret_cast<uintptr_t>(g1) | reinterpret_cast<uintptr_t>(b1) | reinterpret_cast<uintptr_t>(g2) |
               reinterpret_cast<uintptr_t>(b2)) & 15) == 0);
  if (M == 0) return 0;
  CUtensorMap tmHid, tmX, tmWo, tmWe, tmWs;
  int rc;
  if ((rc = tc::make_map_2d(&tmHid, hid, M, C, ld_hid, 64, BM))) return rc;
  if ((rc = tc::make_map_2d(&tmX, x, M, C, ld_x, 64, BM))) return rc;
  if ((rc = tc::make_map_2d(&tmWo, Wo, C, C, C, 64, 256))) return rc;
  if ((rc = tc::make_map_2d(&tmWe, We, HID, C, C, 64, 256))) return rc;
  if ((rc = tc::make_map_2d(&tmWs, Ws, C, HID, HID, 64, 256))) return rc;
  int grid;
  S6_CHECK(s6_persistent_grid(s6_cdiv(M, BM), 1, &grid));
  TailArgs a{bo, g1, b1, be, bs, g2, b2, M, eps};
  S6_CHECK(cudaFuncSetAttribute(tail_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  S6_CHECK(s6_launch_pdl(tail_tc_kernel, dim3(grid), dim3(THREADS), SMEM, s6_stream(stream), tmHid, tmX, tmWo, tmWe, tmWs, a,
                         reinterpret_cast<__nv_bfloat16*>(out), ld_out));
  S6_LAUNCH_CHECK();
  return 0;
}
