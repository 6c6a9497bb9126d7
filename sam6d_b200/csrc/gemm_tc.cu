// gemm_tc.cu -- bf16 tensor-core GEMM on wgmma with fp32 accumulation in registers:
//     C[z] = alpha * A[z] W[z]^T (+ bias) (ReLU) (+ R[z])
// Same contract as sam6d_gemm_f32 (gemm_simt.cu); A and W may be fp32 (converted to bf16 while staging) or bf16, C fp32 or bf16.
//
// CTA = one 128 x 256 output tile, 12 warps, warp-specialised:
//   warps 8-11 producers : coalesced 16-byte global loads -> bf16 -> st.shared into K-major, 128B-swizzled [rows][64] slabs
//                          (the layout a TMA SWIZZLE_128B box would produce), 2-stage mbarrier ring
//   warps 0-7  consumers : warpgroup g owns rows [64 g, 64 g + 64): 4 x wgmma m64n256k16 per 64-wide k-block, then
//                          bias / ReLU / residual -> global straight from the accumulator registers (epilogue.cuh)
#include "epilogue.cuh"
#include "tc.cuh"

namespace {

constexpr int BM = 128, BN = 256, BK = 64, STAGES = 2;
constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int CONSUMERS = 256, NUM_THREADS = CONSUMERS + 128;

struct TcArgs {
  const void* A; const void* W; const float* bias; const float* R; void* C;
  int M, N, K;
  long long lda, ldw, ldc, ldr, sA, sW, sC, sR;
  float alpha;
  int relu;
};

// stage `rows` x 64 of a row-major (rows_total, K) operand into a swizzled slab; zero-fill out-of-range rows / columns.
// All global loads of a batch are issued before the first use (16 x 16-byte loads in flight per thread): with the loads
// interleaved with the conversion every load's latency is exposed.
template <typename T, int ROWS>
__device__ __forceinline__ void stage_tile(const T* __restrict__ base, long long ld, int row0, int rows_total, int k0, int K,
                                           uint8_t* __restrict__ slab, int ptid) {
  if constexpr (sizeof(T) == 4) {
    constexpr int UNITS = ROWS * 16;                 // float4 units
    constexpr int BATCH = 16;
#pragma unroll 1
    for (int i0 = 0; i0 < UNITS / 128; i0 += BATCH) {
      float4 v[BATCH];
#pragma unroll
      for (int i = 0; i < BATCH; ++i) {
        const int u = (i0 + i) * 128 + ptid, r = u >> 4, c = (u & 15) << 2;
        const int gr = row0 + r, gk = k0 + c;
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gr < rows_total && gk < K) v[i] = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + (size_t)gr * ld + gk));
      }
#pragma unroll
      for (int i = 0; i < BATCH; ++i) {
        const int u = (i0 + i) * 128 + ptid, r = u >> 4, c = (u & 15) << 2;
        *reinterpret_cast<uint2*>(slab + tc::sw128_offset(r, c)) = make_uint2(tc::pack_bf16(v[i].x, v[i].y), tc::pack_bf16(v[i].z, v[i].w));
      }
    }
  } else {
    constexpr int UNITS = ROWS * 8;                  // 16-byte units of 8 bf16
    constexpr int BATCH = (UNITS / 128) < 16 ? (UNITS / 128) : 16;
#pragma unroll 1
    for (int i0 = 0; i0 < UNITS / 128; i0 += BATCH) {
      uint4 v[BATCH];
#pragma unroll
      for (int i = 0; i < BATCH; ++i) {
        const int u = (i0 + i) * 128 + ptid, r = u >> 3, c = (u & 7) << 3;
        const int gr = row0 + r, gk = k0 + c;
        v[i] = make_uint4(0u, 0u, 0u, 0u);
        if (gr < rows_total && gk < K) v[i] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(base) + (size_t)gr * ld + gk));
      }
#pragma unroll
      for (int i = 0; i < BATCH; ++i) {
        const int u = (i0 + i) * 128 + ptid, r = u >> 3, c = (u & 7) << 3;
        *reinterpret_cast<uint4*>(slab + tc::sw128_offset(r, c)) = v[i];
      }
    }
  }
}

template <typename AT, typename WT, typename OT, int ACT, bool HAS_BIAS, bool HAS_RES>
__global__ void __launch_bounds__(NUM_THREADS, 1) gemm_tc_kernel(TcArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int z = blockIdx.z, m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const AT* A = reinterpret_cast<const AT*>(g.A) + (size_t)z * g.sA;
  const WT* W = reinterpret_cast<const WT*>(g.W) + (size_t)z * g.sW;
  const int nkb = (g.K + BK - 1) / BK;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full_bar[s], 128); tc::mbar_init(&empty_bar[s], CONSUMERS / 32); }
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (tid >= CONSUMERS) {
    // ------------------------------------------------------------------ producers
    const int ptid = tid - CONSUMERS;
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % STAGES;
      tc::mbar_wait(&empty_bar[s], ((kb / STAGES) & 1) ^ 1);
      uint8_t* a_slab = smem + s * STAGE_BYTES;
      uint8_t* b_slab = a_slab + A_BYTES;
      stage_tile<AT, BM>(A, g.lda, m0, g.M, kb * BK, g.K, a_slab, ptid);
      stage_tile<WT, BN>(W, g.ldw, n0, g.N, kb * BK, g.K, b_slab, ptid);
      tc::fence_proxy_async_smem();
      tc::mbar_arrive(&full_bar[s]);
    }
    return;
  }
  // ------------------------------------------------------------------ consumers: warpgroup wg <-> rows [64 wg, 64 wg + 64)
  const int wg = warp >> 2, w = warp & 3;
  float acc[BN / 2];
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb % STAGES;
    tc::mbar_wait(&full_bar[s], (kb / STAGES) & 1);
    const uint32_t a_addr = tc::smem_u32(smem + s * STAGE_BYTES) + wg * (64 * 128), b_addr = tc::smem_u32(smem + s * STAGE_BYTES) + A_BYTES;
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) tc::wgmma_bf16<BN>(acc, tc::wg_desc(a_addr + k * 32), tc::wg_desc(b_addr + k * 32), (kb | k) ? 1u : 0u);
    tc::wg_commit();
    tc::wg_wait<0>();
    if (lane == 0) tc::mbar_arrive(&empty_bar[s]);
  }
  OT* Cz = reinterpret_cast<OT*>(g.C) + (size_t)z * g.sC;
  const float* Rz = g.R ? g.R + (size_t)z * g.sR : nullptr;
  epi::store_frag<OT, ACT, HAS_BIAS, HAS_RES, float, BN>(acc, w, lane, m0 + wg * 64, g.M, n0, g.N, g.alpha, g.bias, Rz, g.ldr, Cz, g.ldc);
}

template <typename AT, typename WT, typename OT>
int launch(const TcArgs& g, int batch, cudaStream_t st) {
  const size_t smem = STAGES * STAGE_BYTES + 1024;
  dim3 grid(s6_cdiv(g.N, BN), s6_cdiv(g.M, BM), batch);
  cudaError_t e = cudaSuccess;
#define LAUNCH_TC(ACT, HB, HR)                                                                    \
  do {                                                                                            \
    auto kern = gemm_tc_kernel<AT, WT, OT, ACT, HB, HR>;                                          \
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);       \
    if (e != cudaSuccess) return (int)e;                                                          \
    kern<<<grid, NUM_THREADS, smem, st>>>(g);                                                     \
  } while (0)
  EPI_DISPATCH(g.relu, g.bias, g.R, LAUNCH_TC);
#undef LAUNCH_TC
  e = cudaGetLastError();
  return (int)e;
}

}  // namespace

// dtype codes: 0 = fp32, 1 = bf16.  Requires K % 8 == 0 and 16-byte aligned operand rows (lda/ldw multiples of 4 (fp32) or 8 (bf16)).
S6_API int sam6d_gemm_bf16(const void* A, int a_dtype, const void* W, int w_dtype, const float* bias, const float* R, void* C,
                           int c_dtype, int M, int N, int K, long long lda, long long ldw, long long ldc, long long ldr, int batch,
                           long long sA, long long sW, long long sC, long long sR, float alpha, int relu, void* stream) {
  S6_REQUIRE(A && W && C && M >= 0 && N > 0 && K > 0 && batch >= 0 && (K % 8) == 0 && relu >= 0 && relu <= 2);
  if (M == 0 || batch == 0) return 0;
  S6_REQUIRE(batch <= 65535 && s6_cdiv(M, BM) <= 65535);
  const int am = a_dtype ? 8 : 4, wm = w_dtype ? 8 : 4;
  S6_REQUIRE(lda % am == 0 && ldw % wm == 0 && sA % am == 0 && sW % wm == 0);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0);
  TcArgs g{A, W, bias, R, C, M, N, K, lda, ldw, ldc, ldr, sA, sW, sC, sR, alpha, relu};
  cudaStream_t st = s6_stream(stream);
  const int code = (a_dtype ? 4 : 0) | (w_dtype ? 2 : 0) | (c_dtype ? 1 : 0);
  switch (code) {
    case 0: return launch<float, float, float>(g, batch, st);
    case 1: return launch<float, float, __nv_bfloat16>(g, batch, st);
    case 2: return launch<float, __nv_bfloat16, float>(g, batch, st);
    case 3: return launch<float, __nv_bfloat16, __nv_bfloat16>(g, batch, st);
    case 4: return launch<__nv_bfloat16, float, float>(g, batch, st);
    case 5: return launch<__nv_bfloat16, float, __nv_bfloat16>(g, batch, st);
    case 6: return launch<__nv_bfloat16, __nv_bfloat16, float>(g, batch, st);
    default: return launch<__nv_bfloat16, __nv_bfloat16, __nv_bfloat16>(g, batch, st);
  }
}
