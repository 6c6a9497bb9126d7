// tc.cuh -- sm_90a tensor-core plumbing: mbarrier, TMA 2-D tile loads, proxy fences and warpgroup MMA (wgmma) on K-major
// 128-byte-swizzled bf16 operands with fp32 accumulators in registers.  Inline PTX only; the one host part is the encoding of
// the TMA tensor maps that produce those operands.
//
// Accumulator fragment of one m64nN wgmma (the layout every kernel here reads its results in): thread t of the warpgroup
// (warp w = t / 32, lane l) holds d[i], i < N/2, at row 16 w + l/4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (l & 3) + (i & 1)
// (frag_row / frag_col).  A row of the tile lives in the four lanes of a quad, so row reductions are two xor-shuffles.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)   // suspend-time hint: the warp sleeps in the barrier unit instead of
      : "memory");                                         // re-issuing try_wait (a spinning warp costs its sub-partition issue slots)
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------------------------------------------------- fences
// generic-proxy smem writes (st.shared) -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor for a K-major operand tile stored as rows of 64 bf16 (128 bytes) with the 128-byte swizzle
// (16-byte chunk index XOR (row % 8)); 8-row groups are 1024 bytes apart (SBO), tile base 1024-byte aligned.  The k-th 16-wide
// K step of a slab starts 32 k bytes further.  Fields: start>>4 [0,14), LBO>>4 [16,30) (unused when swizzled), SBO>>4 [32,46),
// layout [62,64) = 1 (SWIZZLE_128B).
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// before the first wgmma that reads or writes accumulator registers the warpgroup has touched
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed groups of this warpgroup are still running
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D (64 x N, fp32 fragment) (+)= A (64 x 16, K-major smem) * B (N x 16, K-major smem)^T; all 128 threads of the warpgroup
template <int N>
struct Wgmma;
// the specialisations: register lists "%0, ..." in chunks of eight, "+f" operand lists of the fragment
#define S6_R0 "%0, %1, %2, %3, %4, %5, %6, %7"
#define S6_R1 "%8, %9, %10, %11, %12, %13, %14, %15"
#define S6_R2 "%16, %17, %18, %19, %20, %21, %22, %23"
#define S6_R3 "%24, %25, %26, %27, %28, %29, %30, %31"
#define S6_R4 "%32, %33, %34, %35, %36, %37, %38, %39"
#define S6_R5 "%40, %41, %42, %43, %44, %45, %46, %47"
#define S6_R6 "%48, %49, %50, %51, %52, %53, %54, %55"
#define S6_R7 "%56, %57, %58, %59, %60, %61, %62, %63"
#define S6_R8 "%64, %65, %66, %67, %68, %69, %70, %71"
#define S6_R9 "%72, %73, %74, %75, %76, %77, %78, %79"
#define S6_R10 "%80, %81, %82, %83, %84, %85, %86, %87"
#define S6_R11 "%88, %89, %90, %91, %92, %93, %94, %95"
#define S6_R12 "%96, %97, %98, %99, %100, %101, %102, %103"
#define S6_R13 "%104, %105, %106, %107, %108, %109, %110, %111"
#define S6_R14 "%112, %113, %114, %115, %116, %117, %118, %119"
#define S6_R15 "%120, %121, %122, %123, %124, %125, %126, %127"
#define S6_F4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define S6_F8(i) S6_F4(i), S6_F4(i + 4)
#define S6_F16(i) S6_F8(i), S6_F8(i + 8)
#define S6_F32(i) S6_F16(i), S6_F16(i + 16)
#define S6_F64(i) S6_F32(i), S6_F32(i + 32)
// DA, DB, ACC: the operand numbers that follow the N/2 accumulator registers
#define S6_WGMMA(N, REGS, DA, DB, ACC, ...)                                                                                     \
  template <>                                                                                                                \
  struct Wgmma<N> {                                                                                                          \
    __device__ __forceinline__ static void mma(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc) {                 \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " ACC ", 0;\n\twgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 {" \
                   REGS "}, " DA ", " DB ", p, 1, 1, 0, 0;\n\t}"                                                             \
                   : __VA_ARGS__                                                                                             \
                   : "l"(da), "l"(db), "r"(acc));                                                                            \
    }                                                                                                                        \
  };
S6_WGMMA(16, S6_R0, "%8", "%9", "%10", S6_F8(0))
S6_WGMMA(32, S6_R0 ", " S6_R1, "%16", "%17", "%18", S6_F16(0))
S6_WGMMA(64, S6_R0 ", " S6_R1 ", " S6_R2 ", " S6_R3, "%32", "%33", "%34", S6_F32(0))
S6_WGMMA(80, S6_R0 ", " S6_R1 ", " S6_R2 ", " S6_R3 ", " S6_R4, "%40", "%41", "%42", S6_F32(0), S6_F8(32))
S6_WGMMA(128, S6_R0 ", " S6_R1 ", " S6_R2 ", " S6_R3 ", " S6_R4 ", " S6_R5 ", " S6_R6 ", " S6_R7, "%64", "%65", "%66", S6_F64(0))
S6_WGMMA(256, S6_R0 ", " S6_R1 ", " S6_R2 ", " S6_R3 ", " S6_R4 ", " S6_R5 ", " S6_R6 ", " S6_R7 ", " S6_R8 ", " S6_R9 ", " S6_R10
         ", " S6_R11 ", " S6_R12 ", " S6_R13 ", " S6_R14 ", " S6_R15, "%128", "%129", "%130", S6_F64(0), S6_F64(64))

template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  Wgmma<N>::mma(d, da, db, accumulate);
}

// position of fragment element i inside the 64-row tile of warpgroup thread (warp w of the group, lane l)
__host__ __device__ constexpr int frag_row(int i, int w, int l) { return 16 * w + (l >> 2) + 8 * ((i >> 1) & 1); }
__host__ __device__ constexpr int frag_col(int i, int l) { return 8 * (i >> 2) + 2 * (l & 3) + (i & 1); }

// sum / max over the four lanes of a quad (the four threads that hold one accumulator row)
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// warp-specialised kernels of three warpgroups (one TMA thread + two MMA warpgroups): the TMA warpgroup hands its registers
// to the MMA warpgroups (40 + 2 x 232 per thread of a warpgroup fill the register file at 384 threads)
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs)); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs)); }

__device__ __forceinline__ void named_bar(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// byte offset of element (row, col) inside a [rows][64] bf16 tile with the 128-byte swizzle
__device__ __forceinline__ uint32_t sw128_offset(int row, int col) {
  return (uint32_t)(row * 128 + ((((col >> 3) ^ (row & 7)) << 4) | ((col & 7) << 1)));
}

// ---------------------------------------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_load_2d(const void* tmap, uint64_t* bar, void* smem_dst, int crd0, int crd1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(crd0), "r"(crd1)
               : "memory");
}
__device__ __forceinline__ void tma_load_3d(const void* tmap, uint64_t* bar, void* smem_dst, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_load_4d(const void* tmap, uint64_t* bar, void* smem_dst, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// 1-D bulk copy global -> shared (size multiple of 16 bytes), completion counted on an mbarrier
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gmem_src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}

// Host side: the tensor maps the loads above read.  Every map is bf16 with the 128-byte swizzle (a box of 64 channels lands as
// the K-major slab wg_desc describes), 256-byte L2 promotion and out-of-bounds elements read as zeros.  Both encoders
// return 0, 999 when the driver entry point is unavailable, or 1000 + the CUresult of a rejected map.
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<EncodeFn>(p);
  }
  return fn;
}

// rank-dimensional map: dims, box and element strides estr innermost first; strides_bytes of dimensions 1 .. rank-1
inline int encode_map(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                      const cuuint32_t* box, const cuuint32_t* estr) {
  EncodeFn enc = get_encode();
  if (!enc) return 999;
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), dims, strides_bytes, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 1000 + (int)r;
}

// 2-D row-major (rows, cols) matrix with row stride ld (elements); box = {box_cols, box_rows}
inline int make_map_2d(CUtensorMap* map, const void* ptr, long long rows, long long cols, long long ld, int box_cols, int box_rows) {
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return encode_map(map, ptr, 2, gdim, gstride, box, estr);
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace tc
