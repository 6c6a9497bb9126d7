// epilogue.cuh -- shared register epilogue of the wgmma GEMMs.
//
// Input: one 64 x N accumulator fragment of a warpgroup (tc.cuh layout: a thread holds column pairs of four rows).  Per
// element: alpha * acc (+ bias) (activation) (+ residual) -> OT.  A thread writes its two adjacent columns with one 8-byte
// (fp32) or 4-byte (bf16) store, so the four lanes of a quad fill 8 adjacent columns of a row and every 32-byte sector of
// an fp32 output is written whole.
// Everything that can be decided at compile time is (activation, bias / residual presence): a runtime activation switch
// if-converts into ~50 predicated erff instructions per element.
#pragma once
#include "tc.cuh"

namespace epi {

template <int ACT>
__device__ __forceinline__ float act_fn(float x) {
  if constexpr (ACT == 1) return fmaxf(x, 0.f);
  if constexpr (ACT == 2) return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
  return x;
}

template <typename T>
struct ident { using type = T; };   // keeps RT out of template argument deduction (callers pass nullptr)
__device__ __forceinline__ float ld_res(const float* p) { return *p; }
__device__ __forceinline__ float ld_res(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float2 ld_res2(const float* p) { return *reinterpret_cast<const float2*>(p); }
__device__ __forceinline__ float2 ld_res2(const __nv_bfloat16* p) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p)); }
__device__ __forceinline__ void st1(float* p, float a) { *p = a; }
__device__ __forceinline__ void st1(__nv_bfloat16* p, float a) { *p = __float2bfloat16(a); }
__device__ __forceinline__ void st2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
__device__ __forceinline__ void st2(__nv_bfloat16* p, float a, float b) { *reinterpret_cast<uint32_t*>(p) = tc::pack_bf16(a, b); }

// d: this thread's fragment of a 64 x N accumulator whose row 0 is global row `row0` and column 0 global column `col0`;
// w: warp index inside the warpgroup.  Only the 8-column groups j in [j_lo, j_hi) are written; rows >= M and columns >= N_lim
// are skipped.  RT: residual element type.  C, R and bias must allow 2-element accesses at even columns (even ldc / ldr).
template <typename OT, int ACT, bool HAS_BIAS, bool HAS_RES, typename RT = float, int N>
__device__ __forceinline__ void store_frag(const float (&d)[N / 2], int w, int lane, int row0, int M, int col0, int N_lim, float alpha,
                                           const float* __restrict__ bias, const typename ident<RT>::type* __restrict__ R, long long ldr,
                                           OT* __restrict__ C, long long ldc, int j_lo = 0, int j_hi = N / 8) {
  const bool pairs = ((ldc & 1) == 0) && (!HAS_RES || (ldr & 1) == 0);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int col = col0 + tc::frag_col(4 * j, lane);
    if (j < j_lo || j >= j_hi || col >= N_lim) continue;
    const bool two = col + 1 < N_lim;
    float b0 = 0.f, b1 = 0.f;
    if constexpr (HAS_BIAS) { b0 = __ldg(bias + col); if (two) b1 = __ldg(bias + col + 1); }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + tc::frag_row(2 * h, w, lane);
      if (row >= M) continue;
      float x0 = act_fn<ACT>(fmaf(d[4 * j + 2 * h], alpha, b0)), x1 = act_fn<ACT>(fmaf(d[4 * j + 2 * h + 1], alpha, b1));
      const size_t rc = (size_t)row * ldc + col;
      if (two && pairs) {
        if constexpr (HAS_RES) { const float2 r = ld_res2(R + (size_t)row * ldr + col); x0 += r.x; x1 += r.y; }
        st2(C + rc, x0, x1);
      } else {
        if constexpr (HAS_RES) x0 += ld_res(R + (size_t)row * ldr + col);
        st1(C + rc, x0);
        if (two) {
          if constexpr (HAS_RES) x1 += ld_res(R + (size_t)row * ldr + col + 1);
          st1(C + rc + 1, x1);
        }
      }
    }
  }
}

// Gated (SwiGLU) epilogue of a 64 x 256 fragment: columns [0, 128) of the tile are the gate pre-activations x1 of 128 hidden
// units, columns [128, 256) the matching "up" pre-activations x2 (the W rows are interleaved in blocks of 128 on the host).
// Column 8j + 2(lane&3) + e and column 8(j+16) + 2(lane&3) + e sit in the same thread (d[4j + 2h + e], d[4(j+16) + 2h + e]),
// so hidden = silu(x1) * x2 is formed in registers and 128 bf16 columns are written from out_col0 on.  bias: the packed
// (interleaved) bias, indexed by the tile's column col0.  C must allow 2-element stores at even columns (even ldc).
__device__ __forceinline__ void store_frag_swiglu(const float (&d)[128], int w, int lane, int row0, int M, int col0, int out_col0,
                                                  float alpha, const float* __restrict__ bias, __nv_bfloat16* __restrict__ C,
                                                  long long ldc) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = tc::frag_col(4 * j, lane);
    const float g0 = __ldg(bias + col0 + c), g1 = __ldg(bias + col0 + c + 1);
    const float u0 = __ldg(bias + col0 + 128 + c), u1 = __ldg(bias + col0 + 128 + c + 1);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + tc::frag_row(2 * h, w, lane);
      if (row >= M) continue;
      const float x0 = fmaf(d[4 * j + 2 * h], alpha, g0), x1 = fmaf(d[4 * j + 2 * h + 1], alpha, g1);
      const float y0 = fmaf(d[4 * (j + 16) + 2 * h], alpha, u0), y1 = fmaf(d[4 * (j + 16) + 2 * h + 1], alpha, u1);
      st2(C + (size_t)row * ldc + out_col0 + c, x0 / (1.f + __expf(-x0)) * y0, x1 / (1.f + __expf(-x1)) * y1);
    }
  }
}

// run-time -> compile-time dispatch of (ACT, HAS_BIAS, HAS_RES)
#define EPI_DISPATCH(ACT_V, BIAS_P, RES_P, ...)                                              \
  do {                                                                                       \
    const int a__ = (ACT_V);                                                                 \
    const bool b__ = (BIAS_P) != nullptr, r__ = (RES_P) != nullptr;                          \
    if (a__ == 0) {                                                                          \
      if (b__) { if (r__) { __VA_ARGS__(0, true, true); } else { __VA_ARGS__(0, true, false); } } \
      else     { if (r__) { __VA_ARGS__(0, false, true); } else { __VA_ARGS__(0, false, false); } } \
    } else if (a__ == 1) {                                                                   \
      if (b__) { if (r__) { __VA_ARGS__(1, true, true); } else { __VA_ARGS__(1, true, false); } } \
      else     { if (r__) { __VA_ARGS__(1, false, true); } else { __VA_ARGS__(1, false, false); } } \
    } else {                                                                                 \
      if (b__) { if (r__) { __VA_ARGS__(2, true, true); } else { __VA_ARGS__(2, true, false); } } \
      else     { if (r__) { __VA_ARGS__(2, false, true); } else { __VA_ARGS__(2, false, false); } } \
    }                                                                                        \
  } while (0)

}  // namespace epi
