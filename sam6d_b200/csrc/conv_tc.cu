// conv_tc.cu -- implicit-GEMM convolution on wgmma for NHWC bf16 activations (every 1x1 and 3x3 convolution of YOLOv8-seg).
//
//   M = output pixels (tiles of 8 rows x 16 columns of one frame), N = Cout (tiles of 128), K = taps x Cin (slabs of 64 channels).
//
// No im2col buffer exists.  The A operand of K slab (tap (ky, kx), channels [64 c, 64 c + 64)) for the output tile at (oy0, ox0)
// is one TMA box of a 4-D tensor map over the input slice (C, W, H, N): start (64 c, s ox0 - p + kx, s oy0 - p + ky, n), box
// (64, 16 s, 8 s, 1) with element strides (1, s, s, 1), so the unit fetches exactly the 8 x 16 input pixels the tap reads, in
// output-pixel order, as 128 K-major rows of 128 bytes with the 128-byte swizzle (the wgmma layout).  Out-of-bounds elements are
// zero-filled: negative / too-large coordinates are the convolution's zero padding, channels >= Cin the ragged K tail (Cin = 80,
// 160, ...), so the weight slab may run past the tap's Cin columns (they are zeros of the weight map too).  The B operand is a
// 3-D map over the weights (Cin, taps, Cout), K-major per tap.
//
// Structure as gemm_tma.cu: persistent CTAs, one TMA thread feeding a 4-stage ring, two consumer warpgroups of 64 rows each
// (wgmma m64n128k16, fp32 accumulators in registers).  Epilogue: + bias (folded BatchNorm), optional SiLU, optional bf16 residual,
// store as bf16 or fp32 into a channel slice (row stride ldy >= Cout) through the output mapping
//   Y[n * y_bs + ((sy * y + oy) * Wy + sx * x + ox) * ldy + c]
// (identity for ordinary layers; sy = sx = 2 and (oy, ox) = tap for one tap of a 2x2 stride-2 transposed convolution).
#include "tc.cuh"

namespace {

constexpr int TY = 8, TX = 16, BM = TY * TX, BN = 128, BK = 64, STAGES = 4;
constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int CONSUMERS = 256, THREADS = CONSUMERS + 128;
constexpr int SMEM = STAGES * STAGE_BYTES + 1024;

struct ConvArgs {
  const float* bias;
  const __nv_bfloat16* R;
  void* Y;
  int Ho, Wo, Cout, Cin, kw, stride, pad;
  int tiles_x, tiles_y, m_tiles, n_tiles, nimg;
  long long ldr, r_bs, ldy, y_bs;
  int Wy, sy, sx, oy, ox;
};

__device__ __forceinline__ float silu(float x) { return x / (1.f + expf(-x)); }
__device__ __forceinline__ void st1(float* p, float a) { *p = a; }
__device__ __forceinline__ void st1(__nv_bfloat16* p, float a) { *p = __float2bfloat16(a); }
__device__ __forceinline__ void st2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
__device__ __forceinline__ void st2(__nv_bfloat16* p, float a, float b) { *reinterpret_cast<uint32_t*>(p) = tc::pack_bf16(a, b); }

template <typename OT, bool SILU, bool HAS_RES>
__global__ void __launch_bounds__(THREADS, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                                                            ConvArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long ntiles = (long long)g.m_tiles * g.n_tiles;
  const int ncc = (g.Cin + BK - 1) / BK, taps = g.kw * g.kw, nkb = taps * ncc;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], CONSUMERS / 32); }
    tc::mbar_fence_init();
    tc::tma_prefetch_desc(&tmX);
    tc::tma_prefetch_desc(&tmW);
  }
  s6_pdl_trigger();
  __syncthreads();
  s6_pdl_wait();                                   // the input / residual come from the kernel before us

  if (warp >= CONSUMERS / 32) {
    // ------------------------------------------------------------------ TMA producer (one thread of the third warpgroup)
    tc::producer_regs();
    if (tid == CONSUMERS) {
      long long gk = 0;
      for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int mt = (int)(tile % g.m_tiles), n0 = (int)(tile / g.m_tiles) * BN;
        const int tx = mt % g.tiles_x, ty = (mt / g.tiles_x) % g.tiles_y, img = mt / (g.tiles_x * g.tiles_y);
        const int ix0 = tx * TX * g.stride - g.pad, iy0 = ty * TY * g.stride - g.pad;
        for (int kb = 0; kb < nkb; ++kb, ++gk) {
          const int s = (int)(gk % STAGES);
          const int tap = kb / ncc, cc = kb - tap * ncc, ky = tap / g.kw, kx = tap - ky * g.kw;
          tc::mbar_wait(&empty_bar[s], (uint32_t)(((gk / STAGES) & 1) ^ 1));
          tc::mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
          uint8_t* a_slab = smem + s * STAGE_BYTES;
          tc::tma_load_4d(&tmX, &full_bar[s], a_slab, cc * BK, ix0 + kx, iy0 + ky, img);
          tc::tma_load_3d(&tmW, &full_bar[s], a_slab + A_BYTES, cc * BK, tap, n0);
        }
      }
    }
    return;
  }
  // ------------------------------------------------------------------ consumers: warpgroup wg <-> tile rows [64 wg, 64 wg + 64)
  tc::consumer_regs();
  const int wg = warp >> 2, w = warp & 3;
  float acc[BN / 2];
  long long gk = 0;
  OT* Y = reinterpret_cast<OT*>(g.Y);
  const bool pairs = ((g.ldy & 1) == 0) && (!HAS_RES || (g.ldr & 1) == 0);
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int mt = (int)(tile % g.m_tiles), n0 = (int)(tile / g.m_tiles) * BN;
    const int tx = mt % g.tiles_x, ty = (mt / g.tiles_x) % g.tiles_y, img = mt / (g.tiles_x * g.tiles_y);
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

    // ---- epilogue straight from the registers
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = wg * 64 + tc::frag_row(2 * h, w, lane);
      const int y = ty * TY + (r >> 4), x = tx * TX + (r & 15);
      if (y >= g.Ho || x >= g.Wo) continue;
      const long long pix = (long long)img * g.y_bs + ((long long)(g.sy * y + g.oy) * g.Wy + (g.sx * x + g.ox)) * g.ldy;
      const long long rpix = HAS_RES ? (long long)img * g.r_bs + ((long long)(g.sy * y + g.oy) * g.Wy + (g.sx * x + g.ox)) * g.ldr : 0;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + tc::frag_col(4 * j, lane);
        if (col >= g.Cout) continue;
        const bool two = col + 1 < g.Cout;
        float x0 = acc[4 * j + 2 * h] + __ldg(g.bias + col), x1 = two ? acc[4 * j + 2 * h + 1] + __ldg(g.bias + col + 1) : 0.f;
        if constexpr (SILU) { x0 = silu(x0); x1 = silu(x1); }
        if constexpr (HAS_RES) {
          x0 += __bfloat162float(g.R[rpix + col]);
          if (two) x1 += __bfloat162float(g.R[rpix + col + 1]);
        }
        if (two && pairs) st2(Y + pix + col, x0, x1);
        else {
          st1(Y + pix + col, x0);
          if (two) st1(Y + pix + col + 1, x1);
        }
      }
    }
  }
}

}  // namespace

// x (B, Hi, Wi, ldx) bf16 NHWC: channels [0, Cin) of each pixel row are the input (a channel slice: offset the pointer);
// w (Cout, k, k, Cin) bf16; bias (Cout) f32; k in {1, 3}, stride in {1, 2}, padding k / 2; silu 0 / 1; r bf16 residual or NULL,
// addressed like y with (ldr, r_bs); y bf16 (y_is_f32 = 0) or f32 (1) through the output mapping above (Wy = width of the output
// tensor, y_bs = elements between frames).  Cin % 8 == 0, ldx % 8 == 0, 16-byte aligned x and w.
S6_API int sam6d_conv2d_tc(const void* x, long long ldx, int B, int Hi, int Wi, int Cin, const void* w, int k, int stride, int Cout,
                           const float* bias, int silu, const void* r, long long ldr, long long r_bs, void* y, int y_is_f32, long long ldy,
                           long long y_bs, int Wy, int sy, int sx, int oy, int ox, void* stream) {
  S6_REQUIRE(x && w && bias && y && B >= 0 && Hi > 0 && Wi > 0 && Cin > 0 && Cout > 0 && (k == 1 || k == 3) && (stride == 1 || stride == 2));
  S6_REQUIRE((Cin % 8) == 0 && (ldx % 8) == 0 && ldx >= Cin && ldy >= Cout && (!r || ldr >= Cout) && Wy > 0 && sy >= 1 && sx >= 1);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(y) & (y_is_f32 ? 7 : 3)) == 0 && (!r || (reinterpret_cast<uintptr_t>(r) & 3) == 0));
  if (B == 0) return 0;
  const int pad = k / 2, Ho = (Hi + 2 * pad - k) / stride + 1, Wo = (Wi + 2 * pad - k) / stride + 1;
  CUtensorMap tmX, tmW;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)Wi, (cuuint64_t)Hi, (cuuint64_t)B};
    cuuint64_t str[3] = {(cuuint64_t)ldx * 2, (cuuint64_t)Wi * ldx * 2, (cuuint64_t)Hi * Wi * ldx * 2};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)(TX * stride), (cuuint32_t)(TY * stride), 1};
    cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    int rc = tc::encode_map(&tmX, x, 4, dims, str, box, estr);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)(k * k), (cuuint64_t)Cout};
    cuuint64_t str[2] = {(cuuint64_t)Cin * 2, (cuuint64_t)k * k * Cin * 2};
    cuuint32_t box[3] = {(cuuint32_t)BK, 1, (cuuint32_t)BN};
    cuuint32_t estr[3] = {1, 1, 1};
    int rc = tc::encode_map(&tmW, w, 3, dims, str, box, estr);
    if (rc) return rc;
  }
  ConvArgs g;
  g.bias = bias; g.R = reinterpret_cast<const __nv_bfloat16*>(r); g.Y = y;
  g.Ho = Ho; g.Wo = Wo; g.Cout = Cout; g.Cin = Cin; g.kw = k; g.stride = stride; g.pad = pad;
  g.tiles_x = s6_cdiv(Wo, TX); g.tiles_y = s6_cdiv(Ho, TY); g.nimg = B;
  const long long m_tiles = (long long)g.tiles_x * g.tiles_y * B;
  S6_REQUIRE(m_tiles < (1LL << 30));
  g.m_tiles = (int)m_tiles; g.n_tiles = s6_cdiv(Cout, BN);
  g.ldr = ldr; g.r_bs = r_bs; g.ldy = ldy; g.y_bs = y_bs; g.Wy = Wy; g.sy = sy; g.sx = sx; g.oy = oy; g.ox = ox;
  int grid;
  S6_CHECK(s6_persistent_grid(m_tiles * g.n_tiles, 1, &grid));
  cudaStream_t st = s6_stream(stream);
#define CONV_LAUNCH(OT, SL, HR)                                                                                      \
  do {                                                                                                               \
    auto kern = conv_tc_kernel<OT, SL, HR>;                                                                          \
    S6_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));                         \
    S6_CHECK(s6_launch_pdl(kern, dim3(grid), dim3(THREADS), SMEM, st, tmX, tmW, g));                                 \
  } while (0)
  if (y_is_f32) {
    S6_REQUIRE(!r);                                  // the fp32 outputs are the heads' last convolutions (Proto.cv3 has SiLU)
    if (silu) CONV_LAUNCH(float, true, false); else CONV_LAUNCH(float, false, false);
  } else if (silu) {
    if (r) CONV_LAUNCH(__nv_bfloat16, true, true); else CONV_LAUNCH(__nv_bfloat16, true, false);
  } else {
    if (r) CONV_LAUNCH(__nv_bfloat16, false, true); else CONV_LAUNCH(__nv_bfloat16, false, false);
  }
#undef CONV_LAUNCH
  S6_LAUNCH_CHECK();
  return 0;
}
