// gemm_simt.cu -- fp32 CUDA-core GEMM  C = act(A W^T + bias) (+ R)  with strided batches.
//
// This is the exact-precision path (and the comparator for the wgmma bf16 path): every Linear /
// 1x1-conv of the matching stage maps onto it.  A is (M,K) row-major with row stride lda, W is
// (N,K) row-major (nn.Linear layout) with row stride ldw, C is (M,N) with row stride ldc.  A batch
// index z = blockIdx.z offsets A, W, C, R by their batch strides (0 = shared operand).
#include "common.cuh"

namespace {

constexpr int BM = 128, BN = 64, BK = 16, TM = 8, TN = 4;  // 256 threads, each an 8x4 micro tile

struct GemmArgs {
  const float* A; const float* W; const float* bias; const float* R; float* C;
  int M, N, K;
  long long lda, ldw, ldc, ldr;
  long long sA, sW, sC, sR;   // batch strides (elements)
  float alpha;                // C = alpha * (A W^T) + bias ...
  int relu;
};

__global__ void __launch_bounds__(256) gemm_tn_kernel(GemmArgs g) {
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Ws[2][BK][BN + 4];
  const int z = blockIdx.z;
  const float* A = g.A + (size_t)z * g.sA;
  const float* W = g.W + (size_t)z * g.sW;
  float* C = g.C + (size_t)z * g.sC;
  const float* R = g.R ? g.R + (size_t)z * g.sR : nullptr;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;  // 16 x 16 thread grid: ty -> rows (8 each), tx -> cols (4 each)

  // global -> smem loaders: A tile 128x16 = 512 float4 (2 per thread), W tile 64x16 = 256 float4 (1 per thread)
  const int a_row = tid >> 2, a_k4 = (tid & 3) * 4;  // rows 0..63 (+64), k offset 0,4,8,12
  const int w_row = tid >> 2, w_k4 = (tid & 3) * 4;
  const bool k_vec = ((g.K & 3) == 0) && ((g.lda & 3) == 0) && ((g.ldw & 3) == 0) &&
                     ((((uintptr_t)A) & 15) == 0) && ((((uintptr_t)W) & 15) == 0);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float4 ra[2], rw;
  auto load_tile = [&](int k0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int r = m0 + a_row + h * 64, k = k0 + a_k4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < g.M) {
        const float* p = A + (size_t)r * g.lda + k;
        if (k_vec && k + 3 < g.K) v = *reinterpret_cast<const float4*>(p);
        else {
          if (k + 0 < g.K) v.x = p[0];
          if (k + 1 < g.K) v.y = p[1];
          if (k + 2 < g.K) v.z = p[2];
          if (k + 3 < g.K) v.w = p[3];
        }
      }
      ra[h] = v;
    }
    {
      int r = n0 + w_row, k = k0 + w_k4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < g.N) {
        const float* p = W + (size_t)r * g.ldw + k;
        if (k_vec && k + 3 < g.K) v = *reinterpret_cast<const float4*>(p);
        else {
          if (k + 0 < g.K) v.x = p[0];
          if (k + 1 < g.K) v.y = p[1];
          if (k + 2 < g.K) v.z = p[2];
          if (k + 3 < g.K) v.w = p[3];
        }
      }
      rw = v;
    }
  };
  auto store_tile = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int r = a_row + h * 64;
      As[buf][a_k4 + 0][r] = ra[h].x;
      As[buf][a_k4 + 1][r] = ra[h].y;
      As[buf][a_k4 + 2][r] = ra[h].z;
      As[buf][a_k4 + 3][r] = ra[h].w;
    }
    Ws[buf][w_k4 + 0][w_row] = rw.x;
    Ws[buf][w_k4 + 1][w_row] = rw.y;
    Ws[buf][w_k4 + 2][w_row] = rw.z;
    Ws[buf][w_k4 + 3][w_row] = rw.w;
  };

  const int nk = (g.K + BK - 1) / BK;
  load_tile(0);
  store_tile(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tile((kt + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * TM]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * TM + 4]);
      float4 w = *reinterpret_cast<const float4*>(&Ws[buf][kk][tx * TN]);
      float av[TM] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float wv[TN] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    if (kt + 1 < nk) store_tile(buf ^ 1);
    __syncthreads();
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int r = m0 + ty * TM + i;
    if (r >= g.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int c = n0 + tx * TN + j;
      if (c >= g.N) continue;
      float v = acc[i][j] * g.alpha;
      if (g.bias) v += g.bias[c];
      v = s6_act(v, g.relu);
      if (R) v += R[(size_t)r * g.ldr + c];
      C[(size_t)r * g.ldc + c] = v;
    }
  }
}

}  // namespace

// C[z] = alpha * A[z] W[z]^T (+bias) (relu) (+R[z]);  all pointers device fp32.
S6_API int sam6d_gemm_f32(const float* A, const float* W, const float* bias, const float* R, float* C, int M, int N, int K,
                          long long lda, long long ldw, long long ldc, long long ldr, int batch, long long sA,
                          long long sW, long long sC, long long sR, float alpha, int relu, void* stream) {
  S6_REQUIRE(A && W && C && M >= 0 && N > 0 && K > 0 && batch >= 0);
  if (M == 0 || batch == 0) return 0;
  S6_REQUIRE(batch <= 65535);
  GemmArgs g{A, W, bias, R, C, M, N, K, lda, ldw, ldc, ldr, sA, sW, sC, sR, alpha, relu};
  dim3 grid(s6_cdiv(N, BN), s6_cdiv(M, BM), batch);
  S6_REQUIRE(grid.y <= 65535);
  gemm_tn_kernel<<<grid, 256, 0, s6_stream(stream)>>>(g);
  S6_LAUNCH_CHECK();
  return 0;
}
