// rowops.cu -- one-warp-per-token kernels over C-channel rows (C = 256 in PEM, 1280 in SAM ViT-H; any multiple of 32 up to 2048):
// LayerNorm, L2 normalisation, the focused-linear-attention feature map, and the rigid warp of a point cloud.
//
// Rows are addressed as  base + (r / rows_per_batch) * batch_stride + (r % rows_per_batch) * ld  so that the
// dense-token view "rows 1..N of a (B, N+1, C) sequence" needs no copy.
#include "common.cuh"

namespace {

struct RowView {
  long long rpb, bstride, ld;
  __device__ __forceinline__ size_t off(long long r) const {
    long long b = r / rpb, i = r - b * rpb;
    return (size_t)(b * bstride + i * ld);
  }
};

constexpr int MAXV_LIMIT = 64;  // per-lane values: C / 32 <= 64 (C <= 2048); kernels are instantiated for 8 / 32 / 64

// LayerNorm(x) * gamma + beta, eps as nn.LayerNorm (PEM/model/transformer.py:156,188: nn.LayerNorm(d_model)).
__device__ __forceinline__ void st_out(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_out(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }

__device__ __forceinline__ float ld_in(const float* p) { return *p; }
__device__ __forceinline__ float ld_in(const __nv_bfloat16* p) { return __bfloat162float(*p); }

template <int MAXV, typename OT, typename IT = float>
__global__ void __launch_bounds__(256) layernorm_kernel(const IT* __restrict__ x, RowView xv, OT* __restrict__ y, RowView yv,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        long long rows, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  s6_pdl_trigger();
  s6_pdl_wait();
  if (r >= rows) return;
  const IT* xp = x + xv.off(r);
  OT* yp = y + yv.off(r);
  const int nv = C >> 5;
  float v[MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (i < nv) { v[i] = ld_in(xp + lane + 32 * i); s += v[i]; }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (i < nv) { float d = v[i] - mean; q += d * d; }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (i < nv) { int c = lane + 32 * i; st_out(yp + c, (v[i] - mean) * rstd * gamma[c] + beta[c]); }
}

// C = 256 bf16 rows (every LayerNorm of the bf16 PEM path): a row is 32 lanes x 16 bytes, one load and one store per lane
__global__ void __launch_bounds__(256) layernorm256_bf16_kernel(const __nv_bfloat16* __restrict__ x, RowView xv, __nv_bfloat16* __restrict__ y,
                                                                RowView yv, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                long long rows, float eps) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  s6_pdl_trigger();
  const float4 g0 = *reinterpret_cast<const float4*>(gamma + lane * 8), g1 = *reinterpret_cast<const float4*>(gamma + lane * 8 + 4);
  const float4 b0 = *reinterpret_cast<const float4*>(beta + lane * 8), b1 = *reinterpret_cast<const float4*>(beta + lane * 8 + 4);
  s6_pdl_wait();
  if (r >= rows) return;
  const uint4 raw = *reinterpret_cast<const uint4*>(x + xv.off(r) + lane * 8);
  const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
  float v[8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[2 * i] = __uint_as_float(w[i] << 16);
    v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    s += v[2 * i] + v[2 * i + 1];
  }
  const float mean = warp_sum(s) * (1.f / 256.f);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { const float d = v[i] - mean; q = fmaf(d, d, q); }
  const float rstd = rsqrtf(warp_sum(q) * (1.f / 256.f) + eps);
  const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float a = (v[2 * i] - mean) * rstd * gg[2 * i] + bb[2 * i], c = (v[2 * i + 1] - mean) * rstd * gg[2 * i + 1] + bb[2 * i + 1];
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, c);
    o[i] = *reinterpret_cast<const uint32_t*>(&h);
  }
  *reinterpret_cast<uint4*>(y + yv.off(r) + lane * 8) = make_uint4(o[0], o[1], o[2], o[3]);
}

// fp32 rows -> bf16 rows with C % 128 == 0 (the ViT-H LayerNorms, C = 1280): lane l owns floats [128 i + 4 l, +4), 16-byte
// loads and 8-byte stores instead of the 4 / 2-byte accesses of the generic kernel
template <int NV>
__global__ void __launch_bounds__(256) layernorm_vec_f32_bf16_kernel(const float* __restrict__ x, RowView xv, __nv_bfloat16* __restrict__ y,
                                                                     RowView yv, const float* __restrict__ gamma,
                                                                     const float* __restrict__ beta, long long rows, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  s6_pdl_trigger();
  s6_pdl_wait();
  if (r >= rows) return;
  const float* xp = x + xv.off(r) + lane * 4;
  __nv_bfloat16* yp = y + yv.off(r) + lane * 4;
  const int nv = C >> 7;
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (i < nv) { v[i] = *reinterpret_cast<const float4*>(xp + 128 * i); s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (i < nv) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (i < nv) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + lane * 4 + 128 * i));
      const float4 b = __ldg(reinterpret_cast<const float4*>(beta + lane * 4 + 128 * i));
      const __nv_bfloat162 lo = __floats2bfloat162_rn((v[i].x - mean) * rstd * g.x + b.x, (v[i].y - mean) * rstd * g.y + b.y);
      const __nv_bfloat162 hi = __floats2bfloat162_rn((v[i].z - mean) * rstd * g.z + b.z, (v[i].w - mean) * rstd * g.w + b.w);
      uint2 o;
      o.x = *reinterpret_cast<const uint32_t*>(&lo);
      o.y = *reinterpret_cast<const uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(yp + 128 * i) = o;
    }
}

// F.normalize(x, p=2, dim=-1): x / max(||x||, 1e-12)   (PEM/utils/model_utils.py:124-126)
template <int MAXV, typename OT = float>
__global__ void __launch_bounds__(256) l2norm_kernel(const float* __restrict__ x, RowView xv, OT* __restrict__ y, RowView yv,
                                                     long long rows, int C) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* xp = x + xv.off(r);
  OT* yp = y + yv.off(r);
  const int nv = C >> 5;
  float v[MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (i < nv) { v[i] = xp[lane + 32 * i]; s += v[i] * v[i]; }
  const float n = fmaxf(sqrtf(warp_sum(s)), 1e-12f);
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (i < nv) st_out(yp + lane + 32 * i, v[i] / n);
}

// Focused linear attention feature map (PEM/model/transformer.py:541-550):
//   q = relu(x) + 1e-6;  q = q / softplus(scale);  n = ||q||;  q = q^3;  q = q / ||q|| * n
template <int MAXV>
__global__ void __launch_bounds__(256) focus_kernel(const float* __restrict__ x, RowView xv, float* __restrict__ y, RowView yv,
                                                    const float* __restrict__ sp_scale, long long rows, int C) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* xp = x + xv.off(r);
  float* yp = y + yv.off(r);
  const int nv = C >> 5;
  float v[MAXV];
  float s1 = 0.f, s3 = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (i < nv) {
      int c = lane + 32 * i;
      float q = (fmaxf(xp[c], 0.f) + 1e-6f) / sp_scale[c];
      s1 += q * q;
      q = q * q * q;
      s3 += q * q;
      v[i] = q;
    }
  const float n1 = sqrtf(warp_sum(s1)), n3 = sqrtf(warp_sum(s3));
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (i < nv) yp[lane + 32 * i] = (v[i] / n3) * n1;
}

// out[b,i,:] = (p[b,i,:] - t[b]) @ R[b]        (PEM/model/fine_point_matching.py:44)
__global__ void rigid_warp_kernel(const float* __restrict__ p, const float* __restrict__ R, const float* __restrict__ t, int n,
                                  long long total, float* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int b = (int)(i / n);
  const float* Rb = R + (size_t)b * 9;
  const float* tb = t + (size_t)b * 3;
  float x = p[i * 3 + 0] - tb[0], y = p[i * 3 + 1] - tb[1], z = p[i * 3 + 2] - tb[2];
  out[i * 3 + 0] = x * Rb[0] + y * Rb[3] + z * Rb[6];
  out[i * 3 + 1] = x * Rb[1] + y * Rb[4] + z * Rb[7];
  out[i * 3 + 2] = x * Rb[2] + y * Rb[5] + z * Rb[8];
}

// per-cloud radius normalisation (PEM/model/feature_extraction.py:139-142):
//   radius[b] = max_i ||po[b,i]||;  pm /= radius + 1e-6;  po /= radius + 1e-6;  model /= radius + 1e-6
__global__ void __launch_bounds__(256) radius_kernel(const float* __restrict__ po, int n, float* __restrict__ radius) {
  __shared__ float red[8];
  const int b = blockIdx.x;
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) {
    const float* q = po + ((size_t)b * n + i) * 3;
    m = fmaxf(m, sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]));
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
    radius[b] = m;
  }
}
__global__ void scale_by_radius_kernel(const float* __restrict__ src, const float* __restrict__ radius, long long per_batch,
                                       long long total, float* __restrict__ dst) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  dst[i] = src[i] / (radius[i / per_batch] + 1e-6f);
}

}  // namespace

#define ROW_ARGS_OK(C) ((C) % 32 == 0 && (C) <= 32 * MAXV_LIMIT && (C) > 0)
#define ROW_DISPATCH(C, KERNEL, ...)                                   \
  do {                                                                 \
    if ((C) <= 256) KERNEL<8 ROW_EXTRA> __VA_ARGS__;                   \
    else if ((C) <= 1024) KERNEL<32 ROW_EXTRA> __VA_ARGS__;            \
    else KERNEL<64 ROW_EXTRA> __VA_ARGS__;                             \
  } while (0)
// LayerNorm goes through the PDL launch (see common.cuh)
#define LN_DISPATCH(C, IT, OT, ...)                                                                                          \
  do {                                                                                                                       \
    if ((C) <= 256) S6_CHECK(s6_launch_pdl(layernorm_kernel<8, OT, IT>, __VA_ARGS__));                                       \
    else if ((C) <= 1024) S6_CHECK(s6_launch_pdl(layernorm_kernel<32, OT, IT>, __VA_ARGS__));                                \
    else S6_CHECK(s6_launch_pdl(layernorm_kernel<64, OT, IT>, __VA_ARGS__));                                                 \
  } while (0)

#define ROW_EXTRA , float
S6_API int sam6d_layernorm(const float* x, long long x_rpb, long long x_bstride, long long x_ld, float* y, long long y_rpb,
                           long long y_bstride, long long y_ld, const float* gamma, const float* beta, long long rows, int C,
                           float eps, void* stream) {
  S6_REQUIRE(x && y && gamma && beta && rows >= 0 && ROW_ARGS_OK(C));
  if (rows == 0) return 0;
  LN_DISPATCH(C, float, float, dim3(s6_cdiv(rows, 8)), dim3(256), 0, s6_stream(stream), x, RowView{x_rpb, x_bstride, x_ld}, y,
              RowView{y_rpb, y_bstride, y_ld}, gamma, beta, rows, C, eps);
  S6_LAUNCH_CHECK();
  return 0;
}

#undef ROW_EXTRA
#define ROW_EXTRA , __nv_bfloat16
// same, writing bf16 rows (the A operand of the next tensor-core GEMM)
S6_API int sam6d_layernorm_bf16(const float* x, long long x_rpb, long long x_bstride, long long x_ld, void* y, long long y_rpb,
                                long long y_bstride, long long y_ld, const float* gamma, const float* beta, long long rows, int C,
                                float eps, void* stream) {
  S6_REQUIRE(x && y && gamma && beta && rows >= 0 && ROW_ARGS_OK(C));
  if (rows == 0) return 0;
  if ((C % 128) == 0 && (x_ld % 4) == 0 && (y_ld % 4) == 0 && (x_bstride % 4) == 0 && (y_bstride % 4) == 0 &&
      (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 7) == 0 &&
      ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15) == 0) {
    const RowView xv{x_rpb, x_bstride, x_ld}, yv{y_rpb, y_bstride, y_ld};
    __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(y);
    if (C <= 512) S6_CHECK(s6_launch_pdl(layernorm_vec_f32_bf16_kernel<4>, dim3(s6_cdiv(rows, 8)), dim3(256), 0, s6_stream(stream), x, xv, yb, yv, gamma, beta, rows, C, eps));
    else if (C <= 1280) S6_CHECK(s6_launch_pdl(layernorm_vec_f32_bf16_kernel<10>, dim3(s6_cdiv(rows, 8)), dim3(256), 0, s6_stream(stream), x, xv, yb, yv, gamma, beta, rows, C, eps));
    else S6_CHECK(s6_launch_pdl(layernorm_vec_f32_bf16_kernel<16>, dim3(s6_cdiv(rows, 8)), dim3(256), 0, s6_stream(stream), x, xv, yb, yv, gamma, beta, rows, C, eps));
    S6_LAUNCH_CHECK();
    return 0;
  }
  LN_DISPATCH(C, float, __nv_bfloat16, dim3(s6_cdiv(rows, 8)), dim3(256), 0, s6_stream(stream), x, RowView{x_rpb, x_bstride, x_ld},
              reinterpret_cast<__nv_bfloat16*>(y), RowView{y_rpb, y_bstride, y_ld}, gamma, beta, rows, C, eps);
  S6_LAUNCH_CHECK();
  return 0;
}
#undef ROW_EXTRA
#define ROW_EXTRA , __nv_bfloat16, __nv_bfloat16
// bf16 rows in, bf16 rows out (statistics in fp32): the all-bf16 activation flow of the dense PEM layers
S6_API int sam6d_layernorm_bf16io(const void* x, long long x_rpb, long long x_bstride, long long x_ld, void* y, long long y_rpb,
                                  long long y_bstride, long long y_ld, const float* gamma, const float* beta, long long rows, int C,
                                  float eps, void* stream) {
  S6_REQUIRE(x && y && gamma && beta && rows >= 0 && ROW_ARGS_OK(C));
  if (rows == 0) return 0;
  if (C == 256 && (x_ld % 8) == 0 && (y_ld % 8) == 0 && (x_bstride % 8) == 0 && (y_bstride % 8) == 0 &&
      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15) == 0) {
    S6_CHECK(s6_launch_pdl(layernorm256_bf16_kernel, dim3(s6_cdiv(rows, 8)), dim3(256), 0, s6_stream(stream),
                           reinterpret_cast<const __nv_bfloat16*>(x), RowView{x_rpb, x_bstride, x_ld}, reinterpret_cast<__nv_bfloat16*>(y),
                           RowView{y_rpb, y_bstride, y_ld}, gamma, beta, rows, eps));
    S6_LAUNCH_CHECK();
    return 0;
  }
  LN_DISPATCH(C, __nv_bfloat16, __nv_bfloat16, dim3(s6_cdiv(rows, 8)), dim3(256), 0, s6_stream(stream),
              reinterpret_cast<const __nv_bfloat16*>(x), RowView{x_rpb, x_bstride, x_ld}, reinterpret_cast<__nv_bfloat16*>(y),
              RowView{y_rpb, y_bstride, y_ld}, gamma, beta, rows, C, eps);
  S6_LAUNCH_CHECK();
  return 0;
}
#undef ROW_EXTRA
#define ROW_EXTRA

S6_API int sam6d_l2norm_rows(const float* x, long long x_rpb, long long x_bstride, long long x_ld, float* y, long long y_rpb,
                             long long y_bstride, long long y_ld, long long rows, int C, void* stream) {
  S6_REQUIRE(x && y && rows >= 0 && ROW_ARGS_OK(C));
  if (rows == 0) return 0;
  ROW_DISPATCH(C, l2norm_kernel, <<<s6_cdiv(rows, 8), 256, 0, s6_stream(stream)>>>(x, RowView{x_rpb, x_bstride, x_ld}, y,
               RowView{y_rpb, y_bstride, y_ld}, rows, C));
  S6_LAUNCH_CHECK();
  return 0;
}

#undef ROW_EXTRA
#define ROW_EXTRA , __nv_bfloat16
// same, bf16 result: the operands of the tensor-core score GEMM
S6_API int sam6d_l2norm_rows_bf16(const float* x, long long x_rpb, long long x_bstride, long long x_ld, void* y, long long y_rpb,
                                  long long y_bstride, long long y_ld, long long rows, int C, void* stream) {
  S6_REQUIRE(x && y && rows >= 0 && ROW_ARGS_OK(C));
  if (rows == 0) return 0;
  ROW_DISPATCH(C, l2norm_kernel, <<<s6_cdiv(rows, 8), 256, 0, s6_stream(stream)>>>(x, RowView{x_rpb, x_bstride, x_ld},
               reinterpret_cast<__nv_bfloat16*>(y), RowView{y_rpb, y_bstride, y_ld}, rows, C));
  S6_LAUNCH_CHECK();
  return 0;
}
#undef ROW_EXTRA
#define ROW_EXTRA

S6_API int sam6d_focus_rows(const float* x, long long x_rpb, long long x_bstride, long long x_ld, float* y, long long y_rpb,
                            long long y_bstride, long long y_ld, const float* softplus_scale, long long rows, int C,
                            void* stream) {
  S6_REQUIRE(x && y && softplus_scale && rows >= 0 && ROW_ARGS_OK(C));
  if (rows == 0) return 0;
  ROW_DISPATCH(C, focus_kernel, <<<s6_cdiv(rows, 8), 256, 0, s6_stream(stream)>>>(x, RowView{x_rpb, x_bstride, x_ld}, y,
               RowView{y_rpb, y_bstride, y_ld}, softplus_scale, rows, C));
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_rigid_warp(const float* p, const float* R, const float* t, int b, int n, float* out, void* stream) {
  // an empty batch is nothing to do, whatever the (possibly null) addresses of its empty arrays
  S6_REQUIRE(b >= 0 && n >= 0);
  long long total = (long long)b * n;
  if (total == 0) return 0;
  S6_REQUIRE(p && R && t && out);
  rigid_warp_kernel<<<s6_cdiv(total, 256), 256, 0, s6_stream(stream)>>>(p, R, t, n, total, out);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_cloud_radius(const float* po, int b, int n, float* radius, void* stream) {
  S6_REQUIRE(b >= 0 && n > 0);
  if (b == 0) return 0;
  S6_REQUIRE(po && radius);
  radius_kernel<<<b, 256, 0, s6_stream(stream)>>>(po, n, radius);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_scale_by_radius(const float* src, const float* radius, int b, long long per_batch, float* dst, void* stream) {
  S6_REQUIRE(b >= 0 && per_batch >= 0);
  long long total = (long long)b * per_batch;
  if (total == 0) return 0;
  S6_REQUIRE(src && radius && dst);
  scale_by_radius_kernel<<<s6_cdiv(total, 256), 256, 0, s6_stream(stream)>>>(src, radius, per_batch, total, dst);
  S6_LAUNCH_CHECK();
  return 0;
}
