// linattn_tc.cu -- the dense side of the focused linear attention (PEM/model/transformer.py:541-559) on wgmma:
//
//   q' = focus(q)                       q = relu(x)+1e-6; q /= softplus(scale); n = ||q||; q = q^3; q = q/||q|| * n
//   x_h = (q'_h KV_h) / (q'_h . ksum_h + 1e-6)       per head h (4 heads x 64 channels), KV_h = sum_j k'_j v_j^T
//
// The (B, N, 256) dense token matrix is 65 k - 131 k rows; per row the reference does a 256-wide feature map and four 64x64
// mat-vecs.  One CTA handles 128 token rows of one cloud:
//   * all 8 warps: read the bf16 q rows (lane = 8 channels), apply the feature map in fp32 (two warp reductions), compute the
//     normaliser q'_h . ksum_h in fp32 (3-step reduction inside the 8 lanes of a head), and write q' as bf16 straight into the
//     swizzled wgmma A slabs (one [128][64] slab per head)
//   * KV_h^T arrives as a ready-made bf16 wgmma B image (4 x [64][64], SWIZZLE_128B) written by linattn_kv_pack_kernel,
//     pulled with one cp.async.bulk
//   * per head, each of the two warpgroups runs 4 x wgmma m64n64k16 on its 64 rows; the result is scaled by 1/normaliser and
//     stored as bf16 straight from the registers.
// 99 KB of shared memory per CTA: two CTAs per SM overlap the feature-map phase of one with the MMA/epilogue of the other.
// HBM traffic: q in, x out (2 x rows x 512 B).
#include "tc.cuh"

namespace {

constexpr int H = 4, D = 64, C = H * D;
constexpr int A_SLAB = 128 * 128;            // [128 rows][64 ch] bf16
constexpr int B_SLAB = 64 * 128;             // [64 e][64 d] bf16
constexpr int BLOB_BYTES = H * B_SLAB;       // per cloud
constexpr int LT_THREADS = 256;
constexpr int LT_SMEM = H * A_SLAB + H * B_SLAB + 128 * H * 4 + 1024;

// grid = B*H, 1024 threads.  Kf: focused keys, V: values, both (B, J, ld) fp32 views.  Writes the bf16 B-operand image of KV_h^T
// and ksum.  Thread (d, e0..e0+3) walks the J sparse tokens: a 196-step chain of 4 FMAs (a 256-thread version with 16
// accumulators per thread is bound by dependent-issue latency).
__global__ void __launch_bounds__(1024) linattn_kv_pack_kernel(const float* __restrict__ Kf, long long k_ld, long long k_bs,
                                                               const float* __restrict__ V, long long v_ld, long long v_bs, int J,
                                                               uint8_t* __restrict__ blob, float* __restrict__ KS) {
  extern __shared__ __align__(16) float sm[];
  float* ks = sm;           // J * D
  float* vs = ks + J * D;   // J * D
  const int bh = blockIdx.x, b = bh / H, h = bh - b * H, tid = threadIdx.x;
  for (int e = tid; e < J * D; e += 1024) {
    int j = e / D, c = e - j * D;
    ks[e] = Kf[(size_t)b * k_bs + (size_t)j * k_ld + h * D + c];
    vs[e] = V[(size_t)b * v_bs + (size_t)j * v_ld + h * D + c];
  }
  __syncthreads();
  const int d = tid >> 4, e0 = (tid & 15) * 4;   // KV[d][e0 .. e0+4)
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float ksum = 0.f;
#pragma unroll 4
  for (int j = 0; j < J; ++j) {
    const float kd = ks[j * D + d];
    const float4 v = *reinterpret_cast<const float4*>(vs + j * D + e0);
    ksum += kd;
    acc.x = fmaf(kd, v.x, acc.x); acc.y = fmaf(kd, v.y, acc.y); acc.z = fmaf(kd, v.z, acc.z); acc.w = fmaf(kd, v.w, acc.w);
  }
  uint8_t* slab = blob + (size_t)b * BLOB_BYTES + h * B_SLAB;     // row = e (the MMA's N), column = d (its K)
  *reinterpret_cast<__nv_bfloat16*>(slab + tc::sw128_offset(e0 + 0, d)) = __float2bfloat16(acc.x);
  *reinterpret_cast<__nv_bfloat16*>(slab + tc::sw128_offset(e0 + 1, d)) = __float2bfloat16(acc.y);
  *reinterpret_cast<__nv_bfloat16*>(slab + tc::sw128_offset(e0 + 2, d)) = __float2bfloat16(acc.z);
  *reinterpret_cast<__nv_bfloat16*>(slab + tc::sw128_offset(e0 + 3, d)) = __float2bfloat16(acc.w);
  if ((tid & 15) == 0) KS[(size_t)bh * D + d] = ksum;
}

struct LtArgs {
  const __nv_bfloat16* Q; long long q_ld, q_bs;
  const uint8_t* blob; const float* KS; const float* sp_scale;
  __nv_bfloat16* X; long long x_ld, x_bs;
  int rpb, tiles_per_cloud;
};

__global__ void __launch_bounds__(LT_THREADS, 2) linattn_tc_kernel(LtArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_s = smem;                                  // 4 head slabs [128 rows][64 ch]
  uint8_t* b_s = smem + H * A_SLAB;
  float* zs = reinterpret_cast<float*>(b_s + H * B_SLAB);   // [128][4] reciprocal normalisers
  __shared__ __align__(8) uint64_t blob_bar;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.x / a.tiles_per_cloud, tile = blockIdx.x - b * a.tiles_per_cloud;
  if (tid == 0) {
    tc::mbar_init(&blob_bar, 1);
    tc::mbar_fence_init();
    tc::mbar_arrive_expect_tx(&blob_bar, BLOB_BYTES);
    tc::bulk_load_1d(b_s, a.blob + (size_t)b * BLOB_BYTES, BLOB_BYTES, &blob_bar);
  }

  // ---------------------------------------------------------------- feature map: warp <-> rows warp, warp+8, ...
  float rs[8], ksv[8];
  {
    const float4 s0 = *reinterpret_cast<const float4*>(a.sp_scale + lane * 8), s1 = *reinterpret_cast<const float4*>(a.sp_scale + lane * 8 + 4);
    rs[0] = 1.f / s0.x; rs[1] = 1.f / s0.y; rs[2] = 1.f / s0.z; rs[3] = 1.f / s0.w;
    rs[4] = 1.f / s1.x; rs[5] = 1.f / s1.y; rs[6] = 1.f / s1.z; rs[7] = 1.f / s1.w;
    const float4 k0 = *reinterpret_cast<const float4*>(a.KS + (size_t)b * C + lane * 8), k1 = *reinterpret_cast<const float4*>(a.KS + (size_t)b * C + lane * 8 + 4);
    ksv[0] = k0.x; ksv[1] = k0.y; ksv[2] = k0.z; ksv[3] = k0.w; ksv[4] = k1.x; ksv[5] = k1.y; ksv[6] = k1.z; ksv[7] = k1.w;
  }
  const int head = lane >> 3, piece = lane & 7;
  const __nv_bfloat16* qbase = a.Q + (size_t)b * a.q_bs + (size_t)tile * 128 * a.q_ld + lane * 8;
  const int rows_left = a.rpb - tile * 128;
#pragma unroll 1
  for (int i0 = warp; i0 < 128; i0 += 32) {             // 4 rows in flight per warp
    uint4 raw[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = i0 + u * 8;
      raw[u] = (i < rows_left) ? *reinterpret_cast<const uint4*>(qbase + (size_t)i * a.q_ld) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = i0 + u * 8;
      const uint32_t w[4] = {raw[u].x, raw[u].y, raw[u].z, raw[u].w};
      float q[8];
      float s1 = 0.f, s3 = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        q[2 * e] = __uint_as_float(w[e] << 16);
        q[2 * e + 1] = __uint_as_float(w[e] & 0xffff0000u);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float t = (fmaxf(q[e], 0.f) + 1e-6f) * rs[e];
        s1 = fmaf(t, t, s1);
        t = t * t * t;
        s3 = fmaf(t, t, s3);
        q[e] = t;
      }
      s1 = warp_sum(s1);
      s3 = warp_sum(s3);
      const float n = sqrtf(s1) * rsqrtf(s3);
      float zp = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) { q[e] *= n; zp = fmaf(q[e], ksv[e], zp); }
      zp += __shfl_xor_sync(0xffffffffu, zp, 1);
      zp += __shfl_xor_sync(0xffffffffu, zp, 2);
      zp += __shfl_xor_sync(0xffffffffu, zp, 4);
      const bool valid = i < rows_left;
      if (piece == 0) zs[i * H + head] = valid ? 1.f / (zp + 1e-6f) : 0.f;
      uint4 o = make_uint4(0u, 0u, 0u, 0u);
      if (valid) o = make_uint4(tc::pack_bf16(q[0], q[1]), tc::pack_bf16(q[2], q[3]), tc::pack_bf16(q[4], q[5]), tc::pack_bf16(q[6], q[7]));
      *reinterpret_cast<uint4*>(a_s + head * A_SLAB + i * 128 + ((piece ^ (i & 7)) << 4)) = o;
    }
  }
  tc::fence_proxy_async_smem();
  __syncthreads();

  // ---------------------------------------------------------------- x = q' KV / z: warpgroup wg <-> rows [64 wg, 64 wg + 64)
  const int wg = warp >> 2, w = warp & 3;
  tc::mbar_wait(&blob_bar, 0);
  __nv_bfloat16* xb = a.X + (size_t)b * a.x_bs;         // rows of this cloud
#pragma unroll 1
  for (int h = 0; h < H; ++h) {
    float acc[D / 2];
    const uint32_t a_addr = tc::smem_u32(a_s + h * A_SLAB) + wg * (64 * 128), b_addr = tc::smem_u32(b_s + h * B_SLAB);
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k) tc::wgmma_bf16<D>(acc, tc::wg_desc(a_addr + k * 32), tc::wg_desc(b_addr + k * 32), k ? 1u : 0u);
    tc::wg_commit();
    tc::wg_wait<0>();
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int r = wg * 64 + tc::frag_row(2 * hr, w, lane), row = tile * 128 + r;
      if (row >= a.rpb) continue;
      const float z = zs[r * H + h];
#pragma unroll
      for (int j = 0; j < D / 8; ++j)
        *reinterpret_cast<uint32_t*>(xb + (size_t)row * a.x_ld + h * D + tc::frag_col(4 * j, lane)) =
            tc::pack_bf16(acc[4 * j + 2 * hr] * z, acc[4 * j + 2 * hr + 1] * z);
    }
  }
}

}  // namespace

// Kf, V: (B,J,4*64) fp32 views (row stride ld, cloud stride bs) -> blob (B x 32 KB bf16 wgmma image of KV_h^T), KS (B,4,64) fp32
S6_API int sam6d_linattn_kv_pack(const float* Kf, long long k_ld, long long k_bs, const float* V, long long v_ld, long long v_bs,
                                 int B, int J, void* blob, float* KS, void* stream) {
  S6_REQUIRE(Kf && V && blob && KS && B >= 0 && J > 0);
  if (B == 0) return 0;
  size_t smem = (size_t)2 * J * D * sizeof(float);
  S6_REQUIRE(smem <= 200 * 1024);
  S6_CHECK(cudaFuncSetAttribute(linattn_kv_pack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  linattn_kv_pack_kernel<<<B * H, 1024, smem, s6_stream(stream)>>>(Kf, k_ld, k_bs, V, v_ld, v_bs, J, reinterpret_cast<uint8_t*>(blob), KS);
  S6_LAUNCH_CHECK();
  return 0;
}

// Q: B clouds x rpb token rows x 256 bf16 (row stride q_ld, cloud stride q_bs), the raw query projection -> X likewise, bf16:
// X[b,i,h*64:(h+1)*64] = (focus(Q[b,i])_h KV[b,h]) / (focus(Q[b,i])_h . KS[b,h] + 1e-6)
S6_API int sam6d_linattn_tc(const void* Q, long long q_ld, long long q_bs, const void* blob, const float* KS,
                            const float* softplus_scale, int B, int rpb, void* X, long long x_ld, long long x_bs, void* stream) {
  S6_REQUIRE(Q && blob && KS && softplus_scale && X && B >= 0 && rpb >= 0 && (q_ld % 8) == 0 && (x_ld % 8) == 0 &&
             (q_bs % 8) == 0 && (x_bs % 8) == 0);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(Q) & 15) == 0 && (reinterpret_cast<uintptr_t>(X) & 15) == 0 &&
             (reinterpret_cast<uintptr_t>(blob) & 15) == 0 && (long long)B * rpb < 2000000000LL);
  if (B == 0 || rpb == 0) return 0;
  S6_CHECK(cudaFuncSetAttribute(linattn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LT_SMEM));
  LtArgs a{reinterpret_cast<const __nv_bfloat16*>(Q), q_ld, q_bs, reinterpret_cast<const uint8_t*>(blob), KS, softplus_scale,
           reinterpret_cast<__nv_bfloat16*>(X), x_ld, x_bs, rpb, s6_cdiv(rpb, 128)};
  linattn_tc_kernel<<<B * a.tiles_per_cloud, LT_THREADS, LT_SMEM, s6_stream(stream)>>>(a);
  S6_LAUNCH_CHECK();
  return 0;
}
