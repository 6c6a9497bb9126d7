// geo.cu -- GeometricStructureEmbedding (PEM/model/transformer.py:286-349).
//
//   E[b,i,j,:] = proj_d(sin_emb(d_ij / sigma_d)) + max_k proj_a(sin_emb(angle_ijk * factor_a))
//
// Stage 1 (geo_indices): pairwise distances in the reference's expanded form, 3 nearest neighbours per
// anchor, the three triplet angles and the distance index -> T[b,i,j,4] = {a0, a1, a2, d}.
// Stage 2 (geo_embed_f32): the two 256x256 projections applied to sinusoidal embeddings that are generated
// on the fly (never materialised), max over the three angle rows fused in the epilogue.  This file holds the
// exact fp32 CUDA-core version; geo_tc.cu holds the wgmma bf16 version.
#include "common.cuh"

namespace {

// one CTA per (anchor i, cloud b)
__global__ void __launch_bounds__(256) geo_indices_kernel(const float* __restrict__ pts, int S, float inv_sigma_d_den,
                                                          float factor_a, float* __restrict__ T) {
  extern __shared__ float sm[];
  float* px = sm;            // S
  float* py = px + S;
  float* pz = py + S;
  float* dist = pz + S;      // S
  __shared__ float red_v[8];
  __shared__ int red_i[8];
  __shared__ int knn[4];

  const int i = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* p = pts + (size_t)b * S * 3;
  for (int j = tid; j < S; j += 256) { px[j] = p[j * 3]; py[j] = p[j * 3 + 1]; pz[j] = p[j * 3 + 2]; }
  __syncthreads();
  const float xi = px[i], yi = py[i], zi = pz[i];
  const float x2 = xi * xi + yi * yi + zi * zi;
  for (int j = tid; j < S; j += 256) {
    // pairwise_distance (PEM/utils/model_utils.py:98-111): x2 - 2 xy + y2, clamp(min=0); then sqrt (transformer.py:315)
    float xj = px[j], yj = py[j], zj = pz[j];
    float y2 = xj * xj + yj * yj + zj * zj;
    float xy = xi * xj + yi * yj + zi * zj;
    float sq = fmaxf(x2 - 2.f * xy + y2, 0.f);
    dist[j] = sqrtf(sq);
  }
  __syncthreads();
  // 4 smallest distances (value, then index), ascending: topk(k+1, largest=False); entry 0 is dropped
  for (int round = 0; round < 4; ++round) {
    float bv = INFINITY;
    int bi = 0x7fffffff;
    for (int j = tid; j < S; j += 256) {
      bool taken = false;
      for (int q = 0; q < round; ++q) taken |= (knn[q] == j);
      float v = dist[j];
      if (!taken && (v < bv || (v == bv && j < bi))) { bv = v; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float v2 = __shfl_xor_sync(0xffffffffu, bv, o);
      int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
      if (v2 < bv || (v2 == bv && i2 < bi)) { bv = v2; bi = i2; }
    }
    if (lane == 0) { red_v[warp] = bv; red_i[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < 8; ++w)
        if (red_v[w] < bv || (red_v[w] == bv && red_i[w] < bi)) { bv = red_v[w]; bi = red_i[w]; }
      knn[round] = (bi == 0x7fffffff) ? 0 : bi;
    }
    __syncthreads();
  }
  float rx[3], ry[3], rz[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int q = knn[k + 1];
    rx[k] = px[q] - xi; ry[k] = py[q] - yi; rz[k] = pz[q] - zi;
  }
  float* Trow = T + ((size_t)b * S + i) * S * 4;
  for (int j = tid; j < S; j += 256) {
    float ax = px[j] - xi, ay = py[j] - yi, az = pz[j] - zi;
    float4 o;
    float a[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      float cx = ry[k] * az - rz[k] * ay;
      float cy = rz[k] * ax - rx[k] * az;
      float cz = rx[k] * ay - ry[k] * ax;
      float sinv = sqrtf(cx * cx + cy * cy + cz * cz);
      // + 0.0f: torch.sum starts from +0, so an all-(-0) product sum (anchor == query, negative ref vector) is +0 there and
      // atan2(0, +0) = 0; without it the FMA chain yields -0 and atan2f(0, -0) = pi
      float cosv = (rx[k] * ax + ry[k] * ay + rz[k] * az) + 0.0f;
      a[k] = atan2f(sinv, cosv) * factor_a;
    }
    o.x = a[0]; o.y = a[1]; o.z = a[2];
    o.w = dist[j] / inv_sigma_d_den;
    reinterpret_cast<float4*>(Trow)[j] = o;
  }
}

// fp32 embedding + projection.  One CTA = TP pairs x 256 output channels; thread = output channel.
constexpr int TP = 16;

__global__ void __launch_bounds__(256) geo_embed_f32_kernel(const float* __restrict__ T, long long npairs,
                                                            const float* __restrict__ div_term,
                                                            const float* __restrict__ WaT,  // (256 k, 256 c)
                                                            const float* __restrict__ WdT,  // (256 k, 256 c)
                                                            const float* __restrict__ bias, // b_a + b_d, (256)
                                                            float* __restrict__ E) {
  extern __shared__ __align__(16) float semb[];  // [256 k][TP*4]
  const int tid = threadIdx.x;
  const long long p0 = (long long)blockIdx.x * TP;
  // sinusoidal embeddings of the 4*TP scalars: token q = pair*4 + type, frequency f -> (sin, cos) at k = 2f, 2f+1
  for (int e = tid; e < TP * 4 * 128; e += 256) {
    int q = e & (TP * 4 - 1), f = e / (TP * 4);
    long long pair = p0 + (q >> 2);
    float x = (pair < npairs) ? T[pair * 4 + (q & 3)] : 0.f;
    float s, c;
    sincosf(x * div_term[f], &s, &c);
    semb[(2 * f) * (TP * 4) + q] = s;
    semb[(2 * f + 1) * (TP * 4) + q] = c;
  }
  __syncthreads();
  float acc[TP][4];
#pragma unroll
  for (int i = 0; i < TP; ++i)
#pragma unroll
    for (int t = 0; t < 4; ++t) acc[i][t] = 0.f;
#pragma unroll 2
  for (int k = 0; k < 256; ++k) {
    const float wa = WaT[k * 256 + tid], wd = WdT[k * 256 + tid];
    const float4* row = reinterpret_cast<const float4*>(semb + k * (TP * 4));
#pragma unroll
    for (int i = 0; i < TP; ++i) {
      float4 v = row[i];
      acc[i][0] = fmaf(wa, v.x, acc[i][0]);
      acc[i][1] = fmaf(wa, v.y, acc[i][1]);
      acc[i][2] = fmaf(wa, v.z, acc[i][2]);
      acc[i][3] = fmaf(wd, v.w, acc[i][3]);
    }
  }
  const float bc = bias[tid];
#pragma unroll
  for (int i = 0; i < TP; ++i) {
    long long pair = p0 + i;
    if (pair < npairs) E[pair * 256 + tid] = acc[i][3] + fmaxf(fmaxf(acc[i][0], acc[i][1]), acc[i][2]) + bc;
  }
}

}  // namespace

// pts (b,S,3) f32 -> T (b,S,S,4) f32 = {a_idx k=0..2, d_idx}   (transformer.py:302-332)
S6_API int sam6d_geo_indices(const float* pts, int b, int S, float sigma_d, float factor_a, float* T, void* stream) {
  S6_REQUIRE(pts && T && b >= 0 && S >= 4 && S <= 4096);
  if (b == 0) return 0;
  dim3 grid(S, b);
  const size_t smem = (size_t)S * 4 * sizeof(float);          // 64 KB at S = 4096: above the 48 KB default, opt in on every call
  S6_CHECK(cudaFuncSetAttribute(geo_indices_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   // (per device, cheap)
  geo_indices_kernel<<<grid, 256, smem, s6_stream(stream)>>>(pts, S, sigma_d, factor_a, T);
  S6_LAUNCH_CHECK();
  return 0;
}

// T (npairs,4) -> E (npairs,256) f32.  WaT/WdT are the transposed (in,out) copies of proj_a/proj_d weights,
// bias = proj_a.bias + proj_d.bias.   (transformer.py:334-349, reduction_a = 'max', hidden_dim = 256)
S6_API int sam6d_geo_embed_f32(const float* T, long long npairs, const float* div_term, const float* WaT, const float* WdT,
                               const float* bias, float* E, void* stream) {
  S6_REQUIRE(T && div_term && WaT && WdT && bias && E && npairs >= 0);
  if (npairs == 0) return 0;
  const size_t smem = 256 * TP * 4 * sizeof(float);
  // unconditionally: the attribute is per device, a process-wide flag would leave a second GPU of the same process without it
  S6_CHECK(cudaFuncSetAttribute(geo_embed_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  geo_embed_f32_kernel<<<s6_cdiv(npairs, TP), 256, smem, s6_stream(stream)>>>(T, npairs, div_term, WaT, WdT, bias, E);
  S6_LAUNCH_CHECK();
  return 0;
}
