// pn2.cu -- point-cloud sampling / grouping kernels (replaces the reference's pointnet2._ext for
// the four ops PEM inference calls; PEM/model/pointnet2/_ext_src/src/{sampling,ball_query,group_points}_gpu.cu).
//
// Index outputs are bit-exact with the reference kernels: the squared-distance expression is
// evaluated with the same contraction nvcc applies there (FMUL, FFMA, FFMA) and argmax ties
// follow the reference's reduction tree (smallest bit-reversed k mod block_size, then smallest k).
#include "common.cuh"

// ------------------------------------------------------------------------------------------
// furthest point sampling
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float sqdist_ref(float x1, float y1, float z1, float x2, float y2, float z2) {
  float dx = x2 - x1, dy = y2 - y1, dz = z2 - z1;
  float d = __fmul_rn(dx, dx);
  d = __fmaf_rn(dy, dy, d);
  d = __fmaf_rn(dz, dz, d);
  return d;
}

struct FpsCand {
  float d;
  int k;
};

// Total order equivalent to the reference's per-thread scan + shared-memory tree (sampling_gpu.cu:64-70,113-170).
// Thread t = k mod block_size keeps its first maximal k (strict '>').  The tree then folds slot t+s into slot t for
// s = bs/2 ... 1 and a tie keeps slot t, so between two tied threads the one with a 0 at the LOWEST differing bit of
// t survives: ties go to the smallest bit-reversed thread id, then to the smallest k.
__device__ __forceinline__ bool fps_better(float d2, int k2, float d1, int k1, int bs_mask) {
  if (d2 != d1) return d2 > d1;
  unsigned t2 = __brev((unsigned)(k2 & bs_mask)), t1 = __brev((unsigned)(k1 & bs_mask));
  if (t2 != t1) return t2 < t1;
  return k2 < k1;
}

// One CTA per cloud, all points and running min-distances in registers (n <= THREADS*PPT <= 4096).
// The order of fps_better is folded into one pair of unsigned keys per candidate -- hi = bits of the (non-negative) distance,
// lo = 2^21 - ((bit-reversed thread slot << 12) | k), 0 for "no candidate" -- so the arg-max of a round is two redux.sync per
// level (max of hi, then max of lo among the lanes that hold it) instead of a five-step shuffle tree of compares: the 195
// serial rounds are pure latency.
template <int THREADS, int PPT>
__global__ void __launch_bounds__(THREADS) fps_reg_kernel(const float* __restrict__ xyz, int n, int m,
                                                           int bs_ref, int* __restrict__ idx) {
  extern __shared__ float sm[];
  float* sx = sm;
  float* sy = sm + n;
  float* sz = sm + 2 * n;
  constexpr int NW = THREADS / 32;
  __shared__ unsigned red_hi[2][NW], red_lo[2][NW];

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* p = xyz + (size_t)b * n * 3;
  int* out = idx + (size_t)b * m;
  for (int i = tid; i < n * 3; i += THREADS) {
    float v = p[i];
    int k = i / 3, c = i - k * 3;
    (c == 0 ? sx : (c == 1 ? sy : sz))[k] = v;
  }
  __syncthreads();
  const int bs_mask = bs_ref - 1, nb = 31 - __clz(bs_ref);      // bs_ref is a power of two
  float px[PPT], py[PPT], pz[PPT], tmp[PPT];
  unsigned lo[PPT];
#pragma unroll
  for (int i = 0; i < PPT; ++i) {
    int k = tid + i * THREADS;
    bool ok = k < n;
    px[i] = ok ? sx[k] : 0.f;
    py[i] = ok ? sy[k] : 0.f;
    pz[i] = ok ? sz[k] : 0.f;
    tmp[i] = 1e10f;
    const unsigned slot = nb ? (__brev((unsigned)(k & bs_mask)) >> (32 - nb)) : 0u;
    lo[i] = ok ? (1u << 21) - ((slot << 12) | (unsigned)k) : 0u;
  }
  int old = 0;
  if (tid == 0) out[0] = 0;
  for (int j = 1; j < m; ++j) {
    float x1 = sx[old], y1 = sy[old], z1 = sz[old];
    unsigned bh = 0u, bl = 0u;
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
      if (lo[i]) {
        float d = sqdist_ref(x1, y1, z1, px[i], py[i], pz[i]);
        float d2 = fminf(d, tmp[i]);
        tmp[i] = d2;
        const unsigned h = __float_as_uint(d2);
        if (h > bh || (h == bh && lo[i] > bl)) { bh = h; bl = lo[i]; }
      }
    }
    unsigned wh = __reduce_max_sync(0xffffffffu, bh);
    unsigned wl = __reduce_max_sync(0xffffffffu, bh == wh ? bl : 0u);
    const int buf = j & 1;
    if (lane == 0) { red_hi[buf][warp] = wh; red_lo[buf][warp] = wl; }
    __syncthreads();
    bh = lane < NW ? red_hi[buf][lane] : 0u;
    bl = lane < NW ? red_lo[buf][lane] : 0u;
    wh = __reduce_max_sync(0xffffffffu, bh);
    wl = __reduce_max_sync(0xffffffffu, bh == wh ? bl : 0u);
    old = (int)(((1u << 21) - wl) & 0xfffu);
    if (tid == 0) out[j] = old;
  }
}

// General n: running min-distances in a caller-provided scratch (b,n) f32, points from global/L2.
template <int THREADS>
__global__ void __launch_bounds__(THREADS) fps_big_kernel(const float* __restrict__ xyz, int n, int m, int bs_ref,
                                                           float* __restrict__ temp, int* __restrict__ idx) {
  __shared__ float red_d[2][THREADS / 32];
  __shared__ int red_k[2][THREADS / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* p = xyz + (size_t)b * n * 3;
  float* tmp = temp + (size_t)b * n;
  int* out = idx + (size_t)b * m;
  for (int k = tid; k < n; k += THREADS) tmp[k] = 1e10f;
  const int bs_mask = bs_ref - 1;
  int old = 0;
  if (tid == 0) out[0] = 0;
  for (int j = 1; j < m; ++j) {
    float x1 = p[old * 3 + 0], y1 = p[old * 3 + 1], z1 = p[old * 3 + 2];
    float best = -1.f;
    int besti = 0;
    for (int k = tid; k < n; k += THREADS) {
      float d = sqdist_ref(x1, y1, z1, p[k * 3 + 0], p[k * 3 + 1], p[k * 3 + 2]);
      float d2 = fminf(d, tmp[k]);
      tmp[k] = d2;
      if (best < 0.f || fps_better(d2, k, best, besti, bs_mask)) { best = d2; besti = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float d2 = __shfl_xor_sync(0xffffffffu, best, o);
      int k2 = __shfl_xor_sync(0xffffffffu, besti, o);
      if (d2 >= 0.f && (best < 0.f || fps_better(d2, k2, best, besti, bs_mask))) { best = d2; besti = k2; }
    }
    const int buf = j & 1;
    if (lane == 0) { red_d[buf][warp] = best; red_k[buf][warp] = besti; }
    __syncthreads();
    best = red_d[buf][0];
    besti = red_k[buf][0];
#pragma unroll
    for (int w = 1; w < THREADS / 32; ++w) {
      float d2 = red_d[buf][w];
      int k2 = red_k[buf][w];
      if (d2 >= 0.f && (best < 0.f || fps_better(d2, k2, best, besti, bs_mask))) { best = d2; besti = k2; }
    }
    old = besti;
    if (tid == 0) out[j] = old;
  }
}

// Large clouds (the 210 000-point template bank of get_obj_feats, PEM/model/feature_extraction.py:170-181): one thread-block
// CLUSTER per cloud.  Each of the CS CTAs keeps its slice of the points and running min-distances in shared memory (SoA, up to
// 13 312 points = 208 KB), finds its local arg-max with two redux.sync per level on packed keys, publishes (distance bits, tie
// key) into every CTA's distributed shared memory, and one barrier.cluster per round later each CTA reduces the CS entries on its
// own -- no global-memory round trip, no grid sync.  The slots are double-buffered by round parity, so one cluster barrier per
// round suffices.  Tie order as above (bs_ref = 512 for these sizes): key = 2^27 - ((bit-reversed (k mod 512) << 18) | k), k < 2^18.
constexpr int FPSC_THREADS = 1024, FPSC_MAX_PER_CTA = 13 * 1024;
__device__ __forceinline__ unsigned cluster_ctarank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void st_cluster_u64(const void* local_smem, unsigned cta, unsigned long long v) {
  unsigned la = (unsigned)__cvta_generic_to_shared(local_smem), ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(cta));
  asm volatile("st.shared::cluster.u64 [%0], %1;" ::"r"(ra), "l"(v) : "memory");
}

template <int CS>
__global__ void __launch_bounds__(FPSC_THREADS, 1) fps_cluster_kernel(const float* __restrict__ xyz, int n, int m, int* __restrict__ idx) {
  extern __shared__ float sm[];
  __shared__ unsigned red_hi[2][FPSC_THREADS / 32], red_lo[2][FPSC_THREADS / 32];
  __shared__ unsigned long long slot[2][CS];          // written by every CTA of the cluster through DSMEM
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned rank = cluster_ctarank();
  const int b = blockIdx.x / CS;
  const int chunk = (n + CS - 1) / CS;                // points [rank*chunk, min(n, (rank+1)*chunk)) live in this CTA
  const int k0 = rank * chunk, cnt = max(0, min(chunk, n - k0));
  float* sx = sm;
  float* sy = sm + chunk;
  float* sz = sm + 2 * chunk;
  float* st = sm + 3 * chunk;
  const float* p = xyz + (size_t)b * n * 3;
  int* out = idx + (size_t)b * m;
  for (int i = tid; i < cnt; i += FPSC_THREADS) {
    const float* q = p + (size_t)(k0 + i) * 3;
    sx[i] = q[0]; sy[i] = q[1]; sz[i] = q[2]; st[i] = 1e10f;
  }
  __syncthreads();
  cluster_sync_all();                                 // every CTA's shared memory exists before anyone writes into it
  int old = 0;
  if (rank == 0 && tid == 0) out[0] = 0;
  for (int j = 1; j < m; ++j) {
    const float x1 = __ldg(p + (size_t)old * 3), y1 = __ldg(p + (size_t)old * 3 + 1), z1 = __ldg(p + (size_t)old * 3 + 2);
    unsigned bh = 0u, bl = 0u;
    for (int i = tid; i < cnt; i += FPSC_THREADS) {
      const float d = sqdist_ref(x1, y1, z1, sx[i], sy[i], sz[i]);
      const float d2 = fminf(d, st[i]);
      st[i] = d2;
      const unsigned k = (unsigned)(k0 + i);
      const unsigned key = (1u << 27) - (((__brev(k & 511u) >> 23) << 18) | k);
      const unsigned h = __float_as_uint(d2);
      if (h > bh || (h == bh && key > bl)) { bh = h; bl = key; }
    }
    unsigned wh = __reduce_max_sync(0xffffffffu, bh);
    unsigned wl = __reduce_max_sync(0xffffffffu, bh == wh ? bl : 0u);
    const int buf = j & 1;
    if (lane == 0) { red_hi[buf][warp] = wh; red_lo[buf][warp] = wl; }
    __syncthreads();
    if (warp == 0) {
      bh = red_hi[buf][lane]; bl = red_lo[buf][lane];
      wh = __reduce_max_sync(0xffffffffu, bh);
      wl = __reduce_max_sync(0xffffffffu, bh == wh ? bl : 0u);
      if (lane < CS) st_cluster_u64(&slot[buf][rank], (unsigned)lane, ((unsigned long long)wh << 32) | wl);
    }
    cluster_sync_all();
    unsigned long long best = 0ull;
#pragma unroll
    for (int c = 0; c < CS; ++c) best = max(best, slot[buf][c]);   // (distance bits, tie key) in one unsigned compare
    old = (int)(((1u << 27) - (unsigned)(best & 0xffffffffull)) & 0x3ffffu);
    if (rank == 0 && tid == 0) out[j] = old;
  }
  cluster_sync_all();                                 // no CTA exits while a peer may still write into its slots
}

template <int CS>
static int launch_fps_cluster(const float* xyz, int b, int n, int m, int* idx, cudaStream_t st) {
  const int chunk = (n + CS - 1) / CS;
  const size_t smem = (size_t)chunk * 4 * sizeof(float);
  auto kern = fps_cluster_kernel<CS>;
  S6_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (CS > 8) S6_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(b * CS); cfg.blockDim = dim3(FPSC_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = CS; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  S6_CHECK(cudaLaunchKernelEx(&cfg, kern, xyz, n, m, idx));
  return 0;
}

static int ref_block_size(int n) {  // cuda_utils.h:20-24
  int p = 1;
  while (p * 2 <= n && p * 2 <= 512) p *= 2;
  return p;
}

// Replaces _ext.furthest_point_sampling (bindings.cpp:14, sampling.cpp:67-91).
// xyz (b,n,3) f32, idx (b,m) i32; temp: scratch (b,n) f32, only needed when n > 4096 (may be null otherwise).
S6_API int sam6d_fps(const float* xyz, int b, int n, int m, float* temp, int* idx, void* stream) {
  S6_REQUIRE(xyz && idx && b >= 0 && n > 0 && m >= 0);
  if (b == 0 || m == 0) return 0;
  const int bs_ref = ref_block_size(n);
  cudaStream_t st = s6_stream(stream);
  if (n <= 4096) {
    size_t smem = (size_t)n * 3 * sizeof(float);
    if (n <= 1024) {
      fps_reg_kernel<256, 4><<<b, 256, smem, st>>>(xyz, n, m, bs_ref, idx);
    } else if (n <= 2048) {
      fps_reg_kernel<512, 4><<<b, 512, smem, st>>>(xyz, n, m, bs_ref, idx);
    } else {
      S6_CHECK(cudaFuncSetAttribute(fps_reg_kernel<512, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      fps_reg_kernel<512, 8><<<b, 512, smem, st>>>(xyz, n, m, bs_ref, idx);
    }
  } else if (n <= 8 * FPSC_MAX_PER_CTA) {
    int rc = launch_fps_cluster<8>(xyz, b, n, m, idx, st);        // 4097 .. 106 496 points: 8 CTAs (portable cluster size)
    if (rc) return rc;
  } else if (n <= 16 * FPSC_MAX_PER_CTA) {
    int rc = launch_fps_cluster<16>(xyz, b, n, m, idx, st);       // .. 212 992 points (the 42 x 5000 template bank): 16 CTAs
    if (rc) {                                                     // a 16-CTA cluster needs a GPC with 16 free SMs: else one CTA
      (void)cudaGetLastError();
      S6_REQUIRE(temp != nullptr);
      fps_big_kernel<1024><<<b, 1024, 0, st>>>(xyz, n, m, bs_ref, temp, idx);
    }
  } else {
    S6_REQUIRE(temp != nullptr);
    fps_big_kernel<1024><<<b, 1024, 0, st>>>(xyz, n, m, bs_ref, temp, idx);
  }
  S6_LAUNCH_CHECK();
  return 0;
}

// the single-CTA general-n kernel on its own (comparator of the cluster kernel in tests / profiles); temp (b,n) f32 scratch
S6_API int sam6d_fps_single_cta(const float* xyz, int b, int n, int m, float* temp, int* idx, void* stream) {
  S6_REQUIRE(xyz && idx && temp && b >= 0 && n > 0 && m >= 0);
  if (b == 0 || m == 0) return 0;
  fps_big_kernel<1024><<<b, 1024, 0, s6_stream(stream)>>>(xyz, n, m, ref_block_size(n), temp, idx);
  S6_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// gathers
// ------------------------------------------------------------------------------------------
// channel-last row gather: out[b,j,:] = src[b, idx[b,j], :]; rows are C floats (C % 4 == 0 -> float4 path)
__global__ void gather_rows_kernel(const float* __restrict__ src, const int* __restrict__ idx, int n, int m, int c,
                                   long long src_bstride, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int c4 = c >> 2;
  const long long total = (long long)m * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int j = (int)(i / c4), q = (int)(i - (long long)j * c4);
    int a = idx[(size_t)b * m + j];
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);            // negative index = padding row (zeros)
    if (a >= 0) v = reinterpret_cast<const float4*>(src + (size_t)b * src_bstride + (size_t)a * c)[q];
    reinterpret_cast<float4*>(out + ((size_t)b * m + j) * c)[q] = v;
  }
}
__global__ void gather_rows_scalar_kernel(const float* __restrict__ src, const int* __restrict__ idx, int n, int m, int c,
                                          long long src_bstride, float* __restrict__ out) {
  const int b = blockIdx.y;
  const long long total = (long long)m * c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int j = (int)(i / c), q = (int)(i - (long long)j * c);
    int a = idx[(size_t)b * m + j];
    out[((size_t)b * m + j) * c + q] = (a >= 0) ? src[(size_t)b * src_bstride + (size_t)a * c + q] : 0.f;
  }
}

// bf16 source rows widened to fp32 (the sparse tokens picked out of the bf16 dense sequence); c % 8 == 0
__global__ void gather_rows_bf16_f32_kernel(const __nv_bfloat16* __restrict__ src, const int* __restrict__ idx, int m, int c,
                                            long long src_bstride, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int c8 = c >> 3;
  const long long total = (long long)m * c8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int j = (int)(i / c8), q = (int)(i - (long long)j * c8);
    int a = idx[(size_t)b * m + j];
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (a >= 0) v = reinterpret_cast<const uint4*>(src + (size_t)b * src_bstride + (size_t)a * c)[q];
    float4* o = reinterpret_cast<float4*>(out + ((size_t)b * m + j) * c + q * 8);
    o[0] = make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xffff0000u), __uint_as_float(v.y << 16),
                       __uint_as_float(v.y & 0xffff0000u));
    o[1] = make_float4(__uint_as_float(v.z << 16), __uint_as_float(v.z & 0xffff0000u), __uint_as_float(v.w << 16),
                       __uint_as_float(v.w & 0xffff0000u));
  }
}
S6_API int sam6d_gather_rows_bf16_f32(const void* src, const int* idx, int b, int n, int m, int c, long long src_bstride,
                                      float* out, void* stream) {
  S6_REQUIRE(src && idx && out && b >= 0 && n > 0 && m >= 0 && c > 0 && (c % 8) == 0 && (src_bstride % 8) == 0);
  S6_REQUIRE((((uintptr_t)src | (uintptr_t)out) % 16) == 0);
  if (b == 0 || m == 0) return 0;
  long long total = (long long)m * (c / 8);
  dim3 grid((unsigned)min((long long)1024, (total + 255) / 256), b);
  gather_rows_bf16_f32_kernel<<<grid, 256, 0, s6_stream(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(src), idx, m, c,
                                                                   src_bstride, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// src (b,n,c) f32 with batch stride src_bstride (elements), idx (b,m) i32 -> out (b,m,c)
S6_API int sam6d_gather_rows(const float* src, const int* idx, int b, int n, int m, int c, long long src_bstride,
                             float* out, void* stream) {
  S6_REQUIRE(src && idx && out && b >= 0 && n > 0 && m >= 0 && c > 0);
  if (b == 0 || m == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  bool vec = (c % 4 == 0) && (src_bstride % 4 == 0) && (((uintptr_t)src | (uintptr_t)out) % 16 == 0);
  long long total = (long long)m * (vec ? c / 4 : c);
  dim3 grid((unsigned)min((long long)1024, (total + 255) / 256), b);
  if (vec) gather_rows_kernel<<<grid, 256, 0, st>>>(src, idx, n, m, c, src_bstride, out);
  else gather_rows_scalar_kernel<<<grid, 256, 0, st>>>(src, idx, n, m, c, src_bstride, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// channel-first gather, the reference ABI: points (b,c,n), idx (b,m) -> out (b,c,m)   (sampling_gpu.cu:13-25)
__global__ void gather_points_cf_kernel(const float* __restrict__ points, const int* __restrict__ idx, int c, int n, int m,
                                        float* __restrict__ out) {
  const int b = blockIdx.z, l = blockIdx.y;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x)
    out[((size_t)b * c + l) * m + j] = points[((size_t)b * c + l) * n + idx[(size_t)b * m + j]];
}
S6_API int sam6d_gather_points(const float* points, const int* idx, int b, int c, int n, int m, float* out, void* stream) {
  S6_REQUIRE(points && idx && out && b >= 0 && c > 0 && n > 0 && m >= 0);
  if (b == 0 || m == 0) return 0;
  S6_REQUIRE(c <= 65535 && b <= 65535);
  dim3 grid(s6_cdiv(m, 256), c, b);
  gather_points_cf_kernel<<<grid, 256, 0, s6_stream(stream)>>>(points, idx, c, n, m, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// ball query: one warp per query, ballot + prefix popcount keeps the reference's ascending-k order
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ball_query_kernel(const float* __restrict__ new_xyz, const float* __restrict__ xyz,
                                                         int n, int m, float radius2, int nsample, int* __restrict__ idx,
                                                         int* __restrict__ cnt_out) {
  extern __shared__ float sp[];  // tile of xyz, 3 * TILE floats
  const int TILE = 1024;
  const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = blockIdx.x * 8 + warp;
  const float* p = xyz + (size_t)b * n * 3;
  float nx = 0.f, ny = 0.f, nz = 0.f;
  if (j < m) {
    const float* q = new_xyz + ((size_t)b * m + j) * 3;
    nx = q[0]; ny = q[1]; nz = q[2];
  }
  int* o = (j < m) ? idx + ((size_t)b * m + j) * nsample : nullptr;
  int cnt = 0, first = 0;
  for (int base = 0; base < n; base += TILE) {
    int tn = min(TILE, n - base);
    __syncthreads();
    for (int i = threadIdx.x; i < tn * 3; i += blockDim.x) sp[i] = p[(size_t)base * 3 + i];
    __syncthreads();
    if (j < m && cnt < nsample) {
      for (int k0 = 0; k0 < tn && cnt < nsample; k0 += 32) {
        int k = k0 + lane;
        bool hit = false;
        if (k < tn) {
          float dx = nx - sp[k * 3 + 0], dy = ny - sp[k * 3 + 1], dz = nz - sp[k * 3 + 2];
          float d2 = __fmul_rn(dx, dx);
          d2 = __fmaf_rn(dy, dy, d2);
          d2 = __fmaf_rn(dz, dz, d2);
          hit = d2 < radius2;
        }
        unsigned mask = __ballot_sync(0xffffffffu, hit);
        if (mask) {
          if (cnt == 0) first = base + k0 + __ffs(mask) - 1;
          int pos = cnt + __popc(mask & ((1u << lane) - 1u));
          if (hit && pos < nsample) o[pos] = base + k;
          cnt += __popc(mask);
        }
      }
    }
  }
  if (j < m) {
    int c = min(cnt, nsample);
    // pad with the first hit; all zeros when the ball is empty (the output is defined as pre-zeroed)
    for (int l = c + lane; l < nsample; l += 32) o[l] = (cnt > 0) ? first : 0;
    if (cnt_out && lane == 0) cnt_out[(size_t)b * m + j] = c;
  }
}

// Replaces _ext.ball_query (bindings.cpp:18, ball_query.cpp:11-35).  cnt (b,m) i32 is optional:
// the number of distinct hits kept (<= nsample), which lets the fused PE kernel skip padding.
S6_API int sam6d_ball_query(const float* new_xyz, const float* xyz, int b, int n, int m, float radius, int nsample,
                            int* idx, int* cnt, void* stream) {
  S6_REQUIRE(new_xyz && xyz && idx && b >= 0 && n > 0 && m >= 0 && nsample > 0);
  if (b == 0 || m == 0) return 0;
  dim3 grid(s6_cdiv(m, 8), b);
  ball_query_kernel<<<grid, 256, 1024 * 3 * sizeof(float), s6_stream(stream)>>>(new_xyz, xyz, n, m, radius * radius,
                                                                               nsample, idx, cnt);
  S6_LAUNCH_CHECK();
  return 0;
}

// Two concentric ball queries over the same clouds in one sweep (PositionalEncoding groups every point at r1/ns1 and r2/ns2,
// fine_point_matching.py:104-109).  THREAD per query, candidates broadcast from shared memory as (x, y, z, -) quadruples: one
// LDS.128 serves 32 queries and a candidate costs ~9 issue slots per warp (3 subtractions, the reference's mul/fma/fma chain,
// two compares) against ~25 per 32 candidates for the warp-per-query ballot scan it replaces (that one is issue-bound).  Hits are rare (a few per cent), so the list bookkeeping sits behind a branch.
// The order of a list is the scan order, i.e. ascending index, as in ball_query_gpu.cu:17-49.
constexpr int BQP_THREADS = 256, BQP_TILE = 2048;
__global__ void __launch_bounds__(BQP_THREADS) ball_query_pair_kernel(const float* __restrict__ new_xyz, const float* __restrict__ xyz, int n,
                                                                      int m, float ra2, int nsa, float rb2, int nsb, int* __restrict__ idxa,
                                                                      int* __restrict__ idxb, int* __restrict__ cnta_out,
                                                                      int* __restrict__ cntb_out) {
  __shared__ float4 sp[BQP_TILE];
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int j = blockIdx.x * BQP_THREADS + threadIdx.x;
  const bool live = j < m;
  const float* p = xyz + (size_t)b * n * 3;
  float nx = 0.f, ny = 0.f, nz = 0.f;
  if (live) {
    const float* q = new_xyz + ((size_t)b * m + j) * 3;
    nx = q[0]; ny = q[1]; nz = q[2];
  }
  int* oa = idxa + ((size_t)b * m + (live ? j : 0)) * nsa;
  int* ob = idxb + ((size_t)b * m + (live ? j : 0)) * nsb;
  int ca = 0, cb = 0, fa = 0, fb = 0;
  for (int base = 0; base < n; base += BQP_TILE) {
    const int tn = min(BQP_TILE, n - base);
    __syncthreads();
    for (int i = threadIdx.x; i < tn; i += BQP_THREADS) {
      const float* q = p + (size_t)(base + i) * 3;
      sp[i] = make_float4(q[0], q[1], q[2], 0.f);
    }
    __syncthreads();
    if (live) {
      // eight candidates per step, branch-free distances, ONE test for "any hit among the eight" (hits are a few per cent, so
      // the list bookkeeping below is rarely entered and the distance chains of a step overlap)
      auto dist2 = [&](const float4 c) {
        const float dx = nx - c.x, dy = ny - c.y, dz = nz - c.z;
        float d = __fmul_rn(dx, dx);
        d = __fmaf_rn(dy, dy, d);
        return __fmaf_rn(dz, dz, d);
      };
      auto take = [&](float d, int k) {
        if (d < rb2) {
          if (cb < nsb) {
            if (cb == 0) fb = k;
            ob[cb] = k;
          }
          ++cb;
          if (d < ra2) {
            if (ca < nsa) {
              if (ca == 0) fa = k;
              oa[ca] = k;
            }
            ++ca;
          }
        }
      };
      int k = 0;
      for (; k + 8 <= tn; k += 8) {
        float d[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) d[u] = dist2(sp[k + u]);
        // A lane's hits of the step as a bit mask, then one bookkeeping pass per SET bit: a warp sees ~9 hits among its 256
        // tests of a step, so "any lane hit" is almost always true, but no single lane has more than one or two
        unsigned hb = 0, ha = 0;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          hb |= (d[u] < rb2) ? (1u << u) : 0u;
          ha |= (d[u] < ra2) ? (1u << u) : 0u;
        }
        while (hb) {
          const int u = __ffs(hb) - 1;
          hb &= hb - 1;
          const int kk = base + k + u;
          if (cb < nsb) {
            if (cb == 0) fb = kk;
            ob[cb] = kk;
          }
          ++cb;
          if ((ha >> u) & 1u) {
            if (ca < nsa) {
              if (ca == 0) fa = kk;
              oa[ca] = kk;
            }
            ++ca;
          }
        }
      }
      for (; k < tn; ++k) take(dist2(sp[k]), base + k);
    }
  }
  // pad the lists with their first entry (0 when empty), warp-cooperatively so that the stores are contiguous
  ca = min(ca, nsa); cb = min(cb, nsb);
  if (live) {
    if (cnta_out) cnta_out[(size_t)b * m + j] = ca;
    if (cntb_out) cntb_out[(size_t)b * m + j] = cb;
  }
  const int j0 = j - lane;
  for (int q = 0; q < 32; ++q) {
    if (j0 + q >= m) break;
    const int qa = __shfl_sync(0xffffffffu, ca, q), qfa = __shfl_sync(0xffffffffu, fa, q);
    const int qb = __shfl_sync(0xffffffffu, cb, q), qfb = __shfl_sync(0xffffffffu, fb, q);
    int* la = idxa + ((size_t)b * m + j0 + q) * nsa;
    int* lb = idxb + ((size_t)b * m + j0 + q) * nsb;
    for (int l = qa + lane; l < nsa; l += 32) la[l] = qfa;
    for (int l = qb + lane; l < nsb; l += 32) lb[l] = qfb;
  }
}

// radius_a <= radius_b.  Same outputs as two sam6d_ball_query calls.
S6_API int sam6d_ball_query_pair(const float* new_xyz, const float* xyz, int b, int n, int m, float radius_a, int nsample_a,
                                 float radius_b, int nsample_b, int* idx_a, int* idx_b, int* cnt_a, int* cnt_b, void* stream) {
  S6_REQUIRE(new_xyz && xyz && idx_a && idx_b && b >= 0 && n > 0 && m >= 0 && nsample_a > 0 && nsample_b > 0 &&
             radius_a <= radius_b);
  if (b == 0 || m == 0) return 0;
  dim3 grid(s6_cdiv(m, BQP_THREADS), b);
  ball_query_pair_kernel<<<grid, BQP_THREADS, 0, s6_stream(stream)>>>(
      new_xyz, xyz, n, m, radius_a * radius_a, nsample_a, radius_b * radius_b, nsample_b, idx_a, idx_b, cnt_a, cnt_b);
  S6_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// group points, the reference ABI: points (b,c,n), idx (b,np,ns) -> out (b,c,np,ns)  (group_points_gpu.cu:13-33)
// ------------------------------------------------------------------------------------------
__global__ void group_points_kernel(const float* __restrict__ points, const int* __restrict__ idx, int c, int n, int np,
                                    int ns, float* __restrict__ out) {
  const int b = blockIdx.z, l = blockIdx.y;
  const long long total = (long long)np * ns;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    out[((size_t)b * c + l) * total + i] = points[((size_t)b * c + l) * n + idx[(size_t)b * total + i]];
}
S6_API int sam6d_group_points(const float* points, const int* idx, int b, int c, int n, int np, int ns, float* out,
                              void* stream) {
  S6_REQUIRE(points && idx && out && b >= 0 && c > 0 && n > 0 && np >= 0 && ns > 0);
  if (b == 0 || np == 0) return 0;
  S6_REQUIRE(c <= 65535 && b <= 65535);
  dim3 grid(min(4096, s6_cdiv((long long)np * ns, 256)), c, b);
  group_points_kernel<<<grid, 256, 0, s6_stream(stream)>>>(points, idx, c, n, np, ns, out);
  S6_LAUNCH_CHECK();
  return 0;
}
