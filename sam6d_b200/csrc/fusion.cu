// fusion.cu -- object models from posed RGB-D views (not in the reference; sam6d_b200/fusion.py, oracle/fusion_oracle.py)
//   1. tsdf_integrate  : one thread per voxel visits T views in index order -> truncated signed distance, weight, colour sums
//   2. tsdf_mesh_count : marching tetrahedra, pass 1: one thread per cube marks the lattice edges its triangles use and counts
//                        its triangles; one thread per lattice point counts its marked edges (the host prefix-sums both)
//   3. tsdf_mesh_emit  : pass 2: one thread per lattice point writes its vertices, one thread per cube writes its triangles
// The exact rules are at the declarations in include/sam6d_b200.h.  Every per-voxel and per-vertex operation is an explicit
// round-to-nearest op in the documented order (the build contracts a * b + c into an FMA otherwise), so a numpy float32
// restatement reproduces the results bit for bit.
#include "common.cuh"

namespace {

constexpr int FU_THREADS = 256;
constexpr int FU_VIEW_TILE = 128;        // views staged in shared memory at a time: (4 + 12) floats each
constexpr int FU_MAX_DIM = 512;

// the 6 Kuhn tetrahedra of a cube, corners numbered by bits x = 1, y = 2, z = 4: the path 0 -> e_a -> e_a + e_b -> 7 for the
// axis permutations (a, b, c) in lexicographic order.  kKuhnOdd: the permutation is odd, so the path's signed volume is negative.
__constant__ int kKuhn[6][4] = {{0, 1, 3, 7}, {0, 1, 5, 7}, {0, 2, 3, 7}, {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 6, 7}};
__constant__ int kKuhnOdd[6] = {0, 1, 1, 0, 0, 1};
// even permutations of the tetrahedron's corners (0..3) led by each corner (one corner on its own) ...
__constant__ int kLead1[4][4] = {{0, 1, 2, 3}, {1, 0, 3, 2}, {2, 0, 1, 3}, {3, 0, 2, 1}};
// ... and led by each pair (two corners inside), indexed by the 4-bit inside mask
__constant__ int kLead2[16][4] = {{0}, {0}, {0}, {0, 1, 2, 3}, {0}, {0, 2, 3, 1}, {1, 2, 0, 3}, {0}, {0}, {0, 3, 1, 2},
                                  {1, 3, 2, 0}, {0}, {2, 3, 0, 1}, {0}, {0}, {0}};

__device__ __forceinline__ float fu_coord(int i, float lo, float voxel) {
  return __fadd_rn(lo, __fmul_rn(__fadd_rn((float)i, 0.5f), voxel));   // (float)i + 0.5 is exact for i <= 512
}

// tsdf <- (tsdf w + obs) / (w + 1), w <- w + 1
__device__ __forceinline__ void fu_update(float& tsdf, int& w, float obs) {
  tsdf = __fdiv_rn(__fadd_rn(__fmul_rn(tsdf, (float)w), obs), (float)(w + 1));
  ++w;
}

__global__ void __launch_bounds__(FU_THREADS) tsdf_integrate_kernel(
    const unsigned char* __restrict__ rgb, const float* __restrict__ depth, const unsigned char* __restrict__ mask,
    const float* __restrict__ K, const float* __restrict__ pose, int T, int H, int W, float bx, float by, float bz, float voxel,
    float trunc, float znear, int nx, int ny, int nz, float* __restrict__ tsdf, int* __restrict__ weight,
    unsigned* __restrict__ csum, int* __restrict__ ccount) {
  __shared__ float sk[FU_VIEW_TILE][4];
  __shared__ float sp[FU_VIEW_TILE][12];
  const long long N = (long long)nx * ny * nz;
  const long long v = (long long)blockIdx.x * FU_THREADS + threadIdx.x;
  const bool live = v < N;
  const int ix = live ? (int)(v % nx) : 0, iy = live ? (int)((v / nx) % ny) : 0, iz = live ? (int)(v / ((long long)nx * ny)) : 0;
  const float px = fu_coord(ix, bx, voxel), py = fu_coord(iy, by, voxel), pz = fu_coord(iz, bz, voxel);
  float s = 0.f;
  int w = 0, cnt = 0;
  unsigned c0 = 0, c1 = 0, c2 = 0;
  if (live) { s = tsdf[v]; w = weight[v]; c0 = csum[v * 3]; c1 = csum[v * 3 + 1]; c2 = csum[v * 3 + 2]; cnt = ccount[v]; }
  const float ntrunc = -trunc;
  for (int k0 = 0; k0 < T; k0 += FU_VIEW_TILE) {
    const int nk = min(FU_VIEW_TILE, T - k0);
    __syncthreads();
    for (int j = threadIdx.x; j < nk * 16; j += FU_THREADS) {
      const int k = j >> 4, e = j & 15;
      if (e < 4) sk[k][e] = K[(size_t)(k0 + k) * 4 + e];
      else sp[k][e - 4] = pose[(size_t)(k0 + k) * 12 + e - 4];
    }
    __syncthreads();
    if (!live) continue;
    for (int k = 0; k < nk; ++k) {
      const float* P = sp[k];
      const float qz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[6], px), __fmul_rn(P[7], py)), __fmul_rn(P[8], pz)), P[11]);
      if (!(qz > znear)) continue;
      const float qx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[0], px), __fmul_rn(P[1], py)), __fmul_rn(P[2], pz)), P[9]);
      const float qy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[3], px), __fmul_rn(P[4], py)), __fmul_rn(P[5], pz)), P[10]);
      const float u = __fadd_rn(__fdiv_rn(__fmul_rn(sk[k][0], qx), qz), sk[k][2]);
      const float vv = __fadd_rn(__fdiv_rn(__fmul_rn(sk[k][1], qy), qz), sk[k][3]);
      const float c = floorf(__fadd_rn(u, 0.5f)), r = floorf(__fadd_rn(vv, 0.5f));
      if (!(c >= 0.f && c < (float)W && r >= 0.f && r < (float)H)) continue;
      const size_t pix = ((size_t)(k0 + k) * H + (size_t)r) * W + (size_t)c;
      const float d = depth[pix];
      if (mask == nullptr || mask[pix] != 0) {
        if (d == 0.f) continue;
        const float sdf = __fsub_rn(d, qz);
        if (sdf < ntrunc) continue;
        fu_update(s, w, fminf(1.f, __fdiv_rn(sdf, trunc)));
        if (fabsf(sdf) < trunc) {
          c0 += rgb[pix * 3]; c1 += rgb[pix * 3 + 1]; c2 += rgb[pix * 3 + 2];
          ++cnt;
        }
      } else {
        if (d > 0.f && qz > __fsub_rn(d, trunc)) continue;   // the voxel may lie behind what this pixel sees
        fu_update(s, w, 1.f);                                 // seen through: free space
      }
    }
  }
  if (live) { tsdf[v] = s; weight[v] = w; csum[v * 3] = c0; csum[v * 3 + 1] = c1; csum[v * 3 + 2] = c2; ccount[v] = cnt; }
}

__device__ __forceinline__ long long fu_corner(long long cube_pt, int corner, int nx, long long nxy) {
  return cube_pt + (corner & 1) + ((corner >> 1) & 1) * (long long)nx + ((corner >> 2) & 1) * nxy;
}

// the cube's corner signs and the active tetrahedra: bit t of the result = tetrahedron t emits triangles
__device__ __forceinline__ int fu_cube(const float* __restrict__ tsdf, const int* __restrict__ weight, long long pt, int nx,
                                       long long nxy, int min_weight, int& inside) {
  int ok = 0;
  inside = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const long long q = fu_corner(pt, c, nx, nxy);
    inside |= (tsdf[q] < 0.f) << c;
    ok |= (weight[q] >= min_weight) << c;
  }
  int act = 0;
#pragma unroll
  for (int t = 0; t < 6; ++t) {
    int in = 0, good = 1;
#pragma unroll
    for (int j = 0; j < 4; ++j) { in |= ((inside >> kKuhn[t][j]) & 1) << j; good &= (ok >> kKuhn[t][j]) & 1; }
    act |= (good && in != 0 && in != 15) << t;
  }
  return act;
}

__device__ __forceinline__ int fu_tet_inside(int inside, int t) {
  int in = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) in |= ((inside >> kKuhn[t][j]) & 1) << j;
  return in;
}

__device__ __forceinline__ void fu_cube_xyz(long long cube, int cx, int cy, int& x, int& y, int& z) {
  x = (int)(cube % cx);
  y = (int)((cube / cx) % cy);
  z = (int)(cube / ((long long)cx * cy));
}

// pass 1, one thread per cube: emask[point] |= 1 << (direction - 1) for every sign-changing edge of an active tetrahedron
// (edges keyed by their lower lattice point and direction bits), tcount[cube] = the cube's triangles
__global__ void __launch_bounds__(FU_THREADS) tsdf_mesh_mark_kernel(const float* __restrict__ tsdf, const int* __restrict__ weight,
                                                                    int nx, int ny, int nz, int min_weight,
                                                                    unsigned* __restrict__ emask, int* __restrict__ tcount) {
  const int cx = nx - 1, cy = ny - 1;
  const long long ncube = (long long)cx * cy * (nz - 1);
  const long long cube = (long long)blockIdx.x * FU_THREADS + threadIdx.x;
  if (cube >= ncube) return;
  int x, y, z;
  fu_cube_xyz(cube, cx, cy, x, y, z);
  const long long nxy = (long long)nx * ny, pt = ((long long)z * ny + y) * nx + x;
  int inside;
  const int act = fu_cube(tsdf, weight, pt, nx, nxy, min_weight, inside);
  unsigned long long m = 0;     // 7 edge bits per corner, corner c at bits 8c..8c+6 (a register, not a local array)
  int ntri = 0;
#pragma unroll
  for (int t = 0; t < 6; ++t) {
    if (!((act >> t) & 1)) continue;
    const int in = fu_tet_inside(inside, t), n = __popc(in);
    ntri += (n == 2) ? 2 : 1;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = i + 1; j < 4; ++j)
        if (((in >> i) ^ (in >> j)) & 1) {
          const int a = kKuhn[t][i], b = kKuhn[t][j];      // a's bits are a subset of b's along the path
          m |= 1ull << (8 * a + (a ^ b) - 1);
        }
  }
  tcount[cube] = ntri;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const unsigned mc = (unsigned)(m >> (8 * c)) & 0x7fu;
    if (mc) atomicOr(&emask[fu_corner(pt, c, nx, nxy)], mc);
  }
}

__global__ void __launch_bounds__(FU_THREADS) tsdf_mesh_popc_kernel(const unsigned* __restrict__ emask, long long N,
                                                                    int* __restrict__ vcount) {
  const long long p = (long long)blockIdx.x * FU_THREADS + threadIdx.x;
  if (p < N) vcount[p] = __popc(emask[p]);
}

// mean colour of a voxel's observations, channel k
__device__ __forceinline__ float fu_mean(const unsigned* __restrict__ csum, const int* __restrict__ ccount, long long p, int k) {
  return __fdiv_rn((float)csum[p * 3 + k], (float)ccount[p]);
}

__device__ __forceinline__ unsigned char fu_u8(float c) { return (unsigned char)min(255, max(0, __float2int_rn(c))); }

// pass 2a, one thread per lattice point: its marked edges in direction order -> vertex position (mm) and colour
__global__ void __launch_bounds__(FU_THREADS) tsdf_mesh_vertex_kernel(
    const float* __restrict__ tsdf, const unsigned* __restrict__ csum, const int* __restrict__ ccount, int nx, int ny, int nz,
    float bx, float by, float bz, float voxel, const unsigned* __restrict__ emask, const int* __restrict__ voff,
    float* __restrict__ verts, unsigned char* __restrict__ vcol) {
  const long long N = (long long)nx * ny * nz;
  const long long p = (long long)blockIdx.x * FU_THREADS + threadIdx.x;
  if (p >= N) return;
  const unsigned m = emask[p];
  if (!m) return;
  const int ix = (int)(p % nx), iy = (int)((p / nx) % ny), iz = (int)(p / ((long long)nx * ny));
  const long long nxy = (long long)nx * ny;
  long long o = voff[p] - __popc(m);
  const float ta = tsdf[p];
  const bool ha = ccount[p] > 0;
  for (int d = 1; d < 8; ++d) {
    if (!((m >> (d - 1)) & 1)) continue;
    const long long q = fu_corner(p, d, nx, nxy);
    const float tb = tsdf[q];
    const float t = __fdiv_rn(ta, __fsub_rn(ta, tb));
    verts[o * 3] = __fadd_rn(bx, __fmul_rn(__fadd_rn(__fadd_rn((float)ix, 0.5f), (d & 1) ? t : 0.f), voxel));
    verts[o * 3 + 1] = __fadd_rn(by, __fmul_rn(__fadd_rn(__fadd_rn((float)iy, 0.5f), (d & 2) ? t : 0.f), voxel));
    verts[o * 3 + 2] = __fadd_rn(bz, __fmul_rn(__fadd_rn(__fadd_rn((float)iz, 0.5f), (d & 4) ? t : 0.f), voxel));
    const bool hb = ccount[q] > 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      float c = 128.f;
      if (ha && hb) {
        const float ma = fu_mean(csum, ccount, p, k), mb = fu_mean(csum, ccount, q, k);
        c = __fadd_rn(ma, __fmul_rn(t, __fsub_rn(mb, ma)));
      } else if (ha) {
        c = fu_mean(csum, ccount, p, k);
      } else if (hb) {
        c = fu_mean(csum, ccount, q, k);
      }
      vcol[o * 3 + k] = fu_u8(c);
    }
    ++o;
  }
}

// the vertex index of the edge (corner a -> corner b, a's bits a subset of b's) of the cube at lattice point pt
__device__ __forceinline__ int fu_vid(const unsigned* __restrict__ emask, const int* __restrict__ voff, long long pt, int a, int b,
                                      int nx, long long nxy) {
  const long long q = fu_corner(pt, a, nx, nxy);
  const unsigned m = emask[q];
  return voff[q] - __popc(m) + __popc(m & ((1u << ((a ^ b) - 1)) - 1u));
}

// the vertex on the tetrahedron t's edge between its corners i and j
__device__ __forceinline__ int fu_tet_vid(const unsigned* __restrict__ emask, const int* __restrict__ voff, long long pt, int t,
                                          int i, int j, int nx, long long nxy) {
  const int a = kKuhn[t][min(i, j)], b = kKuhn[t][max(i, j)];
  return fu_vid(emask, voff, pt, a, b, nx, nxy);
}

// pass 2b, one thread per cube: its triangles at toff in tetrahedron order, wound so (b - a) x (c - a) points to larger tsdf
__global__ void __launch_bounds__(FU_THREADS) tsdf_mesh_face_kernel(const float* __restrict__ tsdf, const int* __restrict__ weight,
                                                                    int nx, int ny, int nz, int min_weight,
                                                                    const unsigned* __restrict__ emask, const int* __restrict__ voff,
                                                                    const int* __restrict__ toff, int* __restrict__ faces) {
  const int cx = nx - 1, cy = ny - 1;
  const long long ncube = (long long)cx * cy * (nz - 1);
  const long long cube = (long long)blockIdx.x * FU_THREADS + threadIdx.x;
  if (cube >= ncube) return;
  int x, y, z;
  fu_cube_xyz(cube, cx, cy, x, y, z);
  const long long nxy = (long long)nx * ny, pt = ((long long)z * ny + y) * nx + x;
  int inside;
  const int act = fu_cube(tsdf, weight, pt, nx, nxy, min_weight, inside);
  if (!act) return;
  long long o = toff[cube];
  {
    // toff is inclusive: step back over this cube's own triangles
    int ntri = 0;
    for (int t = 0; t < 6; ++t)
      if ((act >> t) & 1) ntri += (__popc(fu_tet_inside(inside, t)) == 2) ? 2 : 1;
    o -= ntri;
  }
  for (int t = 0; t < 6; ++t) {
    if (!((act >> t) & 1)) continue;
    const int in = fu_tet_inside(inside, t), n = __popc(in);
    const bool flip = kKuhnOdd[t];
    if (n == 1 || n == 3) {
      // the lone corner i leads the even permutation (i, j, k, l); (x_ij, x_ik, x_il) faces away from i
      const int lone = (n == 1) ? __ffs(in) - 1 : __ffs(~in & 15) - 1;
      const int* L = kLead1[lone];
      int A = fu_tet_vid(emask, voff, pt, t, L[0], L[1], nx, nxy);
      int B = fu_tet_vid(emask, voff, pt, t, L[0], L[2], nx, nxy);
      int C = fu_tet_vid(emask, voff, pt, t, L[0], L[3], nx, nxy);
      if (flip != (n == 3)) { const int s = B; B = C; C = s; }
      faces[o * 3] = A; faces[o * 3 + 1] = B; faces[o * 3 + 2] = C;
      ++o;
    } else {
      // inside pair (i, j), outside (k, l), (i, j, k, l) even: the quad x_ik, x_il, x_jl, x_jk faces the outside pair; it is split
      // along the diagonal x_ik - x_jl into (x_ik, x_il, x_jl) and (x_ik, x_jl, x_jk)
      const int* L = kLead2[in];
      const int A = fu_tet_vid(emask, voff, pt, t, L[0], L[2], nx, nxy);
      int B = fu_tet_vid(emask, voff, pt, t, L[0], L[3], nx, nxy);
      const int C = fu_tet_vid(emask, voff, pt, t, L[1], L[3], nx, nxy);
      int D = fu_tet_vid(emask, voff, pt, t, L[1], L[2], nx, nxy);
      if (flip) { const int s = B; B = D; D = s; }
      faces[o * 3] = A; faces[o * 3 + 1] = B; faces[o * 3 + 2] = C;
      faces[o * 3 + 3] = A; faces[o * 3 + 4] = C; faces[o * 3 + 5] = D;
      o += 2;
    }
  }
}

bool fu_dims_ok(int nx, int ny, int nz) {
  return nx >= 2 && ny >= 2 && nz >= 2 && nx <= FU_MAX_DIM && ny <= FU_MAX_DIM && nz <= FU_MAX_DIM;
}

bool fu_pos_finite(float x) { return isfinite(x) && x > 0.f; }

}  // namespace

S6_API int sam6d_tsdf_integrate(const unsigned char* rgb, const float* depth, const unsigned char* mask, const float* K,
                                const float* pose, int T, int H, int W, float bx, float by, float bz, float voxel, float trunc,
                                float znear, int nx, int ny, int nz, float* tsdf, int* weight, unsigned* csum, int* ccount,
                                void* stream) {
  S6_REQUIRE(fu_dims_ok(nx, ny, nz));
  S6_REQUIRE(fu_pos_finite(voxel) && fu_pos_finite(trunc) && isfinite(znear) && isfinite(bx) && isfinite(by) && isfinite(bz));
  S6_REQUIRE(T >= 1 && H >= 1 && W >= 1);
  S6_REQUIRE(rgb && depth && K && pose && tsdf && weight && csum && ccount);
  const long long N = (long long)nx * ny * nz;
  tsdf_integrate_kernel<<<s6_cdiv(N, FU_THREADS), FU_THREADS, 0, s6_stream(stream)>>>(
      rgb, depth, mask, K, pose, T, H, W, bx, by, bz, voxel, trunc, znear, nx, ny, nz, tsdf, weight, csum, ccount);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_tsdf_mesh_count(const float* tsdf, const int* weight, int nx, int ny, int nz, int min_weight, unsigned* emask,
                                 int* vcount, int* tcount, void* stream) {
  S6_REQUIRE(fu_dims_ok(nx, ny, nz) && min_weight >= 1);
  S6_REQUIRE(tsdf && weight && emask && vcount && tcount);
  const long long N = (long long)nx * ny * nz, ncube = (long long)(nx - 1) * (ny - 1) * (nz - 1);
  cudaStream_t st = s6_stream(stream);
  S6_CHECK(cudaMemsetAsync(emask, 0, N * sizeof(unsigned), st));
  tsdf_mesh_mark_kernel<<<s6_cdiv(ncube, FU_THREADS), FU_THREADS, 0, st>>>(tsdf, weight, nx, ny, nz, min_weight, emask, tcount);
  S6_LAUNCH_CHECK();
  tsdf_mesh_popc_kernel<<<s6_cdiv(N, FU_THREADS), FU_THREADS, 0, st>>>(emask, N, vcount);
  S6_LAUNCH_CHECK();
  return 0;
}

S6_API int sam6d_tsdf_mesh_emit(const float* tsdf, const int* weight, const unsigned* csum, const int* ccount, int nx, int ny, int nz,
                                float bx, float by, float bz, float voxel, int min_weight, const unsigned* emask, const int* voff,
                                const int* toff, float* verts, unsigned char* vcol, int* faces, void* stream) {
  S6_REQUIRE(fu_dims_ok(nx, ny, nz) && min_weight >= 1);
  S6_REQUIRE(fu_pos_finite(voxel) && isfinite(bx) && isfinite(by) && isfinite(bz));
  S6_REQUIRE(tsdf && weight && csum && ccount && emask && voff && toff && verts && vcol && faces);
  const long long N = (long long)nx * ny * nz, ncube = (long long)(nx - 1) * (ny - 1) * (nz - 1);
  cudaStream_t st = s6_stream(stream);
  tsdf_mesh_vertex_kernel<<<s6_cdiv(N, FU_THREADS), FU_THREADS, 0, st>>>(tsdf, csum, ccount, nx, ny, nz, bx, by, bz, voxel, emask,
                                                                         voff, verts, vcol);
  S6_LAUNCH_CHECK();
  tsdf_mesh_face_kernel<<<s6_cdiv(ncube, FU_THREADS), FU_THREADS, 0, st>>>(tsdf, weight, nx, ny, nz, min_weight, emask, voff, toff,
                                                                           faces);
  S6_LAUNCH_CHECK();
  return 0;
}
