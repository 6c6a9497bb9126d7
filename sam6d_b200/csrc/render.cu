// render.cu -- batched triangle rasteriser for CAD template views (SIMT; sam6d_b200/render.py, oracle/render_oracle.py).
//
// O meshes x T views each, one K and H x W.  Visibility is exact and independent of scheduling, so the numpy oracle
// reproduces it bit for bit:
//   vertex pass   p = R x + t and u = fx*x/z + cx, v = fy*y/z + cy with explicit round-to-nearest ops (the build contracts
//                 FMAs), snapped to 1/256 px fixed point; a vertex with z <= znear or |u|, |v| > 2^14 px is invalid;
//   coverage      pixel centres at (x+1/2, y+1/2), int64 edge functions, top-left fill rule, both windings (a negative-area
//                 triangle has its 2nd and 3rd vertex swapped), zero-area triangles skipped, triangles with an invalid vertex
//                 dropped and counted per mesh (no clipping);
//   depth         1/z interpolated with fp32 barycentrics E_i / area; one 64-bit atomicMin per covered pixel on
//                 (float bits of z) << 32 | face id: nearest wins, an exact depth tie goes to the lower face id;
//   resolve       recomputes the winner's barycentrics the same way, interpolates object coordinates and colour / UV
//                 perspective-correctly and shades with ambient + Lambert from a point light at -1.5 t (camera frame).
// Small triangles are rasterised by the thread that set them up; those with a bounding box over RS_BIG_PIXELS pixels go
// to a list that a grid-stride kernel works off with one CTA per triangle.
#include "common.cuh"
#include <cuda_fp16.h>

namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_BIG_PIXELS = 256;
constexpr int RS_BIG_CTAS = 1056;            // 8 per SM of an H100 SXM; the list length is only known on the device
constexpr float RS_GUARD = 16384.f;
constexpr unsigned long long RS_EMPTY = ~0ull;

// mesh_info row: first vertex, vertex count, first face, face count, colour mode, texture height, texture width, unused
enum { MI_V0, MI_NV, MI_F0, MI_NF, MI_MODE, MI_TH, MI_TW, MI_STRIDE = 8 };

// largest o with T * info[o][field] <= idx (meshes are packed in order, so this is the mesh that owns item idx)
__device__ __forceinline__ int rs_find(const int* info, int O, int field, long long T, long long idx) {
  int lo = 0, hi = O - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (T * info[mid * MI_STRIDE + field] <= idx) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ float rs_dot_rn(const float* r, float x, float y, float z, float t) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], x), __fmul_rn(r[1], y)), __fmul_rn(r[2], z)), t);
}

__global__ void __launch_bounds__(RS_THREADS) rs_vertex_kernel(const float* __restrict__ verts, const int* __restrict__ info, int O, int T,
                                                               const float* __restrict__ poses, float fx, float fy, float cx, float cy,
                                                               float znear, long long total, int4* __restrict__ vrec) {
  long long idx = (long long)blockIdx.x * RS_THREADS + threadIdx.x;
  if (idx >= total) return;
  int o = rs_find(info, O, MI_V0, T, idx);
  const int* mi = info + o * MI_STRIDE;
  long long rel = idx - (long long)T * mi[MI_V0];
  int t = (int)(rel / mi[MI_NV]), i = (int)(rel % mi[MI_NV]);
  const float* P = poses + ((long long)o * T + t) * 16;
  const float* v = verts + ((long long)mi[MI_V0] + i) * 3;
  float x = v[0], y = v[1], z = v[2];
  float px = rs_dot_rn(P, x, y, z, P[3]), py = rs_dot_rn(P + 4, x, y, z, P[7]), pz = rs_dot_rn(P + 8, x, y, z, P[11]);
  float u = __fadd_rn(__fdiv_rn(__fmul_rn(fx, px), pz), cx);
  float w = __fadd_rn(__fdiv_rn(__fmul_rn(fy, py), pz), cy);
  bool ok = pz > znear && fabsf(u) <= RS_GUARD && fabsf(w) <= RS_GUARD;
  vrec[idx] = ok ? make_int4(__float2int_rn(__fmul_rn(u, 256.f)), __float2int_rn(__fmul_rn(w, 256.f)), __float_as_int(pz), 1)
                 : make_int4(0, 0, 0, 0);
}

// one triangle of one view in fixed point, normalised to positive area
struct RsTri {
  int ax, ay, bx, by, cx, cy;
  long long area;
  float iza, izb, izc;
};

// 1 = rasterise, 0 = zero area or outside the image, -1 = an index is out of range or a vertex is invalid (dropped)
__device__ __forceinline__ int rs_setup(const int* __restrict__ faces, const int4* __restrict__ vr, const int* mi, int f, RsTri& tr,
                                        int* fi) {
  const int* fc = faces + ((long long)mi[MI_F0] + f) * 3;
  int nv = mi[MI_NV];
  int i0 = fc[0], i1 = fc[1], i2 = fc[2];
  if ((unsigned)i0 >= (unsigned)nv || (unsigned)i1 >= (unsigned)nv || (unsigned)i2 >= (unsigned)nv) return -1;
  int4 a = vr[i0], b = vr[i1], c = vr[i2];
  if (!a.w || !b.w || !c.w) return -1;
  long long area = (long long)(b.x - a.x) * (c.y - a.y) - (long long)(b.y - a.y) * (c.x - a.x);
  if (area == 0) return 0;
  if (area < 0) { int4 s = b; b = c; c = s; int si = i1; i1 = i2; i2 = si; area = -area; }
  tr.ax = a.x; tr.ay = a.y; tr.bx = b.x; tr.by = b.y; tr.cx = c.x; tr.cy = c.y; tr.area = area;
  tr.iza = __fdiv_rn(1.f, __int_as_float(a.z));
  tr.izb = __fdiv_rn(1.f, __int_as_float(b.z));
  tr.izc = __fdiv_rn(1.f, __int_as_float(c.z));
  if (fi) { fi[0] = i0; fi[1] = i1; fi[2] = i2; }
  return 1;
}

__device__ __forceinline__ long long rs_edge(int ax, int ay, int bx, int by, long long px, long long py) {
  return (long long)(bx - ax) * (py - ay) - (long long)(by - ay) * (px - ax);
}
// top-left rule: a pixel centre exactly on an edge belongs to the triangle when the edge is a top edge (dy == 0, dx > 0)
// or a left edge (dy < 0) in this orientation; the two triangles that share an edge traverse it in opposite directions,
// so exactly one of them owns it
__device__ __forceinline__ bool rs_inside(long long e, int dx, int dy) { return e > 0 || (e == 0 && (dy < 0 || (dy == 0 && dx > 0))); }

// perspective-correct weights of a covered pixel; returns false when the centre is outside
__device__ __forceinline__ bool rs_cover(const RsTri& tr, int x, int y, float& q0, float& q1, float& q2, float& invz) {
  long long px = (long long)x * 256 + 128, py = (long long)y * 256 + 128;
  long long e0 = rs_edge(tr.bx, tr.by, tr.cx, tr.cy, px, py);
  long long e1 = rs_edge(tr.cx, tr.cy, tr.ax, tr.ay, px, py);
  long long e2 = rs_edge(tr.ax, tr.ay, tr.bx, tr.by, px, py);
  if (!rs_inside(e0, tr.cx - tr.bx, tr.cy - tr.by) || !rs_inside(e1, tr.ax - tr.cx, tr.ay - tr.cy) ||
      !rs_inside(e2, tr.bx - tr.ax, tr.by - tr.ay))
    return false;
  float fa = __ll2float_rn(tr.area);
  q0 = __fmul_rn(__fdiv_rn(__ll2float_rn(e0), fa), tr.iza);
  q1 = __fmul_rn(__fdiv_rn(__ll2float_rn(e1), fa), tr.izb);
  q2 = __fmul_rn(__fdiv_rn(__ll2float_rn(e2), fa), tr.izc);
  invz = __fadd_rn(__fadd_rn(q0, q1), q2);
  return true;
}

// pixel range whose centres can lie in the triangle, clipped to the image
__device__ __forceinline__ bool rs_box(const RsTri& tr, int H, int W, int& x0, int& x1, int& y0, int& y1) {
  int mnx = min(tr.ax, min(tr.bx, tr.cx)), mxx = max(tr.ax, max(tr.bx, tr.cx));
  int mny = min(tr.ay, min(tr.by, tr.cy)), mxy = max(tr.ay, max(tr.by, tr.cy));
  x0 = max(0, -((128 - mnx) >> 8)); x1 = min(W - 1, (mxx - 128) >> 8);
  y0 = max(0, -((128 - mny) >> 8)); y1 = min(H - 1, (mxy - 128) >> 8);
  return x0 <= x1 && y0 <= y1;
}

__device__ __forceinline__ void rs_plot(const RsTri& tr, int x, int y, int f, unsigned long long* vis_view, int W) {
  float q0, q1, q2, invz;
  if (!rs_cover(tr, x, y, q0, q1, q2, invz)) return;
  float z = __fdiv_rn(1.f, invz);
  atomicMin(vis_view + (long long)y * W + x, ((unsigned long long)__float_as_uint(z) << 32) | (unsigned)f);
}

__global__ void __launch_bounds__(RS_THREADS) rs_setup_kernel(const int* __restrict__ faces, const int* __restrict__ info, int O, int T,
                                                              const int4* __restrict__ vrec, long long total, int H, int W,
                                                              unsigned long long* __restrict__ vis, int2* __restrict__ big, int big_cap,
                                                              int* __restrict__ counters) {
  long long idx = (long long)blockIdx.x * RS_THREADS + threadIdx.x;
  if (idx >= total) return;
  int o = rs_find(info, O, MI_F0, T, idx);
  const int* mi = info + o * MI_STRIDE;
  long long rel = idx - (long long)T * mi[MI_F0];
  int t = (int)(rel / mi[MI_NF]), f = (int)(rel % mi[MI_NF]);
  const int4* vr = vrec + (long long)T * mi[MI_V0] + (long long)t * mi[MI_NV];
  RsTri tr;
  int s = rs_setup(faces, vr, mi, f, tr, nullptr);
  if (s < 0) atomicAdd(counters + 1 + o, 1);
  int x0, x1, y0, y1;
  if (s <= 0 || !rs_box(tr, H, W, x0, x1, y0, y1)) return;
  int view = o * T + t;
  if ((long long)(x1 - x0 + 1) * (y1 - y0 + 1) > RS_BIG_PIXELS) {
    int slot = atomicAdd(counters, 1);
    if (slot < big_cap) { big[slot] = make_int2(view, f); return; }
  }
  unsigned long long* vv = vis + (long long)view * H * W;
  for (int y = y0; y <= y1; ++y)
    for (int x = x0; x <= x1; ++x) rs_plot(tr, x, y, f, vv, W);
}

__global__ void __launch_bounds__(RS_THREADS) rs_big_kernel(const int* __restrict__ faces, const int* __restrict__ info, int T,
                                                            const int4* __restrict__ vrec, int H, int W, unsigned long long* __restrict__ vis,
                                                            const int2* __restrict__ big, int big_cap, const int* __restrict__ counters) {
  int n = min(counters[0], big_cap);
  for (int e = blockIdx.x; e < n; e += gridDim.x) {
    int2 item = big[e];
    int o = item.x / T, t = item.x % T, f = item.y;
    const int* mi = info + o * MI_STRIDE;
    RsTri tr;
    rs_setup(faces, vrec + (long long)T * mi[MI_V0] + (long long)t * mi[MI_NV], mi, f, tr, nullptr);
    int x0, x1, y0, y1;
    rs_box(tr, H, W, x0, x1, y0, y1);
    int bw = x1 - x0 + 1, np = bw * (y1 - y0 + 1);
    unsigned long long* vv = vis + (long long)item.x * H * W;
    for (int p = threadIdx.x; p < np; p += RS_THREADS) rs_plot(tr, x0 + p % bw, y0 + p / bw, f, vv, W);
  }
}

__device__ __forceinline__ float3 rs_texel(const unsigned char* tex, int th, int tw, int x, int y) {
  x = min(max(x, 0), tw - 1); y = min(max(y, 0), th - 1);
  const unsigned char* p = tex + ((long long)y * tw + x) * 3;
  return make_float3(p[0], p[1], p[2]);
}

__global__ void __launch_bounds__(RS_THREADS) rs_resolve_kernel(const float* __restrict__ verts, const int* __restrict__ faces,
                                                                const int* __restrict__ info, int T, const unsigned char* __restrict__ vcol,
                                                                const float* __restrict__ uv, const unsigned char* __restrict__ tex,
                                                                const long long* __restrict__ tex_off, const float* __restrict__ base_color,
                                                                const float* __restrict__ poses, const int4* __restrict__ vrec,
                                                                const unsigned long long* __restrict__ vis, long long total, int H, int W,
                                                                float ambient, unsigned char* __restrict__ rgb, unsigned char* __restrict__ mask,
                                                                __half* __restrict__ xyz, int* __restrict__ tri, float* __restrict__ depth) {
  long long pix = (long long)blockIdx.x * RS_THREADS + threadIdx.x;
  if (pix >= total) return;
  unsigned long long key = vis[pix];
  if (key == RS_EMPTY) {
    rgb[pix * 3] = rgb[pix * 3 + 1] = rgb[pix * 3 + 2] = 0;
    mask[pix] = 0;
    xyz[pix * 3] = xyz[pix * 3 + 1] = xyz[pix * 3 + 2] = __float2half_rn(0.f);
    tri[pix] = -1;
    depth[pix] = 0.f;
    return;
  }
  long long hw = (long long)H * W;
  int view = (int)(pix / hw), o = view / T, t = view % T;
  int rem = (int)(pix % hw), y = rem / W, x = rem % W;
  int f = (int)(unsigned)(key & 0xffffffffu);
  const int* mi = info + o * MI_STRIDE;
  RsTri tr;
  int fi[3];
  rs_setup(faces, vrec + (long long)T * mi[MI_V0] + (long long)t * mi[MI_NV], mi, f, tr, fi);
  float q[3], invz;
  rs_cover(tr, x, y, q[0], q[1], q[2], invz);
  float w[3];
  const float* vp[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    w[k] = __fdiv_rn(q[k], invz);
    vp[k] = verts + ((long long)mi[MI_V0] + fi[k]) * 3;
  }
  float X[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) X[c] = __fadd_rn(__fadd_rn(__fmul_rn(w[0], vp[0][c]), __fmul_rn(w[1], vp[1][c])), __fmul_rn(w[2], vp[2][c]));
  xyz[pix * 3] = __float2half_rn(X[0]);
  xyz[pix * 3 + 1] = __float2half_rn(X[1]);
  xyz[pix * 3 + 2] = __float2half_rn(X[2]);
  mask[pix] = 255;
  tri[pix] = f;
  depth[pix] = __uint_as_float((unsigned)(key >> 32));

  // albedo in [0, 1]
  int mode = mi[MI_MODE];
  float3 alb;
  if (mode == 1 && vcol) {
    const unsigned char* c0 = vcol + ((long long)mi[MI_V0] + fi[0]) * 3;
    const unsigned char* c1 = vcol + ((long long)mi[MI_V0] + fi[1]) * 3;
    const unsigned char* c2 = vcol + ((long long)mi[MI_V0] + fi[2]) * 3;
    alb = make_float3((w[0] * c0[0] + w[1] * c1[0] + w[2] * c2[0]) / 255.f, (w[0] * c0[1] + w[1] * c1[1] + w[2] * c2[1]) / 255.f,
                      (w[0] * c0[2] + w[1] * c1[2] + w[2] * c2[2]) / 255.f);
  } else if (mode == 2 && uv && tex && tex_off) {
    const float* t0 = uv + ((long long)mi[MI_V0] + fi[0]) * 2;
    const float* t1 = uv + ((long long)mi[MI_V0] + fi[1]) * 2;
    const float* t2 = uv + ((long long)mi[MI_V0] + fi[2]) * 2;
    float su = w[0] * t0[0] + w[1] * t1[0] + w[2] * t2[0], sv = w[0] * t0[1] + w[1] * t1[1] + w[2] * t2[1];
    int th = mi[MI_TH], tw = mi[MI_TW];
    // texel centres at (i + 1/2) / size; v = 0 is the bottom row of the image (the PLY / OpenGL convention)
    float tx = fminf(fmaxf(su * tw - 0.5f, -1.f), (float)tw), ty = fminf(fmaxf((1.f - sv) * th - 0.5f, -1.f), (float)th);
    float fx0 = floorf(tx), fy0 = floorf(ty), ax = tx - fx0, ay = ty - fy0;
    int ix = (int)fx0, iy = (int)fy0;
    const unsigned char* tp = tex + tex_off[o];
    float3 a = rs_texel(tp, th, tw, ix, iy), b = rs_texel(tp, th, tw, ix + 1, iy);
    float3 c = rs_texel(tp, th, tw, ix, iy + 1), d = rs_texel(tp, th, tw, ix + 1, iy + 1);
    alb.x = ((1.f - ay) * ((1.f - ax) * a.x + ax * b.x) + ay * ((1.f - ax) * c.x + ax * d.x)) / 255.f;
    alb.y = ((1.f - ay) * ((1.f - ax) * a.y + ax * b.y) + ay * ((1.f - ax) * c.y + ax * d.y)) / 255.f;
    alb.z = ((1.f - ay) * ((1.f - ax) * a.z + ax * b.z) + ay * ((1.f - ax) * c.z + ax * d.z)) / 255.f;
  } else {
    alb = make_float3(base_color[o * 3], base_color[o * 3 + 1], base_color[o * 3 + 2]);
  }

  // ambient + Lambert; the normal of the face in the camera frame, turned towards the camera
  const float* P = poses + (long long)view * 16;
  float pc[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r) pc[k][r] = P[r * 4] * vp[k][0] + P[r * 4 + 1] * vp[k][1] + P[r * 4 + 2] * vp[k][2] + P[r * 4 + 3];
  float e1[3] = {pc[1][0] - pc[0][0], pc[1][1] - pc[0][1], pc[1][2] - pc[0][2]};
  float e2[3] = {pc[2][0] - pc[0][0], pc[2][1] - pc[0][1], pc[2][2] - pc[0][2]};
  float n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
  float s[3], l[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    s[r] = P[r * 4] * X[0] + P[r * 4 + 1] * X[1] + P[r * 4 + 2] * X[2] + P[r * 4 + 3];
    l[r] = -1.5f * P[r * 4 + 3] - s[r];
  }
  float nn = n[0] * n[0] + n[1] * n[1] + n[2] * n[2], ll = l[0] * l[0] + l[1] * l[1] + l[2] * l[2];
  float ndl = 0.f;
  if (nn > 0.f && ll > 0.f) {
    if (n[0] * s[0] + n[1] * s[1] + n[2] * s[2] > 0.f) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
    ndl = fmaxf(0.f, (n[0] * l[0] + n[1] * l[1] + n[2] * l[2]) * rsqrtf(nn) * rsqrtf(ll));
  }
  float shade = ambient + (1.f - ambient) * ndl;
  rgb[pix * 3] = (unsigned char)fminf(255.f, floorf(alb.x * shade * 255.f + 0.5f));
  rgb[pix * 3 + 1] = (unsigned char)fminf(255.f, floorf(alb.y * shade * 255.f + 0.5f));
  rgb[pix * 3 + 2] = (unsigned char)fminf(255.f, floorf(alb.z * shade * 255.f + 0.5f));
}

}  // namespace

S6_API int sam6d_render_meshes(const float* verts, const int* faces, const int* mesh_info, int O, int n_verts, int n_faces,
                               const unsigned char* vcol, const float* uv, const unsigned char* tex, const long long* tex_off,
                               const float* base_color, const float* poses, int T, float fx, float fy, float cx, float cy, int H, int W,
                               float znear, float ambient, int* vrec, unsigned long long* vis, int* big, int big_cap, int* counters,
                               unsigned char* rgb, unsigned char* mask, void* xyz, int* tri, float* depth, void* stream) {
  S6_REQUIRE(verts && faces && mesh_info && base_color && poses && vrec && vis && counters && rgb && mask && xyz && tri && depth);
  S6_REQUIRE(O > 0 && T > 0 && n_verts > 0 && n_faces > 0 && H > 0 && W > 0 && H <= 16384 && W <= 16384 && big_cap >= 0);
  S6_REQUIRE(big || big_cap == 0);
  S6_REQUIRE((long long)O * T <= 0x7fffffffLL);
  cudaStream_t st = s6_stream(stream);
  long long pixels = (long long)O * T * H * W, nv = (long long)T * n_verts, nf = (long long)T * n_faces;
  S6_CHECK(cudaMemsetAsync(vis, 0xff, pixels * sizeof(unsigned long long), st));
  S6_CHECK(cudaMemsetAsync(counters, 0, (O + 1) * sizeof(int), st));
  rs_vertex_kernel<<<s6_cdiv(nv, RS_THREADS), RS_THREADS, 0, st>>>(verts, mesh_info, O, T, poses, fx, fy, cx, cy, znear, nv,
                                                                   reinterpret_cast<int4*>(vrec));
  S6_LAUNCH_CHECK();
  rs_setup_kernel<<<s6_cdiv(nf, RS_THREADS), RS_THREADS, 0, st>>>(faces, mesh_info, O, T, reinterpret_cast<const int4*>(vrec), nf, H, W,
                                                                  vis, reinterpret_cast<int2*>(big), big_cap, counters);
  S6_LAUNCH_CHECK();
  rs_big_kernel<<<RS_BIG_CTAS, RS_THREADS, 0, st>>>(faces, mesh_info, T, reinterpret_cast<const int4*>(vrec), H, W, vis,
                                                    reinterpret_cast<const int2*>(big), big_cap, counters);
  S6_LAUNCH_CHECK();
  rs_resolve_kernel<<<s6_cdiv(pixels, RS_THREADS), RS_THREADS, 0, st>>>(verts, faces, mesh_info, T, vcol, uv, tex, tex_off, base_color, poses,
                                                                        reinterpret_cast<const int4*>(vrec), vis, pixels, H, W, ambient, rgb,
                                                                        mask, reinterpret_cast<__half*>(xyz), tri, depth);
  S6_LAUNCH_CHECK();
  return 0;
}
