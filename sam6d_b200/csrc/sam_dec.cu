// sam_dec.cu -- the small kernels of the SAM prompt encoder / mask decoder / automatic mask generator (SURVEY.md 8f row N4;
// ISM/segment_anything/modeling/{prompt_encoder,mask_decoder,transformer}.py, automatic_mask_generator.py, utils/amg.py).
// The Linears of the decoder (token and image side, the two transposed convolutions written as GEMMs) run on the wgmma GEMMs
// (sam6d_gemm_tma / sam6d_gemm_bf16); this file holds what is not a GEMM:
//   sam_pe_encode          random-Fourier positional encoding of point prompts / of the dense 64 x 64 grid
//   sam_mask_embed         PromptEncoder.mask_downscaling: (B,256,256) mask logits -> (B,4096,256) dense-embedding token rows
//   sam_self_attn          self-attention of the T <= 32 prompt tokens (8 heads x 32)
//   sam_tok2img_attn       prompt tokens attend to the 4096 image tokens (8 heads x 16): scores in shared memory, two passes,
//                          at most 8 tokens per CTA
//   sam_img2tok_attn       image tokens attend to the T <= 32 prompt tokens (softmax over T keys per pixel and head)
//   sam_ln2d_gelu          LayerNorm2d (eps 1e-6) + GELU over 64-channel pixel rows after the first transposed convolution
//   sam_mask_dot(_range)   GELU'd 32-channel upscaled embedding x hypernetwork vectors -> (B,nm,256,256) mask logits of mask
//                          tokens m0 .. m0+nm-1, with the pixel shuffle of both transposed convolutions folded into the output index
//   sam_mask_stats         Sam.postprocess_masks (256 -> 1024 bilinear, crop, -> original size bilinear) evaluated on the fly per
//                          output pixel + stability counts + box extremes per mask (the (64,3,1024,1024) tensor never exists)
//   sam_mask_upscale       the same evaluation written out as logits (Sam.postprocess_masks)
//   sam_mask_binarize      the kept masks at the original resolution
//   sam_nms                box NMS (torchvision semantics) over score-sorted boxes
#include "common.cuh"

namespace {

constexpr int HD_X = 16;      // head dim of the cross attentions (internal dim 128 / 8 heads)
constexpr int NH = 8;
constexpr int TOK_SMALL = 8;  // token bound of the automatic mask generator's shapes (5 output tokens + point + padding point = 7)
constexpr int TOK_MAX = 32;   // 5 output tokens + up to 27 prompt tokens (26 clicks + padding point, or 25 clicks + a box)
constexpr int TOK_CHUNK = 8;  // tokens per CTA of sam_tok2img_attn (their scores over all L keys live in shared memory)

__device__ __forceinline__ float bf2f(__nv_bfloat16 v) { return __bfloat162float(v); }

// ---- positional encoding: out[row, 0:128] = sin(2 pi ((2c-1) G)), out[row, 128:256] = cos(...) --------------------------------
__global__ void sam_pe_encode_kernel(const float* __restrict__ coords, const float* __restrict__ G, int rows, float* __restrict__ out) {
  const int r = blockIdx.x, f = threadIdx.x;     // 128 threads
  if (r >= rows) return;
  const float cx = 2.f * coords[r * 2] - 1.f, cy = 2.f * coords[r * 2 + 1] - 1.f;
  const float v = 6.283185307179586f * (cx * G[f] + cy * G[128 + f]);
  out[(size_t)r * 256 + f] = sinf(v);
  out[(size_t)r * 256 + 128 + f] = cosf(v);
}

// ---- mask prompt -> dense embedding: PromptEncoder.mask_downscaling ------------------------------------------------------------------
// Conv2d 1->4 (k2 s2) -> LayerNorm2d(4) -> GELU -> Conv2d 4->16 (k2 s2) -> LayerNorm2d(16) -> GELU -> Conv2d 16->256 (1x1), fp32.
// Output pixel (y, x) of the 64 x 64 grid depends on input rows 4y .. 4y+3, columns 4x .. 4x+3 only, so the 4- and 16-channel
// intermediates stay in registers / shared memory.  params (ME_NPARAM floats, see sam6d_sam_mask_embed) in the module's order.
constexpr int ME_C1W = 0, ME_C1B = 16, ME_L1W = 20, ME_L1B = 24, ME_C2W = 28, ME_C2B = 284, ME_L2W = 300, ME_L2B = 316, ME_C3W = 332,
              ME_C3B = 4428, ME_NPARAM = 4684;

// LayerNorm2d over n channels (biased variance, eps 1e-6) + affine + erf GELU, in place
template <int n>
__device__ __forceinline__ void ln_gelu(float* v, const float* __restrict__ w, const float* __restrict__ b) {
  float u = 0.f;
#pragma unroll
  for (int i = 0; i < n; ++i) u += v[i];
  u *= 1.f / n;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < n; ++i) var = fmaf(v[i] - u, v[i] - u, var);
  const float sd = sqrtf(var * (1.f / n) + 1e-6f);
#pragma unroll
  for (int i = 0; i < n; ++i) v[i] = s6_act(fmaf(w[i], (v[i] - u) / sd, b[i]), 2);
}

// grid (64 rows of the embedding, B), 256 threads: threads 0..63 take one pixel of the row through the two 2x2 convolutions; then
// thread c writes channel c of all 64 pixels (consecutive threads, consecutive channels: 1 KB per pixel row)
__global__ void __launch_bounds__(256) sam_mask_embed_kernel(const float* __restrict__ masks, const float* __restrict__ prm,
                                                             float* __restrict__ out) {
  __shared__ float p[ME_C3W];
  __shared__ float hs[64][17];
  const int y = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  for (int i = tid; i < ME_C3W; i += 256) p[i] = prm[i];
  __syncthreads();
  if (tid < 64) {
    const float* m = masks + (size_t)b * 65536 + (size_t)(4 * y) * 256 + 4 * tid;
    float in[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float4 v = *reinterpret_cast<const float4*>(m + r * 256);
      in[r][0] = v.x; in[r][1] = v.y; in[r][2] = v.z; in[r][3] = v.w;
    }
    float a[4][4];                                   // [2x2 position (ky, kx)][channel]
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int ky = q >> 1, kx = q & 1;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float s = p[ME_C1B + c];
#pragma unroll
        for (int d = 0; d < 4; ++d) s = fmaf(p[ME_C1W + c * 4 + d], in[2 * ky + (d >> 1)][2 * kx + (d & 1)], s);
        a[q][c] = s;
      }
      ln_gelu<4>(a[q], p + ME_L1W, p + ME_L1B);
    }
    float h[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float s = p[ME_C2B + c];
#pragma unroll
      for (int ci = 0; ci < 4; ++ci)
#pragma unroll
        for (int q = 0; q < 4; ++q) s = fmaf(p[ME_C2W + (c * 4 + ci) * 4 + q], a[q][ci], s);
      h[c] = s;
    }
    ln_gelu<16>(h, p + ME_L2W, p + ME_L2B);
#pragma unroll
    for (int c = 0; c < 16; ++c) hs[tid][c] = h[c];
  }
  __syncthreads();
  float w3[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) w3[k] = __ldg(prm + ME_C3W + tid * 16 + k);
  const float b3 = __ldg(prm + ME_C3B + tid);
  float* o = out + ((size_t)b * 4096 + (size_t)y * 64) * 256 + tid;
  for (int x = 0; x < 64; ++x) {
    float s = b3;
#pragma unroll
    for (int k = 0; k < 16; ++k) s = fmaf(w3[k], hs[x][k], s);
    o[(size_t)x * 256] = s;
  }
}

// ---- prompt-token self-attention: q, k, v (B,T,256) f32 (already projected), 8 heads x 32; one warp per (b, h) ----------------------
template <int MAXT>
__global__ void __launch_bounds__(256) sam_self_attn_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                                            int B, int T, float* __restrict__ out) {
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= B * NH) return;
  const int b = w / NH, h = w % NH;
  const size_t base = (size_t)b * T * 256 + h * 32 + lane;
  float kk[MAXT], vv[MAXT];
  for (int t = 0; t < T; ++t) { kk[t] = k[base + (size_t)t * 256]; vv[t] = v[base + (size_t)t * 256]; }
  const float scale = 0.17677669529663687f;      // 1 / sqrt(32)
  for (int t1 = 0; t1 < T; ++t1) {
    const float qv = q[base + (size_t)t1 * 256];
    float s[MAXT], mx = -INFINITY;
    for (int t2 = 0; t2 < T; ++t2) { s[t2] = warp_sum(qv * kk[t2]) * scale; mx = fmaxf(mx, s[t2]); }
    float den = 0.f, acc = 0.f;
    for (int t2 = 0; t2 < T; ++t2) { const float p = __expf(s[t2] - mx); den += p; acc += p * vv[t2]; }
    out[base + (size_t)t1 * 256] = acc / den;
  }
}

// ---- tokens -> image: Q (B,T,128) f32; K, V (kv_bs = 0: shared (L,128), else (B,L,128)) bf16; out (B,T,128) f32 -----------------------
// grid = B * 8 * ceil(T / 8) (prompt, head, chunk of at most 8 tokens), 256 threads, dynamic smem min(T, 8) * L floats (scores) +
// reductions; the CTAs of one (prompt, head) are adjacent, so the chunks after the first read K and V from L2.  At T <= 8 there is
// one chunk and the CTA computes what it did before tokens were chunked.
__global__ void __launch_bounds__(256) sam_tok2img_attn_kernel(const float* __restrict__ Q, const __nv_bfloat16* __restrict__ K,
                                                               const __nv_bfloat16* __restrict__ V, long long kv_bs, int T, int L,
                                                               float* __restrict__ out) {
  constexpr int MAXT = TOK_CHUNK;
  extern __shared__ float sc[];                  // [Tc][L]
  __shared__ float red[MAXT][8];
  __shared__ float stat[MAXT][2];
  __shared__ float part[16][MAXT][HD_X];
  __shared__ float qs[MAXT][HD_X];
  const int nc = (T + MAXT - 1) / MAXT, c = blockIdx.x % nc, bh = blockIdx.x / nc;
  const int b = bh / NH, h = bh % NH, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int t0 = c * MAXT, Tc = min(MAXT, T - t0);
  const __nv_bfloat16* Kb = K + (size_t)b * kv_bs + h * HD_X;
  const __nv_bfloat16* Vb = V + (size_t)b * kv_bs + h * HD_X;
  if (tid < MAXT * HD_X) {
    const int t = tid / HD_X, d = tid % HD_X;
    qs[t][d] = t < Tc ? Q[((size_t)b * T + t0 + t) * 128 + h * HD_X + d] * 0.25f : 0.f;      // 1 / sqrt(16)
  }
  __syncthreads();
  float mx[MAXT];
#pragma unroll
  for (int t = 0; t < MAXT; ++t) mx[t] = -INFINITY;
  for (int j = tid; j < L; j += 256) {
    const uint4* kp = reinterpret_cast<const uint4*>(Kb + (size_t)j * 128);
    const uint4 a = kp[0], c = kp[1];
    const uint32_t wv[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
    float kf[HD_X];
#pragma unroll
    for (int i = 0; i < 8; ++i) { kf[2 * i] = __uint_as_float(wv[i] << 16); kf[2 * i + 1] = __uint_as_float(wv[i] & 0xffff0000u); }
#pragma unroll
    for (int t = 0; t < MAXT; ++t) {
      if (t < Tc) {
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < HD_X; ++d) s = fmaf(qs[t][d], kf[d], s);
        sc[(size_t)t * L + j] = s;
        mx[t] = fmaxf(mx[t], s);
      }
    }
  }
#pragma unroll
  for (int t = 0; t < MAXT; ++t) { const float m = warp_max(mx[t]); if (lane == 0) red[t][warp] = m; }
  __syncthreads();
  if (tid < MAXT) { float m = red[tid][0]; for (int w = 1; w < 8; ++w) m = fmaxf(m, red[tid][w]); stat[tid][0] = m; }
  __syncthreads();
  float sm[MAXT];
#pragma unroll
  for (int t = 0; t < MAXT; ++t) sm[t] = 0.f;
  for (int j = tid; j < L; j += 256) {
#pragma unroll
    for (int t = 0; t < MAXT; ++t)
      if (t < Tc) { const float p = __expf(sc[(size_t)t * L + j] - stat[t][0]); sc[(size_t)t * L + j] = p; sm[t] += p; }
  }
#pragma unroll
  for (int t = 0; t < MAXT; ++t) { const float v = warp_sum(sm[t]); if (lane == 0) red[t][warp] = v; }
  __syncthreads();
  if (tid < MAXT) { float v = 0.f; for (int w = 0; w < 8; ++w) v += red[tid][w]; stat[tid][1] = v; }
  __syncthreads();
  // out[t][d] = sum_j p[t][j] v_j[d]: thread = (key group g of 16, channel d)
  const int g = tid >> 4, d = tid & 15;
  float acc[MAXT];
#pragma unroll
  for (int t = 0; t < MAXT; ++t) acc[t] = 0.f;
  for (int j = g; j < L; j += 16) {
    const float vv = bf2f(Vb[(size_t)j * 128 + d]);
#pragma unroll
    for (int t = 0; t < MAXT; ++t)
      if (t < Tc) acc[t] = fmaf(sc[(size_t)t * L + j], vv, acc[t]);
  }
#pragma unroll
  for (int t = 0; t < MAXT; ++t) part[g][t][d] = acc[t];
  __syncthreads();
  if (tid < Tc * HD_X) {
    const int t = tid / HD_X, dd = tid % HD_X;
    float v = 0.f;
    for (int gg = 0; gg < 16; ++gg) v += part[gg][t][dd];
    out[((size_t)b * T + t0 + t) * 128 + h * HD_X + dd] = v / stat[t][1];
  }
}

// ---- image -> tokens: Qimg (q_bs = 0: shared (L,128), else (B,L,128)) bf16; Kt, Vt (B,T,128) f32; out (B,L,128) bf16 -------------------
// grid (L / 32, B), 256 threads: thread = (pixel of the 32, head)
template <int MAXT>
__global__ void __launch_bounds__(256) sam_img2tok_attn_kernel(const __nv_bfloat16* __restrict__ Q, long long q_bs, const float* __restrict__ Kt,
                                                               const float* __restrict__ Vt, int T, int L, __nv_bfloat16* __restrict__ out) {
  __shared__ float ks[MAXT][128], vs[MAXT][128];
  const int b = blockIdx.y, tid = threadIdx.x;
  for (int i = tid; i < T * 128; i += 256) { ks[i / 128][i % 128] = Kt[(size_t)b * T * 128 + i]; vs[i / 128][i % 128] = Vt[(size_t)b * T * 128 + i]; }
  __syncthreads();
  const int px = blockIdx.x * 32 + (tid >> 3), h = tid & 7;
  if (px >= L) return;
  const uint4* qp = reinterpret_cast<const uint4*>(Q + (size_t)b * q_bs + (size_t)px * 128 + h * HD_X);
  const uint4 a = qp[0], c = qp[1];
  const uint32_t wv[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
  float q[HD_X];
#pragma unroll
  for (int i = 0; i < 8; ++i) { q[2 * i] = __uint_as_float(wv[i] << 16); q[2 * i + 1] = __uint_as_float(wv[i] & 0xffff0000u); }
  float s[MAXT], mx = -INFINITY;
  for (int t = 0; t < T; ++t) {
    float v = 0.f;
#pragma unroll
    for (int d = 0; d < HD_X; ++d) v = fmaf(q[d], ks[t][h * HD_X + d], v);
    s[t] = v * 0.25f;
    mx = fmaxf(mx, s[t]);
  }
  float den = 0.f, o[HD_X];
#pragma unroll
  for (int d = 0; d < HD_X; ++d) o[d] = 0.f;
  for (int t = 0; t < T; ++t) {
    const float p = __expf(s[t] - mx);
    den += p;
#pragma unroll
    for (int d = 0; d < HD_X; ++d) o[d] = fmaf(p, vs[t][h * HD_X + d], o[d]);
  }
  const float inv = 1.f / den;
  uint32_t pk[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    __nv_bfloat162 hh = __floats2bfloat162_rn(o[2 * i] * inv, o[2 * i + 1] * inv);
    pk[i] = *reinterpret_cast<uint32_t*>(&hh);
  }
  uint4* op = reinterpret_cast<uint4*>(out + ((size_t)b * L + px) * 128 + h * HD_X);
  op[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
  op[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
}

// ---- LayerNorm2d (over 64 channels of a pixel, eps 1e-6) + GELU: rows of 64 bf16 -> bf16; one warp per row -----------------------------
__global__ void __launch_bounds__(256) sam_ln2d_gelu_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, long long rows, __nv_bfloat16* __restrict__ y) {
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const __nv_bfloat162 v2 = *reinterpret_cast<const __nv_bfloat162*>(x + r * 64 + lane * 2);
  const float a = __bfloat162float(v2.x), c = __bfloat162float(v2.y);
  const float mean = warp_sum(a + c) * (1.f / 64.f);
  const float da = a - mean, dc = c - mean;
  const float var = warp_sum(da * da + dc * dc) * (1.f / 64.f);
  const float rstd = rsqrtf(var + 1e-6f);
  const float ya = s6_act(gamma[lane * 2] * (da * rstd) + beta[lane * 2], 2), yc = s6_act(gamma[lane * 2 + 1] * (dc * rstd) + beta[lane * 2 + 1], 2);
  *reinterpret_cast<__nv_bfloat162*>(y + r * 64 + lane * 2) = __floats2bfloat162_rn(ya, yc);
}

// ---- mask logits: up (B*L*4 rows = (b, y, x, i, j), 128 cols = (i', j', o)) bf16 already GELU'd; hyper (B,4,32) f32 --------------------
// masks[b, m-m0, 4y + 2i + i', 4x + 2j + j'] = sum_o hyper[b, m, o] up[row, (i',j',o)]   for m = m0 .. m0+nm-1
// (m0 = 1, nm = 3: the multimask slice; m0 = 0, nm = 1: the single-mask output); thread = (row, sub-position (i',j')); grid covers
// B*L*4*4 threads
__global__ void __launch_bounds__(256) sam_mask_dot_kernel(const __nv_bfloat16* __restrict__ up, const float* __restrict__ hyper, int B, int G,
                                                           int m0, int nm, float* __restrict__ masks) {
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  const long long total = (long long)B * G * G * 16;
  if (t >= total) return;
  const int sub = (int)(t & 3);
  const long long row = t >> 2;
  const int ij = (int)(row & 3);
  const long long pix = row >> 2;
  const int x = (int)(pix % G), y = (int)((pix / G) % G), b = (int)(pix / ((long long)G * G));
  const uint4* p = reinterpret_cast<const uint4*>(up + row * 128 + sub * 32);
  float u[32];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint4 a = p[q];
    const uint32_t wv[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { u[q * 8 + 2 * i] = __uint_as_float(wv[i] << 16); u[q * 8 + 2 * i + 1] = __uint_as_float(wv[i] & 0xffff0000u); }
  }
  const int Y = 4 * y + 2 * (ij >> 1) + (sub >> 1), X = 4 * x + 2 * (ij & 1) + (sub & 1);
  const int S = 4 * G;
  for (int m = m0; m < m0 + nm; ++m) {
    const float* hv = hyper + ((size_t)b * 4 + m) * 32;
    float s = 0.f;
#pragma unroll
    for (int o = 0; o < 32; ++o) s = fmaf(__ldg(hv + o), u[o], s);
    masks[(((size_t)b * nm + (m - m0)) * S + Y) * S + X] = s;
  }
}

// ---- postprocess_masks on the fly ---------------------------------------------------------------------------------------------------
// torch bilinear, align_corners = False: src = scale * (dst + 0.5) - 0.5 clamped at 0, i1 = i0 + (i0 < in - 1)
__device__ __forceinline__ void lin_src(int dst, float scale, int in, int& i0, int& i1, float& l0, float& l1) {
  float s = scale * ((float)dst + 0.5f) - 0.5f;
  s = s < 0.f ? 0.f : s;
  i0 = (int)s;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = s - (float)i0;
  l0 = 1.f - l1;
}
__device__ __forceinline__ float bil(const float* __restrict__ src, int W, int y0, int y1, int x0, int x1, float ly0, float ly1, float lx0, float lx1) {
  return ly0 * (lx0 * src[y0 * W + x0] + lx1 * src[y0 * W + x1]) + ly1 * (lx0 * src[y1 * W + x0] + lx1 * src[y1 * W + x1]);
}
// value of the 1024 x 1024 stage at (Y, X) from the low-res S x S mask
__device__ __forceinline__ float stage1(const float* __restrict__ low, int S, int big, int Y, int X) {
  int y0, y1, x0, x1; float ly0, ly1, lx0, lx1;
  const float sc = (float)S / (float)big;
  lin_src(Y, sc, S, y0, y1, ly0, ly1);
  lin_src(X, sc, S, x0, x1, lx0, lx1);
  return bil(low, S, y0, y1, x0, x1, ly0, ly1, lx0, lx1);
}
__device__ __forceinline__ float mask_logit(const float* __restrict__ low, int S, int big, int in_h, int in_w, int H, int W, int y, int x) {
  int y0, y1, x0, x1; float ly0, ly1, lx0, lx1;
  lin_src(y, (float)in_h / (float)H, in_h, y0, y1, ly0, ly1);
  lin_src(x, (float)in_w / (float)W, in_w, x0, x1, lx0, lx1);
  const float v00 = stage1(low, S, big, y0, x0), v01 = stage1(low, S, big, y0, x1), v10 = stage1(low, S, big, y1, x0), v11 = stage1(low, S, big, y1, x1);
  return ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11);
}

// stats (N,8) i32: 0 count(logit > thr + off), 1 count(logit > thr - off), 2 xmin, 3 ymin, 4 xmax, 5 ymax of (logit > thr)
// grid (ceil(H*W/256), N)
__global__ void __launch_bounds__(256) sam_mask_stats_kernel(const float* __restrict__ low, int N, int S, int big, int in_h, int in_w, int H, int W,
                                                             float thr, float off, int* __restrict__ stats) {
  const int n = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
  bool hi = false, lo = false, on = false;
  int y = 0, x = 0;
  if (i < H * W) {
    y = i / W; x = i - y * W;
    const float v = mask_logit(low + (size_t)n * S * S, S, big, in_h, in_w, H, W, y, x);
    hi = v > thr + off; lo = v > thr - off; on = v > thr;
  }
  const unsigned bh = __ballot_sync(0xffffffffu, hi), bl = __ballot_sync(0xffffffffu, lo), bo = __ballot_sync(0xffffffffu, on);
  int xmin = on ? x : 0x7fffffff, xmax = on ? x : -1, ymin = on ? y : 0x7fffffff, ymax = on ? y : -1;
  if (bo) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      xmin = min(xmin, __shfl_xor_sync(0xffffffffu, xmin, o)); xmax = max(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
      ymin = min(ymin, __shfl_xor_sync(0xffffffffu, ymin, o)); ymax = max(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
    int* s = stats + (size_t)n * 8;
    if (bh) atomicAdd(s + 0, __popc(bh));
    if (bl) atomicAdd(s + 1, __popc(bl));
    if (bo) { atomicMin(s + 2, xmin); atomicMin(s + 3, ymin); atomicMax(s + 4, xmax); atomicMax(s + 5, ymax); }
  }
}

__global__ void sam_stats_init_kernel(int* __restrict__ stats, int N) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * 8) return;
  const int f = i & 7;
  stats[i] = (f == 2 || f == 3) ? 0x7fffffff : ((f == 4 || f == 5) ? -1 : 0);
}

// the kept masks at the original resolution: sel (K) indices into the N low-res masks -> out (K,H,W) u8
__global__ void __launch_bounds__(256) sam_mask_binarize_kernel(const float* __restrict__ low, const int* __restrict__ sel, int S, int big, int in_h,
                                                                int in_w, int H, int W, float thr, unsigned char* __restrict__ out) {
  const int k = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
  if (i >= H * W) return;
  const int y = i / W, x = i - y * W;
  out[(size_t)k * H * W + i] = mask_logit(low + (size_t)sel[k] * S * S, S, big, in_h, in_w, H, W, y, x) > thr ? 1 : 0;
}

// Sam.postprocess_masks written out: low (N,S,S) -> out (N,H,W) f32; the values sam_mask_binarize thresholds
__global__ void __launch_bounds__(256) sam_mask_upscale_kernel(const float* __restrict__ low, int S, int big, int in_h, int in_w, int H, int W,
                                                               float* __restrict__ out) {
  const int n = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
  if (i >= H * W) return;
  const int y = i / W, x = i - y * W;
  out[(size_t)n * H * W + i] = mask_logit(low + (size_t)n * S * S, S, big, in_h, in_w, H, W, y, x);
}

// ---- NMS over boxes sorted by decreasing score (torchvision.ops.nms): keep[i] = 1 for survivors; one CTA -----------------------------------
__global__ void __launch_bounds__(1024) sam_nms_kernel(const float* __restrict__ boxes, int N, float thr, unsigned char* __restrict__ keep) {
  extern __shared__ unsigned char dead[];       // N
  for (int i = threadIdx.x; i < N; i += 1024) dead[i] = 0;
  __syncthreads();
  for (int i = 0; i < N; ++i) {
    if (!dead[i]) {                              // uniform across the block (read after the barrier below)
      const float x1 = boxes[i * 4], y1 = boxes[i * 4 + 1], x2 = boxes[i * 4 + 2], y2 = boxes[i * 4 + 3];
      const float ai = (x2 - x1) * (y2 - y1);
      for (int j = i + 1 + threadIdx.x; j < N; j += 1024) {
        if (dead[j]) continue;
        const float a1 = boxes[j * 4], b1 = boxes[j * 4 + 1], a2 = boxes[j * 4 + 2], b2 = boxes[j * 4 + 3];
        const float iw = fmaxf(fminf(x2, a2) - fmaxf(x1, a1), 0.f), ih = fmaxf(fminf(y2, b2) - fmaxf(y1, b1), 0.f);
        const float inter = iw * ih, aj = (a2 - a1) * (b2 - b1);
        if (inter / (ai + aj - inter) > thr) dead[j] = 1;
      }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < N; i += 1024) keep[i] = dead[i] ? 0 : 1;
}

}  // namespace

// coords (rows,2) f32 already normalised to [0,1]; G (2,128) f32 -> out (rows,256) f32   (PositionEmbeddingRandom._pe_encoding)
S6_API int sam6d_sam_pe_encode(const float* coords, const float* G, int rows, float* out, void* stream) {
  S6_REQUIRE(coords && G && out && rows >= 0);
  if (rows == 0) return 0;
  sam_pe_encode_kernel<<<rows, 128, 0, s6_stream(stream)>>>(coords, G, rows, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// masks (B,256,256) f32 mask logits, params (ME_NPARAM) f32 -> out (B,4096,256) f32 dense-embedding token rows (row = y*64 + x)
S6_API int sam6d_sam_mask_embed(const float* masks, const float* params, int B, float* out, void* stream) {
  S6_REQUIRE(masks && params && out && B >= 0 && B <= 65535 && (reinterpret_cast<uintptr_t>(masks) & 15) == 0);
  if (B == 0) return 0;
  sam_mask_embed_kernel<<<dim3(64, B), 256, 0, s6_stream(stream)>>>(masks, params, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// q, k, v, out (B,T,256) f32, T <= 32: Attention.forward core of the prompt-token self attention (8 heads x 32)
S6_API int sam6d_sam_self_attn(const float* q, const float* k, const float* v, int B, int T, float* out, void* stream) {
  S6_REQUIRE(q && k && v && out && B >= 0 && T > 0 && T <= TOK_MAX);
  if (B == 0) return 0;
  if (T <= TOK_SMALL)
    sam_self_attn_kernel<TOK_SMALL><<<s6_cdiv(B * NH, 8), 256, 0, s6_stream(stream)>>>(q, k, v, B, T, out);
  else
    sam_self_attn_kernel<TOK_MAX><<<s6_cdiv(B * NH, 8), 256, 0, s6_stream(stream)>>>(q, k, v, B, T, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// Q (B,T,128) f32; K, V bf16 (L,128) shared by every prompt (kv_bs = 0) or (B,L,128) (kv_bs = L*128) -> out (B,T,128) f32; T <= 32
S6_API int sam6d_sam_tok2img_attn(const float* Q, const void* K, const void* V, long long kv_bs, int B, int T, int L, float* out, void* stream) {
  S6_REQUIRE(Q && K && V && out && B >= 0 && T > 0 && T <= TOK_MAX && L > 0 && (size_t)min(T, TOK_CHUNK) * L * 4 <= 200 * 1024);
  if (B == 0) return 0;
  const size_t smem = (size_t)min(T, TOK_CHUNK) * L * sizeof(float);
  S6_CHECK(cudaFuncSetAttribute(sam_tok2img_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int chunks = (T + TOK_CHUNK - 1) / TOK_CHUNK;
  sam_tok2img_attn_kernel<<<B * NH * chunks, 256, smem, s6_stream(stream)>>>(Q, reinterpret_cast<const __nv_bfloat16*>(K),
                                                                            reinterpret_cast<const __nv_bfloat16*>(V), kv_bs, T, L, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// Q bf16 (L,128) shared (q_bs = 0) or (B,L,128); Kt, Vt (B,T,128) f32 -> out (B,L,128) bf16; T <= 32
S6_API int sam6d_sam_img2tok_attn(const void* Q, long long q_bs, const float* Kt, const float* Vt, int B, int T, int L, void* out, void* stream) {
  S6_REQUIRE(Q && Kt && Vt && out && B >= 0 && T > 0 && T <= TOK_MAX && L > 0 && B <= 65535);
  if (B == 0) return 0;
  const dim3 grid(s6_cdiv(L, 32), B);
  const __nv_bfloat16* q = reinterpret_cast<const __nv_bfloat16*>(Q);
  __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
  if (T <= TOK_SMALL)
    sam_img2tok_attn_kernel<TOK_SMALL><<<grid, 256, 0, s6_stream(stream)>>>(q, q_bs, Kt, Vt, T, L, o);
  else
    sam_img2tok_attn_kernel<TOK_MAX><<<grid, 256, 0, s6_stream(stream)>>>(q, q_bs, Kt, Vt, T, L, o);
  S6_LAUNCH_CHECK();
  return 0;
}

// x, y (rows,64) bf16; gamma, beta (64) f32: LayerNorm2d(eps 1e-6) + GELU of output_upscaling.{1,2}
S6_API int sam6d_sam_ln2d_gelu(const void* x, const float* gamma, const float* beta, long long rows, void* y, void* stream) {
  S6_REQUIRE(x && gamma && beta && y && rows >= 0);
  if (rows == 0) return 0;
  sam_ln2d_gelu_kernel<<<s6_cdiv(rows, 8), 256, 0, s6_stream(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(x), gamma, beta, rows,
                                                                       reinterpret_cast<__nv_bfloat16*>(y));
  S6_LAUNCH_CHECK();
  return 0;
}

// up (B*G*G*4, 128) bf16, hyper (B,4,32) f32 -> masks (B,nm,4G,4G) f32: the logits of mask tokens m0 .. m0+nm-1
S6_API int sam6d_sam_mask_dot_range(const void* up, const float* hyper, int B, int G, int m0, int nm, float* masks, void* stream) {
  S6_REQUIRE(up && hyper && masks && B >= 0 && G > 0 && m0 >= 0 && nm > 0 && m0 + nm <= 4);
  if (B == 0) return 0;
  const long long total = (long long)B * G * G * 16;
  sam_mask_dot_kernel<<<s6_cdiv(total, 256), 256, 0, s6_stream(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(up), hyper, B, G, m0, nm, masks);
  S6_LAUNCH_CHECK();
  return 0;
}

// up (B*G*G*4, 128) bf16, hyper (B,4,32) f32 -> masks (B,3,4G,4G) f32 (the multimask slice)
S6_API int sam6d_sam_mask_dot(const void* up, const float* hyper, int B, int G, float* masks, void* stream) {
  return sam6d_sam_mask_dot_range(up, hyper, B, G, 1, 3, masks, stream);
}

// low (N,S,S) f32 low-res logits -> stats (N,8) i32 (see the kernel) at original size (H,W) through the big x big stage cropped to (in_h,in_w)
S6_API int sam6d_sam_mask_stats(const float* low, int N, int S, int big, int in_h, int in_w, int H, int W, float thr, float off, int* stats,
                                void* stream) {
  S6_REQUIRE(low && stats && N >= 0 && S > 1 && big >= S && in_h > 0 && in_w > 0 && in_h <= big && in_w <= big && H > 0 && W > 0 && N <= 65535);
  if (N == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  sam_stats_init_kernel<<<s6_cdiv(N * 8, 256), 256, 0, st>>>(stats, N);
  S6_LAUNCH_CHECK();
  sam_mask_stats_kernel<<<dim3(s6_cdiv((long long)H * W, 256), N), 256, 0, st>>>(low, N, S, big, in_h, in_w, H, W, thr, off, stats);
  S6_LAUNCH_CHECK();
  return 0;
}

// sel (K) i32 indices into low (N,S,S) -> out (K,H,W) u8 = logit > thr
S6_API int sam6d_sam_mask_binarize(const float* low, const int* sel, int K, int S, int big, int in_h, int in_w, int H, int W, float thr,
                                   unsigned char* out, void* stream) {
  S6_REQUIRE(low && sel && out && K >= 0 && S > 1 && K <= 65535);
  if (K == 0) return 0;
  sam_mask_binarize_kernel<<<dim3(s6_cdiv((long long)H * W, 256), K), 256, 0, s6_stream(stream)>>>(low, sel, S, big, in_h, in_w, H, W, thr, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// low (N,S,S) f32 -> out (N,H,W) f32: S -> big bilinear, crop to (in_h,in_w), -> (H,W) bilinear (Sam.postprocess_masks)
S6_API int sam6d_sam_mask_upscale(const float* low, int N, int S, int big, int in_h, int in_w, int H, int W, float* out, void* stream) {
  S6_REQUIRE(low && out && N >= 0 && S > 1 && big >= S && in_h > 0 && in_w > 0 && in_h <= big && in_w <= big && H > 0 && W > 0 && N <= 65535);
  if (N == 0) return 0;
  sam_mask_upscale_kernel<<<dim3(s6_cdiv((long long)H * W, 256), N), 256, 0, s6_stream(stream)>>>(low, S, big, in_h, in_w, H, W, out);
  S6_LAUNCH_CHECK();
  return 0;
}

// boxes (N,4) f32 xyxy sorted by decreasing score -> keep (N) u8; N <= 65536
S6_API int sam6d_sam_nms(const float* boxes, int N, float thr, unsigned char* keep, void* stream) {
  S6_REQUIRE(boxes && keep && N >= 0 && N <= 65536);
  if (N == 0) return 0;
  S6_CHECK(cudaFuncSetAttribute(sam_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
  sam_nms_kernel<<<1, 1024, N, s6_stream(stream)>>>(boxes, N, thr, keep);
  S6_LAUNCH_CHECK();
  return 0;
}
