// yolo.cu -- the parts of YOLOv8-seg (FastSAM-x) that are not convolutions on wgmma (those are csrc/conv_tc.cu):
//   stem      letterboxed u8 frame -> channel flip, /255 -> 3x3 stride-2 conv (3 -> C, BatchNorm folded) + SiLU -> NHWC bf16
//             (C = 80 for FastSAM-x, 32 for FastSAM-s)
//   sppf      the three cascaded 5x5 max-pools of SPPF written into their concat slices
//   upsample  nearest x2 into a concat slice
//   decode    Detect / Segment head decode (DFL, dist2bbox, sigmoid) + confidence filter with an ordered compaction
//   masks     sigmoid(coeffs . proto) cropped by the box on the 1/4 grid -> bilinear to the letterboxed frame -> > 0.5 as u8
#include "common.cuh"

namespace {

constexpr int HEAD_W = 64 + 1 + 32, ROW_W = 6 + 32, NM = 32;

__device__ __forceinline__ float silu(float x) { return x / (1.f + expf(-x)); }
__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// thread = one output pixel x 16 output channels (blockIdx.y picks the group of 16); C output channels per pixel
template <int C>
__global__ void __launch_bounds__(128) yolo_stem_kernel(const uint8_t* __restrict__ img, int B, int H, int W, int Ho, int Wo,
                                                        const float* __restrict__ w, const float* __restrict__ bias,
                                                        __nv_bfloat16* __restrict__ out) {
  __shared__ float ws[16 * 27];
  const int o0 = blockIdx.y * 16;
  for (int i = threadIdx.x; i < 16 * 27; i += blockDim.x) ws[i] = w[o0 * 27 + i];
  __syncthreads();
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (long long)B * Ho * Wo) return;
  const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho), n = (int)(p / ((long long)Wo * Ho));
  float v[27];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int iy = 2 * oy - 1 + ky, ix = 2 * ox - 1 + kx;
      const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
      const uint8_t* px = img + (((long long)n * H + (in ? iy : 0)) * W + (in ? ix : 0)) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) v[(ky * 3 + kx) * 3 + c] = in ? (float)px[2 - c] / 255.f : 0.f;   // network channel c = frame channel 2 - c
    }
  uint32_t packed[8];
#pragma unroll
  for (int o = 0; o < 16; o += 2) {
    float a0 = bias[o0 + o], a1 = bias[o0 + o + 1];
#pragma unroll
    for (int t = 0; t < 27; ++t) { a0 = fmaf(ws[o * 27 + t], v[t], a0); a1 = fmaf(ws[(o + 1) * 27 + t], v[t], a1); }
    __nv_bfloat162 h = __floats2bfloat162_rn(silu(a0), silu(a1));
    packed[o / 2] = *reinterpret_cast<uint32_t*>(&h);
  }
  uint4* dst = reinterpret_cast<uint4*>(out + p * C + o0);
  dst[0] = make_uint4(packed[0], packed[1], packed[2], packed[3]);
  dst[1] = make_uint4(packed[4], packed[5], packed[6], packed[7]);
}

// thread = one pixel x 2 channels; reads slice [0, C), writes the 5x5, 9x9 and 13x13 maxima to slices [C, 2C), [2C, 3C), [3C, 4C)
__global__ void yolo_sppf_kernel(__nv_bfloat16* buf, long long ld, int B, int H, int W, int C) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x, half = C / 2;
  if (t >= (long long)B * H * W * half) return;
  const int c = (int)(t % half) * 2;
  const long long p = t / half;
  const int x = (int)(p % W), y = (int)((p / W) % H), n = (int)(p / ((long long)W * H));
  const __nv_bfloat162 ninf = __floats2bfloat162_rn(-INFINITY, -INFINITY);
  __nv_bfloat162 m5 = ninf, m9 = ninf, m13 = ninf;
  for (int dy = -6; dy <= 6; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int dx = -6; dx <= 6; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W) continue;
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(buf + (((long long)n * H + yy) * W + xx) * ld + c);
      m13 = __hmax2(m13, v);
      if (abs(dy) <= 4 && abs(dx) <= 4) m9 = __hmax2(m9, v);
      if (abs(dy) <= 2 && abs(dx) <= 2) m5 = __hmax2(m5, v);
    }
  }
  __nv_bfloat16* o = buf + p * ld + c;
  *reinterpret_cast<__nv_bfloat162*>(o + C) = m5;
  *reinterpret_cast<__nv_bfloat162*>(o + 2 * C) = m9;
  *reinterpret_cast<__nv_bfloat162*>(o + 3 * C) = m13;
}

// thread = one output pixel x 8 channels
__global__ void yolo_upsample2x_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int B, int H, int W, int C,
                                       __nv_bfloat16* __restrict__ y, long long ldy) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x, chunks = C / 8;
  if (t >= (long long)B * 4 * H * W * chunks) return;
  const int c = (int)(t % chunks) * 8;
  const long long p = t / chunks;
  const int X = (int)(p % (2 * W)), Y = (int)((p / (2 * W)) % (2 * H)), n = (int)(p / (4LL * W * H));
  *reinterpret_cast<uint4*>(y + p * ldy + c) = *reinterpret_cast<const uint4*>(x + (((long long)n * H + Y / 2) * W + X / 2) * ldx + c);
}

// One CTA per frame.  Head row of anchor i: 64 DFL logits (l, t, r, b x 16 bins), 1 class logit, 32 mask coefficients.  The box
// arithmetic follows DFL / dist2bbox / the NMS's xywh2xyxy operation by operation with explicit round-to-nearest ops (no FMA
// contraction), so candidates agree with the fp32 restatement to the last bits of the softmax expectation.
constexpr int DEC_THREADS = 256;
__global__ void __launch_bounds__(DEC_THREADS) yolo_decode_kernel(const float* __restrict__ head, long long ld, long long bs, int A,
                                                                   int3 lv_h, int3 lv_w, float thr, float* __restrict__ cand,
                                                                   int* __restrict__ count) {
  __shared__ int warp_cnt[DEC_THREADS / 32];
  __shared__ int base_s;
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* hb = head + n * bs;
  float* cb = cand + (long long)n * A * ROW_W;
  if (tid == 0) base_s = 0;
  __syncthreads();
  const int n0 = lv_h.x * lv_w.x, n1 = n0 + lv_h.y * lv_w.y;
  for (int i0 = 0; i0 < A; i0 += DEC_THREADS) {
    const int i = i0 + tid;
    float conf = 0.f;
    if (i < A) conf = sigmoid(hb[(long long)i * ld + 64]);
    const bool keep = i < A && conf > thr;
    const unsigned ball = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_cnt[warp] = __popc(ball);
    __syncthreads();
    int off = base_s;
    for (int k = 0; k < warp; ++k) off += warp_cnt[k];
    off += __popc(ball & ((1u << lane) - 1u));
    if (keep) {
      const float* h = hb + (long long)i * ld;
      int j = i, wl = lv_w.x;
      float s = 8.f;
      if (i >= n1) { j = i - n1; wl = lv_w.z; s = 32.f; }
      else if (i >= n0) { j = i - n0; wl = lv_w.y; s = 16.f; }
      const float ax = (float)(j % wl) + 0.5f, ay = (float)(j / wl) + 0.5f;
      float d[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float m = h[16 * k];
#pragma unroll
        for (int b = 1; b < 16; ++b) m = fmaxf(m, h[16 * k + b]);
        float e[16], sum = 0.f;
#pragma unroll
        for (int b = 0; b < 16; ++b) { e[b] = expf(h[16 * k + b] - m); sum = __fadd_rn(sum, e[b]); }
        float acc = 0.f;
#pragma unroll
        for (int b = 1; b < 16; ++b) acc = __fadd_rn(acc, __fmul_rn((float)b, __fdiv_rn(e[b], sum)));
        d[k] = acc;
      }
      const float x1 = __fsub_rn(ax, d[0]), y1 = __fsub_rn(ay, d[1]), x2 = __fadd_rn(ax, d[2]), y2 = __fadd_rn(ay, d[3]);
      const float cx = __fmul_rn(__fdiv_rn(__fadd_rn(x1, x2), 2.f), s), cy = __fmul_rn(__fdiv_rn(__fadd_rn(y1, y2), 2.f), s);
      const float bw = __fmul_rn(__fsub_rn(x2, x1), s), bh = __fmul_rn(__fsub_rn(y2, y1), s);
      float* o = cb + (long long)off * ROW_W;
      o[0] = __fsub_rn(cx, __fdiv_rn(bw, 2.f));
      o[1] = __fsub_rn(cy, __fdiv_rn(bh, 2.f));
      o[2] = __fadd_rn(cx, __fdiv_rn(bw, 2.f));
      o[3] = __fadd_rn(cy, __fdiv_rn(bh, 2.f));
      o[4] = conf;
      o[5] = 0.f;
#pragma unroll 8
      for (int k = 0; k < NM; ++k) o[6 + k] = h[65 + k];
    }
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int k = 0; k < DEC_THREADS / 32; ++k) tot += warp_cnt[k];
      base_s += tot;
    }
    __syncthreads();
  }
  if (tid == 0) count[n] = base_s;
}

// low (N, mh, mw) = crop_mask(sigmoid(coeffs . proto), box * (kx, ky)); blockIdx.y = mask
__global__ void yolo_mask_lowres_kernel(const float* __restrict__ proto, int mh, int mw, const float* __restrict__ rows, long long row_ld,
                                        float kx, float ky, float* __restrict__ low) {
  __shared__ float c[NM];
  __shared__ float box[4];
  const int m = blockIdx.y;
  if (threadIdx.x < NM) c[threadIdx.x] = rows[m * row_ld + 6 + threadIdx.x];
  if (threadIdx.x < 4) box[threadIdx.x] = __fmul_rn(rows[m * row_ld + threadIdx.x], (threadIdx.x & 1) ? ky : kx);
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= mh * mw) return;
  const int r = p % mw, q = p / mw;                  // r: column, q: row (crop_mask's r and c)
  const float4* pp = reinterpret_cast<const float4*>(proto + (long long)p * NM);
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < NM / 4; ++k) {
    const float4 v = pp[k];
    acc = fmaf(c[4 * k], v.x, acc); acc = fmaf(c[4 * k + 1], v.y, acc); acc = fmaf(c[4 * k + 2], v.z, acc); acc = fmaf(c[4 * k + 3], v.w, acc);
  }
  const bool in = (float)r >= box[0] && (float)r < box[2] && (float)q >= box[1] && (float)q < box[3];
  low[(long long)m * mh * mw + p] = in ? sigmoid(acc) : 0.f;
}

// F.interpolate(bilinear, align_corners=False) of low to (ih, iw), then > 0.5; thread = one output pixel
__global__ void yolo_mask_up_kernel(const float* __restrict__ low, int N, int mh, int mw, int ih, int iw, uint8_t* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)N * ih * iw) return;
  const int X = (int)(t % iw), Y = (int)((t / iw) % ih), m = (int)(t / ((long long)iw * ih));
  const float sh = (float)mh / (float)ih, sw = (float)mw / (float)iw;
  const float fy = fmaxf(__fsub_rn(__fmul_rn(sh, (float)Y + 0.5f), 0.5f), 0.f), fx = fmaxf(__fsub_rn(__fmul_rn(sw, (float)X + 0.5f), 0.5f), 0.f);
  const int y0 = (int)fy, x0 = (int)fx, y1 = y0 + (y0 < mh - 1), x1 = x0 + (x0 < mw - 1);
  const float ly1 = fy - (float)y0, lx1 = fx - (float)x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
  const float* L = low + (long long)m * mh * mw;
  const float v = ly0 * (lx0 * L[y0 * mw + x0] + lx1 * L[y0 * mw + x1]) + ly1 * (lx0 * L[y1 * mw + x0] + lx1 * L[y1 * mw + x1]);
  out[t] = v > 0.5f ? 1 : 0;
}

}  // namespace

// img (B,H,W,3) u8 letterboxed frames (channel order as given: the network sees channel 2 - c as its channel c); w (C,3,3,3)
// f32 folded weights in (out, ky, kx, in) order, bias (C) f32 -> out (B, ceil(H/2), ceil(W/2), C) bf16; C in {16, 32, 48, 64, 80}
S6_API int sam6d_yolo_stem_c(const unsigned char* img, int B, int H, int W, int C, const float* w, const float* bias, void* out, void* stream) {
  S6_REQUIRE(img && w && bias && out && B >= 0 && H > 0 && W > 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0);
  S6_REQUIRE(C > 0 && C <= 80 && (C % 16) == 0);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long long P = (long long)B * Ho * Wo;
  if (P == 0) return 0;
  const dim3 grid(s6_cdiv(P, 128), C / 16);
  __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
  cudaStream_t st = s6_stream(stream);
  switch (C) {
    case 16: yolo_stem_kernel<16><<<grid, 128, 0, st>>>(img, B, H, W, Ho, Wo, w, bias, o); break;
    case 32: yolo_stem_kernel<32><<<grid, 128, 0, st>>>(img, B, H, W, Ho, Wo, w, bias, o); break;
    case 48: yolo_stem_kernel<48><<<grid, 128, 0, st>>>(img, B, H, W, Ho, Wo, w, bias, o); break;
    case 64: yolo_stem_kernel<64><<<grid, 128, 0, st>>>(img, B, H, W, Ho, Wo, w, bias, o); break;
    default: yolo_stem_kernel<80><<<grid, 128, 0, st>>>(img, B, H, W, Ho, Wo, w, bias, o); break;
  }
  S6_LAUNCH_CHECK();
  return 0;
}

// sam6d_yolo_stem_c at C = 80 (FastSAM-x)
S6_API int sam6d_yolo_stem(const unsigned char* img, int B, int H, int W, const float* w, const float* bias, void* out, void* stream) {
  return sam6d_yolo_stem_c(img, B, H, W, 80, w, bias, out, stream);
}

// buf (B,H,W,ld) bf16: channels [0, C) in, [C, 4C) out (MaxPool2d(5, 1, 2) applied once, twice, three times == 5x5, 9x9, 13x13)
S6_API int sam6d_yolo_sppf(void* buf, long long ld, int B, int H, int W, int C, void* stream) {
  S6_REQUIRE(buf && B >= 0 && H > 0 && W > 0 && C > 0 && (C % 2) == 0 && (ld % 2) == 0 && ld >= 4 * C);
  const long long T = (long long)B * H * W * (C / 2);
  if (T == 0) return 0;
  yolo_sppf_kernel<<<s6_cdiv(T, 256), 256, 0, s6_stream(stream)>>>(reinterpret_cast<__nv_bfloat16*>(buf), ld, B, H, W, C);
  S6_LAUNCH_CHECK();
  return 0;
}

// x (B,H,W,ldx) bf16 channels [0, C) -> y (B,2H,2W,ldy) channels [0, C), nearest; C, ldx, ldy multiples of 8, 16-byte aligned
S6_API int sam6d_yolo_upsample2x(const void* x, long long ldx, int B, int H, int W, int C, void* y, long long ldy, void* stream) {
  S6_REQUIRE(x && y && B >= 0 && H > 0 && W > 0 && C > 0 && (C % 8) == 0 && (ldx % 8) == 0 && (ldy % 8) == 0);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0);
  const long long T = (long long)B * 4 * H * W * (C / 8);
  if (T == 0) return 0;
  yolo_upsample2x_kernel<<<s6_cdiv(T, 256), 256, 0, s6_stream(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx, B, H, W, C,
                                                                         reinterpret_cast<__nv_bfloat16*>(y), ldy);
  S6_LAUNCH_CHECK();
  return 0;
}

// head (B, A, ld) f32 rows [64 DFL logits | class logit | 32 coefficients], frame stride bs; the A anchors are the three levels'
// grids (h0 x w0 at stride 8, h1 x w1 at 16, h2 x w2 at 32) row-major in that order -> cand (B, A, 38) f32 rows
// (x1, y1, x2, y2, conf, cls = 0, 32 coefficients) of the anchors with sigmoid(class logit) > conf_thr, in anchor order;
// count (B) i32 = rows written per frame
S6_API int sam6d_yolo_decode(const float* head, long long ld, long long bs, int B, int h0, int w0, int h1, int w1, int h2, int w2, float conf_thr,
                             float* cand, int* count, void* stream) {
  S6_REQUIRE(head && cand && count && B >= 0 && ld >= HEAD_W && h0 > 0 && w0 > 0 && h1 > 0 && w1 > 0 && h2 > 0 && w2 > 0);
  const int A = h0 * w0 + h1 * w1 + h2 * w2;
  S6_REQUIRE(bs >= (long long)A * ld);
  if (B == 0) return 0;
  yolo_decode_kernel<<<B, DEC_THREADS, 0, s6_stream(stream)>>>(head, ld, bs, A, make_int3(h0, h1, h2), make_int3(w0, w1, w2), conf_thr, cand,
                                                                count);
  S6_LAUNCH_CHECK();
  return 0;
}

// process_mask(upsample=True) for N detections of one frame: proto (mh, mw, 32) f32 NHWC, rows (N, row_ld) f32 candidate rows
// (box in letterboxed pixels at 0..3, coefficients at 6..37), kx = mw / iw, ky = mh / ih; low (N, mh, mw) f32 scratch ->
// out (N, ih, iw) u8 = bilinear(crop(sigmoid(coeffs . proto))) > 0.5
S6_API int sam6d_yolo_masks(const float* proto, int mh, int mw, const float* rows, long long row_ld, int N, int ih, int iw, float kx, float ky,
                            float* low, unsigned char* out, void* stream) {
  S6_REQUIRE(proto && rows && low && out && mh > 0 && mw > 0 && ih > 0 && iw > 0 && N >= 0 && row_ld >= ROW_W);
  S6_REQUIRE((reinterpret_cast<uintptr_t>(proto) & 15) == 0);
  if (N == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  yolo_mask_lowres_kernel<<<dim3(s6_cdiv((long long)mh * mw, 256), N), 256, 0, st>>>(proto, mh, mw, rows, row_ld, kx, ky, low);
  S6_LAUNCH_CHECK();
  const long long T = (long long)N * ih * iw;
  yolo_mask_up_kernel<<<s6_cdiv(T, 256), 256, 0, st>>>(low, N, mh, mw, ih, iw, out);
  S6_LAUNCH_CHECK();
  return 0;
}
