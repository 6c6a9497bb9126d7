// ism_pbr.cu -- ISM reference crops from BOP PBR frames (rendering_type: pbr; ISM/provider/bop_pbr.py BOPTemplatePBR.__getitem__):
//   * mask_bbox       : PIL Image.getbbox of every visible mask: the box of its nonzero pixels, exclusive max
//   * pbr_crop        : Image.composite(rgb, black, mask) / 255, the mask / 255, CropResizePad(T) of both (crop_geom.cuh, the
//                       index math of sam6d_crop_resize_pad) and T.Normalize(ImageNet) of the padded RGB crop -- every reference of
//                       a chunk in one launch, each cut from its frame of a shared stack, instead of one PIL + torch pass per image
#include "common.cuh"
#include "crop_geom.cuh"

namespace {

constexpr int BBOX_THREADS = 512;

__device__ __forceinline__ void bbox_add(int i, int W, int& x0, int& y0, int& x1, int& y1) {
  const int y = i / W, x = i - y * W;
  x0 = min(x0, x); x1 = max(x1, x); y0 = min(y0, y); y1 = max(y1, y);
}

// one CTA per mask (H*W u8, nonzero = object) -> box (x0, y0, x1 + 1, y1 + 1), or (0, 0, 0, 0) for an empty mask
__global__ void __launch_bounds__(BBOX_THREADS) mask_bbox_kernel(const unsigned char* __restrict__ masks, int H, int W, int* __restrict__ boxes) {
  const int r = blockIdx.x, tid = threadIdx.x;
  const long long n = (long long)H * W;
  const unsigned char* m = masks + (size_t)r * n;
  int x0 = INT_MAX, y0 = INT_MAX, x1 = -1, y1 = -1;
  if ((n & 15) == 0 && (reinterpret_cast<size_t>(masks) & 15) == 0) {
    const uint4* v = reinterpret_cast<const uint4*>(m);
    for (long long j = tid; j < n / 16; j += BBOX_THREADS) {
      const uint4 q = __ldg(v + j);
      if ((q.x | q.y | q.z | q.w) == 0u) continue;
      const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int k = 0; k < 16; ++k)
        if ((w[k >> 2] >> ((k & 3) * 8)) & 0xffu) bbox_add((int)(j * 16 + k), W, x0, y0, x1, y1);
    }
  } else {
    for (long long i = tid; i < n; i += BBOX_THREADS)
      if (m[i]) bbox_add((int)i, W, x0, y0, x1, y1);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    x0 = min(x0, __shfl_xor_sync(0xffffffffu, x0, o)); y0 = min(y0, __shfl_xor_sync(0xffffffffu, y0, o));
    x1 = max(x1, __shfl_xor_sync(0xffffffffu, x1, o)); y1 = max(y1, __shfl_xor_sync(0xffffffffu, y1, o));
  }
  __shared__ int red[4][BBOX_THREADS / 32];
  const int lane = tid & 31, warp = tid >> 5;
  if (lane == 0) { red[0][warp] = x0; red[1][warp] = y0; red[2][warp] = x1; red[3][warp] = y1; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < BBOX_THREADS / 32; ++w) {
      x0 = min(x0, red[0][w]); y0 = min(y0, red[1][w]); x1 = max(x1, red[2][w]); y1 = max(y1, red[3][w]);
    }
    const bool empty = x1 < 0;
    boxes[r * 4 + 0] = empty ? 0 : x0; boxes[r * 4 + 1] = empty ? 0 : y0;
    boxes[r * 4 + 2] = empty ? 0 : x1 + 1; boxes[r * 4 + 3] = empty ? 0 : y1 + 1;
  }
}

// grid (T, R), block T threads (rounded up to a warp): reference r, output row oy, column ox.
//   rgb[r, c]  = (composite / 255 - mean[c]) / std[c], composite = DIV255(frame * mask) as PIL's paste through an L mask rounds it;
//                the padding is (0 - mean[c]) / std[c] (Normalize runs after the pad)
//   pmask[r]   = mask / 255 on the crop, 0 on the padding
// Both /255 are float64 divisions rounded to float32, as np.array(image) / 255 followed by .float() computes them.
__global__ void pbr_crop_kernel(const unsigned char* __restrict__ frames, int F, int H, int W, const int* __restrict__ frame_idx,
                                const unsigned char* __restrict__ masks, const int* __restrict__ boxes, int T, float* __restrict__ rgb,
                                float* __restrict__ pmask) {
  const int r = blockIdx.y, oy = blockIdx.x, ox = threadIdx.x;
  if (ox >= T) return;
  const int f = frame_idx[r];
  int sy, sx;
  const bool inside = (unsigned)f < (unsigned)F &&
                      crop_resize_pad_src(boxes[r * 4], boxes[r * 4 + 1], boxes[r * 4 + 2], boxes[r * 4 + 3], T, oy, ox, sy, sx);
  const unsigned m = inside ? masks[((size_t)r * H + sy) * W + sx] : 0u;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, sd[3] = {0.229f, 0.224f, 0.225f};
  const size_t plane = (size_t)T * T, o = (size_t)oy * T + ox;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = 0.f;
    if (inside) {
      const unsigned t = (unsigned)frames[(((size_t)f * H + sy) * W + sx) * 3 + c] * m + 128u;
      v = (float)((double)((t + (t >> 8)) >> 8) / 255.0);
    }
    rgb[((size_t)r * 3 + c) * plane + o] = __fdiv_rn(__fsub_rn(v, mean[c]), sd[c]);
  }
  pmask[(size_t)r * plane + o] = inside ? (float)((double)m / 255.0) : 0.f;
}

}  // namespace

S6_API int sam6d_pbr_reference_crops(const unsigned char* frames, int F, int H, int W, const int* frame_idx, const unsigned char* masks, int R,
                                     int T, int* boxes, float* rgb, float* pmask, void* stream) {
  S6_REQUIRE(frames && frame_idx && masks && boxes && rgb && pmask && F > 0 && H > 0 && W > 0 && R >= 0 && R <= 65535 && T > 0 && T <= 1024 &&
             (long long)H * W < (1ll << 31));
  if (R == 0) return 0;
  cudaStream_t st = s6_stream(stream);
  mask_bbox_kernel<<<R, BBOX_THREADS, 0, st>>>(masks, H, W, boxes);
  pbr_crop_kernel<<<dim3(T, R), ((T + 31) / 32) * 32, 0, st>>>(frames, F, H, W, frame_idx, masks, boxes, T, rgb, pmask);
  S6_LAUNCH_CHECK();
  return 0;
}
