// crop_geom.cuh -- the index math of CropResizePad (ISM/utils/bbox_utils.py:89-126): which source pixel of the box feeds output
// pixel (oy, ox) of the T x T crop.  Shared by every kernel that crops a box to the descriptor's input, so they agree bit for bit.
#pragma once

// F.interpolate(mode='nearest', scale_factor=s): out = floor(in * s) (double), src = min(floor(dst * (1/s) as float), in - 1)
__device__ __forceinline__ int nearest_src(int dst, float inv_scale, int in_size) { return min((int)floorf((float)dst * inv_scale), in_size - 1); }

// box (x1, y1, x2, y2), exclusive max -> true and the source pixel (sy, sx) when output pixel (oy, ox) lies on the resized crop,
// false when it lies on the zero padding.  An empty box (x2 <= x1 or y2 <= y1) has no crop: every pixel is padding.
__device__ __forceinline__ bool crop_resize_pad_src(int x1, int y1, int x2, int y2, int T, int oy, int ox, int& sy, int& sx) {
  const int bw = x2 - x1, bh = y2 - y1;
  sy = sx = 0;
  if (bw <= 0 || bh <= 0) return false;
  // scale_factor = target_max / max(box size) as a float32 tensor element, .item() -> double (bbox_utils.py:99-105)
  // `target_max / tensor` is torch.Tensor.__rtruediv__ = tensor.reciprocal() * target_max: two float32 roundings
  const float scale_f = __fmul_rn(__frcp_rn((float)max(bw, bh)), (float)T);
  const double scale = (double)scale_f;
  const int rh = (int)floor((double)bh * scale), rw = (int)floor((double)bw * scale);
  const float inv = (float)(1.0 / scale);                 // ATen: scale = 1 / scale_factor, computed in double, used as float
  // padding (bbox_utils.py:111-118); a square resized crop (target ratio == original ratio) is not padded
  int pt = 0, pl = 0, side = rh;                          // side of the (square) image after the optional padding
  if ((double)rw / (double)rh != 1.0) { pt = max((T - rh) / 2, 0); pl = max((T - rw) / 2, 0); side = T; }
  // final F.interpolate(scale_factor = T / side) (:122-124): the identity unless an unpadded square crop came out one pixel short
  int py = oy, px = ox;
  if (side != T) {
    const float inv2 = (float)(1.0 / ((double)T / (double)side));
    py = nearest_src(oy, inv2, side); px = nearest_src(ox, inv2, side);
  }
  const int yy = py - pt, xx = px - pl;
  if (!(yy >= 0 && yy < rh && xx >= 0 && xx < rw)) return false;
  sy = y1 + nearest_src(yy, inv, bh); sx = x1 + nearest_src(xx, inv, bw);
  return true;
}
