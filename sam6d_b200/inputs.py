"""PEM input builder on the GPU -- drop-in for get_test_data / the detection loop of PEM/run_inference_custom.py:165-253
(SURVEY.md 8f row N3).  The reference decodes every detection's mask, crops, samples and resizes in numpy / cv2 on one host
core; here two C-ABI calls (csrc/inputs.cu) do it for all detections of a frame on the device, and only 10 ints per detection
come back in between so that the host can draw the sample indices with numpy's RNG exactly as the reference does.

    ret_dict, whole_image, whole_pts, model_points, all_dets = get_test_data(dets, image, depth, cam_K, depth_scale, model_points, ...)

ret_dict carries the reference's keys: pts (P,2048,3), rgb (P,3,224,224), rgb_choose (P,2048) int64, score (P), model, K."""
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib

ST = 12   # ints per detection in the stats array (csrc/inputs.cu)


def pack_rle(dets: Sequence[Dict], H: int, W: int):
    """uncompressed COCO RLE of every detection ({"counts": [...], "size": [h, w]}, ISM/model/utils.py:25-43) -> (cumulative run
    ends concatenated, offsets) as int32 arrays"""
    cums, off = [], [0]
    for d in dets:
        seg = d["segmentation"]
        if list(seg["size"]) != [H, W]:
            raise ValueError(f"segmentation size {seg['size']} does not match the frame {(H, W)}")
        counts = seg["counts"]
        if isinstance(counts, (str, bytes)):
            raise NotImplementedError("compressed COCO RLE strings: SAM-6D's ISM writes uncompressed counts (mask_to_rle)")
        c = np.cumsum(np.asarray(counts, dtype=np.int64))
        if len(c) and c[-1] != H * W:
            raise ValueError("RLE counts do not cover the image")
        cums.append(c.astype(np.int32))
        off.append(off[-1] + len(c))
    cum = np.concatenate(cums) if cums else np.zeros(0, np.int32)
    return np.ascontiguousarray(cum, dtype=np.int32), np.asarray(off, dtype=np.int32)


class FrameInputs:
    """device-side state of one frame between the two stages.  radius: the object radius (one number for every detection) or
    one radius per detection (several objects in a frame).

    BOPTestset.get_instance (sam6d_b200/bop.py) uses the same stages with its own rules: depth_m, the (H,W) float32 depth map in
    metres that replaces the custom path's (depth_raw then only gives the frame size), thr, the float64 radius threshold of every
    detection that replaces radius * 1.2, and min_count, the pixel count a mask must exceed (kept() takes the rest of the rule)."""

    def __init__(self, dets, image_u8: np.ndarray, depth_raw: np.ndarray, cam_K, depth_scale: float, radius, device=None,
                 depth_m: Optional[np.ndarray] = None, thr: Optional[np.ndarray] = None, min_count: int = 32):
        self.device = torch.device(device if device is not None else "cuda")
        self.dets = list(dets)
        if image_u8.ndim == 2:                                                     # run_inference_custom.py:177-178
            image_u8 = np.concatenate([image_u8[:, :, None]] * 3, axis=2)
        self.H, self.W = depth_raw.shape
        K = np.asarray(cam_K, dtype=np.float64).reshape(3, 3)
        self.K = K
        if depth_m is None:
            whole_depth = depth_raw.astype(np.float32) * depth_scale / 1000.0      # :179 (float32 * python floats)
        else:
            whole_depth = depth_m
        self.depth = torch.from_numpy(np.ascontiguousarray(whole_depth, dtype=np.float32)).to(self.device)
        self.image = torch.from_numpy(np.ascontiguousarray(image_u8, dtype=np.uint8)).to(self.device)
        P = len(self.dets)
        if thr is None:
            radius = np.broadcast_to(np.asarray(radius, dtype=np.float32), (P,))
            self.thr = (radius * np.float32(1.2)).astype(np.float64)               # :209 under numpy >= 2 (weak python scalar)
        else:
            self.thr = np.array(np.broadcast_to(np.asarray(thr, dtype=np.float64), (P,)))
        cum, off = pack_rle(self.dets, self.H, self.W)
        self.cap = min(self.H, self.W) ** 2
        dev = self.device
        self.mask = torch.empty(P, self.H, self.W, dtype=torch.uint8, device=dev)
        self.stats = torch.empty(P, ST, dtype=torch.int32, device=dev)
        self.choose1 = torch.empty(P, self.cap, dtype=torch.int32, device=dev)
        self.choose2 = torch.empty(P, self.cap, dtype=torch.int32, device=dev)
        self.cloud2 = torch.empty(P, self.cap, 3, dtype=torch.float32, device=dev)
        if P:
            cum_d = torch.from_numpy(cum).to(dev) if len(cum) else torch.zeros(1, dtype=torch.int32, device=dev)
            off_d = torch.from_numpy(off).to(dev)
            thr_d = torch.from_numpy(self.thr).to(dev)
            _lib.call("sam6d_inputs_stage_a_min", cum_d, off_d, P, self.H, self.W, self.depth, float(K[0, 0]), float(K[1, 1]),
                      float(K[0, 2]), float(K[1, 2]), thr_d, int(min_count), self.mask, self.stats, self.cap, self.choose1, self.choose2,
                      self.cloud2)
        self.stats_host = self.stats.cpu().numpy() if P else np.zeros((0, ST), np.int32)

    # what the reference's loop decides per detection (run_inference_custom.py:199-212: more than 32 pixels, at least 4 points
    # after the radius filter; BOPTestset.get_instance: 8 and 8)
    def kept(self, min_count: int = 32, min_valid: int = 4) -> np.ndarray:
        s = self.stats_host
        return np.flatnonzero((s[:, 4] > min_count) & (s[:, 9] >= min_valid)) if len(s) else np.zeros(0, np.int64)

    def n_valid(self) -> np.ndarray:
        return self.stats_host[:, 9]

    def bbox(self) -> np.ndarray:
        return self.stats_host[:, 5:9]

    def sample(self, keep: np.ndarray, choose_idx: np.ndarray, img_size: int = 224, rgb_mask_flag: bool = True, want_u8: bool = False):
        """choose_idx (Q, n_sample) indices into each kept detection's filtered point list -> pts, rgb_choose, rgb (, rgb_u8)"""
        Q, ns = choose_idx.shape
        dev = self.device
        pts = torch.empty(Q, ns, 3, dtype=torch.float32, device=dev)
        rgb_choose = torch.empty(Q, ns, dtype=torch.int64, device=dev)
        rgb = torch.empty(Q, 3, img_size, img_size, dtype=torch.float32, device=dev)
        u8 = torch.empty(Q, img_size, img_size, 3, dtype=torch.uint8, device=dev) if want_u8 else None
        if Q:
            keep_d = torch.from_numpy(np.ascontiguousarray(keep, dtype=np.int32)).to(dev)
            ci = torch.from_numpy(np.ascontiguousarray(choose_idx, dtype=np.int32)).to(dev)
            _lib.call("sam6d_inputs_stage_b", self.stats, keep_d, Q, self.H, self.W, self.cap, self.choose2, self.cloud2, ci, ns, img_size,
                      self.image, self.mask, int(rgb_mask_flag), pts, rgb_choose, rgb, u8)
        return pts, rgb_choose, rgb, u8

    def rows(self, keep: np.ndarray) -> SimpleNamespace:
        """the device state pose verification reads, without a copy: depth (H,W) f32 metres, mask (P,H,W) u8 (the RLE AND
        depth > 0) and mrow (Q,) int64, the mask row of each kept detection"""
        return SimpleNamespace(depth=self.depth, mask=self.mask, mrow=np.asarray(keep, dtype=np.int64))

    def whole_points(self) -> torch.Tensor:
        """get_point_cloud_from_depth of the frame, (H*W, 3) float32 (visualisation only in the reference)"""
        ys, xs = torch.meshgrid(torch.arange(self.H, device=self.device), torch.arange(self.W, device=self.device), indexing="ij")
        z = self.depth.double()
        x = (xs.float().double() - self.K[0, 2]) * z / self.K[0, 0]
        y = (ys.float().double() - self.K[1, 2]) * z / self.K[1, 1]
        return torch.stack([x, y, z], dim=-1).reshape(-1, 3).float()


def draw_choose_idx(n_valid: Sequence[int], n_sample: int, rng=None) -> np.ndarray:
    """run_inference_custom.py:213-216: np.random.choice(np.arange(n), n_sample[, replace=False]) per kept detection"""
    rng = rng if rng is not None else np.random
    out = np.empty((len(n_valid), n_sample), dtype=np.int64)
    for i, n in enumerate(n_valid):
        out[i] = rng.choice(np.arange(n), n_sample) if n <= n_sample else rng.choice(np.arange(n), n_sample, replace=False)
    return out


def get_test_data(dets: List[Dict], whole_image: np.ndarray, depth_raw: np.ndarray, cam_K, depth_scale: float, model_points: np.ndarray,
                  det_score_thresh: float = 0.2, n_sample_observed_point: int = 2048, img_size: int = 224, rgb_mask_flag: bool = True,
                  choose_idx: Optional[np.ndarray] = None, rng=None, device=None, det_obj: Optional[Sequence[int]] = None,
                  frame_rows: bool = False):
    """The reference's get_test_data after its file reads (the caller loads rgb / depth / camera / detections / CAD samples).
    model_points: (n,3) float32 CAD samples in metres (the reference draws them with trimesh, :182-184).
    -> (ret_dict, whole_image, whole_pts (H*W,3), model_points, all_dets) like the reference.
    Several objects: model_points (O,n,3) and det_obj the object index of every detection in `dets`.  Each detection then gets
    its object's radius filter and `model` rows; ret_dict["obj"] (P) int64 holds the object index of every kept one and
    ret_dict["choose_idx"] the sample indices drawn for it.
    frame_rows=True appends frame_rows(), the frame's device depth and decoded masks with the kept detections' rows."""
    sel = [i for i, d in enumerate(dets) if d["score"] > det_score_thresh]           # :168-171
    dets = [dets[i] for i in sel]
    model_points = np.asarray(model_points, dtype=np.float32)
    if det_obj is None:
        radius = np.max(np.linalg.norm(model_points, axis=1))                        # :184
    else:
        det_obj = np.asarray(det_obj, dtype=np.int64)[sel]
        radius = np.asarray([np.max(np.linalg.norm(m, axis=1)) for m in model_points])[det_obj]
    frame = FrameInputs(dets, whole_image, depth_raw, cam_K, depth_scale, radius, device)
    keep = frame.kept()
    if choose_idx is None:
        choose_idx = draw_choose_idx(frame.n_valid()[keep], n_sample_observed_point, rng)
    pts, rgb_choose, rgb, _ = frame.sample(keep, np.asarray(choose_idx), img_size, rgb_mask_flag)
    dev = frame.device
    n = len(keep)
    if det_obj is None:
        model = torch.from_numpy(model_points).to(dev).unsqueeze(0).repeat(n, 1, 1)
    else:
        obj = torch.from_numpy(det_obj[keep]).to(dev)
        model = torch.from_numpy(model_points).to(dev)[obj]
    ret = dict(pts=pts, rgb=rgb, rgb_choose=rgb_choose,
               score=torch.tensor([dets[i]["score"] for i in keep], dtype=torch.float32, device=dev), model=model,
               K=torch.tensor(np.asarray(cam_K, dtype=np.float64).reshape(3, 3), dtype=torch.float32, device=dev).unsqueeze(0).repeat(n, 1, 1))
    if det_obj is not None:
        ret["obj"], ret["choose_idx"] = obj, np.asarray(choose_idx)
    if frame_rows:
        return ret, whole_image, frame.whole_points(), model_points, [dets[i] for i in keep], frame.rows(keep)
    return ret, whole_image, frame.whole_points(), model_points, [dets[i] for i in keep]


def _square_bbox(mask: np.ndarray):
    """get_bbox (PEM/utils/data_utils.py:127-160) on a host mask"""
    H, W = mask.shape
    rows, cols = np.flatnonzero(mask.any(axis=1)), np.flatnonzero(mask.any(axis=0))
    rmin, rmax, cmin, cmax = int(rows[0]), int(rows[-1]) + 1, int(cols[0]), int(cols[-1]) + 1
    b = min(max(rmax - rmin, cmax - cmin), min(H, W))
    cy, cx, hb = (rmin + rmax) // 2, (cmin + cmax) // 2, b // 2
    rmin, rmax, cmin, cmax = cy - hb, cy + hb, cx - hb, cx + hb
    if rmin < 0:
        rmax, rmin = rmax - rmin, 0
    if cmin < 0:
        cmax, cmin = cmax - cmin, 0
    if rmax > H:
        rmin, rmax = rmin - (rmax - H), H
    if cmax > W:
        cmin, cmax = cmin - (cmax - W), W
    return [rmin, rmax, cmin, cmax]


def get_templates_from_arrays(rgbs: Sequence[np.ndarray], masks: Sequence[np.ndarray], xyzs_mm: Sequence[np.ndarray],
                              n_sample_template_point: int = 5000, img_size: int = 224, rgb_mask_flag: bool = True, choose_idx=None,
                              rng=None, device=None):
    """_get_template (PEM/run_inference_custom.py:117-146) for all template views after their file reads: rgb (H,W,3) uint8 as
    loaded, mask (H,W) uint8 (255 = object), xyz (H,W,3) object coordinates in mm.
    -> (all_tem, all_tem_pts, all_tem_choose): lists of (1,3,S,S) f32, (1,n,3) f32, (1,n) int64 like get_templates (:149-162)"""
    dev = torch.device(device if device is not None else "cuda")
    T = len(rgbs)
    H, W = masks[0].shape
    m = np.stack([np.ascontiguousarray(x == 255) for x in masks])
    bbox = np.asarray([_square_bbox(mm) for mm in m], dtype=np.int32)
    img_d = torch.from_numpy(np.ascontiguousarray(np.stack(rgbs), dtype=np.uint8)).to(dev)
    mask_d = torch.from_numpy(m.astype(np.uint8)).to(dev)
    bbox_d = torch.from_numpy(bbox).to(dev)
    rgb = torch.empty(T, 3, img_size, img_size, dtype=torch.float32, device=dev)
    _lib.call("sam6d_crop_resize_normalize", img_d, mask_d, bbox_d, T, H, W, img_size, int(rgb_mask_flag), rgb, None)
    rng = rng if rng is not None else np.random
    all_tem, all_pts, all_choose = [], [], []
    for t in range(T):
        y1, y2, x1, x2 = bbox[t].tolist()
        crop = mask_d[t, y1:y2, x1:x2].reshape(-1)
        choose = torch.nonzero(crop, as_tuple=False).reshape(-1)                      # row-major, ascending like numpy's nonzero
        n = int(choose.numel())
        if choose_idx is not None:
            ci = np.asarray(choose_idx[t])
        else:
            ci = rng.choice(np.arange(n), n_sample_template_point) if n <= n_sample_template_point else \
                rng.choice(np.arange(n), n_sample_template_point, replace=False)
        choose = choose[torch.from_numpy(np.ascontiguousarray(ci, dtype=np.int64)).to(dev)]
        xyz = torch.from_numpy(np.ascontiguousarray(xyzs_mm[t][y1:y2, x1:x2, :], dtype=np.float32)).to(dev).reshape(-1, 3) / 1000.0
        cw = x2 - x1
        ratio_h, ratio_w = img_size / (y2 - y1), img_size / cw
        rc = (torch.floor((choose // cw).double() * ratio_h) * img_size + torch.floor((choose % cw).double() * ratio_w)).long()
        all_tem.append(rgb[t:t + 1])
        all_pts.append(xyz[choose].unsqueeze(0))
        all_choose.append(rc.unsqueeze(0))
    return all_tem, all_pts, all_choose
