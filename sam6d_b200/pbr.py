"""ISM references from BOP PBR frames: onboarding_config.rendering_type "pbr" (ISM/provider/bop_pbr.py BOPTemplatePBR).

For every template view the ISM takes, instead of a render of the CAD model, the photo-realistic frame of a BOP `train_pbr` split
whose object pose is nearest that view, cut out with the object's visible mask.

    rows = scan_split(root)                                  # load_metaData + shuffle + visibility filter (host)
    sel = select_references(rows, obj_ids, view_poses, rng)  # load_processed_metaData: one row per (object, template) (host)
    ref_cls, ref_patch = reference_features(desc, rows, sel, device)   # decode with PIL, crop on the GPU, DINOv2 descriptors

The crops come from one kernel per chunk (csrc/ism_pbr.cu: sam6d_pbr_reference_crops).  Each distinct row is decoded, cropped
and described once, however many templates it serves; the frames of a chunk stay within FRAME_BUDGET_BYTES on the device.

Quirks of the reference kept on purpose: a scene contributes max_num_frames + 2 frames (its break comes after the rows are
added); max_num_frames is 1000 (the data config's 500 never reaches the class); the visibility filter is strict (> 0.8); the
5000 draws per object come from the caller's RNG (the reference: numpy's global one); the padding of the RGB crops is
normalised with the rest of the crop, so it holds -mean/std (the custom-template path feeds un-normalised crops)."""
import json
import os
import time
from dataclasses import dataclass
from pathlib import Path

import numpy as np
import torch

from . import _lib

MAX_NUM_SCENES = 10
MAX_NUM_FRAMES = 1000
MIN_VISIB_FRACT = 0.8
N_DRAWS = 5000                   # rows drawn (with replacement) per object before the nearest-view search
SHUFFLE_SEED = 2021              # metaData.sample(frac=1, random_state=2021)
# decoded frames (u8 RGB) of one kernel call stay within this many bytes on the device; more frames go to further calls
FRAME_BUDGET_BYTES = 1 << 28
MAX_ROWS_PER_CALL = 256          # crops of one call: 256 x (3 + 1) x 224 x 224 f32 = 205 MB, plus the descriptors' activations


@dataclass
class PbrRows:
    """the rows of a scanned split, one per object instance of a frame: scene_id (the scene directory's name), frame_id, rgb_path,
    visib_fract, obj_id, idx_obj (the instance's position in the frame's scene_gt list) and poses (N,4,4) float64, the
    object -> camera pose (cam_R_m2c, cam_t_m2c in mm).  root and split locate the mask_visib files."""
    root: str
    split: str
    scene_id: np.ndarray
    frame_id: np.ndarray
    rgb_path: np.ndarray
    visib_fract: np.ndarray
    obj_id: np.ndarray
    idx_obj: np.ndarray
    poses: np.ndarray

    def __len__(self):
        return len(self.obj_id)

    def take(self, index) -> "PbrRows":
        index = np.asarray(index, dtype=np.int64)
        return PbrRows(self.root, self.split, self.scene_id[index], self.frame_id[index], self.rgb_path[index], self.visib_fract[index],
                       self.obj_id[index], self.idx_obj[index], self.poses[index])

    def mask_path(self, i: int) -> str:
        return os.path.join(self.root, self.split, f"{int(self.scene_id[i]):06d}", "mask_visib",
                            f"{int(self.frame_id[i]):06d}_{int(self.idx_obj[i]):06d}.png")


def list_scenes(root: str, split: str = "train_pbr"):
    """BaseBOP.load_list_scene: the scene directories of the split but `models`, sorted"""
    folder = os.path.join(root, split)
    if not os.path.isdir(folder):
        raise FileNotFoundError(f"BOP split directory {folder} not found")
    return sorted(os.path.join(folder, s) for s in os.listdir(folder) if os.path.isdir(os.path.join(folder, s)) and s != "models")


def scan_rows(root: str, split: str = "train_pbr", max_num_scenes: int = MAX_NUM_SCENES, max_num_frames: int = MAX_NUM_FRAMES) -> PbrRows:
    """BOPTemplatePBR.load_metaData before its shuffle: the first max_num_scenes scenes; in each, the frames of rgb/*.[pj][pn][g]
    (gray/*.tif without rgb/), sorted, each adding one row per instance of scene_gt.json / scene_gt_info.json.  A scene stops
    after the frame whose position exceeds max_num_frames, so it gives up to max_num_frames + 2 frames."""
    cols = {k: [] for k in ("scene_id", "frame_id", "rgb_path", "visib_fract", "obj_id", "idx_obj", "poses")}
    for scene in list_scenes(root, split)[:max_num_scenes]:
        scene_id = scene.split("/")[-1]
        if os.path.exists(os.path.join(scene, "rgb")):
            paths = sorted(Path(scene).glob("rgb/*.[pj][pn][g]"))
        else:
            paths = sorted(Path(scene).glob("gray/*.tif"))
        with open(os.path.join(scene, "scene_gt_info.json")) as fh:
            gt_info = json.load(fh)
        with open(os.path.join(scene, "scene_gt.json")) as fh:
            gt = json.load(fh)
        for idx_frame, path in enumerate(paths):
            frame_id = int(str(path).split("/")[-1].split(".")[0])
            insts, infos = gt[f"{frame_id}"], gt_info[f"{frame_id}"]
            if len(insts) != len(infos):
                raise ValueError(f"{scene}: frame {frame_id} has {len(insts)} scene_gt and {len(infos)} scene_gt_info entries")
            for k, (x, info) in enumerate(zip(insts, infos)):
                pose = np.eye(4)
                pose[:3, :3] = np.array(x["cam_R_m2c"]).reshape(3, 3)
                pose[:3, 3] = np.array(x["cam_t_m2c"]).reshape(-1)
                cols["scene_id"].append(scene_id)
                cols["frame_id"].append(frame_id)
                cols["rgb_path"].append(str(path))
                cols["visib_fract"].append(float(info["visib_fract"]))
                cols["obj_id"].append(int(x["obj_id"]))
                cols["idx_obj"].append(k)
                cols["poses"].append(pose)
            if idx_frame > max_num_frames:
                break
    return PbrRows(root, split, np.array(cols["scene_id"], dtype=object), np.array(cols["frame_id"], dtype=np.int64),
                   np.array(cols["rgb_path"], dtype=object), np.array(cols["visib_fract"], dtype=np.float64),
                   np.array(cols["obj_id"], dtype=np.int64), np.array(cols["idx_obj"], dtype=np.int64),
                   np.array(cols["poses"], dtype=np.float64).reshape(-1, 4, 4))


def shuffle_order(n: int) -> np.ndarray:
    """the row order of DataFrame.sample(frac=1, random_state=2021) on n rows: RandomState(2021).permutation(n)"""
    return np.random.RandomState(SHUFFLE_SEED).permutation(n)


def scan_split(root: str, split: str = "train_pbr", max_num_scenes: int = MAX_NUM_SCENES, max_num_frames: int = MAX_NUM_FRAMES,
               min_visib_fract: float = MIN_VISIB_FRACT) -> PbrRows:
    """load_metaData and the filter of load_processed_metaData: scan_rows, shuffled, then the rows with visib_fract >
    min_visib_fract (strictly) in that order"""
    rows = scan_rows(root, split, max_num_scenes, max_num_frames)
    rows = rows.take(shuffle_order(len(rows)))
    return rows.take(np.flatnonzero(rows.visib_fract > min_visib_fract))


def select_references(rows: PbrRows, obj_ids, view_poses: np.ndarray, rng=None, n_draws: int = N_DRAWS) -> np.ndarray:
    """load_processed_metaData's selection -> (O,T) int64 row indices into `rows`: for each object in the order given,
    rng.choice(its rows, n_draws) (with replacement; rng defaults to numpy's global RNG), then for each of the T views of
    view_poses (T,4,4) object -> camera the draw whose OpenGL camera axis (third row of opencv2opengl(pose)[:3, :3], so
    rotation only) is nearest in float64 Euclidean distance (scipy cdist), the first draw on a tie.  A row may serve
    several views."""
    from scipy.spatial.distance import cdist
    rng = rng if rng is not None else np.random
    tmpl = -np.asarray(view_poses, dtype=np.float64)[:, 2, :3]
    out = np.empty((len(obj_ids), len(tmpl)), dtype=np.int64)
    for o, obj_id in enumerate(obj_ids):
        cand = np.flatnonzero(rows.obj_id == int(obj_id))
        if len(cand) == 0:
            raise ValueError(f"object {int(obj_id)}: no row of {os.path.join(rows.root, rows.split)} shows it with visib_fract > "
                             f"{MIN_VISIB_FRACT} in the scanned scenes")
        draw = rng.choice(cand, n_draws)
        out[o] = draw[np.argmin(cdist(tmpl, -rows.poses[draw][:, 2, :3]), axis=-1)]
    return out


# ---- crops (BOPTemplatePBR.__getitem__) ---------------------------------------------------------------------------------------
def decode_rgb(path: str) -> np.ndarray:
    """a frame as PIL decodes it -> (H,W,3) u8 RGB"""
    from PIL import Image
    with Image.open(path) as im:
        return np.array(im.convert("RGB"))


def decode_mask(path: str) -> np.ndarray:
    """a visible mask -> (H,W) u8 as stored (an 8-bit grey PNG; any value 0..255)"""
    from PIL import Image
    with Image.open(path) as im:
        if im.mode != "L":
            raise ValueError(f"{path}: visible masks must be 8-bit grey images, got mode {im.mode}")
        return np.array(im)


def crop_frames(frames: torch.Tensor, frame_idx: torch.Tensor, masks: torch.Tensor, target: int = 224):
    """the kernel: frames (F,H,W,3) u8, frame_idx (R,) i32, masks (R,H,W) u8, all CUDA -> (boxes (R,4) i32 Image.getbbox of each
    mask, rgb (R,3,T,T) f32 Normalize(CropResizePad(composite / 255)), mask (R,T,T) f32 CropResizePad(mask / 255))"""
    for t, dt, nd in ((frames, torch.uint8, 4), (frame_idx, torch.int32, 1), (masks, torch.uint8, 3)):
        if not t.is_cuda or t.dtype != dt or t.dim() != nd:
            raise RuntimeError(f"crop_frames: expected CUDA {dt} tensors of frames (F,H,W,3), frame_idx (R,), masks (R,H,W)")
    F, H, W, C = frames.shape
    R = frame_idx.shape[0]
    if C != 3 or tuple(masks.shape) != (R, H, W):
        raise RuntimeError(f"crop_frames: frames {tuple(frames.shape)} and masks {tuple(masks.shape)} do not match")
    if R and (int(frame_idx.min()) < 0 or int(frame_idx.max()) >= F):
        raise ValueError(f"crop_frames: frame_idx outside [0, {F})")
    dev = frames.device
    boxes = torch.empty(R, 4, dtype=torch.int32, device=dev)
    rgb = torch.empty(R, 3, target, target, dtype=torch.float32, device=dev)
    pmask = torch.empty(R, target, target, dtype=torch.float32, device=dev)
    frames, frame_idx, masks = frames.contiguous(), frame_idx.contiguous(), masks.contiguous()
    _lib.call("sam6d_pbr_reference_crops", frames, F, H, W, frame_idx, masks, R, target, boxes, rgb, pmask)
    return boxes, rgb, pmask


def _tick(timings, key, t0, sync=False):
    if timings is None:
        return t0
    if sync:
        torch.cuda.synchronize()
    t1 = time.perf_counter()
    timings[key] = timings.get(key, 0.0) + (t1 - t0)
    return t1


def iter_crops(rows: PbrRows, index, target: int = 224, device=None, max_rows: int = None, frame_budget_bytes: int = None,
               timings=None):
    """crops of rows[index] (distinct row indices) in chunks -> yields (positions into `index` (n,) int64, boxes (n,4) i32,
    rgb (n,3,T,T) f32, mask (n,T,T) f32), the tensors on `device`.  The rows are visited frame after frame; a chunk holds at
    most max_rows rows (MAX_ROWS_PER_CALL) and frames of at most frame_budget_bytes (FRAME_BUDGET_BYTES) of decoded RGB, and
    every frame is decoded once.  An empty visible mask raises.  timings: a dict to which the seconds spent decoding
    ("decode") and in the kernel ("crop") are added (the device is synchronised for that)."""
    max_rows = MAX_ROWS_PER_CALL if max_rows is None else int(max_rows)
    budget = FRAME_BUDGET_BYTES if frame_budget_bytes is None else int(frame_budget_bytes)
    device = torch.device(device if device is not None else "cuda")
    index = np.asarray(index, dtype=np.int64)
    order = sorted(range(len(index)), key=lambda k: (rows.rgb_path[index[k]], int(rows.idx_obj[index[k]])))
    decoded = {}                                   # rgb path -> frame, for the frames of the current and the next chunk
    pos = 0
    while pos < len(order):
        t0 = time.perf_counter()
        chunk, paths, nbytes = [], [], 0
        while pos < len(order) and len(chunk) < max_rows:
            path = rows.rgb_path[index[order[pos]]]
            if path not in paths:
                if path not in decoded:
                    decoded[path] = decode_rgb(path)
                if paths and nbytes + decoded[path].nbytes > budget:
                    break
                paths.append(path)
                nbytes += decoded[path].nbytes
            chunk.append(order[pos])
            pos += 1
        masks = [decode_mask(rows.mask_path(index[k])) for k in chunk]
        t0 = _tick(timings, "decode", t0)
        # one kernel call per frame size: BOP frames of a split share one size, hand-made ones need not
        shapes = sorted({decoded[p].shape for p in paths})
        for shape in shapes:
            group_paths = [p for p in paths if decoded[p].shape == shape]
            slot = {p: i for i, p in enumerate(group_paths)}
            sub = [j for j, k in enumerate(chunk) if rows.rgb_path[index[k]] in slot]
            for j in sub:
                if masks[j].shape != shape[:2]:
                    k = chunk[j]
                    raise ValueError(f"{rows.mask_path(index[k])}: mask {masks[j].shape} does not match its frame {shape[:2]}")
            frames = torch.from_numpy(np.stack([decoded[p] for p in group_paths])).to(device)
            fidx = torch.tensor([slot[rows.rgb_path[index[chunk[j]]]] for j in sub], dtype=torch.int32, device=device)
            m = torch.from_numpy(np.stack([masks[j] for j in sub])).to(device)
            boxes, rgb, pmask = crop_frames(frames, fidx, m, target)
            del frames, m
            t0 = _tick(timings, "crop", t0, sync=True)
            empty = (boxes[:, 2] <= boxes[:, 0]).nonzero().flatten().tolist()
            if empty:
                raise ValueError(f"{rows.mask_path(index[chunk[sub[empty[0]]]])}: the visible mask is empty")
            yield np.array([chunk[j] for j in sub], dtype=np.int64), boxes, rgb, pmask
            t0 = time.perf_counter()
        later = {rows.rgb_path[index[k]] for k in order[pos:pos + max_rows]}
        decoded = {p: f for p, f in decoded.items() if p in later}


def reference_features(desc, rows: PbrRows, selection: np.ndarray, device=None, target: int = 224, timings=None, max_rows: int = None,
                       frame_budget_bytes: int = None):
    """the ISM references of selection (O,T) row indices (select_references) -> (ref_cls (O,T,C), ref_patch (O,T,256,C)) of
    desc.compute_cls_and_patch_features on the crops, written chunk by chunk into the preallocated stacks: each distinct row is
    cropped and described once and copied to every (object, template) it serves.  timings as iter_crops, plus "descriptors".
    max_rows, frame_budget_bytes: iter_crops' chunking."""
    device = torch.device(device if device is not None else "cuda")
    selection = np.asarray(selection, dtype=np.int64)
    O, T = selection.shape
    uniq, inverse = np.unique(selection.reshape(-1), return_inverse=True)
    C, G = desc.model.embed_dim, desc.proposal_size // desc.patch_size
    ref_cls = torch.empty(O * T, C, dtype=torch.float32, device=device)
    ref_patch = torch.empty(O * T, G * G, C, dtype=torch.float32, device=device)
    # slots of every distinct row, grouped: slots_of[u] = the (object, template) positions row uniq[u] serves
    by_row = np.argsort(inverse, kind="stable")
    starts = np.searchsorted(inverse[by_row], np.arange(len(uniq) + 1))
    for where, _, rgb, pmask in iter_crops(rows, uniq, target, device, max_rows, frame_budget_bytes, timings):
        t0 = time.perf_counter()
        cls, patch = desc.compute_cls_and_patch_features(rgb, pmask)
        dst = np.concatenate([by_row[starts[u]:starts[u + 1]] for u in where])
        src = np.concatenate([np.full(starts[u + 1] - starts[u], j) for j, u in enumerate(where)])
        for s in range(0, len(dst), len(where)):          # a row may serve many slots: gather at most a chunk's worth at a time
            d, g = torch.from_numpy(dst[s:s + len(where)]).to(device), torch.from_numpy(src[s:s + len(where)]).to(device)
            ref_cls[d] = cls[g]
            ref_patch[d] = patch[g]
        del cls, patch, rgb, pmask
        _tick(timings, "descriptors", t0, sync=True)
    return ref_cls.view(O, T, C), ref_patch.view(O, T, G * G, C)
