"""tools/make_golden_ism_pbr.py -- writes tests/golden/ism_pbr.pt from the reference's own BOPTemplatePBR, imported through
tools/ref_ism_import.py (run it where the reference's sources are available).

A small seeded BOP split is synthesised: three scenes (plus a `models` directory the scan skips), objects 1, 2 and 5 (and 9,
never visible enough), PNG and JPEG frames from 40 x 30 to 640 x 480, non-contiguous frame ids, visible masks touching the image
border, one mask with non-binary values, visib_fract values at exactly 0.8.  The reference's load_processed_metaData then runs
under np.random.seed at level 0 and level 1 (max_num_frames = 4, so the first scene's quirk shows), and its __getitem__ gives
the crops of a few references.

Stored: every file of the split as bytes (tests rebuild the directory exactly), the reference's view sets, the selected
(scene, frame, idx_obj) per (object, template) in the reference's template order, the unshuffled row keys of load_metaData,
and the reference's `templates` / `template_masks` of a few references, losslessly (their distinct float32 values and an
lzma-compressed uint16 index).  File contents are stored as uint8 tensors, which torch.save writes raw."""
import io
import json
import os
import sys
import tempfile
import lzma

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ism_pbr.pt")
OBJ_IDS = [1, 2, 5]
MAX_NUM_FRAMES = 4
SEED = 7
# (scene name, frame ids, (W, H) per frame, file extension per frame)
SCENES = [
    ("000000", [0, 1, 2, 3, 5, 6, 8, 9], [(48, 36)] * 8, ["png"] * 8),
    ("000001", [0, 3, 4, 7], [(40, 30), (64, 48), (64, 48), (40, 30)], ["jpg", "png", "jpg", "png"]),
    ("000003", [1, 2, 4], [(640, 480), (56, 42), (56, 42)], ["jpg", "png", "png"]),
]


def _rotation(rs):
    q = rs.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _frame(rs, w, h):
    """smooth colour ramps plus noise: compressible, and every channel takes many values (the full-size frame is kept smooth
    so that its JPEG stays small)"""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    base = np.stack([xx / w * 255, yy / h * 255, (xx + yy) / (w + h) * 255], axis=-1)
    noise = rs.normal(0, 20, (h, w, 3)) if w < 640 else 40 * np.sin(xx / 23.0)[..., None] * np.cos(yy / 17.0)[..., None]
    return np.clip(base + noise, 0, 255).astype(np.uint8)


def _mask(rs, w, h, kind):
    yy, xx = np.mgrid[0:h, 0:w]
    cx, cy = rs.uniform(0.2, 0.8) * w, rs.uniform(0.2, 0.8) * h
    if kind == "border":                                  # the ellipse runs off the image on two sides
        cx, cy = rs.choice([0.0, w - 1.0]), rs.choice([0.0, h - 1.0])
    ax, ay = rs.uniform(0.15, 0.45) * w, rs.uniform(0.15, 0.45) * h
    inside = ((xx - cx) / ax) ** 2 + ((yy - cy) / ay) ** 2 <= 1.0
    m = np.zeros((h, w), np.uint8)
    if kind == "soft":                                    # every value 0..255 inside the object
        m[inside] = rs.randint(0, 256, int(inside.sum()))
    else:
        m[inside] = 255
    return m


def _encode(img, ext):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, format="JPEG" if ext == "jpg" else "PNG", **({"quality": 90} if ext == "jpg" else {}))
    return buf.getvalue()


def make_split():
    """-> {path relative to the dataset root: file bytes} of the synthetic train_pbr split"""
    rs = np.random.RandomState(SEED)
    files = {"train_pbr/models/models_info.json": b"{}"}
    n_inst = 0
    for scene, frame_ids, sizes, exts in SCENES:
        gt, gt_info = {}, {}
        for fid, (w, h), ext in zip(frame_ids, sizes, exts):
            files[f"train_pbr/{scene}/rgb/{fid:06d}.{ext}"] = _encode(_frame(rs, w, h), ext)
            k = rs.randint(2, 5)
            objs = [int(o) for o in rs.choice([1, 2, 5, 9], k)] if w < 640 else [1, 2, 5]
            gt[str(fid)], gt_info[str(fid)] = [], []
            for i, o in enumerate(objs):
                R = _rotation(rs)
                t = np.array([rs.uniform(-100, 100), rs.uniform(-100, 100), rs.uniform(400, 1200)])
                vf = float(rs.choice([0.8, round(float(rs.uniform(0.3, 1.0)), 6), 1.0]))
                if w == 640:                                      # the full-size frame's instances are all usable
                    vf = 1.0
                if o == 9:
                    vf = min(vf, 0.8)
                gt[str(fid)].append({"cam_R_m2c": R.reshape(-1).tolist(), "cam_t_m2c": t.tolist(), "obj_id": o})
                gt_info[str(fid)].append({"visib_fract": vf, "bbox_visib": [0, 0, w, h]})
                kind = {1: "border", 3: "soft"}.get(n_inst % 5, "plain") if w < 640 else "plain"
                files[f"train_pbr/{scene}/mask_visib/{fid:06d}_{i:06d}.png"] = _encode(_mask(rs, w, h, kind), "png")
                n_inst += 1
        files[f"train_pbr/{scene}/scene_gt.json"] = json.dumps(gt).encode()
        files[f"train_pbr/{scene}/scene_gt_info.json"] = json.dumps(gt_info).encode()
    return files


def write_split(files, root):
    for rel, data in files.items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as fh:
            fh.write(data)


def _pack(t):
    """a crop, losslessly: its distinct float32 values and the lzma-compressed uint16 index of each element's value (a crop
    built from 8-bit images takes at most 256 distinct values per plane)"""
    a = t.detach().cpu().numpy().astype(np.float32)
    values, index = np.unique(a, return_inverse=True)
    assert len(values) <= 1 << 16
    return {"shape": a.shape, "values": torch.from_numpy(values), "index": _blob(lzma.compress(index.astype(np.uint16).tobytes(), preset=9))}


def _blob(data: bytes) -> torch.Tensor:
    """bytes as a uint8 tensor: torch.save writes tensors raw, where a pickled bytes object grows by half"""
    return torch.frombuffer(bytearray(data), dtype=torch.uint8)


def _crop_rows(root, md, n=5):
    """positions in the selection of up to n distinct rows: one with a non-binary mask, one whose mask touches the border, one
    from a JPEG frame, one from the 640 x 480 frame, then the first others"""
    from PIL import Image
    first, props = {}, []
    for i in range(len(md)):
        key = (str(md.iloc[i].scene_id), int(md.iloc[i].frame_id), int(md.iloc[i].idx_obj))
        if key in first:
            continue
        first[key] = i
        m = np.array(Image.open(os.path.join(root, "train_pbr", key[0], "mask_visib", f"{key[1]:06d}_{key[2]:06d}.png")))
        border = m[0].any() or m[-1].any() or m[:, 0].any() or m[:, -1].any()
        props.append((i, {"soft": bool(((m > 0) & (m < 255)).any()), "border": bool(border),
                          "jpeg": str(md.iloc[i].rgb_path).endswith(".jpg"), "large": m.shape == (480, 640)}))
    chosen = []
    for want in ("soft", "border", "jpeg", "large"):
        hit = next((i for i, p in props if p[want] and i not in chosen), None)
        assert hit is not None, f"no selected row is {want}: change SEED"
        chosen.append(hit)
    chosen += [i for i, _ in props if i not in chosen][:n - len(chosen)]
    return sorted(chosen)


def main():
    import ref_ism_import as rii
    rii.import_reference_ism()
    rii._stub("imageio.v2")
    from provider.bop_pbr import BOPTemplatePBR
    from utils.poses.pose_utils import get_obj_poses_from_template_level
    from types import SimpleNamespace

    files = make_split()
    out = {"files": {k: _blob(v) for k, v in files.items()}, "obj_ids": OBJ_IDS, "max_num_frames": MAX_NUM_FRAMES, "seed": SEED, "levels": {}}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "synth")
        write_split(files, root)
        tdir = os.path.join(tmp, "templates")
        for o in OBJ_IDS:
            os.makedirs(os.path.join(tdir, f"obj_{o:06d}"))
        for level in (0, 1):
            ds = BOPTemplatePBR(root_dir=root, template_dir=tdir, obj_ids=None, processing_config=SimpleNamespace(image_size=224),
                                level_templates=level, pose_distribution="all", max_num_frames=MAX_NUM_FRAMES)
            assert ds.obj_ids == OBJ_IDS
            np.random.seed(SEED + level)
            ds.load_processed_metaData(reset_metaData=True)
            md = ds.metaData
            T = len(ds.template_poses)
            keys = [(str(md.iloc[i].scene_id), int(md.iloc[i].frame_id), int(md.iloc[i].idx_obj)) for i in range(len(md))]
            rec = {"template_poses": np.asarray(get_obj_poses_from_template_level(level, "all"), dtype=np.float64),
                   "selected": [keys[o * T:(o + 1) * T] for o in range(len(OBJ_IDS))], "np_seed": SEED + level}
            if level == 0:
                raw = ds.load_metaData(reset_metaData=True)          # the unshuffled rows, and the shuffled frame
                rec["raw_keys"] = [(str(s), int(f), int(k)) for s, f, k in zip(raw["scene_id"], raw["frame_id"], raw["idx_obj"])]
                rec["raw_visib"] = np.asarray(raw["visib_fract"], dtype=np.float64)
                rec["shuffled_keys"] = [(str(ds.metaData.iloc[i].scene_id), int(ds.metaData.iloc[i].frame_id), int(ds.metaData.iloc[i].idx_obj))
                                        for i in range(len(ds.metaData))]
                # the reference's crops of a few selected rows, one row at a time through its own __getitem__ (it stacks the full
                # frames of an object's references, so it needs one frame size per object; the split has several)
                np.random.seed(SEED + level)
                ds.load_processed_metaData(reset_metaData=True)
                md, tp = ds.metaData, ds.template_poses
                crops = []
                for i in _crop_rows(root, md):
                    ds.metaData, ds.template_poses = md.iloc[[i]].reset_index(drop=True), tp[:1]
                    item = ds[0]
                    crops.append({"obj": i // T, "template": i % T, "key": keys[i], "templates": _pack(item["templates"][0]),
                                  "template_masks": _pack(item["template_masks"][0])})
                ds.metaData, ds.template_poses = md, tp
                rec["crops"] = crops
            out["levels"][level] = rec
    torch.save(out, OUT)
    print(f"wrote {OUT}: {len(files)} files, {os.path.getsize(OUT) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
