"""tools/make_golden_bop_test.py -- writes tests/golden/bop_test.pt from the reference's own BOP test code (run it where the
reference's sources are available).

A small seeded synthetic BOP dataset "lmo" (so the category-id quirk shows) is built: objects 1 and 5 (models_info diameters,
ASCII PLY files, 42 template views each), three test scenes -- PNG rgb with depth_scale 0.1, JPEG rgb with depth_scale 1.0,
and a gray/*.tif scene -- u16 depth with holes, and a detection JSON whose scores sit around 0.25 and whose masks sit around
the 8-point limits (8 and 9 pixels, masks whose points mostly fall outside 0.6 x diameter).  Then the reference runs on it:

- PEM/provider/bop_test_dataset.py BOPTestset.__getitem__ (get_instance, get_bop_image, get_bop_depth_map) on every image of
  the detection file; the sample indices its np.random.choice calls return are recorded;
- PEM/test_bop.py test() with a stub Net (seeded outputs) and a stub DataLoader-free setting: the CSV lines it writes;
- ISM/model/utils.py Detections.save_to_file + convert_npz_to_json on synthetic detections, for "lmo" and "ycbv".

pycocotools, trimesh, gorilla and imageio are not installed here, so they are stubbed: cocomask.decode of an uncompressed RLE
is the reference's own numpy rle_to_binary_mask (PEM/utils/data_utils.py), trimesh's mesh.sample returns model points this
script draws (they are stored), imageio.imread is PIL's decode.

Everything is stored losslessly and compressed (tests/_bop_golden.py reads it back): the split's files as lzma-compressed bytes,
integer arrays as lzma-compressed bytes, point clouds as their distinct float32 values plus a compressed index, and each
normalised crop as the u8 crop it was made from (checked here to give the reference's crop back through ToTensor + Normalize)."""
import importlib
import io
import json
import lzma
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "bop_test.pt")
PEM = "/root/reference/SAM-6D/Pose_Estimation_Model"
SEED = 11
DATASET = "lmo"
OBJ_IDS = [1, 5]
DIAMETERS = {1: 120.0, 5: 90.0}
W, H = 64, 48
K = [60.0, 0.0, 31.5, 0.0, 60.0, 23.5, 0.0, 0.0, 1.0]
# scene -> (frame ids, image kind, depth_scale)
SCENES = {2: ([3], "png", 0.1), 7: ([1, 2], "jpg", 1.0), 9: ([4], "tif", 0.1)}
EMPTY = (7, 2)            # every detection of this image is dropped (the reference fails on it)
N_MODEL_POINTS = 1024


def _encode(img, fmt):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, format=fmt, **({"quality": 90} if fmt == "JPEG" else {}))
    return buf.getvalue()


def _ply(rs):
    """a small closed mesh (octahedron, mm) as ASCII PLY; its content does not matter to the instances"""
    v = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64) * rs.uniform(30, 50)
    f = [[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]]
    s = "ply\nformat ascii 1.0\nelement vertex 6\nproperty float x\nproperty float y\nproperty float z\nelement face 8\n" \
        "property list uchar int vertex_indices\nend_header\n"
    s += "".join("%f %f %f\n" % tuple(x) for x in v) + "".join("3 %d %d %d\n" % tuple(x) for x in f)
    return s.encode()


def _ellipse(cx, cy, ax, ay, h=H, w=W):
    yy, xx = np.mgrid[0:h, 0:w]
    return ((xx - cx) / ax) ** 2 + ((yy - cy) / ay) ** 2 <= 1.0


def _rle(mask):
    """uncompressed COCO RLE (column-major runs, first run of zeros), as the ISM writes it"""
    flat = mask.ravel(order="F").astype(np.int64)
    change = np.flatnonzero(np.diff(flat)) + 1
    ends = np.concatenate([change, [flat.size]])
    counts = np.diff(np.concatenate([[0], ends])).tolist()
    if flat[0]:
        counts = [0] + counts
    return {"counts": counts, "size": [H, W]}


def make_split():
    """-> ({path relative to the BOP root: bytes}, model points {obj_id: (n,3) f64 mm}, detections)"""
    rs = np.random.RandomState(SEED)
    files, points = {}, {}
    mdir = f"{DATASET}/models"
    files[f"{mdir}/models_info.json"] = json.dumps({str(o): {"diameter": DIAMETERS[o]} for o in OBJ_IDS}).encode()
    for o in OBJ_IDS:
        files[f"{mdir}/obj_{o:06d}.ply"] = _ply(rs)
        points[o] = np.round(rs.uniform(-40, 40, (N_MODEL_POINTS, 3)), 1)
        for v in range(42):                                     # the PEM's template views
            m = _ellipse(16 + rs.uniform(-3, 3), 16 + rs.uniform(-3, 3), rs.uniform(5, 12), rs.uniform(5, 12), 32, 32)
            yy, xx = np.mgrid[0:32, 0:32]
            rgb = np.stack([xx * 7 + v, yy * 7 + 2 * v, (xx + yy) * 3 + 3 * v], -1).astype(np.uint8)
            xyz = (np.stack([xx - 16.0, yy - 16.0, (xx + yy) / 2.0 + v], -1) * 2.5 * m[..., None]).astype(np.float16)
            files[f"BOP-Templates/{DATASET}/obj_{o:06d}/rgb_{v}.png"] = _encode(rgb, "PNG")
            files[f"BOP-Templates/{DATASET}/obj_{o:06d}/mask_{v}.png"] = _encode((m * 255).astype(np.uint8), "PNG")
            buf = io.BytesIO()
            np.save(buf, xyz)
            files[f"BOP-Templates/{DATASET}/obj_{o:06d}/xyz_{v}.npy"] = buf.getvalue()
    dets = []
    yy, xx = np.mgrid[0:H, 0:W]
    for scene, (frame_ids, kind, scale) in SCENES.items():
        sdir = f"{DATASET}/test/{scene:06d}"
        cams = {}
        for fid in frame_ids:
            cams[str(fid)] = {"cam_K": K, "depth_scale": scale}
            img = np.clip(np.stack([xx * 4, yy * 5, (xx + yy) * 2], -1) + 20 * np.sin(xx[..., None] / 2.3 + yy[..., None] / 3.1 + np.arange(3)) + rs.normal(0, 2, (H, W, 3)), 0, 255).astype(np.uint8)
            if kind == "png":
                files[f"{sdir}/rgb/{fid:06d}.png"] = _encode(img, "PNG")
            elif kind == "jpg":
                files[f"{sdir}/rgb/{fid:06d}.jpg"] = _encode(img, "JPEG")
            else:
                files[f"{sdir}/gray/{fid:06d}.tif"] = _encode(img[..., 0], "TIFF")
            depth_mm = 600 + 2.3 * xx + 1.7 * yy + rs.uniform(0, 40, (H, W))
            depth_mm[rs.uniform(size=(H, W)) < 0.08] = 0                     # holes
            depth_mm[30:40, 50:60] += 400                                    # a step: far points inside some masks
            depth_mm[5:9, 5:8] = 650                                         # the 9-pixel mask: no hole
            depth_mm[44, 40:52] = 700
            depth_mm[44, 50:52] += 150                                       # 10-pixel line, two points off the object
            raw = np.round(depth_mm / scale).astype(np.uint16)
            files[f"{sdir}/depth/{fid:06d}.png"] = _encode(raw, "PNG")
            t = float(rs.uniform(0.1, 0.5))
            masks = [_ellipse(20, 20, 8, 6), _ellipse(45, 30, 6, 5), _ellipse(40, 12, 4, 3)]
            tiny9 = np.zeros((H, W), bool)                                   # get_bbox's square crop holds all of it
            tiny9[5:9, 5:7] = True
            tiny9[5, 7] = True
            tiny8 = tiny9.copy()
            tiny8[5, 7] = False
            line = np.zeros((H, W), bool)
            line[44, 42:52] = True
            masks += [tiny9, tiny8, line]
            scores = [0.9, 0.6, 0.25, float(np.nextafter(np.float32(0.25), np.float32(1))), 0.5, 0.7]
            if (scene, fid) == EMPTY:
                scores = [0.2, 0.25, 0.1, 0.25, 0.05, 0.2]
            for k, (m, s) in enumerate(zip(masks, scores)):
                ys, xs = np.nonzero(m)
                dets.append({"scene_id": scene, "image_id": fid, "category_id": [1, 5, 1, 5, 1, 1][k],
                             "bbox": [int(xs.min()), int(ys.min()), int(xs.max() - xs.min()), int(ys.max() - ys.min())],
                             "score": s, "time": t, "segmentation": _rle(m)})
        files[f"{sdir}/scene_camera.json"] = json.dumps(cams).encode()
    rs.shuffle(dets)                                                  # images interleaved: grouping by first appearance
    return files, points, dets


def write_files(files, root):
    for rel, data in files.items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as fh:
            fh.write(data)


def _blob(data: bytes) -> torch.Tensor:
    return torch.frombuffer(bytearray(data), dtype=torch.uint8)


def _xz(a, delta: int = 0):
    """an array, losslessly: its dtype, shape and lzma-compressed bytes (with a byte-delta filter of distance `delta` first, for
    smooth interleaved images)"""
    a = np.ascontiguousarray(a)
    filters = ([{"id": lzma.FILTER_DELTA, "dist": delta}] if delta else []) + [{"id": lzma.FILTER_LZMA2, "preset": 9 | lzma.PRESET_EXTREME}]
    return {"dtype": a.dtype.str, "shape": a.shape, "data": _blob(lzma.compress(a.tobytes(), format=lzma.FORMAT_RAW, filters=filters)),
            "delta": delta}


def _pack(a):
    """float32 values, losslessly: the distinct values and the compressed index of each element"""
    a = np.asarray(a, dtype=np.float32)
    values, index = np.unique(a, return_inverse=True)
    assert len(values) <= 1 << 16
    return {"shape": a.shape, "values": torch.from_numpy(values), "index": _xz(index.astype(np.uint16).reshape(a.shape))}


def _crop_u8(rgb):
    """the reference's normalised crop (3,S,S) f32 -> the (S,S,3) u8 crop it was made from, checked to give it back through
    ToTensor + Normalize exactly as BOPTestset.transform does"""
    import torchvision.transforms as T
    mean, std = np.array([0.485, 0.456, 0.406])[:, None, None], np.array([0.229, 0.224, 0.225])[:, None, None]
    u8 = np.clip(np.round((rgb.astype(np.float64) * std + mean) * 255), 0, 255).astype(np.uint8).transpose(1, 2, 0)
    again = T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])(T.ToTensor()(u8.copy())).numpy()
    assert np.array_equal(again, rgb)
    return u8


def _stub_modules(points_by_path):
    from PIL import Image
    sys.path[:0] = [os.path.join(PEM, d) for d in ("provider", "utils", "model")] + [PEM]
    imageio = types.ModuleType("imageio")
    imageio.imread = lambda p: np.array(Image.open(p))
    sys.modules["imageio"] = imageio
    data_utils = importlib.import_module("data_utils")
    coco = types.ModuleType("pycocotools")
    mask = types.ModuleType("pycocotools.mask")

    def fr_py_objects(seg, h, w):
        raise TypeError("stub: keep the uncompressed RLE")
    mask.frPyObjects = fr_py_objects
    mask.decode = lambda rle: data_utils.rle_to_binary_mask(rle).astype(np.uint8)
    coco.mask = mask
    sys.modules["pycocotools"], sys.modules["pycocotools.mask"] = coco, mask
    trimesh = types.ModuleType("trimesh")

    class Mesh:
        def __init__(self, path):
            self.path = path

        def sample(self, n):
            return points_by_path[os.path.basename(self.path)][:n]
    trimesh.load_mesh = Mesh
    trimesh.Trimesh = Mesh
    sys.modules["trimesh"] = trimesh
    gorilla = types.ModuleType("gorilla")
    sys.modules["gorilla"] = gorilla


def _cfg(root):
    return types.SimpleNamespace(data_dir=root, template_dir=os.path.join(root, "BOP-Templates"), img_size=224, rgb_mask_flag=True,
                                 n_sample_observed_point=2048, n_sample_model_point=N_MODEL_POINTS, n_sample_template_point=5000,
                                 minimum_n_point=8, seg_filter_score=0.25, n_template_view=42, name="bop_test_dataset")


def model_points(points):
    """load_obj's model points: mesh.sample(n).astype(np.float32) / 1000.0"""
    return {o: p.astype(np.float32) / 1000.0 for o, p in points.items()}


def pem_instances(root, det_path, ds_points):
    """BOPTestset.__getitem__ of every image, with the sample indices of its np.random.choice calls"""
    from bop_test_dataset import BOPTestset
    ds = BOPTestset(_cfg(root), DATASET, det_path)
    calls, choice = [], np.random.choice

    def recording_choice(*a, **k):
        out = choice(*a, **k)
        calls.append(np.asarray(out))
        return out
    images = []
    np.random.seed(SEED)
    np.random.choice = recording_choice
    try:
        for i in range(len(ds)):
            dets = ds.dets[ds.det_keys[i]]
            calls.clear()
            try:
                item = ds[i]
            except IndexError:                                       # every detection of the image dropped: instances[0]
                images.append({"key": ds.det_keys[i], "empty": True})
                continue
            obj = item["obj"].reshape(-1)
            assert all(np.array_equal(ob.model_points, model_points({ob.obj_id: ds_points[ob.obj_id]})[ob.obj_id]) for ob in ds.objects)
            # the model rows are the object's model points (stored once, not per instance)
            assert all(torch.equal(item["model"][k], torch.from_numpy(ds.objects[int(o)].model_points)) for k, o in enumerate(obj))
            # pts and rgb_choose are rows of the filtered cloud and its crop indices taken at choose_idx: store those rows once
            ci = np.stack(calls)
            n = int(ci.max()) + 1
            cloud, rc = np.zeros((len(ci), n, 3), np.float32), np.zeros((len(ci), n), np.int32)
            pts, rgb_choose = item["pts"].numpy(), item["rgb_choose"].numpy()
            for k in range(len(ci)):
                cloud[k, ci[k]], rc[k, ci[k]] = pts[k], rgb_choose[k]
                assert np.array_equal(cloud[k, ci[k]], pts[k]) and np.array_equal(rc[k, ci[k]], rgb_choose[k])
            images.append({"key": ds.det_keys[i], "empty": False, "n_dets": len(dets), "choose_idx": _xz(ci.astype(np.int16)),
                           "cloud": _pack(cloud), "rgb_choose_rows": _xz(rc),
                           "rgb_u8": _xz(np.stack([_crop_u8(r) for r in item["rgb"].numpy()]), delta=3),
                           "obj": obj.tolist(), "obj_id": item["obj_id"].reshape(-1).tolist(), "score": item["score"].reshape(-1).tolist(),
                           "seg_time": float(item["seg_time"])})
    finally:
        np.random.choice = choice
    return images


def pem_rows(root, det_path):
    """test_bop.test() with a stub Net whose outputs are seeded draws (recorded), on the CPU: .cuda() is the identity"""
    cfg = types.SimpleNamespace(test_dataset=_cfg(root), test_dataloader=types.SimpleNamespace(bs=2, num_workers=0, shuffle=False,
                                                                                             drop_last=False, pin_memory=False))
    test_bop = importlib.import_module("test_bop")
    outputs = []
    gen = torch.Generator().manual_seed(SEED)

    class FeatureExtraction:
        def get_obj_feats(self, tem, pts, choose):
            return torch.zeros(len(tem[0]), 4, 3), torch.zeros(len(tem[0]), 4, 8)

    class Net:
        feature_extraction = FeatureExtraction()

        def eval(self):
            return self

        def __call__(self, inputs):
            b = inputs["pts"].shape[0]
            out = {"pred_R": torch.rand(b, 3, 3, generator=gen), "pred_t": torch.rand(b, 3, generator=gen) - 0.5,
                   "pred_pose_score": torch.rand(b, generator=gen)}
            outputs.append(out)
            return out
    saved_cuda, saved_sync = torch.Tensor.cuda, torch.cuda.synchronize
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.cuda.synchronize = lambda *a, **k: None
    out_csv = os.path.join(root, "result.csv")
    try:
        np.random.seed(SEED)
        test_bop.test(Net(), cfg, out_csv, DATASET, det_path)
    finally:
        torch.Tensor.cuda, torch.cuda.synchronize = saved_cuda, saved_sync
    return open(out_csv).read().splitlines(keepends=True), {k: torch.cat([o[k] for o in outputs]) for k in outputs[0]}


def ism_records(tmp):
    """Detections.save_to_file + convert_npz_to_json of synthetic detections, for lmo and ycbv"""
    import ref_ism_import as rii
    rii.import_reference_ism()
    from model.utils import Detections, convert_npz_to_json
    rs = np.random.RandomState(SEED)
    n = 5
    masks = np.zeros((n, H, W), np.float32)
    for i in range(n):
        masks[i] = _ellipse(rs.uniform(0, W), rs.uniform(0, H), rs.uniform(3, 20), rs.uniform(3, 20))
    masks[0, 0, 0] = 1.0                                            # a mask whose first pixel is set
    boxes = np.stack([np.concatenate([np.nonzero(m)[1][[0]], np.nonzero(m)[0][[0]], np.nonzero(m)[1][[0]] + 5,
                                      np.nonzero(m)[0][[0]] + 7]) for m in masks]).astype(np.int64)
    scores = rs.uniform(0.1, 0.9, n).astype(np.float32)
    object_ids = np.array([0, 3, 1, 7, 2], dtype=np.int64)
    out = {"masks": _xz(masks.astype(np.uint8)), "boxes": torch.from_numpy(boxes), "scores": torch.from_numpy(scores),
           "object_ids": torch.from_numpy(object_ids), "runtime": 0.123456789, "records": {}}
    for name in ("lmo", "ycbv"):
        det = Detections.__new__(Detections)
        det.boxes, det.scores, det.object_ids, det.masks = boxes, scores, object_ids, masks
        path = os.path.join(tmp, f"scene{name}_frame3")
        det.save_to_file(scene_id=48, frame_id=3, runtime=out["runtime"], file_path=path, dataset_name=name)
        out["records"][name] = convert_npz_to_json(0, [path + ".npz"])
    return out


def main():
    files, points, dets = make_split()
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "bop")
        write_files(files, root)
        det_path = os.path.join(tmp, "dets.json")
        json.dump(dets, open(det_path, "w"))
        _stub_modules({f"obj_{o:06d}.ply": p for o, p in points.items()})
        images = pem_instances(root, det_path, points)
        full = os.path.join(tmp, "dets_full.json")
        json.dump([d for d in dets if (d["scene_id"], d["image_id"]) != EMPTY], open(full, "w"))
        lines, stub_out = pem_rows(root, full)
        ism = ism_records(tmp)
    names = sorted(files)
    out = {"files": {"names": names, "sizes": [len(files[k]) for k in names],
                     "data": _xz(np.frombuffer(b"".join(files[k] for k in names), np.uint8))}, "dataset": DATASET, "obj_ids": OBJ_IDS, "seed": SEED,
           "model_points": {o: _pack(model_points(points)[o]) for o in OBJ_IDS},
           "detections": dets, "images": images, "csv_lines": lines, "stub_out": stub_out, "stub_bs": 2, "ism": ism}
    torch.save(out, OUT)
    print(f"wrote {OUT}: {len(files)} files, {len(images)} images, {sum(len(i.get('obj', [])) for i in images)} instances, "
          f"{len(lines)} csv lines, {os.path.getsize(OUT) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
