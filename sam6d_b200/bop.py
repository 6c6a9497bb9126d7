"""SAM-6D over a BOP test split: the host side of the reference's ISM/run_inference.py (BaseBOPTest, test_step, test_epoch_end)
and PEM/test_bop.py (BOPTestset, load_objs), for SAM6D.run_bop_ism / run_bop_pem (sam6d_b200/pipeline.py).

    frames = scan_test_split(root, "ycbv")                # ISM/provider/base_bop.py load_metaData (mode "query")
    objects = load_objects(root, "ycbv")                  # PEM/utils/bop_object_utils.py load_objs: ids, meshes, diameters
    rgb = round_trip(decode_rgb(frames[0].rgb_path))      # what test_step segments: inv_normalize(normalize(to_tensor(img)))
    groups = group_detections(json.load(open(path)))      # BOPTestset.__init__: per (scene_id, image_id), first appearance

Quirks kept on purpose: category ids in the ISM output are the object index + 1, except on lmo (ISM/model/utils.py:159-170);
the PEM's depth is np.float32(raw / 1000.0 * depth_scale), a float64 product rounded once; the PEM keeps a detection with score
> 0.25 whose mask AND depth > 0 has more than 8 pixels and at least 8 points within 0.6 x diameter of their centroid; CSV
fields are str() of numpy float32 values and the row time adds the float32-rounded ISM time of the image's first detection."""
import glob
import json
import os
from dataclasses import dataclass
from pathlib import Path
from typing import List, Optional

import numpy as np
import torch

from . import pbr

LMO_OBJECT_IDS = np.array([1, 5, 6, 8, 9, 10, 11, 12])      # ISM/model/utils.py: occlusion LINEMOD's ids
SEG_FILTER_SCORE = 0.25                                     # PEM/config/base.yaml test_dataset.seg_filter_score
MINIMUM_N_POINT = 8                                         # test_dataset.minimum_n_point
N_SAMPLE_MODEL_POINT = 1024                                 # test_dataset.n_sample_model_point
PEM_BATCH = 16                                              # test_dataloader.bs: Net.forward's chunk in test_bop.py
RADIUS_FACTOR = 0.6                                         # bop_test_dataset.py:134: |p - centroid| < diameter * 0.6
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def split_name(dataset_name: str) -> str:
    """ISM/run_inference.py:33-36: the test images of hb and tless are those of their primesense sensor"""
    return "test_primesense" if dataset_name in ("hb", "tless") else "test"


def model_dir(dataset_name: str) -> str:
    """bop_test_dataset.py:43-46: tless's CAD models are models_cad"""
    return "models_cad" if dataset_name == "tless" else "models"


# ---- the test split (BaseBOP.load_list_scene + load_metaData, BaseBOPTest.load_depth_img) ------------------------------------
@dataclass
class BopFrame:
    """one image of the test split: scene_id and frame_id as ints, the image and depth paths, cam_K (9 floats) and depth_scale
    of the scene's scene_camera.json"""
    scene_id: int
    frame_id: int
    rgb_path: str
    depth_path: str
    cam_K: list
    depth_scale: float


def depth_path_of(rgb_path: str) -> str:
    """BaseBOPTest.load_depth_img: depth/<frame>.png when the scene has it, else the image path with its rgb directory replaced
    by depth (gray by depth for gray images, itodd).  Only the image's own directory is replaced, not every "rgb" of the path."""
    scene, sub, name = os.path.dirname(os.path.dirname(rgb_path)), os.path.basename(os.path.dirname(rgb_path)), os.path.basename(rgb_path)
    png = os.path.join(scene, "depth", f"{int(name.split('.')[0]):06d}.png")
    if os.path.exists(png):
        return png
    return os.path.join(scene, "depth" if sub in ("rgb", "gray") else sub, name)


def scan_test_split(root: str, dataset_name: str, split: Optional[str] = None) -> List[BopFrame]:
    """the frames of root/dataset_name/<split> (split_name() by default): scenes sorted (pbr.list_scenes), in each the images
    rgb/*.[pj][pn]g, or gray/*.tif without rgb/, sorted; cam_K and depth_scale from the scene's scene_camera.json"""
    split = split_name(dataset_name) if split is None else split
    frames = []
    for scene in pbr.list_scenes(os.path.join(root, dataset_name), split):
        if os.path.exists(os.path.join(scene, "rgb")):
            paths = sorted(Path(scene).glob("rgb/*.[pj][pn]g"))
        else:
            paths = sorted(Path(scene).glob("gray/*.tif"))
        if not paths:
            raise FileNotFoundError(f"{scene} is empty: no rgb/*.[pj][pn]g nor gray/*.tif")
        with open(os.path.join(scene, "scene_camera.json")) as fh:
            camera = json.load(fh)
        for path in paths:
            frame_id = int(path.name.split(".")[0])
            cam = camera[f"{frame_id}"]
            frames.append(BopFrame(int(os.path.basename(scene)), frame_id, str(path), depth_path_of(str(path)), list(cam["cam_K"]),
                                    float(cam["depth_scale"])))
    return frames


def frame_paths(root: str, dataset_name: str, scene_id: int, image_id: int, split: Optional[str] = None):
    """the PEM's file reads of one image (data_utils.get_bop_image / get_bop_depth_map): the image is the first of
    rgb/<id>.jpg, rgb/<id>.png, gray/<id>.tif that exists, the depth depth/<id>.png or else depth/<id>.tif; cam_K and depth_scale
    from scene_camera.json -> (rgb path, depth path, cam_K, depth_scale)"""
    split = split_name(dataset_name) if split is None else split
    scene = os.path.join(root, dataset_name, split, f"{int(scene_id):06d}")
    rgb = next((os.path.join(scene, s) for s in (f"rgb/{image_id:06d}.jpg", f"rgb/{image_id:06d}.png", f"gray/{image_id:06d}.tif")
                if os.path.exists(os.path.join(scene, s))), None)
    if rgb is None:
        raise FileNotFoundError(f"{scene}: no image {image_id:06d} in rgb/ or gray/")
    depth = os.path.join(scene, "depth", f"{image_id:06d}.png")
    if not os.path.exists(depth):
        depth = os.path.join(scene, "depth", f"{image_id:06d}.tif")
    with open(os.path.join(scene, "scene_camera.json")) as fh:
        cam = json.load(fh)[str(image_id)]
    return rgb, depth, list(cam["cam_K"]), float(cam["depth_scale"])


# ---- objects (bop_object_utils.load_objs) -------------------------------------------------------------------------------------
@dataclass
class BopObjects:
    """the dataset's objects in load_objs' order: ids (sorted model ids), ply paths, diameters in metres (models_info / 1000)"""
    ids: List[int]
    ply_paths: List[str]
    diameters: np.ndarray

    def index(self, obj_id: int) -> int:
        """BOPTestset.obj_idxs: a category id of the detection file -> the object's position"""
        try:
            return self.ids.index(int(obj_id))
        except ValueError:
            raise ValueError(f"category_id {obj_id} is not among the dataset's objects {self.ids}") from None


def load_objects(root: str, dataset_name: str) -> BopObjects:
    """the objects of root/dataset_name/models (models_cad for tless): obj_*.ply sorted by id, diameter / 1000 from
    models_info.json"""
    folder = os.path.join(root, dataset_name, model_dir(dataset_name))
    paths = glob.glob(os.path.join(folder, "obj_*.ply"))
    if not paths:
        raise FileNotFoundError(f"no obj_*.ply in {folder}")
    ids = sorted(int(os.path.basename(p)[4:10]) for p in paths)
    with open(os.path.join(folder, "models_info.json")) as fh:
        info = json.load(fh)
    return BopObjects(ids, [os.path.join(folder, f"obj_{i:06d}.ply") for i in ids],
                      np.array([info[str(i)]["diameter"] / 1000.0 for i in ids], dtype=np.float64))


def category_ids(dataset_name: str, n_objects: int) -> List[int]:
    """Detections.save_to_file's category_id of object index 0..n-1: index + 1, or lmo_object_ids[index] on lmo"""
    if dataset_name == "lmo":
        if n_objects > len(LMO_OBJECT_IDS):
            raise ValueError(f"lmo has {len(LMO_OBJECT_IDS)} objects, got {n_objects}")
        return [int(i) for i in LMO_OBJECT_IDS[:n_objects]]
    return list(range(1, n_objects + 1))


def template_views(total_n_view: int, n_view: int = 42) -> List[int]:
    """Obj._get_template: the n_view template files int(total_n_view / n_view * v) of a directory holding total_n_view"""
    return [int(total_n_view / n_view * v) for v in range(n_view)]


def load_templates(template_dir: str, dataset_name: str, obj_id: int, n_view: int = 42):
    """BOP-Templates/<dataset>/obj_XXXXXX: the n_view template views picked by template_views -> (rgbs (H,W,3) u8, masks (H,W)
    u8 with 255 = object, xyzs (H,W,3) f32 in mm) as lists, for inputs.get_templates_from_arrays"""
    from PIL import Image
    path = os.path.join(template_dir, dataset_name, f"obj_{int(obj_id):06d}")
    total = len(glob.glob(os.path.join(path, "rgb_*.png")))
    if total == 0:
        raise FileNotFoundError(f"no template rgb_*.png in {path}")
    rgbs, masks, xyzs = [], [], []
    for i in template_views(total, n_view):
        rgbs.append(np.array(Image.open(os.path.join(path, f"rgb_{i}.png"))).astype(np.uint8)[..., :3])
        masks.append(np.array(Image.open(os.path.join(path, f"mask_{i}.png"))).astype(np.uint8))
        xyzs.append(np.load(os.path.join(path, f"xyz_{i}.npy")).astype(np.float32))
    return rgbs, masks, xyzs


# ---- the ISM's image (provider/bop.py rgb_transform, detector.py:338-344) ------------------------------------------------------
def round_trip_table() -> np.ndarray:
    """(3,256) u8: what test_step segments for byte value v of channel c, np.uint8(clip(inv_normalize(normalize(to_tensor)), 0, 1)
    * 255), with torchvision's float32 ops: ToTensor's v / 255, Normalize's sub_(mean).div_(std), the inverse Normalize with
    mean -m/s and std 1/s (float64 constants rounded to float32)"""
    x = torch.arange(256, dtype=torch.uint8).float().div(255).expand(3, 256).clone()
    mean = torch.tensor(IMAGENET_MEAN, dtype=torch.float32).view(-1, 1)
    std = torch.tensor(IMAGENET_STD, dtype=torch.float32).view(-1, 1)
    x.sub_(mean).div_(std)
    inv_mean = torch.tensor([-m / s for m, s in zip(IMAGENET_MEAN, IMAGENET_STD)], dtype=torch.float32).view(-1, 1)
    inv_std = torch.tensor([1 / s for s in IMAGENET_STD], dtype=torch.float32).view(-1, 1)
    x.sub_(inv_mean).div_(inv_std)
    return np.uint8(x.numpy().clip(0, 1) * 255)


_TABLE = None


def round_trip(rgb_u8: np.ndarray) -> np.ndarray:
    """(H,W,3) u8 -> the image test_step segments, through round_trip_table"""
    global _TABLE
    if _TABLE is None:
        _TABLE = round_trip_table()
    return _TABLE[np.arange(3), rgb_u8]


def decode_rgb(path: str) -> np.ndarray:
    """BaseBOPTest.__getitem__'s Image.open(path).convert("RGB") (gray images become three equal channels) -> (H,W,3) u8"""
    return pbr.decode_rgb(path)


def decode_depth(path: str) -> np.ndarray:
    """a depth image as stored (u16 PNG or TIFF) -> (H,W) array of raw values"""
    from PIL import Image
    with Image.open(path) as im:
        return np.array(im)


def decode_pem_image(path: str) -> np.ndarray:
    """get_bop_image's read: the image as loaded, gray stacked to three channels, [..., :3] -> (H,W,3) u8 (RGB; the crop
    kernel applies the reference's [..., ::-1])"""
    from PIL import Image
    with Image.open(path) as im:
        rgb = np.array(im).astype(np.uint8)
    if rgb.ndim == 2:
        rgb = np.stack([rgb] * 3, axis=2)
    return np.ascontiguousarray(rgb[..., :3])


def pem_depth(raw: np.ndarray, depth_scale: float) -> np.ndarray:
    """get_bop_depth_map(inst) * depth_scale then get_point_cloud_from_depth's astype: float64 raw / 1000.0 * depth_scale rounded
    once to float32 (metres).  The custom path's float32 raw * depth_scale / 1000.0 differs in the last bit for some values."""
    return np.float32(np.asarray(raw) / 1000.0 * depth_scale)


# ---- detections and rows (BOPTestset.__init__, test_bop.py:99-185) -------------------------------------------------------------
def group_detections(dets):
    """-> [((scene_id, image_id), [detections])] in order of the first appearance of each image, detections in file order"""
    groups = {}
    for d in dets:
        groups.setdefault((int(d["scene_id"]), int(d["image_id"])), []).append(d)
    return list(groups.items())


def pem_rand(generator: torch.Generator, n: int, n_rand: int, device, batch: int = PEM_BATCH) -> torch.Tensor:
    """the coarse stage's uniforms of n instances as test_bop.py draws them: torch.rand(chunk, n_rand) for every chunk of `batch`
    instances, from one generator that continues across images -> (n, n_rand) f32"""
    parts = [torch.rand(min(batch, n - s), n_rand, generator=generator, device=device) for s in range(0, n, batch)]
    return torch.cat(parts) if parts else torch.empty(0, n_rand, device=device)


def csv_rows(scene_id: int, image_id: int, obj_ids, scores: np.ndarray, R: np.ndarray, t_mm: np.ndarray, image_time: float) -> List[str]:
    """test_bop.py:166-176: one line per instance, scene_id,im_id,obj_id,score,R (9, space separated),t (3, mm),time; values
    as str() of the float32 numpy values"""
    R = np.asarray(R, dtype=np.float32).reshape(-1, 9)
    t_mm = np.asarray(t_mm, dtype=np.float32).reshape(-1, 3)
    scores = np.asarray(scores, dtype=np.float32)
    return [",".join((str(scene_id), str(image_id), str(int(obj_ids[k])), str(scores[k]), " ".join(str(v) for v in R[k]),
                      " ".join(str(v) for v in t_mm[k]), f"{image_time}\n")) for k in range(len(scores))]


def pem_instances(dets, image_u8: np.ndarray, depth_raw: np.ndarray, cam_K, depth_scale: float, objects: BopObjects,
                  model_points: np.ndarray, rng=None, choose_idx: Optional[np.ndarray] = None, n_sample: int = 2048, img_size: int = 224,
                  device=None, frame_rows: bool = False):
    """BOPTestset.__getitem__ / get_instance for the detections of one image, on the device (inputs.FrameInputs): the detections
    with score > 0.25; the mask is the RLE AND depth > 0 with pem_depth's depth; a detection is kept with more than 8 mask pixels
    and at least 8 points within diameter * 0.6 (float64) of their centroid; observed-point samples drawn from `rng` in
    detection order (or choose_idx (Q,n_sample)).  model_points (O,n,3) f32 in metres, O in objects' order.
    -> (dict of pts (Q,n_sample,3), rgb (Q,3,S,S) (BGR crop, as get_bop_image), rgb_choose (Q,n_sample) i64, model (Q,n,3),
    score (Q) f32, obj (Q) i64 object index; the kept detections; choose_idx), and with frame_rows=True a fourth item,
    inputs.FrameInputs.rows of the kept detections (the device depth and masks pose verification reads)"""
    from . import inputs
    sel = [d for d in dets if d["score"] > SEG_FILTER_SCORE]
    obj = np.array([objects.index(d["category_id"]) for d in sel], dtype=np.int64)
    thr = objects.diameters[obj] * RADIUS_FACTOR
    frame = inputs.FrameInputs(sel, image_u8, depth_raw, cam_K, depth_scale, None, device, depth_m=pem_depth(depth_raw, depth_scale),
                               thr=thr, min_count=MINIMUM_N_POINT)
    keep = frame.kept(MINIMUM_N_POINT, MINIMUM_N_POINT)
    if choose_idx is None:
        choose_idx = inputs.draw_choose_idx(frame.n_valid()[keep], n_sample, rng)
    pts, rgb_choose, rgb, _ = frame.sample(keep, np.asarray(choose_idx), img_size, True)
    dev = frame.device
    o = torch.from_numpy(obj[keep]).to(dev)
    data = dict(pts=pts, rgb=rgb, rgb_choose=rgb_choose, model=torch.from_numpy(np.asarray(model_points, dtype=np.float32)).to(dev)[o],
                score=torch.tensor([sel[i]["score"] for i in keep], dtype=torch.float32, device=dev), obj=o)
    if frame_rows:
        return data, [sel[i] for i in keep], np.asarray(choose_idx), frame.rows(keep)
    return data, [sel[i] for i in keep], np.asarray(choose_idx)
