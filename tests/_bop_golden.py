"""tests/golden/bop_test.pt as tools/make_golden_bop_test.py stores it: lzma-compressed arrays, point clouds as distinct values
plus an index, and the u8 crops behind the reference's normalised crops."""
import lzma
import os

import numpy as np
import torch


def load(golden_dir):
    return torch.load(os.path.join(golden_dir, "bop_test.pt"), weights_only=False)


def unxz(p) -> np.ndarray:
    filters = ([{"id": lzma.FILTER_DELTA, "dist": p["delta"]}] if p["delta"] else []) + [{"id": lzma.FILTER_LZMA2}]
    data = lzma.decompress(p["data"].numpy().tobytes(), format=lzma.FORMAT_RAW, filters=filters)
    return np.frombuffer(data, dtype=np.dtype(p["dtype"])).reshape(p["shape"])


def unpack(p) -> torch.Tensor:
    """a float32 array stored as its distinct values and an index"""
    return torch.from_numpy(p["values"].numpy()[unxz(p["index"]).astype(np.int64)].reshape(p["shape"]))


def write_split(gold, root):
    """the synthetic split's files under root"""
    f = gold["files"]
    data, pos = unxz(f["data"]).tobytes(), 0
    for rel, n in zip(f["names"], f["sizes"]):
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as fh:
            fh.write(data[pos:pos + n])
        pos += n
    return str(root)


def instance(im):
    """one image's instances as BOPTestset.__getitem__ returned them: pts and rgb_choose (the stored rows of the filtered cloud
    and its crop indices, taken at the sample indices), rgb (ToTensor + Normalize of the stored u8 crops, as the reference's
    transform computes it), obj, obj_id, score (float32); and the sample indices its np.random.choice calls returned"""
    import torchvision.transforms as T
    tf = T.Compose([T.ToTensor(), T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])])
    rgb = torch.stack([tf(np.array(u8)) for u8 in unxz(im["rgb_u8"])])
    ci = unxz(im["choose_idx"]).astype(np.int64)
    cloud, rows = unpack(im["cloud"]).numpy(), unxz(im["rgb_choose_rows"]).astype(np.int64)
    q = np.arange(len(ci))[:, None]
    return dict(pts=torch.from_numpy(cloud[q, ci]), rgb=rgb, rgb_choose=torch.from_numpy(rows[q, ci]), choose_idx=ci,
                obj=torch.tensor(im["obj"], dtype=torch.int64), obj_id=torch.tensor(im["obj_id"], dtype=torch.int32),
                score=torch.tensor(im["score"], dtype=torch.float32))
