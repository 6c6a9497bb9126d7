"""numpy / torch-CPU restatement of BOPTemplatePBR.__getitem__ for one reference (ISM/provider/bop_pbr.py), and the synthetic
BOP split of tests/golden/ism_pbr.pt written back to a directory"""
import os
import lzma

import numpy as np
import torch

from oracle.dinov2_oracle import crop_resize_pad

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def composite(rgb_u8: np.ndarray, mask_u8: np.ndarray) -> np.ndarray:
    """Image.composite(rgb, black, mask) with an L mask: PIL's paste blends as DIV255(rgb * mask), rounded to nearest"""
    t = rgb_u8.astype(np.uint32) * mask_u8.astype(np.uint32)[..., None] + 128
    return ((t + (t >> 8)) >> 8).astype(np.uint8)


def getbbox(mask_u8: np.ndarray):
    """Image.getbbox: the box of the nonzero pixels, exclusive max; None when there are none"""
    ys, xs = np.nonzero(mask_u8)
    return None if len(xs) == 0 else (int(xs.min()), int(ys.min()), int(xs.max()) + 1, int(ys.max()) + 1)


def reference_crop(rgb_u8: np.ndarray, mask_u8: np.ndarray, target: int = 224):
    """-> (box (4,) int, templates (3,T,T) f32, template_masks (T,T) f32) as __getitem__ builds them for one reference"""
    box = getbbox(mask_u8)
    image = torch.from_numpy(composite(rgb_u8, mask_u8) / 255).float().permute(2, 0, 1)
    mask = torch.from_numpy(mask_u8 / 255).float()
    b = torch.tensor([box])
    rgb = crop_resize_pad(image[None], b, target)[0]
    m = crop_resize_pad(mask[None, None], b, target)[0, 0]
    rgb = (rgb - torch.tensor(MEAN, dtype=torch.float32).view(3, 1, 1)) / torch.tensor(STD, dtype=torch.float32).view(3, 1, 1)
    return np.array(box), rgb, m


def unpack(rec) -> torch.Tensor:
    """a stored crop: its distinct values gathered by the uint16 index of every element"""
    index = np.frombuffer(lzma.decompress(rec["index"].numpy().tobytes()), dtype=np.uint16)
    return rec["values"][torch.from_numpy(index.astype(np.int64))].reshape(rec["shape"])


def write_split(files, root):
    """the golden's {relative path: file bytes as a uint8 tensor} -> files under root (the BOP dataset directory)"""
    for rel, data in files.items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as fh:
            fh.write(data.numpy().tobytes())
    return root
