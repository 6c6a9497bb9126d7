"""Synthetic workloads for tests and bench.py: seeded weights under the reference's parameter names and inputs of the BASELINE
shapes (SURVEY.md 8d).  There is no network for checkpoints or datasets, so every measured or tested run uses these generators;
they are data, not algorithm -- the CPU restatements of the reference live in oracle/ and are imported by tests, smoke() and the
CPU legs of bench.py only."""
import math
from typing import Dict

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]
FINE_NPOINT = 2048
N_PROPOSAL1 = 6000       # PEM/config/base.yaml: coarse_point_matching.nproposal1 (hypotheses drawn per proposal)


# --------------------------------------------------------------------------------------
# seeded weights with the reference's state_dict layout (SURVEY.md Appendix A)
# --------------------------------------------------------------------------------------
def _init_linear(sd: SD, name: str, out_f: int, in_f: int, g: torch.Generator, bias: bool = True):
    bound = 1.0 / math.sqrt(in_f)
    sd[name + ".weight"] = (torch.rand(out_f, in_f, generator=g) * 2 - 1) * bound
    if bias:
        sd[name + ".bias"] = (torch.rand(out_f, generator=g) * 2 - 1) * bound


def _init_ln(sd: SD, name: str, c: int, g: torch.Generator):
    sd[name + ".weight"] = 1.0 + 0.1 * torch.randn(c, generator=g)
    sd[name + ".bias"] = 0.1 * torch.randn(c, generator=g)


def _init_geo_transformer(sd: SD, p: str, c: int, g: torch.Generator):
    for li, kinds in ((0, "qkvp"), (1, "qkv")):
        a = f"{p}.layers.{li}.attention"
        for kch in kinds:
            _init_linear(sd, f"{a}.attention.proj_{kch}", c, c, g)
        _init_linear(sd, a + ".linear", c, c, g)
        _init_ln(sd, a + ".norm", c, g)
        o = f"{p}.layers.{li}.output"
        _init_linear(sd, o + ".expand", 2 * c, c, g)
        _init_linear(sd, o + ".squeeze", c, 2 * c, g)
        _init_ln(sd, o + ".norm", c, g)


def make_pem_state_dict(seed: int = 1, c: int = 256, nblock: int = 3) -> SD:
    """Seeded random weights under the reference's parameter names (matching path only).
    BatchNorm running statistics and LayerNorm affine terms are randomised so that folding
    and affine paths are exercised (freshly constructed reference modules would hide them)."""
    g = torch.Generator().manual_seed(seed)
    sd: SD = {}
    sd["geo_embedding.embedding.div_term"] = torch.exp(torch.arange(0, c, 2).float() * (-math.log(10000.0) / c))
    _init_linear(sd, "geo_embedding.proj_d", c, c, g)
    _init_linear(sd, "geo_embedding.proj_a", c, c, g)
    for stage in ("coarse_point_matching", "fine_point_matching"):
        _init_linear(sd, stage + ".in_proj", c, c, g)
        _init_linear(sd, stage + ".out_proj", c, c, g)
        sd[stage + ".bg_token"] = torch.randn(1, 1, c, generator=g) * 0.02
    for i in range(nblock):
        _init_geo_transformer(sd, f"coarse_point_matching.transformers.{i}", c, g)
        t = f"fine_point_matching.transformers.{i}"
        _init_geo_transformer(sd, t + ".sparse_layer", c, g)
        a = t + ".dense_layer.attention"
        for kch in "qkv":
            _init_linear(sd, f"{a}.attention.proj_{kch}", c, c, g)
        sd[a + ".attention.scale"] = 0.2 * torch.randn(1, 1, c, generator=g)
        _init_linear(sd, a + ".linear", c, c, g)
        _init_ln(sd, a + ".norm", c, g)
        o = t + ".dense_layer.output"
        _init_linear(sd, o + ".expand", 2 * c, c, g)
        _init_linear(sd, o + ".squeeze", c, 2 * c, g)
        _init_ln(sd, o + ".norm", c, g)
    pe = "fine_point_matching.PE"
    for m in ("mlp1", "mlp2"):
        dims = [6, 32, 64, 128]
        for j in range(3):
            lp = f"{pe}.{m}.layer{j}"
            sd[lp + ".conv.weight"] = torch.randn(dims[j + 1], dims[j], 1, 1, generator=g) * math.sqrt(2.0 / dims[j])
            sd[lp + ".normlayer.bn.weight"] = 1.0 + 0.1 * torch.randn(dims[j + 1], generator=g)
            sd[lp + ".normlayer.bn.bias"] = 0.1 * torch.randn(dims[j + 1], generator=g)
            sd[lp + ".normlayer.bn.running_mean"] = 0.1 * torch.randn(dims[j + 1], generator=g)
            sd[lp + ".normlayer.bn.running_var"] = 0.5 + torch.rand(dims[j + 1], generator=g)
            sd[lp + ".normlayer.bn.num_batches_tracked"] = torch.tensor(1)
    sd[pe + ".mlp3.conv.weight"] = torch.randn(c, c, 1, generator=g) * math.sqrt(2.0 / c)
    sd[pe + ".mlp3.conv.bias"] = 0.1 * torch.randn(c, generator=g)
    return sd


# --------------------------------------------------------------------------------------
# synthetic proposals of the named shapes (SURVEY.md 8d, config #2)
# --------------------------------------------------------------------------------------
def random_rotation(B: int, g: torch.Generator) -> torch.Tensor:
    q = torch.randn(B, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    return torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], dim=1).view(B, 3, 3)


def make_pem_inputs(B: int = 2, n: int = FINE_NPOINT, c: int = 256, n_model: int = 1024, seed: int = 1):
    """Synthetic RGB-D+CAD proposal batch: a blob-shaped CAD template cloud, an observed cloud that
    is the template under a random rigid pose + 1 mm noise + 20% outliers, features correlated
    through the ground-truth correspondence."""
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(B, n + n_model, 3, generator=g)
    d = d / d.norm(dim=2, keepdim=True)
    bump = 1.0 + 0.3 * torch.sin(3.0 * d[..., 0:1]) * torch.cos(2.0 * d[..., 1:2]) + 0.2 * d[..., 2:3]
    axes = 0.6 + 0.4 * torch.rand(B, 1, 3, generator=g)
    size = 0.05 + 0.10 * torch.rand(B, 1, 1, generator=g)
    surf = d * bump * axes * size
    dense_po, model = surf[:, :n].contiguous(), surf[:, n:].contiguous()
    R = random_rotation(B, g)
    t = (torch.rand(B, 3, generator=g) * 0.2 - 0.1) + torch.tensor([0.0, 0.0, 0.8])
    perm = torch.stack([torch.randperm(n, generator=g) for _ in range(B)])
    src = torch.gather(dense_po, 1, perm.unsqueeze(2).expand(B, n, 3))
    pts = src @ R.transpose(1, 2) + t.unsqueeze(1) + 0.001 * torch.randn(B, n, 3, generator=g)
    n_out = n // 5
    pts[:, :n_out] = pts[:, :n_out] + 0.05 * torch.randn(B, n_out, 3, generator=g)
    latent = torch.randn(B, n, c, generator=g)
    dense_fo = latent + 0.5 * torch.randn(B, n, c, generator=g)
    dense_fm = torch.gather(latent, 1, perm.unsqueeze(2).expand(B, n, c)) + 0.5 * torch.randn(B, n, c, generator=g)
    return dict(pts=pts.contiguous(), dense_fm=dense_fm.contiguous(), dense_po=dense_po, dense_fo=dense_fo.contiguous(),
                model=model, gt_R=R, gt_t=t)


# --------------------------------------------------------------------------------------
# SAM ViT-H image encoder (ISM), template descriptors, PEM RGB branch
# --------------------------------------------------------------------------------------
def make_sam_state_dict(embed_dim=1280, depth=2, num_heads=16, global_attn_indexes=(1,), img_size=1024, patch=16, window=14,
                    out_chans=256, seed=1) -> SD:
    """seeded weights under the reference's names; rel-pos tables are NOT zero (the reference zero-inits them, which would
    hide the bias path)"""
    g = torch.Generator().manual_seed(seed)
    hd = embed_dim // num_heads
    grid = img_size // patch

    def lin(name, o, i, bias=True, scale=None):
        s = scale if scale is not None else 1.0 / math.sqrt(i)
        sd[name + ".weight"] = torch.randn(o, i, generator=g) * s
        if bias:
            sd[name + ".bias"] = torch.randn(o, generator=g) * 0.02

    sd: SD = {}
    sd["patch_embed.proj.weight"] = torch.randn(embed_dim, 3, patch, patch, generator=g) / math.sqrt(3 * patch * patch)
    sd["patch_embed.proj.bias"] = torch.randn(embed_dim, generator=g) * 0.02
    sd["pos_embed"] = torch.randn(1, grid, grid, embed_dim, generator=g) * 0.02
    for i in range(depth):
        p = f"blocks.{i}"
        size = grid if i in global_attn_indexes else window
        for n in ("norm1", "norm2"):
            sd[f"{p}.{n}.weight"] = 1.0 + 0.1 * torch.randn(embed_dim, generator=g)
            sd[f"{p}.{n}.bias"] = 0.1 * torch.randn(embed_dim, generator=g)
        lin(p + ".attn.qkv", 3 * embed_dim, embed_dim)
        lin(p + ".attn.proj", embed_dim, embed_dim)
        sd[p + ".attn.rel_pos_h"] = torch.randn(2 * size - 1, hd, generator=g) * 0.05
        sd[p + ".attn.rel_pos_w"] = torch.randn(2 * size - 1, hd, generator=g) * 0.05
        lin(p + ".mlp.lin1", 4 * embed_dim, embed_dim)
        lin(p + ".mlp.lin2", embed_dim, 4 * embed_dim)
    sd["neck.0.weight"] = torch.randn(out_chans, embed_dim, 1, 1, generator=g) / math.sqrt(embed_dim)
    sd["neck.1.weight"] = 1.0 + 0.1 * torch.randn(out_chans, generator=g)
    sd["neck.1.bias"] = 0.1 * torch.randn(out_chans, generator=g)
    sd["neck.2.weight"] = torch.randn(out_chans, out_chans, 3, 3, generator=g) / math.sqrt(9 * out_chans)
    sd["neck.3.weight"] = 1.0 + 0.1 * torch.randn(out_chans, generator=g)
    sd["neck.3.bias"] = 0.1 * torch.randn(out_chans, generator=g)
    return sd


def make_images(B=1, size=1024, seed=1) -> torch.Tensor:
    """Sam.preprocess-like input: normalised uint8 noise with smooth structure, padded region zero (frames are 640x480 ->
    1024x768 -> pad to 1024^2, ISM/segment_anything/modeling/sam.py:164-174)"""
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (B, 3, size * 3 // 4, size), generator=g).float()
    mean = torch.tensor([123.675, 116.28, 103.53]).view(1, 3, 1, 1)
    std = torch.tensor([58.395, 57.12, 57.375]).view(1, 3, 1, 1)
    img = (img - mean) / std
    return F.pad(img, (0, 0, 0, size - img.shape[2])).contiguous()


def make_descriptors(P=64, O=8, T=42, C=1024, seed=1):
    """queries with planted matches: proposal p looks like template (p % T) of object (p % O), plus clutter proposals"""
    g = torch.Generator().manual_seed(seed)
    ref = torch.randn(O, T, C, generator=g)
    obj_mean = torch.randn(O, 1, C, generator=g)
    ref = ref + 1.5 * obj_mean
    q = torch.empty(P, C)
    for p in range(P):
        if p % 5 == 4:
            q[p] = torch.randn(C, generator=g)                     # clutter: should fall under the threshold
        else:
            q[p] = ref[p % O, (3 * p) % T] + 0.6 * torch.randn(C, generator=g)
    return q, ref


def make_vit_state_dict(embed_dim=768, depth=12, out_dim=256, n_patches=196, num_classes=1000, seed=1, prefix="rgb_net.") -> SD:
    g = torch.Generator().manual_seed(seed)
    sd: SD = {}
    v = prefix + "vit."

    def lin(name, o, i, scale=None):
        s = scale if scale is not None else 1.0 / math.sqrt(i)
        sd[name + ".weight"] = (torch.rand(o, i, generator=g) * 2 - 1) * s
        sd[name + ".bias"] = (torch.rand(o, generator=g) * 2 - 1) * s

    def ln(name, c):
        sd[name + ".weight"] = 1.0 + 0.1 * torch.randn(c, generator=g)
        sd[name + ".bias"] = 0.1 * torch.randn(c, generator=g)

    sd[v + "cls_token"] = torch.randn(1, 1, embed_dim, generator=g) * 0.02
    sd[v + "pos_embed"] = torch.randn(1, n_patches + 1, embed_dim, generator=g) * 0.02
    sd[v + "patch_embed.proj.weight"] = (torch.rand(embed_dim, 3, 16, 16, generator=g) * 2 - 1) / math.sqrt(768)
    sd[v + "patch_embed.proj.bias"] = (torch.rand(embed_dim, generator=g) * 2 - 1) / math.sqrt(768)
    for i in range(depth):
        b = f"{v}blocks.{i}."
        ln(b + "norm1", embed_dim)
        lin(b + "attn.qkv", 3 * embed_dim, embed_dim)
        lin(b + "attn.proj", embed_dim, embed_dim)
        ln(b + "norm2", embed_dim)
        lin(b + "mlp.fc1", 4 * embed_dim, embed_dim)
        lin(b + "mlp.fc2", embed_dim, 4 * embed_dim)
    ln(v + "norm", embed_dim)
    if num_classes:
        lin(v + "head", num_classes, embed_dim)
    lin(prefix + "output_upscaling", 16 * out_dim, 4 * embed_dim)
    return sd


def make_dinov2_state_dict(embed_dim=1024, depth=24, num_heads=16, patch=14, img_size=518, seed=1, ffn_layer="mlp") -> SD:
    """seeded weights under the names of `dinov2_vit{s,b,l,g}14_pretrain.pth` (DinoVisionTransformer, ISM/model/vision_transformer.py):
    linear weights ~ trunc-normal-like N(0, 0.02) as the reference initialises them, but NON-trivial biases, LayerNorm affines and
    LayerScale gammas (the reference's zero / one initial values would hide those code paths).  ffn_layer "mlp" (fc1 / fc2) or
    "swiglufused" (w12 / w3, hidden (int(4C * 2/3) + 7) // 8 * 8, ISM/model/layers/swiglu_ffn.py:45-63); the defaults draw the
    ViT-L/14 tensors of tests/golden/dinov2.pt."""
    g = torch.Generator().manual_seed(seed)
    C = embed_dim
    n = (img_size // patch) ** 2
    sd: SD = {}
    sd["cls_token"] = torch.randn(1, 1, C, generator=g) * 0.02
    sd["pos_embed"] = torch.randn(1, n + 1, C, generator=g) * 0.02
    sd["mask_token"] = torch.zeros(1, C)
    sd["patch_embed.proj.weight"] = torch.randn(C, 3, patch, patch, generator=g) * 0.02
    sd["patch_embed.proj.bias"] = torch.randn(C, generator=g) * 0.02

    def lin(name, o, i):
        sd[name + ".weight"] = torch.randn(o, i, generator=g) * 0.02
        sd[name + ".bias"] = torch.randn(o, generator=g) * 0.02

    def ln(name):
        sd[name + ".weight"] = 1.0 + 0.1 * torch.randn(C, generator=g)
        sd[name + ".bias"] = 0.05 * torch.randn(C, generator=g)

    for i in range(depth):
        p = f"blocks.{i}."
        ln(p + "norm1")
        lin(p + "attn.qkv", 3 * C, C)
        lin(p + "attn.proj", C, C)
        sd[p + "ls1.gamma"] = 0.5 + torch.rand(C, generator=g)
        ln(p + "norm2")
        if ffn_layer == "swiglufused":
            hid = (int(4 * C * 2 / 3) + 7) // 8 * 8
            lin(p + "mlp.w12", 2 * hid, C)
            lin(p + "mlp.w3", C, hid)
        else:
            lin(p + "mlp.fc1", 4 * C, C)
            lin(p + "mlp.fc2", C, 4 * C)
        sd[p + "ls2.gamma"] = 0.5 + torch.rand(C, generator=g)
    ln("norm")
    return sd


def make_proposals(P=6, H=480, W=640, seed=1):
    """a synthetic frame with P mask proposals: image (H,W,3) uint8, masks (P,H,W) float32 0/1 (ellipses, boxes with holes, a
    border-clipped one, an exactly square one), boxes (P,4) int64 xyxy = tight bounds of each mask (Detections convention)"""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    base = (torch.sin(xx / 23.0) + torch.cos(yy / 17.0) + 0.002 * (xx + yy)).unsqueeze(-1)
    image = ((base * torch.tensor([40.0, 55.0, 35.0]) + 110 + 25 * torch.randn(H, W, 3, generator=g)).clamp(0, 255)).to(torch.uint8)
    masks = torch.zeros(P, H, W)
    for p in range(P):
        cy, cx = int(torch.randint(60, H - 60, (1,), generator=g)), int(torch.randint(60, W - 60, (1,), generator=g))
        ry, rx = int(torch.randint(12, 110, (1,), generator=g)), int(torch.randint(12, 110, (1,), generator=g))
        kind = p % 4
        if kind == 0:
            m = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1.0
        elif kind == 1:
            m = ((yy - cy).abs() < ry) & ((xx - cx).abs() < rx) & ~(((yy - cy).abs() < ry // 3) & ((xx - cx).abs() < rx // 3))
        elif kind == 2:
            m = (yy > H - 2 * ry) & (xx > W - 2 * rx)                      # clipped at the image border
        else:
            m = ((yy - cy).abs() < ry) & ((xx - cx).abs() < ry)            # square box
        masks[p] = m.float()
    boxes = torch.zeros(P, 4, dtype=torch.int64)
    for p in range(P):
        ys, xs = torch.nonzero(masks[p] > 0, as_tuple=True)
        boxes[p] = torch.tensor([xs.min(), ys.min(), xs.max(), ys.max()])
    return image, masks, boxes


def make_sam_decoder_state_dict(seed=1) -> SD:
    """seeded weights under the names of `sam_vit_h_4b8939.pth` for `prompt_encoder.*` and `mask_decoder.*`
    (ISM/segment_anything/modeling/{prompt_encoder,mask_decoder,transformer}.py).  Scales are chosen so that the automatic mask
    generator's filters (predicted IoU > 0.88, stability >= 0.95) keep a useful share of the masks with random weights: the IoU
    head's last bias is ~0.9 and the mask logits are a few units large."""
    g = torch.Generator().manual_seed(seed)
    sd: SD = {}

    def lin(name, o, i, scale=None, bias_scale=0.02):
        s = scale if scale is not None else 1.0 / math.sqrt(i)
        sd[name + ".weight"] = torch.randn(o, i, generator=g) * s
        sd[name + ".bias"] = torch.randn(o, generator=g) * bias_scale

    def ln(name, c):
        sd[name + ".weight"] = 1.0 + 0.1 * torch.randn(c, generator=g)
        sd[name + ".bias"] = 0.05 * torch.randn(c, generator=g)

    p = "prompt_encoder."
    sd[p + "pe_layer.positional_encoding_gaussian_matrix"] = torch.randn(2, 128, generator=g)
    for i in range(4):
        sd[p + f"point_embeddings.{i}.weight"] = torch.randn(1, 256, generator=g) * 0.5
    sd[p + "not_a_point_embed.weight"] = torch.randn(1, 256, generator=g) * 0.5
    sd[p + "mask_downscaling.0.weight"] = torch.randn(4, 1, 2, 2, generator=g) * 0.5
    sd[p + "mask_downscaling.0.bias"] = torch.randn(4, generator=g) * 0.02
    ln(p + "mask_downscaling.1", 4)
    sd[p + "mask_downscaling.3.weight"] = torch.randn(16, 4, 2, 2, generator=g) * 0.25
    sd[p + "mask_downscaling.3.bias"] = torch.randn(16, generator=g) * 0.02
    ln(p + "mask_downscaling.4", 16)
    sd[p + "mask_downscaling.6.weight"] = torch.randn(256, 16, 1, 1, generator=g) * 0.25
    sd[p + "mask_downscaling.6.bias"] = torch.randn(256, generator=g) * 0.02
    sd[p + "no_mask_embed.weight"] = torch.randn(1, 256, generator=g) * 0.5
    m = "mask_decoder."
    t = m + "transformer."

    def attn(name, internal):
        for q in ("q_proj", "k_proj", "v_proj"):
            lin(f"{name}.{q}", internal, 256)
        lin(f"{name}.out_proj", 256, internal)

    for i in range(2):
        l = t + f"layers.{i}."
        attn(l + "self_attn", 256)
        ln(l + "norm1", 256)
        attn(l + "cross_attn_token_to_image", 128)
        ln(l + "norm2", 256)
        lin(l + "mlp.lin1", 2048, 256)
        lin(l + "mlp.lin2", 256, 2048)
        ln(l + "norm3", 256)
        ln(l + "norm4", 256)
        attn(l + "cross_attn_image_to_token", 128)
    attn(t + "final_attn_token_to_image", 128)
    ln(t + "norm_final_attn", 256)
    sd[m + "iou_token.weight"] = torch.randn(1, 256, generator=g) * 0.5
    sd[m + "mask_tokens.weight"] = torch.randn(4, 256, generator=g) * 0.5
    sd[m + "output_upscaling.0.weight"] = torch.randn(256, 64, 2, 2, generator=g) / 16.0
    sd[m + "output_upscaling.0.bias"] = torch.randn(64, generator=g) * 0.02
    ln(m + "output_upscaling.1", 64)
    sd[m + "output_upscaling.3.weight"] = torch.randn(64, 32, 2, 2, generator=g) / 8.0
    sd[m + "output_upscaling.3.bias"] = torch.randn(32, generator=g) * 0.02
    for i in range(4):
        h = m + f"output_hypernetworks_mlps.{i}.layers."
        lin(h + "0", 256, 256)
        lin(h + "1", 256, 256)
        lin(h + "2", 32, 256, scale=40.0 / 16.0)
    h = m + "iou_prediction_head.layers."
    lin(h + "0", 256, 256)
    lin(h + "1", 256, 256)
    lin(h + "2", 4, 256, scale=0.05 / 16.0)
    sd[h + "2.bias"] = torch.tensor([0.9, 0.9, 0.9, 0.9]) + 0.03 * torch.randn(4, generator=g)
    return sd


def make_image_embedding(seed=1, size=64) -> torch.Tensor:
    """a smooth synthetic (1,256,size,size) image embedding: blobs of different feature directions (so that point prompts in
    different places see different neighbourhoods) plus noise"""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, size), torch.linspace(0, 1, size), indexing="ij")
    emb = 0.3 * torch.randn(256, size, size, generator=g)
    for _ in range(12):
        cy, cx, r = torch.rand(3, generator=g).tolist()
        d = torch.randn(256, generator=g)
        blob = torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * (0.05 + 0.15 * r) ** 2))
        emb += d[:, None, None] * blob[None]
    return emb.unsqueeze(0)


# the heads' last layers in make_fastsam_state_dict: scales of the DFL (cv2), class (cv3) and coefficient (cv4) weights, the
# coefficient bias, and the class bias of each level.  At s the class features of a level vary little around a level-dependent
# mean, so the class weights are scaled up and each level's bias centres its logits near -2.5.
_FASTSAM_HEAD_SCALES = {"x": (20.0, 35.0, 300.0, 0.065, (0.0, 0.0, 0.0)), "s": (20.0, 140.0, 200.0, 20.0, (-19.8, 13.0, 13.6))}


def make_fastsam_state_dict(seed: int = 1, scale: str = "x") -> SD:
    """Seeded YOLOv8{scale}-seg (nc=1) weights under ultralytics' keys (the layout of FastSAM-x.pt / FastSAM-s.pt; the x draw
    is the one this function made before it took a scale).  Convolutions are drawn at
    1/sqrt(fan_in) and BatchNorm statistics are randomised, so activations stay O(1) through the 23 layers and folding is
    exercised.  The heads' last layers are scaled so decoded boxes vary, masks are crisp (few pixels near the 0.5 threshold) and,
    on the test frames, several hundred anchors pass conf 0.25 and more than max_det = 200 survive NMS, so the max_det cut is
    exercised."""
    from .fast_sam import YOLOv8Seg
    g = torch.Generator().manual_seed(seed)
    sd: SD = {}
    for k, v in YOLOv8Seg(scale).state_dict().items():
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.zeros((), dtype=torch.long)
        elif k.endswith("dfl.conv.weight"):
            sd[k] = torch.arange(16, dtype=torch.float32).view(1, 16, 1, 1)
        elif k.endswith("bn.weight"):
            sd[k] = 0.8 + 0.4 * torch.rand(v.shape, generator=g)
        elif k.endswith("bn.bias") or k.endswith("bn.running_mean"):
            sd[k] = 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith("bn.running_var"):
            sd[k] = 0.5 + torch.rand(v.shape, generator=g)
        elif k.endswith("weight"):
            fan_in = v.shape[0] * v.shape[2] * v.shape[3] if "upsample" in k else v[0].numel()
            sd[k] = torch.randn(v.shape, generator=g) * (1.25 if k.endswith("conv.weight") else 1.0) / math.sqrt(fan_in)
        else:
            sd[k] = 0.05 * torch.randn(v.shape, generator=g)
    # the heads' last 1x1 convolutions: zero-sum rows (the SiLU features have a positive mean, which would otherwise give every
    # anchor the same offset), scaled so DFL logits have std ~2.4 and class logits ~N(-2.5, 1.5) (~18 % of anchors pass 0.25);
    # the mask coefficients are scaled and biased so that coeffs . proto is ~0 on average over anchors with std ~1.6 within a mask
    s_box, s_cls, s_mc, b_mc, b_cls = _FASTSAM_HEAD_SCALES[scale]
    for i in range(3):
        for name, f in (("cv2", s_box), ("cv3", s_cls), ("cv4", s_mc)):
            w = sd[f"model.22.{name}.{i}.2.weight"]
            sd[f"model.22.{name}.{i}.2.weight"] = (w - w.mean(dim=1, keepdim=True)) * f
        sd[f"model.22.cv3.{i}.2.bias"].fill_(b_cls[i])
        sd[f"model.22.cv4.{i}.2.bias"].fill_(b_mc)
    return sd


def make_fastsam_frame(H: int = 480, W: int = 640, seed: int = 0):
    """(H,W,3) uint8 RGB test frame: smooth background and a few filled rectangles and discs"""
    import numpy as np
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    img = np.stack([80 + 60 * np.sin(xx / (37 + 11 * c) + c) * np.cos(yy / (53 - 7 * c)) for c in range(3)], -1)
    for _ in range(12):
        col = rs.randint(0, 256, 3)
        y0, x0 = rs.randint(0, H - 20), rs.randint(0, W - 20)
        if rs.rand() < 0.5:
            img[y0:y0 + rs.randint(20, H // 3), x0:x0 + rs.randint(20, W // 3)] = col
        else:
            r = rs.randint(10, min(H, W) // 5)
            img[(yy - y0) ** 2 + (xx - x0) ** 2 < r * r] = col
    img += rs.randn(H, W, 3) * 8
    return np.clip(img, 0, 255).astype(np.uint8)
