"""oracle/sam_predictor_oracle.py -- TEST INFRASTRUCTURE ONLY.

CPU restatement (torch fp32) of the prompt paths of SAM that the automatic mask generator does not use, built on
oracle/sam_dec_oracle.py:
    embed_prompts / mask_downscaling   PromptEncoder.forward with points (pad only without a box), boxes and mask inputs
                                       ISM/segment_anything/modeling/prompt_encoder.py:76-170
    mask_decoder                       MaskDecoder.predict_masks with a per-prompt dense embedding, both multimask_output values
                                       modeling/mask_decoder.py:71-176
    apply_coords / apply_boxes         ResizeLongestSide (utils/transforms.py)
    predict_torch / predict            SamPredictor (predictor.py) on an image embedding that is already set
over a flat state_dict with the reference's key names.  Parity status: PINNED -- tools/make_golden_sam_predictor.py runs the
vendored reference SamPredictor on the same seeded weights and finds this restatement bit-identical; fixture
tests/golden/sam_predictor.pt."""
from typing import Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import sam_dec_oracle as so

SD = so.SD


# ---- prompt encoder ----------------------------------------------------------------------------------------------------
def _pe_with_coords(sd: SD, coords: torch.Tensor, image_size: int = 1024) -> torch.Tensor:
    """PositionEmbeddingRandom.forward_with_coords"""
    c = coords.clone()
    c[:, :, 0] = c[:, :, 0] / image_size
    c[:, :, 1] = c[:, :, 1] / image_size
    return so._pe_encoding(sd, c.to(torch.float))


def embed_points(sd: SD, points: torch.Tensor, labels: torch.Tensor, pad: bool) -> torch.Tensor:
    """_embed_points: labels -1 (not a point: PE zeroed), 0, 1; the padding point only when pad"""
    points = points + 0.5
    if pad:
        points = torch.cat([points, torch.zeros((points.shape[0], 1, 2))], dim=1)
        labels = torch.cat([labels, -torch.ones((labels.shape[0], 1))], dim=1)
    e = _pe_with_coords(sd, points)
    e[labels == -1] = 0.0
    e[labels == -1] += sd["prompt_encoder.not_a_point_embed.weight"]
    e[labels == 0] += sd["prompt_encoder.point_embeddings.0.weight"]
    e[labels == 1] += sd["prompt_encoder.point_embeddings.1.weight"]
    return e


def embed_boxes(sd: SD, boxes: torch.Tensor) -> torch.Tensor:
    """_embed_boxes: corners shifted by 0.5, point_embeddings 2 and 3"""
    e = _pe_with_coords(sd, (boxes + 0.5).reshape(-1, 2, 2))
    e[:, 0, :] += sd["prompt_encoder.point_embeddings.2.weight"]
    e[:, 1, :] += sd["prompt_encoder.point_embeddings.3.weight"]
    return e


def _layer_norm_2d(sd: SD, n: str, x: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + eps)
    return sd[n + ".weight"][:, None, None] * x + sd[n + ".bias"][:, None, None]


def mask_downscaling(sd: SD, masks: torch.Tensor) -> torch.Tensor:
    """(B,1,256,256) -> (B,256,64,64)"""
    p = "prompt_encoder.mask_downscaling"
    x = F.conv2d(masks, sd[p + ".0.weight"], sd[p + ".0.bias"], stride=2)
    x = F.gelu(_layer_norm_2d(sd, p + ".1", x))
    x = F.conv2d(x, sd[p + ".3.weight"], sd[p + ".3.bias"], stride=2)
    x = F.gelu(_layer_norm_2d(sd, p + ".4", x))
    return F.conv2d(x, sd[p + ".6.weight"], sd[p + ".6.bias"])


def embed_prompts(sd: SD, points: Optional[Tuple[torch.Tensor, torch.Tensor]], boxes: Optional[torch.Tensor],
                  masks: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
    """PromptEncoder.forward -> (sparse (B,N,256), dense (B,256,64,64))"""
    bs = points[0].shape[0] if points is not None else boxes.shape[0] if boxes is not None else masks.shape[0] if masks is not None else 1
    sparse = torch.empty((bs, 0, so.C))
    if points is not None:
        sparse = torch.cat([sparse, embed_points(sd, points[0], points[1], pad=boxes is None)], dim=1)
    if boxes is not None:
        sparse = torch.cat([sparse, embed_boxes(sd, boxes)], dim=1)
    if masks is not None:
        dense = mask_downscaling(sd, masks)
    else:
        dense = sd["prompt_encoder.no_mask_embed.weight"].reshape(1, -1, 1, 1).expand(bs, -1, 64, 64)
    return sparse, dense


# ---- mask decoder with a dense embedding per prompt ------------------------------------------------------------------------
def mask_decoder(sd: SD, image_embeddings: torch.Tensor, image_pe: torch.Tensor, sparse: torch.Tensor, dense: torch.Tensor,
                 multimask_output: bool = True):
    """MaskDecoder.forward -> (low-res masks (B,3|1,256,256), iou predictions (B,3|1))"""
    B = sparse.shape[0]
    out_tokens = torch.cat([sd["mask_decoder.iou_token.weight"], sd["mask_decoder.mask_tokens.weight"]], dim=0)
    tokens = torch.cat((out_tokens.unsqueeze(0).expand(B, -1, -1), sparse), dim=1)
    h, w = image_embeddings.shape[-2:]
    src = torch.repeat_interleave(image_embeddings, B, dim=0) + dense
    pos = torch.repeat_interleave(image_pe, B, dim=0)
    hs, src = so.two_way_transformer(sd, src, pos, tokens)
    iou_tok, mask_tok = hs[:, 0, :], hs[:, 1:so.T_OUT, :]
    src = src.transpose(1, 2).view(B, so.C, h, w)
    u = "mask_decoder.output_upscaling"
    x = F.conv_transpose2d(src, sd[u + ".0.weight"], sd[u + ".0.bias"], stride=2)
    x = F.gelu(_layer_norm_2d(sd, u + ".1", x))
    x = F.gelu(F.conv_transpose2d(x, sd[u + ".3.weight"], sd[u + ".3.bias"], stride=2))
    hyper = []
    for i in range(4):
        y = mask_tok[:, i, :]
        for j in range(3):
            y = so._lin(sd, f"mask_decoder.output_hypernetworks_mlps.{i}.layers.{j}", y)
            if j < 2:
                y = F.relu(y)
        hyper.append(y)
    hyper = torch.stack(hyper, dim=1)
    b, c, hh, ww = x.shape
    masks = (hyper @ x.view(b, c, hh * ww)).view(b, -1, hh, ww)
    y = iou_tok
    for j in range(3):
        y = so._lin(sd, f"mask_decoder.iou_prediction_head.layers.{j}", y)
        if j < 2:
            y = F.relu(y)
    sl = slice(1, None) if multimask_output else slice(0, 1)
    return masks[:, sl], y[:, sl]


# ---- predictor ---------------------------------------------------------------------------------------------------------------
def apply_coords(coords: np.ndarray, original_size: Tuple[int, int]) -> np.ndarray:
    return so.apply_coords(np.asarray(coords), original_size)


def apply_boxes(boxes: np.ndarray, original_size: Tuple[int, int]) -> np.ndarray:
    return apply_coords(np.asarray(boxes).reshape(-1, 2, 2), original_size).reshape(-1, 4)


def apply_coords_torch(coords: torch.Tensor, original_size: Tuple[int, int]) -> torch.Tensor:
    """ResizeLongestSide.apply_coords_torch: the scaling in fp32 (apply_coords scales in float64)"""
    new_h, new_w = so.preprocess_shape(*original_size)
    c = coords.clone().to(torch.float)
    c[..., 0] = c[..., 0] * (new_w / original_size[1])
    c[..., 1] = c[..., 1] * (new_h / original_size[0])
    return c


def apply_boxes_torch(boxes: torch.Tensor, original_size: Tuple[int, int]) -> torch.Tensor:
    return apply_coords_torch(boxes.reshape(-1, 2, 2), original_size).reshape(-1, 4)


def predict_torch(sd: SD, features: torch.Tensor, original_size: Tuple[int, int], point_coords=None, point_labels=None, boxes=None,
                  mask_input=None, multimask_output: bool = True, return_logits: bool = False):
    """SamPredictor.predict_torch with prompts in the resized frame -> (masks (B,C,H,W), iou (B,C), low-res logits (B,C,256,256))"""
    points = (point_coords, point_labels) if point_coords is not None else None
    sparse, dense = embed_prompts(sd, points, boxes, mask_input)
    low, iou = mask_decoder(sd, features, so.dense_pe(sd), sparse, dense, multimask_output)
    masks = so.postprocess_masks(low, so.preprocess_shape(*original_size), original_size)
    if not return_logits:
        masks = masks > 0.0
    return masks, iou, low


def predict(sd: SD, features: torch.Tensor, original_size: Tuple[int, int], point_coords=None, point_labels=None, box=None,
            mask_input=None, multimask_output: bool = True, return_logits: bool = False):
    """SamPredictor.predict: numpy prompts in original-image pixels, one prompt -> numpy (masks, iou, low-res logits)"""
    c = l = b = m = None
    if point_coords is not None:
        c = torch.as_tensor(apply_coords(point_coords, original_size), dtype=torch.float)[None, :, :]
        l = torch.as_tensor(point_labels, dtype=torch.int)[None, :]
    if box is not None:
        b = torch.as_tensor(apply_boxes(box, original_size), dtype=torch.float)[None, :]
    if mask_input is not None:
        m = torch.as_tensor(mask_input, dtype=torch.float)[None, :, :, :]
    masks, iou, low = predict_torch(sd, features, original_size, c, l, b, m, multimask_output, return_logits)
    return masks[0].numpy(), iou[0].numpy(), low[0].numpy()


# ---- the fixture's prompt cases (tools/make_golden_sam_predictor.py, tests/test_*sam_predictor*.py) ---------------------------------
def smooth_logits(seed: int, n: int = 1) -> torch.Tensor:
    """(n,1,256,256) low-res logits of the kind an earlier prediction gives: smooth blobs reaching about +-20"""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.randn(n, 1, 8, 8, generator=g) * 12, size=(256, 256), mode="bicubic", align_corners=False)
    return (base + 0.5 * torch.randn(n, 1, 256, 256, generator=g)).clamp(-20, 20).contiguous()


def make_cases(original_size: Tuple[int, int]):
    """nine prompt cases on a frame of original_size (H, W): name -> dict(api = "predict" | "predict_torch", kwargs).  The kwargs of
    "mask_from_case1" name no mask_input: it is case 1's low-res logits of highest predicted IoU (see resolve_kwargs)."""
    H, W = original_size
    rng = np.random.default_rng(H * 10000 + W)
    xy = lambda fx, fy: [fx * W, fy * H]                                  # noqa: E731
    box = np.array(xy(0.22, 0.25) + xy(0.71, 0.8))
    clicks26 = np.stack([rng.uniform(0, W, 26), rng.uniform(0, H, 26)], axis=-1)
    labels26 = rng.integers(0, 2, 26)
    labels26[[5, 17]] = -1                                                 # user-given "not a point" labels
    g = np.stack([rng.uniform(0, 0.6 * W, 16), rng.uniform(0, 0.6 * H, 16)], axis=-1)
    boxes16 = np.concatenate([g, g + np.stack([rng.uniform(40, 0.4 * W, 16), rng.uniform(40, 0.4 * H, 16)], axis=-1)], axis=-1)
    one = np.array([xy(0.55, 0.45)])
    return {
        "click": dict(api="predict", kwargs=dict(point_coords=one, point_labels=np.array([1]), multimask_output=True)),
        "three_clicks": dict(api="predict", kwargs=dict(point_coords=np.array([xy(0.3, 0.3), xy(0.6, 0.5), xy(0.4, 0.7)]),
                                                        point_labels=np.array([1, 0, 1]), multimask_output=False)),
        "box": dict(api="predict", kwargs=dict(box=box, multimask_output=False)),
        "box_two_clicks": dict(api="predict", kwargs=dict(box=box, point_coords=np.array([xy(0.4, 0.5), xy(0.65, 0.3)]),
                                                          point_labels=np.array([1, 0]), multimask_output=False)),
        "mask_from_case1": dict(api="predict", kwargs=dict(point_coords=np.array([xy(0.5, 0.5)]), point_labels=np.array([1]),
                                                           multimask_output=False)),
        "boxes16_torch": dict(api="predict_torch", kwargs=dict(boxes=boxes16, multimask_output=False)),
        "clicks26": dict(api="predict", kwargs=dict(point_coords=clicks26, point_labels=labels26, multimask_output=False)),
        "mask_only": dict(api="predict", kwargs=dict(mask_input=smooth_logits(H + W)[0].numpy(), multimask_output=True)),
        "logits": dict(api="predict", kwargs=dict(point_coords=one, point_labels=np.array([1]), multimask_output=True, return_logits=True)),
    }


def resolve_kwargs(name: str, kwargs: dict, click_out) -> dict:
    """case 5 takes case 1's best low-res logits (click_out = (masks, iou, low) of "click") as mask_input"""
    if name != "mask_from_case1":
        return kwargs
    _, iou, low = click_out
    return dict(kwargs, mask_input=np.asarray(low)[int(np.argmax(np.asarray(iou)))][None])


def run_cases(sd: SD, features: torch.Tensor, original_size: Tuple[int, int]):
    """every case through this restatement -> name -> (masks, iou, low) as torch tensors (predict: one prompt, unbatched)"""
    out = {}
    for name, c in make_cases(original_size).items():
        kw = resolve_kwargs(name, c["kwargs"], out.get("click"))
        if c["api"] == "predict_torch":
            b = apply_boxes_torch(torch.as_tensor(kw["boxes"], dtype=torch.float), original_size)
            r = predict_torch(sd, features, original_size, boxes=b, multimask_output=kw["multimask_output"])
        else:
            r = tuple(torch.as_tensor(a) for a in predict(sd, features, original_size, **kw))
        out[name] = r
    return out
