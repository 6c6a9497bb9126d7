"""float64 restatements of the SAM image encoder's stages (ISM/segment_anything/modeling/image_encoder.py), written with explicit
index tables so that a test can also evaluate plausible wrong variants of the same formula.  Pinned to oracle/sam_oracle.py by
tests/test_sam_encoder_reference_cpu.py; used by tests/test_gpu_sam_encoder_kernels.py."""
import torch
import torch.nn.functional as F


def rel_index(Hs: int, Ws: int, device=None):
    """(ih (L, Hs), iw (L, Ws)) for the L = Hs*Ws queries of a window: the table rows qh - kh + Hs - 1 and qw - kw + Ws - 1 that
    get_rel_pos (image_encoder.py:293-322) gathers"""
    r = torch.arange(Hs * Ws, device=device)
    qh, qw = r // Ws, r % Ws
    ih = qh[:, None] - torch.arange(Hs, device=device)[None, :] + Hs - 1
    iw = qw[:, None] - torch.arange(Ws, device=device)[None, :] + Ws - 1
    return ih, iw


def decomposed_bias(q, rel_h, rel_w, Hs: int, Ws: int, ih=None, iw=None):
    """add_decomposed_rel_pos (image_encoder.py:325-361) as an additive (..., L, L) bias: q (..., L, D) UNSCALED queries,
    bias[n, kh*Ws + kw] = q_n . rel_h[ih[n, kh]] + q_n . rel_w[iw[n, kw]].  ih / iw default to rel_index(Hs, Ws)."""
    L = Hs * Ws
    if ih is None or iw is None:
        dih, diw = rel_index(Hs, Ws, q.device)
        ih = dih if ih is None else ih
        iw = diw if iw is None else iw
    gh = q @ rel_h.transpose(0, 1).to(q.dtype)                       # (..., L, 2Hs-1)
    gw = q @ rel_w.transpose(0, 1).to(q.dtype)
    lead = q.shape[:-2]
    bh = torch.gather(gh, -1, ih.expand(*lead, L, ih.shape[-1]))      # (..., L, Hs)
    bw = torch.gather(gw, -1, iw.expand(*lead, L, iw.shape[-1]))      # (..., L, Ws)
    return (bh[..., :, None] + bw[..., None, :]).reshape(*lead, L, L)


def relpos_logits(q, k, rel_h, rel_w, Hs: int, Ws: int, scale: float):
    """Attention.forward (image_encoder.py:224-240): (q * scale) k^T + the decomposed rel-pos bias of the unscaled q"""
    return (q * scale) @ k.transpose(-1, -2) + decomposed_bias(q, rel_h, rel_w, Hs, Ws)


def relpos_attention(q, k, v, rel_h, rel_w, Hs: int, Ws: int, scale: float):
    """q, k, v (..., L, D) -> softmax(logits) v"""
    return torch.softmax(relpos_logits(q, k, rel_h, rel_w, Hs, Ws, scale), dim=-1) @ v


def layer_norm(x, w, b, eps: float):
    """nn.LayerNorm over the last dim (two-pass statistics, biased variance)"""
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    var = d.pow(2).mean(-1, keepdim=True)
    return d / torch.sqrt(var + eps) * w + b


def partition_ids(B: int, G: int, ws: int):
    """the reference window_partition (image_encoder.py:243-264: F.pad, then the window view) applied to the token ids of a
    B x G x G grid: (B, nwin*nwin*ws*ws) per-image token index, -1 at the zero padding"""
    from oracle import sam_oracle as so
    ids = torch.arange(1, B * G * G + 1, dtype=torch.float64).view(B, G, G, 1)      # 0 marks the padding
    w, (Hp, Wp) = so.window_partition(ids, ws)
    w = w.reshape(B, -1).long() - 1
    base = (torch.arange(B) * G * G)[:, None]
    return torch.where(w >= 0, w - base, torch.full_like(w, -1)), (Hp, Wp)


def unpartition_ids(B: int, G: int, ws: int):
    """the reference window_unpartition (image_encoder.py:267-290) applied to the window-token positions of each image:
    (B, G*G) -> the position in the per-image window sequence that lands on each grid token"""
    from oracle import sam_oracle as so
    Gp = (G + ws - 1) // ws * ws
    n = Gp * Gp
    pos = torch.arange(B * n, dtype=torch.float64).view(B * (Gp // ws) ** 2, ws, ws, 1)
    x = so.window_unpartition(pos, ws, (Gp, Gp), (G, G)).reshape(B, G * G).long()
    return x - (torch.arange(B) * n)[:, None]


def conv3x3_taps(G: int):
    """the 9 neighbourhoods of F.conv2d(padding=1) on a G x G grid, in the weight order (kh, kw): (9, G*G) token index of the
    input that tap (kh, kw) multiplies at each output token, -1 where it reads the zero padding"""
    ids = torch.arange(1, G * G + 1, dtype=torch.float64).view(1, 1, G, G)
    taps = []
    for kh in range(3):
        for kw in range(3):
            wt = torch.zeros(1, 1, 3, 3, dtype=torch.float64)
            wt[0, 0, kh, kw] = 1.0
            taps.append(F.conv2d(ids, wt, padding=1).reshape(-1).long() - 1)
    return torch.stack(taps)
