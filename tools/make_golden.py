"""tools/make_golden.py -- run in the DEV CONTAINER ONLY (needs /root/reference).

Pins the oracle: imports the reference's own Python modules from /root/reference, loads the
oracle's seeded state_dict into them (strict), runs both on identical seeded inputs on the CPU,
asserts agreement, and writes small golden fixtures to tests/golden/.

The reference's `pointnet2._ext` is CUDA-only; under the reference's Python wrappers we plug
oracle/pn2.py (the C restatement of those kernels).  So this script pins every Python-level
function of the path against the reference code itself, and the native ops against their
restatement (those are pinned against the real CUDA kernels on the GPU box, tests/test_gpu_pn2.py).

Usage: python tools/make_golden.py [small full b32 sam ...]   (no argument = all cases)
"""
import builtins
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = "/root/reference/SAM-6D"
PEM = os.path.join(REF, "Pose_Estimation_Model")

from oracle import pem_oracle as po  # noqa: E402
from oracle import pn2  # noqa: E402


def import_reference_pem():
    builtins.__POINTNET2_SETUP__ = True
    for sub in ("model", "utils", os.path.join("model", "pointnet2")):
        sys.path.insert(0, os.path.join(PEM, sub))
    import pointnet2_utils  # noqa
    pointnet2_utils._ext = types.SimpleNamespace(
        furthest_point_sampling=pn2.furthest_point_sampling,
        gather_points=pn2.gather_points,
        ball_query=pn2.ball_query,
        group_points=pn2.group_points,
    )
    import transformer, coarse_point_matching, fine_point_matching, model_utils  # noqa
    return transformer, coarse_point_matching, fine_point_matching, model_utils


def ns(**kw):
    return types.SimpleNamespace(**kw)


class RefMatcher(torch.nn.Module):
    """The reference's Net minus the ViT feature extractor (pose_estimation_model.py:11-53)."""

    def __init__(self, mods, coarse_npoint):
        super().__init__()
        transformer, cpm, fpm, mu = mods
        self.mu = mu
        self.coarse_npoint = coarse_npoint
        self.geo_embedding = transformer.GeometricStructureEmbedding(
            ns(sigma_d=0.2, sigma_a=15, angle_k=3, reduction_a="max", hidden_dim=256))
        self.coarse_point_matching = cpm.CoarsePointMatching(
            ns(nblock=3, input_dim=256, hidden_dim=256, out_dim=256, temp=0.1, sim_type="cosine",
               normalize_feat=True, loss_dis_thres=0.15, nproposal1=6000, nproposal2=300))
        self.fine_point_matching = fpm.FinePointMatching(
            ns(nblock=3, input_dim=256, hidden_dim=256, out_dim=256, pe_radius1=0.1, pe_radius2=0.2,
               focusing_factor=3, temp=0.1, sim_type="cosine", normalize_feat=True, loss_dis_thres=0.15))

    @torch.no_grad()
    def forward(self, inp):
        # ViTEncoder.forward inference branch, feature_extraction.py:135-142
        dense_po = inp["dense_po"].clone()
        radius = torch.norm(dense_po, dim=2).max(1)[0]
        dense_pm = inp["pts"] / (radius.reshape(-1, 1, 1) + 1e-6)
        dense_po = dense_po / (radius.reshape(-1, 1, 1) + 1e-6)
        dense_fm, dense_fo = inp["dense_fm"], inp["dense_fo"]
        ep = {"model": inp["model"]}
        bg_point = torch.ones(dense_pm.size(0), 1, 3).float() * 100
        sp_m, sf_m, idx_m = self.mu.sample_pts_feats(dense_pm, dense_fm, self.coarse_npoint, return_index=True)
        geo_m = self.geo_embedding(torch.cat([bg_point, sp_m], dim=1))
        sp_o, sf_o, idx_o = self.mu.sample_pts_feats(dense_po, dense_fo, self.coarse_npoint, return_index=True)
        geo_o = self.geo_embedding(torch.cat([bg_point, sp_o], dim=1))
        ep = self.coarse_point_matching(sp_m, sf_m, geo_m, sp_o, sf_o, geo_o, radius, ep)
        ep = self.fine_point_matching(dense_pm, dense_fm, geo_m, idx_m, dense_po, dense_fo, geo_o, idx_o, radius, ep)
        ep.update(fps_idx_m=idx_m, fps_idx_o=idx_o, geo_m=geo_m, geo_o=geo_o)
        return ep


def check(name, a, b, atol, rtol=0.0):
    a, b = a.float(), b.float()
    err = (a - b).abs().max().item()
    ok = torch.allclose(a, b, atol=atol, rtol=rtol)
    print(f"  {name:28s} max|diff| = {err:.3e}  {'OK' if ok else 'MISMATCH'}")
    assert ok, name


def run_case(mods, tag, B, n, coarse_npoint, seed, out_dir, store_inputs):
    print(f"case {tag}: B={B} n={n} sparse={coarse_npoint} seed={seed}")
    sd = po.make_state_dict(seed=seed)
    ref = RefMatcher(mods, coarse_npoint).eval()
    missing = ref.load_state_dict(sd, strict=True)
    print("  reference modules accepted the oracle state_dict (strict):", missing)
    inp = po.make_inputs(B=B, n=n, seed=seed)
    torch.manual_seed(1)
    rand = torch.rand(B, po.N_PROPOSAL1 * 3)
    torch.manual_seed(1)
    r = ref(inp)
    o = po.pem_forward(sd, inp["pts"], inp["dense_fm"], inp["dense_po"], inp["dense_fo"], inp["model"],
                       rand=rand, coarse_npoint=coarse_npoint, return_stages=True, completion="both")
    assert torch.equal(r["fps_idx_m"], o["fps_idx_m"]) and torch.equal(r["fps_idx_o"], o["fps_idx_o"])
    check("geo_embedding_m", r["geo_m"], o["geo_m"], 1e-5)
    check("geo_embedding_o", r["geo_o"], o["geo_o"], 1e-5)
    check("init_R", r["init_R"], o["init_R"], 1e-5)
    check("init_t", r["init_t"], o["init_t"], 1e-5)
    check("pred_R", r["pred_R"], o["pred_R"], 1e-5)
    check("pred_t", r["pred_t"], o["pred_t"], 1e-5)
    check("pred_pose_score", r["pred_pose_score"], o["pred_pose_score"], 1e-6)
    well = ~o["init_degenerate"]
    same = (o["det_init_R"] - o["init_R"]).abs().amax(dim=(1, 2)) == 0
    print(f"  reference winner well defined on {int(well.sum())}/{B} proposals; deterministic completion leaves "
          f"{int(same.sum())}/{B} initial poses bit-identical; max |det - ref| pred_R on the others = "
          f"{(o['det_pred_R'] - o['pred_R'])[~same].abs().max().item() if (~same).any() else 0.0:.3e}")
    g = torch.Generator().manual_seed(7)
    S = coarse_npoint + 1
    pick = torch.randint(0, S, (64, 2), generator=g)
    gold = dict(
        meta=dict(B=B, n=n, coarse_npoint=coarse_npoint, seed=seed, torch=torch.__version__,
                  source="reference modules imported from /root/reference (CPU, fp32)"),
        rand=rand if store_inputs else None,
        fps_idx_m=r["fps_idx_m"], fps_idx_o=r["fps_idx_o"],
        geo_pick=pick, geo_m_pick=r["geo_m"][:, pick[:, 0], pick[:, 1], :].clone(),
        geo_o_pick=r["geo_o"][:, pick[:, 0], pick[:, 1], :].clone(),
        geo_m_sum=r["geo_m"].double().sum(dim=(1, 2)).float(),
        init_R=r["init_R"], init_t=r["init_t"], pred_R=r["pred_R"], pred_t=r["pred_t"],
        pred_pose_score=r["pred_pose_score"],
        # is the reference's winning pose hypothesis rank-deficient (its rotation decided by SVD rounding noise)?
        init_degenerate=o["init_degenerate"], init_score=o["init_score"],
        # the oracle with the deterministic completion of rank-deficient hypotheses (the CUDA path's rule; identical to the
        # reference outputs above wherever no such hypothesis wins): the comparator that holds on EVERY proposal
        det_init_R=o["det_init_R"], det_init_t=o["det_init_t"], det_pred_R=o["det_pred_R"], det_pred_t=o["det_pred_t"],
        det_pred_pose_score=o["det_pred_pose_score"], det_init_score=o["det_init_score"],
        det_init_degenerate=o["det_init_degenerate"],
        input_checksum={k: v.double().sum().item() for k, v in inp.items()},
        atten_coarse=o["atten_coarse"] if S <= 64 else o["atten_coarse"][:, :8, :].clone(),
    )
    if store_inputs:
        gold["inputs"] = {k: v for k, v in inp.items()}
    path = os.path.join(out_dir, f"pem_{tag}.pt")
    torch.save(gold, path)
    print(f"  wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


def run_sam_case(out_dir, tag="sam_small", cfg=None, check_oracle=True):
    """SAM image encoder: the vendored reference module against oracle/sam_oracle.py.
    sam_small: 2 blocks of ViT-H width (one windowed, one global), 1024^2 input -- every code path of the 32-block model.
    sam_vith:  the full 32-block ViT-H of build_sam.py:14-21 on one frame (5.96 TFLOP on the CPU).
    sam_vitl / sam_vitb: the full 24-block ViT-L / 12-block ViT-B of build_sam.py:27-44 (head dim 64)."""
    from oracle import sam_oracle as so
    sys.path.insert(0, os.path.join(REF, "Instance_Segmentation_Model"))
    from functools import partial
    from segment_anything.modeling.image_encoder import ImageEncoderViT
    cfg = cfg or dict(embed_dim=1280, depth=2, num_heads=16, global_attn_indexes=(1,))
    print(f"case {tag}:", cfg)
    sd = so.make_state_dict(seed=1, **cfg)
    ref = ImageEncoderViT(depth=cfg["depth"], embed_dim=cfg["embed_dim"], img_size=1024, mlp_ratio=4,
                          norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), num_heads=cfg["num_heads"], patch_size=16,
                          qkv_bias=True, use_rel_pos=True, global_attn_indexes=cfg["global_attn_indexes"], window_size=14,
                          out_chans=256).eval()
    print("  reference ImageEncoderViT accepted the oracle state_dict (strict):", ref.load_state_dict(sd, strict=True))
    img = so.make_images(B=1, seed=1)
    with torch.no_grad():
        r = ref(img)
    if check_oracle:
        o = so.image_encoder(sd, img, cfg["num_heads"], cfg["global_attn_indexes"])
        check("image_encoder output", r, o, 1e-4)
    gold = dict(meta=dict(cfg=cfg, seed=1, img_seed=1, source="segment_anything ImageEncoderViT imported from /root/reference"),
                out_sub=r[:, :, ::4, ::4].clone(), out_sum=r.double().sum().item(), out_abs_mean=r.abs().mean().item(),
                out_abs_max=r.abs().max().item(), out_std=r.std().item())
    path = os.path.join(out_dir, tag + ".pt")
    torch.save(gold, path)
    print(f"  wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


def run_sam_keys_case(out_dir):
    """the (key, shape) list and parameter count of the reference's sam_model_registry[t]() for vit_h, vit_l and vit_b
    (build_sam.py:14-52): the checkpoint layout each backbone's drop-in must load strictly"""
    sys.path.insert(0, os.path.join(REF, "Instance_Segmentation_Model"))
    from segment_anything.build_sam import sam_model_registry
    gold = dict(meta=dict(source="segment_anything sam_model_registry imported from /root/reference"), types={})
    for t in ("vit_h", "vit_l", "vit_b"):
        torch.manual_seed(0)
        model = sam_model_registry[t]()
        keys = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
        n = sum(p.numel() for p in model.parameters())
        gold["types"][t] = dict(keys=keys, n_params=n)
        print(f"  {t}: {len(keys)} state_dict tensors, {n} parameters")
    path = os.path.join(out_dir, "sam_keys.pt")
    torch.save(gold, path)
    print(f"  wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


def main(only=None):
    out_dir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    torch.set_num_threads(8)
    want = lambda name: not only or name in only  # noqa: E731
    if any(want(c) for c in ("small", "full", "b32")):
        mods = import_reference_pem()
    if want("small"):   # inputs stored in the fixture; runs in seconds everywhere
        run_case(mods, "small", B=2, n=256, coarse_npoint=32, seed=3, out_dir=out_dir, store_inputs=True)
    if want("full"):    # full BASELINE shapes for four proposals: inputs regenerated from the seed
        run_case(mods, "full", B=4, n=2048, coarse_npoint=196, seed=1, out_dir=out_dir, store_inputs=False)
    if want("b32"):     # BASELINE config #2 itself: 32 proposals x 2048 x 2048 (the bench workload)
        run_case(mods, "b32", B=32, n=2048, coarse_npoint=196, seed=2, out_dir=out_dir, store_inputs=False)
    if want("sam"):
        run_sam_case(out_dir)
    if want("sam_vith"):
        run_sam_case(out_dir, "sam_vith", dict(embed_dim=1280, depth=32, num_heads=16, global_attn_indexes=(7, 15, 23, 31)))
    if want("sam_vitl"):
        run_sam_case(out_dir, "sam_vitl", dict(embed_dim=1024, depth=24, num_heads=16, global_attn_indexes=(5, 11, 17, 23)))
    if want("sam_vitb"):
        run_sam_case(out_dir, "sam_vitb", dict(embed_dim=768, depth=12, num_heads=12, global_attn_indexes=(2, 5, 8, 11)))
    if want("sam_keys"):
        run_sam_keys_case(out_dir)


if __name__ == "__main__":
    main(sys.argv[1:])
