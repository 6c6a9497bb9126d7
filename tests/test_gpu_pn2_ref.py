"""GPU: pins the point-cloud ops against the REFERENCE's own CUDA kernels.

tests/golden/pn2_ref.json holds what the reference's pointnet2._ext kernels returned on an H100 for the seeded inputs below
(tools/make_golden_pn2.py): the SHA-256 digest of each output's bytes (indices as int32) and 16 sampled elements, which point at
a difference before the digest does.  Both the C restatement (oracle/pn2_oracle.c) and the sam6d_b200 kernels must reproduce
them bit for bit."""
import hashlib
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import pn2     # noqa: E402

FPS_CASES = [(4, 2048, 196, False), (2, 2048, 196, True), (2, 1000, 100, False), (1, 5000, 64, False), (2, 300, 40, True)]
FPS_BIG_CASES = [(1, 210000, 2048), (2, 50000, 512), (3, 4097, 100), (1, 106496, 300), (1, 106497, 300)]
BALL_CASES = [(2048, 0.1, 32), (2048, 0.2, 64), (700, 0.3, 16)]


def digest(t):
    t = t.cpu().contiguous()
    return hashlib.sha256((t if t.is_floating_point() else t.to(torch.int32)).numpy().tobytes()).hexdigest()


@pytest.fixture(scope="module")
def ref(golden_dir):
    gold = json.load(open(os.path.join(golden_dir, "pn2_ref.json")))

    def check(key, got, what):
        want = gold[key]
        flat = got.cpu().reshape(-1)
        assert flat[want["idx"]].tolist() == want["sample"], f"{what} (sampled elements)"
        assert digest(got) == want["sha256"], what
    return check


def clouds(b, n, seed, dup=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, n, 3, generator=g)
    x = x / x.norm(dim=2, keepdim=True) * (0.5 + 0.5 * torch.rand(b, n, 1, generator=g))
    if dup:
        pick = torch.randint(0, n // 6, (b, n), generator=g)
        x = torch.gather(x, 1, pick.unsqueeze(2).expand(b, n, 3))
    return x.contiguous()


def gather_inputs():
    g = torch.Generator().manual_seed(3)
    pts = torch.randn(2, 9, 500, generator=g)
    idx = torch.randint(0, 500, (2, 77), generator=g, dtype=torch.int32)
    gi = torch.randint(0, 500, (2, 77, 8), generator=g, dtype=torch.int32)
    return pts, idx, gi


@pytest.mark.parametrize("b,n,m,dup", FPS_CASES)
def test_fps_matches_reference_kernel(ref, b, n, m, dup):
    from sam6d_b200 import ops
    x = clouds(b, n, n + m, dup)
    key = f"fps/{b}/{n}/{m}/{int(dup)}"
    ref(key, pn2.furthest_point_sampling(x, m), "C restatement != reference CUDA kernel")
    ref(key, ops.furthest_point_sampling(x.cuda(), m), "sam6d_b200 kernel != reference CUDA kernel")


@pytest.mark.parametrize("b,n,m", FPS_BIG_CASES)
def test_fps_cluster_kernel_matches_reference_kernel(ref, b, n, m):
    """large clouds: the thread-block-cluster FPS (8 / 16 CTAs per cloud, points in distributed shared memory) and the one-CTA
    kernel against the reference's own kernel; 210 000 -> 2048 is the template bank of get_obj_feats
    (PEM/model/feature_extraction.py:170-181)."""
    from sam6d_b200 import ops
    x = clouds(b, n, n + m, dup=(n == 50000)).cuda()
    ref(f"fps_big/{b}/{n}/{m}", ops.furthest_point_sampling(x, m), "cluster FPS != reference CUDA kernel")
    ref(f"fps_big/{b}/{n}/{m}", ops.furthest_point_sampling_single_cta(x, m), "one-CTA FPS != reference CUDA kernel")


@pytest.mark.parametrize("n,r,ns", BALL_CASES)
def test_ball_query_matches_reference_kernel(ref, n, r, ns):
    from sam6d_b200 import ops
    x = clouds(3, n, n + ns)
    ref(f"ball/{n}/{r}/{ns}", pn2.ball_query(x, x, r, ns), "C restatement != reference CUDA kernel")
    ref(f"ball/{n}/{r}/{ns}", ops.ball_query(x.cuda(), x.cuda(), r, ns), "sam6d_b200 kernel != reference CUDA kernel")


def test_gather_group_match_reference_kernel(ref):
    from sam6d_b200 import ops
    pts, idx, gi = gather_inputs()
    ref("gather_points", ops.gather_points(pts.cuda(), idx.cuda()), "gather_points")
    ref("group_points", ops.group_points(pts.cuda(), gi.cuda()), "group_points")
