"""CPU: the C-ABI library builds (nvcc cross-compiles sm_90a without a GPU), loads, and exports every symbol that
include/sam6d_b200.h declares; the host-side drop-in classes keep the reference's state_dict layout.  No compute calls."""
import ctypes
import os
import subprocess

import pytest
import torch

from sam6d_b200 import _lib, build


@pytest.fixture(scope="module")
def libpath():
    return build.build()


def test_header_symbols_exported(libpath):
    protos = _lib.parse_header()
    assert len(protos) >= 29
    lib = ctypes.CDLL(libpath)
    for name in protos:
        assert hasattr(lib, name), f"{name} declared in include/sam6d_b200.h but not exported"
    # nothing else leaks out of the library: visibility is hidden by default
    out = subprocess.run(["nm", "-D", "--defined-only", libpath], capture_output=True, text=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    extra = {s for s in exported if not s.startswith("sam6d_") and not s.startswith("_")}
    assert not extra, extra
    assert set(protos) <= exported


def test_library_is_sm90a(libpath):
    out = subprocess.run(["cuobjdump", "-lelf", libpath], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_version_and_loader():
    assert _lib.version().startswith("sam6d_b200")
    assert _lib.launch_count() >= 0


def test_ops_reject_cpu_tensors():
    from sam6d_b200 import ops
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.furthest_point_sampling(torch.zeros(1, 8, 3), 2)
    with pytest.raises(RuntimeError):
        ops.gemm(torch.zeros(2, 2), torch.zeros(2, 2))


def test_call_rejects_cpu_tensor_arguments(libpath):
    """every pointer of the C ABI is a device pointer: a host tensor is refused before the stream is read or anything launches"""
    before = _lib.launch_count()
    with pytest.raises(_lib.Sam6dError, match="device pointer"):
        _lib.call("sam6d_cloud_radius", torch.zeros(1, 8, 3), 1, 8, None)
    assert _lib.launch_count() == before


def test_net_state_dict_layout_matches_reference_names():
    from oracle import pem_oracle as po
    from sam6d_b200.pem import Net
    net = Net().eval()
    sd = po.make_state_dict(seed=1)          # accepted strictly by the reference modules (tools/make_golden.py)
    res = net.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    keys = set(net.state_dict().keys())
    assert "coarse_point_matching.transformers.0.layers.0.attention.attention.proj_p.weight" in keys
    assert "fine_point_matching.PE.mlp2.layer2.normlayer.bn.running_var" in keys
    assert "fine_point_matching.transformers.1.dense_layer.attention.attention.scale" in keys
    with pytest.raises(NotImplementedError):
        Net().train()({})                    # inference-only drop-in


def test_pointnet2_ext_surface():
    import sam6d_b200.pointnet2_ext as _ext
    for name in ("furthest_point_sampling", "gather_points", "ball_query", "group_points", "gather_points_grad",
                 "group_points_grad", "three_nn", "three_interpolate", "three_interpolate_grad"):
        assert callable(getattr(_ext, name))             # bindings.cpp:11-24
    with pytest.raises(NotImplementedError):
        _ext.three_nn(None, None)
