"""Time the point-to-plane ICP refinement (csrc/icp.cu, sam6d_icp_refine) with CUDA events, beside a bf16 Net.forward at the
same batch, on the GPU.

    python tools/icp_bench.py [--batches 1 32 200] [--iters 10] [--reps 20]

Per batch B: N = 2048 observed points and M = 4096 object samples per instance (tests/test_gpu_icp.py's synthetic instances:
two objects, 1 mm noise, 10 % background points, start poses within 5 degrees and 0.02 r), K = --iters iterations with
every instance running all of them (the step tolerance is not reached from these starts in 10 iterations; iters_run is
printed).  Net.forward runs with seeded weights on bench.py's synthetic inputs, captured as a CUDA graph as bench.py does.
Prints the card's name and power limit, then one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def events(fn, n):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 32, 200])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    import test_gpu_icp as tg
    from sam6d_b200 import ops, synth
    from sam6d_b200.pem import Net
    print(f"[icp_bench] card: {card()}")
    golden = os.path.join(ROOT, "tests", "golden")
    meshes, Q, Nn = tg._objects(golden)
    dev = torch.device("cuda")
    net = Net(precision="bf16").to(dev).eval()
    net.load_state_dict(synth.make_pem_state_dict(seed=1), strict=True)
    net.enable_graphs()
    rows = []
    for B in args.batches:
        obj = np.arange(B) % 2
        P, R0, t0, radius = tg._observations(meshes, obj, 2048, np.random.RandomState(B))
        c = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(dt).to(dev)   # noqa: E731
        a = (c(R0), c(t0), c(P), c(Q), c(Nn), c(obj, torch.int32), c(radius))
        res = ops.icp_refine(*a, args.iters)
        ms_icp = events(lambda: ops.icp_refine(*a, args.iters), args.reps)
        iters_run = res[4].cpu().numpy()
        inp = {k: v.to(dev) for k, v in synth.make_pem_inputs(B=B, n=2048, n_model=1024, seed=100).items()
               if k in ("pts", "dense_fm", "dense_po", "dense_fo", "model")}
        rand = torch.rand(B, synth.N_PROPOSAL1 * 3, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
        with torch.no_grad():
            for _ in range(3):                                               # launch by launch, capture, replay
                net(dict(inp), rand=rand)
            ms_fwd = events(lambda: net(dict(inp), rand=rand), max(3, args.reps // 4))
        # distance evaluations of the search: B x N x M per iteration
        gflop = B * 2048 * 4096 * args.iters * 8 / 1e9
        row = dict(B=B, N=2048, M=4096, K=args.iters, icp_ms=round(ms_icp, 4), forward_ms=round(ms_fwd, 3),
                   icp_share_of_forward=round(ms_icp / ms_fwd, 4), search_gflop=round(gflop, 2),
                   search_tflops=round(gflop / ms_icp, 2), iters_run_min=int(iters_run.min()), iters_run_max=int(iters_run.max()))
        print(f"[icp_bench] B={B}: ICP {ms_icp:.3f} ms per call ({row['search_tflops']} TFLOP/s of fp32 search at 8 FLOP per "
              f"distance), Net.forward {ms_fwd:.3f} ms, ICP / forward {ms_icp / ms_fwd:.3f}; iterations run "
              f"{row['iters_run_min']}..{row['iters_run_max']}")
        rows.append(row)
    print(json.dumps(dict(card=card(), rows=rows)))


if __name__ == "__main__":
    main()
