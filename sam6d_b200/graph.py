"""CUDA-graph replay of a fixed-shape forward.

A 32-proposal step of the matching path is ~120 kernel launches of 10-300 us each.  Issued one by one the host pays a ctypes
call, a few tensor allocations and a launch per kernel (3-5 ms of host time per step, next to ~7 ms on the device), and at small
per-GPU batches (strong scaling: 25 proposals per GPU at 8 GPUs) the host becomes the bound.  Every shape on the path is static,
there is no host read-back and no data-dependent control flow, so the whole forward is captured once per input signature with
stream capture (the programmatic-dependent-launch edges between the kernels are kept by the capture) and replayed as ONE graph
launch.

Policy (`StepGraphs.run`): the signature of a call is (name, data pointer, shape, stride, dtype) of every tensor in the
end-points dict.  First sighting of a signature: the forward runs launch by launch (this is also the warm-up that fills the
packed-weight caches).  Second sighting: the forward is captured READING THE CALLER'S TENSORS IN PLACE (no staging copy: a
signature match means the same addresses hold this call's inputs) and replayed; later sightings replay.  A serving loop over a
double-buffered input set settles on two graphs.  The outputs of a replay live in graph memory, so the five small result
tensors are copied out (one copy of 25 floats per proposal) before they are returned, together with any further outputs the
caller names (`keys`: the hyp_* results of a forward with several coarse hypotheses).  The random draws of `compute_coarse_Rt` are
made outside the graph into a fixed buffer (`torch.rand`, as the reference) or copied there when the caller passes them.

Any failure to capture turns the cache off for the module (with a warning) and the call runs launch by launch: same kernels,
same results.
"""
import warnings
from collections import OrderedDict
from typing import Callable, Dict, Optional

import torch

from . import _lib

OUT_KEYS = (("init_R", 9), ("init_t", 3), ("pred_R", 9), ("pred_t", 3), ("pred_pose_score", 1))
OUT_FLOATS = sum(n for _, n in OUT_KEYS)
_OUT_NAMES = frozenset(k for k, _ in OUT_KEYS)
# further results a forward may add (pem.HYP_KEYS); like OUT_KEYS they are not part of a call's signature
_MORE_NAMES = frozenset(("hyp_init_R", "hyp_init_t", "hyp_R", "hyp_t", "hyp_pose_score", "hyp_valid", "hyp_index"))


class _Captured:
    __slots__ = ("graph", "flat", "rand", "launches", "batch", "more")

    def __init__(self, graph, flat, rand, launches, batch, more=()):
        self.graph, self.flat, self.rand, self.launches, self.batch = graph, flat, rand, launches, batch
        self.more = more        # (name, shape, dtype) of every output stored after the OUT_KEYS block


def signature(end_points: Dict[str, torch.Tensor], extra=()) -> Optional[tuple]:
    sig = []
    for k in sorted(end_points):
        v = end_points[k]
        # a dict that went through forward() before carries its results
        if isinstance(v, torch.Tensor) and k not in _OUT_NAMES and k not in _MORE_NAMES:
            if not v.is_cuda:
                return None
            sig.append((k, v.data_ptr(), tuple(v.shape), tuple(v.stride()), v.dtype))
    return tuple(sig) + tuple(extra)


class StepGraphs:
    """per-module cache of captured forwards, least recently used first out"""

    def __init__(self, max_graphs: int = 8):
        self.max_graphs = max_graphs
        self.graphs: "OrderedDict[tuple, _Captured]" = OrderedDict()
        self.seen: "OrderedDict[tuple, int]" = OrderedDict()
        self.pool = None
        self.stream = None
        self.disabled = False
        self.replays = 0
        self.captures = 0

    def _capture(self, fn: Callable, end_points, n_rand: int, keys=()) -> _Captured:
        some = next(v for v in end_points.values() if isinstance(v, torch.Tensor))
        dev = some.device
        B = end_points["pts"].shape[0]
        if self.stream is None:
            self.stream = torch.cuda.Stream(dev)
        rand = torch.empty(B, n_rand, dtype=torch.float32, device=dev)
        g = torch.cuda.CUDAGraph()
        l0 = _lib.launch_count()
        kw = dict(pool=self.pool) if self.pool is not None else {}
        # thread_local: CUDA calls of other host threads (the NCCL watchdog's event queries) do not invalidate the capture
        with torch.cuda.graph(g, stream=self.stream, capture_error_mode="thread_local", **kw):
            out = fn(dict(end_points), rand)
            flat = torch.cat([out[k].reshape(B * n).to(torch.float32) for k, n in OUT_KEYS]   # contiguous block per output
                             + [out[k].reshape(-1).to(torch.float32) for k in keys])          # exact: small ints, 0 / 1 flags
        if self.pool is None:
            self.pool = g.pool()
        self.captures += 1
        launches = _lib.launch_count() - l0
        _lib.add_launches(-launches)                                   # counted while capturing, not launched
        return _Captured(g, flat, rand, launches, B, tuple((k, tuple(out[k].shape), out[k].dtype) for k in keys))

    def run(self, fn: Callable, end_points: Dict[str, torch.Tensor], rand: Optional[torch.Tensor], n_rand: int, extra=(), keys=()):
        """fn(end_points, rand) -> end_points is the launch-by-launch forward.  Returns the updated end_points, or None when
        this call is to run launch by launch (first sighting, capture turned off, CPU tensors in the dict).  keys: outputs of
        fn to return besides OUT_KEYS; a call that names other keys must also pass another `extra`."""
        if self.disabled or torch.cuda.is_current_stream_capturing():
            return None
        sig = signature(end_points, extra)
        if sig is None:
            return None
        cap = self.graphs.get(sig)
        if cap is None:
            n = self.seen.get(sig, 0) + 1
            self.seen[sig] = n
            self.seen.move_to_end(sig)
            while len(self.seen) > 64:
                self.seen.popitem(last=False)
            if n < 2:
                return None
            try:
                cap = self._capture(fn, end_points, n_rand, keys) if keys else self._capture(fn, end_points, n_rand)
            except Exception as e:                                  # same kernels launch by launch from here on
                self.disabled = True
                warnings.warn(f"sam6d_b200: CUDA-graph capture of the forward failed ({type(e).__name__}: {e}); "
                              "running launch by launch")
                return None
            self.graphs[sig] = cap
            while len(self.graphs) > self.max_graphs:
                self.graphs.popitem(last=False)
        else:
            self.graphs.move_to_end(sig)
        if rand is None:
            cap.rand.uniform_()                                      # the reference's torch.rand draw (model_utils.py:199)
        else:
            cap.rand.copy_(rand.reshape(cap.rand.shape), non_blocking=True)
        cap.graph.replay()
        _lib.add_launches(cap.launches)
        self.replays += 1
        res = cap.flat.clone()
        off, B = 0, cap.batch
        for k, n in OUT_KEYS:
            v = res[off:off + B * n]
            end_points[k] = v.view(B, 3, 3) if n == 9 else (v.view(B, 3) if n == 3 else v)
            off += B * n
        for k, shape, dtype in cap.more:
            n = 1
            for d in shape:
                n *= d
            end_points[k] = res[off:off + n].view(shape).to(dtype)
            off += n
        return end_points
