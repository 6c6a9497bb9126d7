"""ctypes binding of libsam6d_b200.so.  Prototypes are parsed from include/sam6d_b200.h, so the header is the single
source of truth for the C ABI.  There is no fallback: if the library is missing or a call fails, we raise."""
import ctypes
import os
import re

import torch

_Tensor = torch.Tensor

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), "include", "sam6d_b200.h")
LIB_PATH = os.path.join(_HERE, "libsam6d_b200.so")

_CTYPES = {
    "int": ctypes.c_int,
    "long long": ctypes.c_longlong,
    "float": ctypes.c_float,
    "double": ctypes.c_double,
}


def parse_header(path: str = HEADER):
    """-> {name: (restype, [(ctype, argname), ...])} for every function the header declares."""
    text = open(path).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = {}
    for m in re.finditer(r"(const char\*|int)\s+(sam6d_\w+)\s*\(([^)]*)\)\s*;", text):
        ret, name, args = m.group(1), m.group(2), m.group(3)
        argl = []
        for a in [x.strip() for x in args.split(",")]:
            if a in ("void", ""):
                continue
            if "*" in a:
                argl.append((ctypes.c_void_p, a.split("*")[-1].strip()))
            else:
                typ, nm = a.rsplit(" ", 1)
                argl.append((_CTYPES[typ.strip()], nm))
        protos[name] = (ctypes.c_char_p if ret != "int" else ctypes.c_int, argl)
    return protos


class Sam6dError(RuntimeError):
    pass


_lib = None
_protos = None
_fns = {}        # name -> (ctypes function, number of parameters before a trailing stream, or -1 if there is none)


def lib():
    global _lib, _protos
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Sam6dError(
                f"{LIB_PATH} not found: build it with `python -m sam6d_b200.build` "
                "(or __graft_entry__.build()); sam6d_b200 has no CPU or eager fallback")
        _lib = ctypes.CDLL(LIB_PATH)
        _protos = parse_header()
        for name, (ret, args) in _protos.items():
            fn = getattr(_lib, name)
            fn.restype = ret
            fn.argtypes = [t for t, _ in args]
            _fns[name] = (fn, len(args) - 1 if args and args[-1][1] == "stream" else -1)
    return _lib


_launches = 0
# entry points that launch more than one kernel
_MULTI = {"sam6d_fine_assign": 6, "sam6d_coarse_select": 2, "sam6d_geo_embed_tc": 2, "sam6d_render_meshes": 4, "sam6d_yolo_masks": 2,
          "sam6d_mask_rle_count": 2, "sam6d_template_score_agg": 2, "sam6d_template_score": 2,
          "sam6d_pbr_reference_crops": 2, "sam6d_track_points": 4,
          "sam6d_track_points_scene": 5, "sam6d_symmetry_agreement": 2, "sam6d_tsdf_mesh_count": 2, "sam6d_tsdf_mesh_emit": 2}
_timed = {}      # name -> list of (start_event, end_event); filled only for names registered with time_kernel()


def launch_count() -> int:
    """number of sam6d_b200 kernels launched so far through the C ABI (bench.py reports the per-step delta)"""
    return _launches


def add_launches(n: int):
    """a captured forward replayed as one CUDA graph launches the kernels counted while it was captured"""
    global _launches
    _launches += int(n)


def time_kernel(name: str, enable: bool = True):
    """bracket every call of C-ABI function `name` with CUDA events on the launching (current) stream"""
    if enable:
        _timed[name] = []
    else:
        _timed.pop(name, None)


def timed_events(name: str):
    return _timed.get(name, [])


def call(name: str, *args):
    """calls C-ABI function `name`.  The trailing stream may be left out, and is then the current CUDA stream.  A tensor
    argument is passed as its device address; it must be a CUDA tensor, since every pointer the header declares is a
    device pointer.  Everything else goes to ctypes as it is: ints, floats, bools and None for NULL."""
    global _launches
    if _lib is None:
        lib()
    fn, n_before_stream = _fns[name]
    args = [(a.data_ptr() if a.is_cuda else _not_device(name, a)) if isinstance(a, _Tensor) else a for a in args]
    if len(args) == n_before_stream:
        args.append(torch.cuda.current_stream().cuda_stream)
    rec = _timed.get(name)
    if rec is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = fn(*args)
        e1.record()
        rec.append((e0, e1))
    else:
        rc = fn(*args)
    _launches += _MULTI.get(name, 1)
    if rc != 0:
        if rc == -22:
            raise Sam6dError(f"{name}: invalid argument (see include/sam6d_b200.h)")
        raise Sam6dError(f"{name}: CUDA error {rc}")
    return rc


def _not_device(name: str, t: torch.Tensor):
    raise Sam6dError(f"{name}: a {t.device} tensor where the C ABI takes a device pointer")


def version() -> str:
    return lib().sam6d_version().decode()
