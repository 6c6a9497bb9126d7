"""Build libsam6d_b200.so in-tree with nvcc for sm_90a (one translation unit per .cu, linked into one C-ABI library)."""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libsam6d_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + [
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stamp(path):
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cuh", ".h")):
            with open(os.path.join(CSRC, f), "rb") as fh:
                h.update(fh.read())
    with open(path, "rb") as fh:
        h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src):
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src[:-3] + ".o")
    stamp_file = obj + ".stamp"
    stamp = _stamp(path)
    if os.path.exists(obj) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return obj, False
    cmd = [NVCC] + FLAGS + ["-c", path, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    with open(stamp_file, "w") as fh:
        fh.write(stamp)
    return obj, True


def build(verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        res = list(ex.map(_compile, _sources()))
    objs = [o for o, _ in res]
    if any(changed for _, changed in res) or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ARCH + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    if verbose:
        print(f"built {LIB} from {len(objs)} objects ({sum(c for _, c in res)} recompiled)")
    return LIB


if __name__ == "__main__":
    build(verbose=True)
    sys.exit(0)
