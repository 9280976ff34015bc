"""Build liblb200.so (hand-written sm_90a CUDA + C ABI) in-tree with nvcc.

    python -m latentblending_b200.build        # or __graft_entry__.build()

nvcc cross-compiles without a GPU.  The .so lands next to this file so it
travels with the repo snapshot to the GPU box; objects go to csrc/_build/.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_build")
LIB = os.path.join(HERE, "liblb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stamp(src):
    h = hashlib.sha1()
    for f in [src] + sorted(os.path.join(CSRC, x) for x in os.listdir(CSRC) if x.endswith((".cuh", ".h"))) + \
            [os.path.join(HERE, "..", "include", "lb200.h")]:
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(name, verbose):
    src = os.path.join(CSRC, name)
    obj = os.path.join(OBJ, name[:-3] + ".o")
    stamp_file = obj + ".stamp"
    stamp = _stamp(src)
    if os.path.exists(obj) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return obj, False, ""
    cmd = [NVCC] + FLAGS + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {name}:\n{r.stdout}\n{r.stderr}")
    with open(stamp_file, "w") as fh:
        fh.write(stamp)
    return obj, True, r.stderr


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    with ThreadPoolExecutor(max_workers=8) as ex:
        results = list(ex.map(lambda n: _compile(n, verbose), _sources()))
    objs = [r[0] for r in results]
    rebuilt = any(r[1] for r in results)
    if verbose:
        for r in results:
            if r[2]:
                print(r[2])
    if rebuilt or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a",
                                                     "-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
