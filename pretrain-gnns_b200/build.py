"""Build libpgnn_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python pretrain-gnns_b200/build.py [--force]

One object per csrc/*.cu (compiled in parallel, skipped when newer than its sources), linked into
`pretrain-gnns_b200/libpgnn_b200.so` with the static CUDA runtime so the library depends on nothing
but the driver.  No torch headers are involved: the boundary is the C ABI of include/pgnn_b200.h.
"""
import concurrent.futures
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# PGNN_BUILD_DIR / PGNN_LIB_OUT: scratch build elsewhere (compile checks that must not touch the in-tree library)
OBJ = os.environ.get("PGNN_BUILD_DIR") or os.path.join(HERE, "csrc", "_obj")
LIB = os.environ.get("PGNN_LIB_OUT") or os.path.join(HERE, "libpgnn_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _newer(target, deps):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def _compile(src, force):
    obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
    deps = [src] + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    if not force and _newer(obj, deps):
        return obj, False
    cmd = [NVCC] + ARCH + FLAGS + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj, True


def build(force=False, verbose=True):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, force), srcs))
    objs = [o for o, _ in res]
    if force or any(c for _, c in res) or not _newer(LIB, objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
        if verbose:
            print("built", LIB)
    elif verbose:
        print("up to date:", LIB)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
