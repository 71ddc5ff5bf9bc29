"""Build libts_b200.so in-tree with nvcc for sm_90a (H100; no torch extension machinery: the library is
a plain C-ABI shared object loaded with ctypes, see tianshou_b200/_cabi.py)."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["capi.cu", "gae.cu", "nstep.cu", "index.cu", "segtree.cu", "mlp.cu", "mlp_tc.cu", "peer.cu", "hostperm.cu", "net_gemm.cu", "net_ops.cu", "ppo_rows.cu", "npg.cu", "gail.cu",
           "discrete_sac.cu", "cql.cu", "td3.cu", "bcq.cu", "discrete_bcq.cu", "discrete_crr.cu", "qrdqn.cu", "iqn.cu", "fqf.cu", "redq.cu", "bdqn.cu", "c51.cu", "rainbow.cu", "lstm.cu", "imitation.cu", "icm.cu", "psrl.cu", "hostperm_simd.cpp"]      # .cpp = host-only, compiled by g++
DIAG_SOURCES = ["umma_selftest.cu"]       # diagnostics library only (-DTS_B200_DIAGNOSTICS: phase timeline + wgmma self-test)
LIB = os.path.join(os.path.dirname(HERE), "libts_b200.so")
DIAG_LIB = os.path.join(os.path.dirname(HERE), "libts_b200_diag.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = os.environ.get("CXX", "g++")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [
    *ARCH,
    "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _newer(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def build(force: bool = False, verbose: bool = False, diag: bool = False) -> str:
    """Product library (default) or, with ``diag``, the diagnostics build ``libts_b200_diag.so`` (same sources compiled with
    -DTS_B200_DIAGNOSTICS plus the wgmma self-test; used by tools/tc_timeline.py and tools/umma_probe.py only)."""
    hdrs = [os.path.join(HERE, "common.cuh"), os.path.join(HERE, "..", "..", "include", "ts_b200.h")]
    hdrs += [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".cuh", ".h"))]
    srcs = [os.path.join(HERE, s) for s in SOURCES + (DIAG_SOURCES if diag else [])]
    lib = DIAG_LIB if diag else LIB
    flags = FLAGS + (["-DTS_B200_DIAGNOSTICS"] if diag else [])
    if not force and _newer(lib, srcs + hdrs + [os.path.abspath(__file__)]):
        return lib
    objdir = os.path.join(HERE, "build_diag" if diag else "build")
    os.makedirs(objdir, exist_ok=True)

    def compile_one(src: str) -> str:
        obj = os.path.join(objdir, os.path.splitext(os.path.basename(src))[0] + ".o")
        if not force and _newer(obj, [src, *hdrs]):
            return obj
        if src.endswith(".cpp"):
            cmd = [CXX, "-O3", "-std=c++17", "-fPIC", "-g1", "-c", src, "-o", obj]
        else:
            cmd = [NVCC, *flags, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(obj + ".log", "w") as f:
            f.write(log)
        if r.returncode != 0:
            sys.stderr.write(log)
            raise RuntimeError(f"compiler failed for {src}")
        if verbose:
            sys.stderr.write(log)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    tmp = lib + ".tmp"      # link next to the target and rename: a reader never sees a half-written library
    cmd = [NVCC, "-shared", "-o", tmp, *objs, *ARCH, "-lcudart", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    os.replace(tmp, lib)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, diag="--diag" in sys.argv))
