"""Build libphc_b200.so (hand-written sm_90a CUDA + the C ABI of include/phc_b200.h) in-tree with nvcc.

    python -m phc_b200.build            # incremental (per-file mtime check)
    python -m phc_b200.build --force

No torch headers are involved: the library is a plain C-ABI shared object (extern "C", raw pointers, a
cudaStream_t as void*); it links only against libcudart.  nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "lib")
OBJ_DIR = os.path.join(OUT_DIR, "obj")
LIB_PATH = os.path.join(OUT_DIR, "libphc_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
          "--expt-relaxed-constexpr"]
# per-file extra flags.  The env-side arithmetic mirrors the reference expression by expression: FMA contraction is off
# in the off-step kernels and, in the fused step kernel, pinned off at the ill-conditioned spots by explicit intrinsics
# (phc_math.cuh explains which and why; PHC_ENV_FMAD=0 builds the step kernel without any contraction for A/B checks).
SOURCES = {
    "phc_api.cu": [],
    "env_step.cu": ["-fmad=false"] if os.environ.get("PHC_ENV_FMAD", "1") == "0" else [],
    "env_step_fast.cu": [],
    "env_step_wide.cu": [],
    "getup.cu": [],
    "motion.cu": ["-fmad=false"],
    "motion_wide.cu": ["-fmad=false"],
    "motion_load.cu": ["-fmad=false"],
    "ppo_scalars.cu": ["-fmad=false"],
    "gemm.cu": [],
    "gemm_wgmma.cu": [],
    "ppo_update.cu": [],
}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _newer(src_files, target) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_files)


def build_variant(name: str, flags, source="env_step.cu") -> str:
    """Experiment builds: the same library with extra -D flags on ONE source file (or a
    list of them), written to lib/alt_<name>/libphc_b200.so; selected at run time with PHC_LIB_PATH.  Never the default."""
    out_dir = os.path.join(OUT_DIR, f"alt_{name}")
    os.makedirs(out_dir, exist_ok=True)
    nvcc = _nvcc()
    sources = [source] if isinstance(source, str) else list(source)
    alt = {}
    for src in sources:
        obj = os.path.join(out_dir, src.replace(".cu", ".o"))
        r = subprocess.run([nvcc] + ARCH + COMMON + SOURCES[src] + list(flags) + ["-c", os.path.join(CSRC, src), "-o", obj],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src} ({name}):\n{r.stderr}")
        alt[src] = obj
    build()
    objs = [alt.get(s, os.path.join(OBJ_DIR, s.replace(".cu", ".o"))) for s in SOURCES]
    lib = os.path.join(out_dir, "libphc_b200.so")
    r = subprocess.run([nvcc] + ARCH + ["-shared", "-o", lib] + objs + ["-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed ({name}):\n{r.stderr}")
    return lib


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = _nvcc()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "phc_b200.h"))
    headers.append(os.path.abspath(__file__))
    objs = []
    for src, extra in SOURCES.items():
        sp = os.path.join(CSRC, src)
        op = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
        objs.append(op)
        if force or _newer([sp] + headers, op):
            cmd = [nvcc] + ARCH + COMMON + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", sp, "-o", op]
            if verbose:
                print(" ".join(cmd))
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
            if verbose:
                print(r.stderr)
    if force or _newer(objs, LIB_PATH):
        cmd = [nvcc] + ARCH + ["-shared", "-o", LIB_PATH] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv or "--verbose" in sys.argv)
    print(p)
