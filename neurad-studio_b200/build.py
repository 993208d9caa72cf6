"""Build libb200nerf.so (sm_90a) in-tree with nvcc.  No JIT cache: build() writes the .so next to the package sources."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libb200nerf.so")
SOURCES = ["b200nerf.cu"]
HEADERS = ["nff_device.h", "nff_lane.h", "tc_mlp.cuh", "rgb_decoder.cuh", "nff_modules.h", "modules.cuh", "nff_params.h", "simt.h", "lidar_eval.cuh", "lidar_loss.cuh", "image_metrics.cuh", "camera_rays.h", "lidar_sim.cuh", os.path.join("..", "..", "include", "b200nerf.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (needed to build libb200nerf.so)")


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile the CUDA library if it is missing or stale; returns its path."""
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH] + SOURCES
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return LIB_PATH


def build_variant(name: str, defines=(), verbose: bool = False) -> str:
    """A/B builds for GPU experiments (tools/perf_probe.py picks one with NFF_LIB=...): the same sources with extra -D
    switches, written to lib/variants/libb200nerf_<name>.so.  Never loaded by the product."""
    out_dir = os.path.join(LIB_DIR, "variants")
    os.makedirs(out_dir, exist_ok=True)
    out = os.path.join(out_dir, f"libb200nerf_{name}.so")
    cmd = [_nvcc()] + NVCC_FLAGS + [f"-D{d}" for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + SOURCES
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return out


if __name__ == "__main__":
    import sys

    if len(sys.argv) > 1:  # python build.py <variant-name> [DEFINE=VALUE ...]
        print(build_variant(sys.argv[1], sys.argv[2:], verbose=True))
    else:
        print(build(force=True, verbose=True))
