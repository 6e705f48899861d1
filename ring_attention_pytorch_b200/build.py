"""In-tree build of the sm_90a extension (``ring_attention_pytorch_b200/_C.so``).

Kernels (.cu) are compiled straight with nvcc for ``compute_90a/sm_90a`` and never include torch
headers, so a kernel edit rebuilds in seconds; only ``bindings.cpp`` sees torch.  The resulting shared
object is loaded with ``torch.ops.load_library`` from the package directory (no JIT cache involved).

    python -m ring_attention_pytorch_b200.build          # incremental
    python -m ring_attention_pytorch_b200.build --force  # rebuild everything
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
BUILD = PKG_DIR / "_build"
SO_PATH = PKG_DIR / "_C.so"

CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")

CU_SOURCES = [
    "attn_fwd_sm90.cu",
    "attn_bwd_sm90.cu",
    "tree_decode_sm90.cu",
    "tree_decode_tc_sm90.cu",
    "elementwise_sm90.cu",
]
CPP_SOURCES = ["tmap.cpp", "symm.cpp"]
TORCH_CPP_SOURCES = ["bindings.cpp"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _headers():
    return sorted(list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")))


def _stale(obj: Path, src: Path) -> bool:
    if not obj.exists():
        return True
    t = obj.stat().st_mtime
    if src.stat().st_mtime > t:
        return True
    return any(h.stat().st_mtime > t for h in _headers())


def _run(cmd, log: Path | None = None):
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if log is not None:
        log.write_text(proc.stdout + proc.stderr)
    if proc.returncode != 0:
        sys.stderr.write(" ".join(map(str, cmd)) + "\n" + proc.stdout + proc.stderr)
        raise RuntimeError(f"build step failed: {cmd[0]} {cmd[-1]}")
    return proc


def _torch_paths():
    import torch  # noqa: F401
    from torch.utils import cpp_extension as ce

    inc = ce.include_paths()
    lib = [str(Path(torch.__file__).parent / "lib")]
    return inc, lib


def build(force: bool = False, verbose: bool = True) -> Path:
    BUILD.mkdir(exist_ok=True)
    sources = [s for s in CU_SOURCES if (CSRC / s).exists()]
    jobs = []
    objs = []
    inc_torch, lib_torch = _torch_paths()
    cxx = os.environ.get("CXX", "g++")
    py_inc = sysconfig.get_paths()["include"]
    abi = None
    try:
        import torch

        abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    except Exception:
        abi = 1

    for s in sources:
        src, obj = CSRC / s, BUILD / (s + ".o")
        objs.append(obj)
        if force or _stale(obj, src):
            cmd = [NVCC, *NVCC_FLAGS, "-I", str(CSRC), "-c", str(src), "-o", str(obj)]
            jobs.append((cmd, BUILD / (s + ".log")))
    for s in CPP_SOURCES:
        src, obj = CSRC / s, BUILD / (s + ".o")
        objs.append(obj)
        if force or _stale(obj, src):
            cmd = [cxx, "-O2", "-std=c++17", "-fPIC", "-I", str(CSRC), "-I", os.path.join(CUDA_HOME, "include"),
                   "-c", str(src), "-o", str(obj)]
            jobs.append((cmd, None))
    for s in TORCH_CPP_SOURCES:
        src, obj = CSRC / s, BUILD / (s + ".o")
        objs.append(obj)
        if force or _stale(obj, src):
            cmd = [cxx, "-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-I", str(CSRC),
                   "-I", os.path.join(CUDA_HOME, "include"), "-I", py_inc]
            for i in inc_torch:
                cmd += ["-isystem", i]
            cmd += ["-c", str(src), "-o", str(obj)]
            jobs.append((cmd, None))

    if jobs:
        if verbose:
            print(f"[build] compiling {len(jobs)} translation unit(s) for sm_90a ...", flush=True)
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(lambda j: _run(j[0], j[1]), jobs))

    need_link = force or bool(jobs) or not SO_PATH.exists()
    if need_link:
        cuda_lib = os.path.join(CUDA_HOME, "lib64")
        cmd = [cxx, "-shared", "-o", str(SO_PATH), *map(str, objs)]
        for l in lib_torch:
            cmd += [f"-L{l}", f"-Wl,-rpath,{l}"]
        cmd += [f"-L{cuda_lib}", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-lcudart"]
        _run(cmd)
        if verbose:
            print(f"[build] linked {SO_PATH}", flush=True)
    return SO_PATH


def ptxas_report() -> str:
    """Concatenated ``ptxas -v`` output (registers / spills / smem) of the last build."""
    out = []
    for log in sorted(BUILD.glob("*.log")):
        out.append(f"== {log.name}\n{log.read_text()}")
    return "\n".join(out)


if __name__ == "__main__":
    if not shutil.which(NVCC) and not os.path.exists(NVCC):
        raise SystemExit(f"nvcc not found at {NVCC}")
    build(force="--force" in sys.argv)
    if "--report" in sys.argv:
        print(ptxas_report())
