"""The one-pass backward kernel keeps its wgmma asynchronous.

ptxas serializes every wgmma of a kernel (a wait after each instruction) when a function call sits anywhere in it
(C7510, e.g. a ``printf`` in a watchdog) or when the asynchronous schedule does not fit the register budget (C7512).
Neither is an error, so nothing else would notice; the one-pass backward then runs at a fraction of its speed.
This reads the ``ptxas -v`` log of ``attn_bwd_sm90.cu`` left by the build, or compiles the file when that log is
missing or older than the sources.
"""
from __future__ import annotations

import os
import re
import shutil
import subprocess

import pytest

from ring_attention_pytorch_b200 import build as ext_build

SRC = ext_build.CSRC / "attn_bwd_sm90.cu"
LOG = ext_build.BUILD / "attn_bwd_sm90.cu.log"


def _ptxas_log(tmp_path) -> str:
    if LOG.exists():
        t = LOG.stat().st_mtime
        if all(f.stat().st_mtime <= t for f in [SRC, *ext_build._headers()]):
            return LOG.read_text()
    if not (shutil.which(ext_build.NVCC) or os.path.exists(ext_build.NVCC)):
        pytest.skip("nvcc not available and no current build log")
    cmd = [ext_build.NVCC, *ext_build.NVCC_FLAGS, "-I", str(ext_build.CSRC), "-c", str(SRC),
           "-o", str(tmp_path / "attn_bwd_sm90.o")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    return proc.stdout + proc.stderr


def test_one_pass_backward_wgmma_not_serialized(tmp_path):
    log = _ptxas_log(tmp_path)
    one_pass = set(re.findall(r"Compiling entry function '(\S*attn_bwd_dkv_kernel\S*AttnBwdFusedParams\S*)'", log))
    assert len(one_pass) == 4, "expected the four one-pass instantiations (bf16/fp16 x documents on/off) in the log"
    serialized = re.findall(r"\((C751\d)\) Potential Performance Loss: wgmma.mma_async instructions are serialized"
                            r".*function '(\S+)'", log)
    bad = [(code, fn) for code, fn in serialized if fn in one_pass]
    assert not bad, f"ptxas serialized the one-pass backward's wgmma: {bad}"
