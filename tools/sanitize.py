#!/usr/bin/env python
"""Run small forward / backward / decode cases under ``compute-sanitizer`` (memcheck, racecheck, synccheck,
initcheck) — the race-detection subsystem the reference lacks (SURVEY §5: it relies on ``tl.debug_barrier()``
work-arounds, triton_flash_attn.py:648-728).

    python tools/sanitize.py                       # all tools, default cases, log in sanitize.log (temporary directory)
    python tools/sanitize.py --tools memcheck --cases fwd_d128_causal_n1000

Cases are the names of ``tools/gpu_dev_check.py``; every case runs in its own process so one report cannot hide
another.  The exit code is non-zero if any tool reports an error.
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_CASES = "fwd_d128_causal_n1000,ring3_kmask,bwd_d128_causal_n1000,rbwd4_striped_causal"
DEFAULT_TOOLS = "memcheck,racecheck,synccheck"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tools", default=DEFAULT_TOOLS)
    ap.add_argument("--cases", default=DEFAULT_CASES)
    ap.add_argument("--timeout", type=int, default=420, help="seconds per (tool, case)")
    ap.add_argument("--log", default=os.path.join(tempfile.gettempdir(), "sanitize.log"))
    args = ap.parse_args()
    os.makedirs(os.path.dirname(args.log), exist_ok=True)
    sanitizer = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "compute-sanitizer")
    failed = 0
    with open(args.log, "w") as log:
        for tool in args.tools.split(","):
            for case in args.cases.split(","):
                cmd = [sanitizer, "--tool", tool, "--print-limit", "20", "--error-exitcode", "99", sys.executable,
                       os.path.join(ROOT, "tools", "gpu_dev_check.py"), "--case", case]
                t0 = time.time()
                try:
                    proc = subprocess.run(cmd, capture_output=True, text=True, timeout=args.timeout, cwd=ROOT)
                    out, code = proc.stdout + proc.stderr, proc.returncode
                except subprocess.TimeoutExpired as e:
                    out = ((e.stdout or b"").decode(errors="replace") if isinstance(e.stdout, bytes) else (e.stdout or ""))
                    code = -1
                m = re.search(r"ERROR SUMMARY: (\d+) error", out)
                errors = int(m.group(1)) if m else None
                if errors is None:  # racecheck prints "RACECHECK SUMMARY: N hazards displayed (E errors, W warnings)"
                    m = re.search(r"RACECHECK SUMMARY: (\d+) hazard", out)
                    errors = int(m.group(1)) if m else None
                ok_line = next((l[7:] for l in out.splitlines() if l.startswith("RESULT ")), "")
                status = "timeout" if code == -1 else ("clean" if errors == 0 and code == 0 else "ERRORS")
                line = f"[{tool}] {case}: {status} (errors={errors}, exit={code}, {time.time() - t0:.0f}s) {ok_line}"
                print(line, flush=True)
                log.write(line + "\n")
                if status == "ERRORS":
                    failed += 1
                    log.write(out[-6000:] + "\n")
                log.flush()
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
