"""In-tree build of libtce_b200.so (nvcc, sm_90a only)."""
from __future__ import annotations

import os
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
LIB = PKG / "lib" / "libtce_b200.so"


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA source of the package for sm_90a (cross-compiles without a GPU)."""
    if force:
        subprocess.run(["make", "-C", str(PKG / "csrc"), "clean"], check=True, capture_output=not verbose)
    jobs = str(max(1, min(8, os.cpu_count() or 1)))
    r = subprocess.run(["make", "-C", str(PKG / "csrc"), "-j", jobs], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("libtce_b200 build failed:\n" + r.stdout[-4000:] + r.stderr[-4000:])
    if verbose:
        print(r.stdout)
    if not LIB.exists():
        raise RuntimeError(f"build finished but {LIB} is missing")
    return LIB
