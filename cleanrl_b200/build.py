"""Compile libb200rl.so in-tree with nvcc for sm_90a (no JIT cache, no torch headers).

``python -m cleanrl_b200.build`` or ``__graft_entry__.build()``.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libb200rl.so"
STAMP = PKG / ".libb200rl.stamp"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-DB200RL_ARCH=90",
]


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _digest():
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "b200rl.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def find_nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libb200rl.so")
    return nvcc


def build(force=False, verbose=False):
    """Build (or reuse an up-to-date) cleanrl_b200/libb200rl.so; returns its path."""
    dig = _digest()
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == dig:
        return LIB
    nvcc = find_nvcc()
    cmd = [nvcc] + NVCC_FLAGS + [str(s) for s in _sources()] + ["-o", str(LIB)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), file=sys.stderr)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr, file=sys.stderr)
    STAMP.write_text(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
