"""Builds libtokenhmr_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU), and next to the test suite
the probe library tests/libthmr_probe.so (tests/csrc/kernel_probe.cu: test-only wrappers around the internal launchers
of every mode, the fused SMPLify-inverse's loss and Adam kernels, and the skeleton overlay's span generator run on the
host), the GEMM plan probe tests/libthmr_gemm_probe.so (tests/csrc/gemm_probe.cu: forced epilogue kinds, plan
queries and the per-tile timeline kernels, which the product does not compile) and the head-training probe
tests/libthmr_head_train_probe.so (tests/csrc/head_train_probe.cu: the training kernels of csrc/head_train.cuh and
csrc/token_head_train.cuh)."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libtokenhmr_b200.so"
STAMP = PKG_DIR / ".libtokenhmr_b200.stamp"
PROBE_SRC = PKG_DIR.parent / "tests" / "csrc" / "kernel_probe.cu"
PROBE_PATH = PKG_DIR.parent / "tests" / "libthmr_probe.so"
PROBE_STAMP = PKG_DIR.parent / "tests" / ".libthmr_probe.stamp"
GEMM_PROBE_SRC = PKG_DIR.parent / "tests" / "csrc" / "gemm_probe.cu"
GEMM_PROBE_PATH = PKG_DIR.parent / "tests" / "libthmr_gemm_probe.so"
GEMM_PROBE_STAMP = PKG_DIR.parent / "tests" / ".libthmr_gemm_probe.stamp"
HEAD_PROBE_SRC = PKG_DIR.parent / "tests" / "csrc" / "head_train_probe.cu"
HEAD_PROBE_PATH = PKG_DIR.parent / "tests" / "libthmr_head_train_probe.so"
HEAD_PROBE_STAMP = PKG_DIR.parent / "tests" / ".libthmr_head_train_probe.stamp"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC", "-shared",
]
# The probe is loaded into the same process as the library and compiles the same inline functions, whose static locals
# (e.g. the "kernel attributes configured" flags of the launchers) would otherwise be merged with the library's by the
# dynamic linker.  Hidden visibility keeps every one of them private to the probe; its wrappers are exported explicitly.
PROBE_FLAGS = ["-Xcompiler", "-fvisibility=hidden"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def source_hash(probe: bool = False) -> str:
    h = hashlib.sha256()
    files = sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cuh")) + sorted((PKG_DIR.parent / "include").glob("*.h"))
    if probe:
        files += sorted(PROBE_SRC.parent.glob("*.cu"))
    for f in files:
        h.update(f.name.encode())
        h.update(f.read_bytes())
    h.update(" ".join(NVCC_FLAGS + (PROBE_FLAGS if probe else [])).encode())
    return h.hexdigest()


def _compile(src: Path, out: Path, stamp: Path, flags: list, want: str, force: bool, verbose: bool) -> Path:
    if not force and out.exists() and stamp.exists() and stamp.read_text().strip() == want:
        return out
    cmd = [_nvcc(), *flags, "-o", str(out), str(src)]  # cudart linked statically (nvcc default)
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), file=sys.stderr)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed ({res.returncode}):\n{res.stdout}\n{res.stderr}")
    if verbose:
        print(res.stderr, file=sys.stderr)
    stamp.write_text(want)
    return out


def build_probe(force: bool = False, verbose: bool = False) -> Path:
    """Compile tests/csrc/kernel_probe.cu -> tests/libthmr_probe.so, tests/csrc/gemm_probe.cu ->
    tests/libthmr_gemm_probe.so and tests/csrc/head_train_probe.cu -> tests/libthmr_head_train_probe.so (each a no-op
    when sources are unchanged)."""
    for src, out, stamp in ((GEMM_PROBE_SRC, GEMM_PROBE_PATH, GEMM_PROBE_STAMP),
                            (HEAD_PROBE_SRC, HEAD_PROBE_PATH, HEAD_PROBE_STAMP)):
        if src.exists():
            _compile(src, out, stamp, NVCC_FLAGS + PROBE_FLAGS, source_hash(probe=True), force, verbose)
    return _compile(PROBE_SRC, PROBE_PATH, PROBE_STAMP, NVCC_FLAGS + PROBE_FLAGS, source_hash(probe=True), force,
                    verbose)


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile csrc/tokenhmr_b200.cu -> libtokenhmr_b200.so, and the probe library when the test sources are present
    (no-op when sources are unchanged)."""
    path = _compile(CSRC / "tokenhmr_b200.cu", LIB_PATH, STAMP, NVCC_FLAGS, source_hash(), force, verbose)
    if PROBE_SRC.exists():
        build_probe(force, verbose)
    return path


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
