"""The test-only probe of the regression head's training kernels (tests/csrc/head_train_probe.cu) builds with the
library, loads on a CPU-only host and exports exactly the wrappers tests/head_train_probe.py binds, with the HlGemm
layout the binding mirrors, and none of the library's internals (no compute calls here)."""
import ctypes
import re
import shutil
import subprocess
from pathlib import Path

import pytest

import head_train_probe

CSRC = Path(__file__).resolve().parent / "csrc" / "head_train_probe.cu"


def test_head_train_probe_builds_and_exports_every_bound_wrapper(built_lib):
    from tokenhmr_b200 import _build
    assert _build.HEAD_PROBE_PATH == head_train_probe.PROBE_PATH and head_train_probe.PROBE_PATH.exists()
    assert _build.HEAD_PROBE_STAMP.read_text().strip() == _build.source_hash(probe=True)
    defined = set(re.findall(r"^HEAD_PROBE_API\s+[\w\s\*]+?\b(head_probe_\w+)\s*\(", CSRC.read_text(), flags=re.M))
    assert defined == set(head_train_probe.SIGNATURES), defined ^ set(head_train_probe.SIGNATURES)
    L = head_train_probe.lib()
    for name in head_train_probe.SIGNATURES:
        assert hasattr(L, name), f"{name} is bound in tests/head_train_probe.py but not exported"
    assert L.head_probe_hl_gemm_desc_size() == ctypes.sizeof(head_train_probe.HlGemm)
    assert L.head_probe_hl_split_floats() == 264 * 64 * 64          # kSplitTarget x one 64 x 64 tile


def test_head_train_probe_keeps_the_library_internals_private(built_lib):
    """Its launchers' static state (rh_configure's 'attributes set' flag) must not merge with the library's."""
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("no nm")
    out = subprocess.run([nm, "-D", "--defined-only", str(head_train_probe.PROBE_PATH)], check=True,
                         capture_output=True, text=True).stdout
    names = [ln.split()[-1] for ln in out.splitlines() if ln.strip()]
    assert set(head_train_probe.SIGNATURES) <= set(names), set(head_train_probe.SIGNATURES) - set(names)
    leaked = [n for n in names if "thmr" in n]
    assert not leaked, leaked[:10]
