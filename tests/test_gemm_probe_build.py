"""The test-only GEMM plan probe (tests/csrc/gemm_probe.cu) builds with the library, loads on a CPU-only host and
exports exactly the wrappers tests/gemm_probe.py binds, with the descriptor layout the binding mirrors (no compute
calls here)."""
import ctypes
import re
from pathlib import Path

import gemm_probe

CSRC = Path(__file__).resolve().parent / "csrc" / "gemm_probe.cu"


def test_gemm_probe_builds_and_exports_every_bound_wrapper(built_lib):
    from tokenhmr_b200 import _build
    assert _build.GEMM_PROBE_PATH == gemm_probe.PROBE_PATH and gemm_probe.PROBE_PATH.exists()
    assert _build.GEMM_PROBE_STAMP.read_text().strip() == _build.source_hash(probe=True)
    defined = set(re.findall(r"^GEMM_PROBE_API\s+[\w\s\*]+?\b(gemm_probe_\w+)\s*\(", CSRC.read_text(), flags=re.M))
    assert defined == set(gemm_probe.SIGNATURES), defined ^ set(gemm_probe.SIGNATURES)
    L = gemm_probe.lib()
    for name in gemm_probe.SIGNATURES:
        assert hasattr(L, name), f"{name} is bound in tests/gemm_probe.py but not exported"
    assert L.gemm_probe_desc_size() == ctypes.sizeof(gemm_probe.GemmDesc)
