"""The test-only kernel probe (tests/csrc/kernel_probe.cu) builds with the library, loads on a CPU-only host and exports
exactly the wrappers tests/probe.py binds (no compute calls here)."""
import ctypes
import re
from pathlib import Path

import probe

CSRC = Path(__file__).resolve().parent / "csrc" / "kernel_probe.cu"


def test_probe_builds_and_exports_every_bound_wrapper(built_lib):
    from tokenhmr_b200 import _build
    assert _build.PROBE_PATH == probe.PROBE_PATH and probe.PROBE_PATH.exists()
    assert _build.PROBE_STAMP.read_text().strip() == _build.source_hash(probe=True)
    defined = set(re.findall(r"^PROBE_API\s+[\w\s\*]+?\b(probe_\w+)\s*\(", CSRC.read_text(), flags=re.M))
    assert defined == set(probe.SIGNATURES), defined ^ set(probe.SIGNATURES)
    L = probe.lib()
    for name in probe.SIGNATURES:
        assert hasattr(L, name), f"{name} is bound in tests/probe.py but not exported"
    assert L.probe_gemm_desc_size() == ctypes.sizeof(probe.GemmDesc)


def test_probe_keeps_the_library_internals_private(built_lib):
    """Only the probe_* wrappers are exported: the probe compiles the same inline launchers as the library, and a shared
    symbol would let one library's static state (e.g. a launcher's 'kernel attributes configured' flag) stand in for
    the other's."""
    import shutil
    import subprocess
    nm = shutil.which("nm")
    if nm is None:
        import pytest
        pytest.skip("no nm")
    out = subprocess.run([nm, "-D", "--defined-only", str(probe.PROBE_PATH)], check=True, capture_output=True,
                         text=True).stdout
    names = [ln.split()[-1] for ln in out.splitlines() if ln.strip()]
    leaked = [n for n in names if "thmr" in n]
    assert not leaked, leaked[:10]
