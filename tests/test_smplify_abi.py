"""thmr_smplify_desc (include/tokenhmr_b200.h) and its ctypes mirror _lib.SmplifyDesc agree field for field and in size,
and thmr_smplify_workspace_bytes is pure arithmetic that rejects bad sizes (no compute calls here)."""
import ctypes
import re
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def test_smplify_desc_fields_in_header_order():
    from tokenhmr_b200 import _lib
    text = (ROOT / "include" / "tokenhmr_b200.h").read_text()
    body = re.search(r"typedef struct thmr_smplify_desc \{(.*?)\} thmr_smplify_desc;", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    declared = re.findall(r"\b([A-Za-z_0-9]+)\s*(?=[,;])", body)
    assert declared == [n for n, _ in _lib.SmplifyDesc._fields_]


def test_smplify_desc_size_matches_c(tmp_path):
    from tokenhmr_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "size.c"
    src.write_text(f'#include <stdio.h>\n#include "{ROOT / "include" / "tokenhmr_b200.h"}"\n'
                   'int main(void) { printf("%zu", sizeof(thmr_smplify_desc)); return 0; }\n')
    exe = tmp_path / "size"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-o", str(exe), str(src)], check=True, capture_output=True)
    assert int(subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout) == \
        ctypes.sizeof(_lib.SmplifyDesc)


def test_smplify_workspace_rejects_bad_sizes(built_lib):
    assert built_lib.thmr_smplify_workspace_bytes(None, 4, 10) == 0
