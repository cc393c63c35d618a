"""og_rows_field / og_rows_series / og_rows_desc / og_rows_info: the ctypes mirrors in _lib.py match include/ogpu.h (no GPU needed)."""
import ctypes as C
import os
import subprocess

import pytest

from opengemini_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("struct,mirror", [("og_rows_field", L.RowsField), ("og_rows_series", L.RowsSeries),
                                           ("og_rows_desc", L.RowsDesc), ("og_rows_info", L.RowsInfo)])
def test_rows_layout_matches_the_header(tmp_path, struct, mirror):
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "ogpu.h")}"', "int main(void) {",
             f'  printf("size %zu\\n", sizeof({struct}));']
    for name, _t in mirror._fields_:
        lines.append(f'  printf("{name} %zu\\n", offsetof({struct}, {name}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "ri.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "ri"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)
    seen = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.strip().splitlines())
    assert int(seen["size"]) == C.sizeof(mirror)
    for name, _t in mirror._fields_:
        assert int(seen[name]) == getattr(mirror, name).offset, name
