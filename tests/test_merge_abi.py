"""og_merge_info: the ctypes mirror in _lib.py matches include/ogpu.h (no GPU needed)."""
import ctypes as C
import os
import subprocess

from opengemini_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_merge_info_layout_matches_the_header(tmp_path):
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "ogpu.h")}"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(og_merge_info));',
             '  printf("flag %u\\n", (unsigned)OG_FILE_OUT_OF_ORDER);']
    for name, _t in L.MergeInfo._fields_:
        lines.append(f'  printf("{name} %zu\\n", offsetof(og_merge_info, {name}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "mi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "mi"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)
    seen = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.strip().splitlines())
    assert int(seen["size"]) == C.sizeof(L.MergeInfo)
    assert int(seen["flag"]) == L.FILE_OUT_OF_ORDER
    for name, _t in L.MergeInfo._fields_:
        assert int(seen[name]) == getattr(L.MergeInfo, name).offset, name
