"""The ctypes mirrors of shb_cross_strand_result and shb_chimeric_result against include/shasta_b200.h, and the two new
symbols of the library."""
import ctypes as C
import os
import re
import subprocess

from shasta_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = {"shb_cross_strand_result": capi.CrossStrandResult, "shb_chimeric_result": capi.ChimericResult}


def test_struct_sizes_and_offsets(tmp_path):
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "shasta_b200.h"', 'int main(void) {']
    for cname, cls in PAIRS.items():
        lines.append(f'printf("{cname} size %zu\\n", sizeof({cname}));')
        for field, _ in cls._fields_:
            lines.append(f'printf("{cname} {field} %zu\\n", offsetof({cname}, {field}));')
    lines += ['return 0; }']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    seen = 0
    for line in subprocess.check_output([str(exe)], text=True).splitlines():
        cname, what, value = re.match(r"(\w+) (\w+) (\d+)", line).groups()
        cls = PAIRS[cname]
        assert (C.sizeof(cls) if what == "size" else getattr(cls, what).offset) == int(value), (cname, what)
        seen += 1
    assert seen == sum(len(c._fields_) + 1 for c in PAIRS.values())


def test_symbols_exported():
    lib = capi.lib()
    for name in ("shb_flag_cross_strand_read_graph_edges1", "shb_flag_chimeric_reads"):
        assert hasattr(lib, name), name
