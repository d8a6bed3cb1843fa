"""The ctypes mirrors in shasta_b200/capi.py against include/shasta_b200.h: sizes and field offsets as gcc lays the C structs out,
for every struct the header defines."""
import ctypes as C
import os
import re
import subprocess

from shasta_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = {"shb_lowhash_params": capi.LowHashParams, "shb_lowhash_result": capi.LowHashResult, "shb_align_options": capi.AlignOptions,
         "shb_align_result": capi.AlignResult, "shb_marker_result": capi.MarkerResult, "shb_dist_timing": capi.DistTiming,
         "shb_read_graph2_criteria": capi.ReadGraph2Criteria, "shb_cross_strand_result": capi.CrossStrandResult,
         "shb_chimeric_result": capi.ChimericResult, "shb_palindromic_params": capi.PalindromicParams,
         "shb_palindromic_result": capi.PalindromicResult, "shb_marker_graph_params": capi.MarkerGraphParams,
         "shb_marker_graph_result": capi.MarkerGraphResult}


def test_every_header_struct_has_a_mirror():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "shasta_b200.h")).read(), flags=re.S)
    defined = set(re.findall(r"typedef\s+struct\s*\w*\s*\{[^}]*\}\s*(shb_\w+)\s*;", text))
    assert "shb_context" not in defined      # opaque: declared, never defined
    assert len(defined) == 13 and defined == set(PAIRS)


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
    out = subprocess.check_output([str(exe)], text=True)
    seen = 0
    for line in out.splitlines():
        cname, what, value = re.match(r"(\w+) (\w+) (\d+)", line).groups()
        cls = PAIRS[cname]
        if what == "size":
            assert C.sizeof(cls) == int(value), cname
        else:
            assert getattr(cls, what).offset == int(value), (cname, what)
        seen += 1
    assert seen == sum(len(c._fields_) + 1 for c in PAIRS.values())
