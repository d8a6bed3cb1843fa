"""createMarkerGraphEdges, its source and target tables and findMarkerGraphReverseComplementEdges: the C restatement
(oracle/markergraph_edges_oracle.c) against the reference's own MarkerGraph, MultithreadedObject and MemoryMapped containers
driven in the members' control flow (oracle/ref_glue/ref_markergraph_edges.cpp). With one thread the reference's output is
fully determined and the restatement must equal it byte for byte, except the unnamed flag bits of each Edge; with every
core it must equal it in canonical form. The reference's outputs are stored in tests/golden/reference_markergraph_edges.npz,
each with a digest of its input; arrays above 4096 elements as their SHA-256."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import markergraph_edges_bindings as EB
import support  # noqa: F401  (tests/golden on sys.path)

from markergraph_edges_inputs import digest, rc_failure_inputs, vertex_cases
from reference_outputs import recorded, shrink

CASES = vertex_cases()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def exact_form(s):
    """The one-thread output: named Edge fields, interval toc and data, both tables as stored."""
    return dict(fields=EB.named_fields(s["edges"]), itoc=s["intervalsToc"], idata=s["intervalsData"], stoc=s["bySourceToc"],
                sdata=s["bySourceData"], ttoc=s["byTargetToc"], tdata=s["byTargetData"])


def canonical_form(s, rc=None):
    f, itoc, idata, stoc, sdata, ttoc, tdata, nrc = EB.canonical(s, rc)
    out = dict(fields=f, itoc=itoc, idata=idata, stoc=stoc, sdata=sdata, ttoc=ttoc, tdata=tdata)
    if nrc is not None:
        out["rc"] = nrc
    return out


def _input_digest(d):
    return digest(d["toc"], d["table"], d["vtoc"], d["vdata"])


def _ref_case(name):
    d = CASES[name]
    one = EB.ref_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"], threads=1)
    assert one["status"] == 0
    out = {f"one/{k}": shrink(v, 4096) for k, v in exact_form(one).items()}
    many = EB.ref_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"], threads=0)
    rc_many = None
    if d["rc"] is not None:
        msg, rc = EB.ref_find_rc_edges(d["toc"], d["rc"], one, threads=1)
        out["rc_message"] = msg or ""
        out["one/rc"] = shrink(rc if rc is not None else np.zeros(0, np.uint64), 4096)
        msg_many, rc_many = EB.ref_find_rc_edges(d["toc"], d["rc"], many, threads=0)
        assert msg_many == msg or (msg and msg_many)
    out.update({f"all/{k}": shrink(v, 4096) for k, v in canonical_form(many, rc_many).items()})
    out["input"] = _input_digest(d)
    return out


def _check(got, ref, prefix):
    for k, v in got.items():
        assert np.array_equal(shrink(v, 4096).reshape(-1), np.asarray(ref[f"{prefix}/{k}"]).reshape(-1)), f"{prefix}/{k}"


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference(name):
    d = CASES[name]
    ref = recorded("markergraph_edges", name, _ref_case, name)
    assert np.array_equal(ref["input"], _input_digest(d)), "the recorded input differs from this input"
    o = EB.oracle_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"])
    assert o["status"] == 0
    _check(exact_form(o), ref, "one")
    rc = None
    if d["rc"] is not None:
        msg, rc = EB.oracle_find_rc_edges(d["toc"], d["rc"], o)
        assert (msg or "") == ref["rc_message"]
        if rc is not None:
            assert np.array_equal(shrink(rc, 4096).reshape(-1), np.asarray(ref["one/rc"]).reshape(-1))
    _check(canonical_form(o, rc), ref, "all")


def test_cases_reach_every_branch():
    """Self-loops, capped coverage, long gaps, reads without vertices, zero vertices, permuted numberings and parallel-free
    (source, target) pairs: what the comparison above is meant to cover."""
    seen = set()
    for name, d in CASES.items():
        o = EB.oracle_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"])
        f = EB.named_fields(o["edges"])
        pairs = {tuple(x) for x in f[:, :2].tolist()}
        assert len(pairs) == len(f), name
        if (f[:, 0] == f[:, 1]).any():
            seen.add("self_loop")
        if (f[:, 2] == 255).any() and o["saturated"]:
            seen.add("saturated")
        if len(d["vtoc"]) == 1:
            seen.add("zero")
        gaps = np.asarray(o["intervalsData"], np.int64)
        if len(gaps) and (gaps[:, 2] - gaps[:, 1]).max() > 20000:
            seen.add("long_gap")
        first = np.asarray(d["vdata"])[np.asarray(d["vtoc"][:-1], np.int64)]
        if (np.diff(first.astype(np.int64)) < 0).any():
            seen.add("permuted")
    assert {"self_loop", "saturated", "zero", "long_gap", "permuted"} <= seen


def _ref_rc_failure(i):
    name, d, s = rc_failure_inputs(CASES["genome/cov2"])[i]
    msg, _ = EB.ref_find_rc_edges(d["toc"], d["rc"], s, threads=1)
    return dict(message=msg or "", input=digest(s["edges"], s["intervalsToc"], s["intervalsData"], s["bySourceToc"], s["bySourceData"]))


@pytest.mark.parametrize("i", [0, 1])
def test_rc_failures_give_the_reference_messages(i):
    name, d, s = rc_failure_inputs(CASES["genome/cov2"])[i]
    ref = recorded("markergraph_edges", f"rc_failure/{name}", _ref_rc_failure, i)
    assert np.array_equal(ref["input"], digest(s["edges"], s["intervalsToc"], s["intervalsData"], s["bySourceToc"], s["bySourceData"]))
    msg, rc = EB.oracle_find_rc_edges(d["toc"], d["rc"], s)
    assert rc is None and msg == str(ref["message"])
    assert msg.startswith("Unable to locate" if name == "missing_interval" else "Reverse complement edge check failed")


def test_rc_assertion_on_a_row_of_another_source():
    d = CASES["genome/cov2"]
    o = EB.oracle_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"])
    stoc = o["bySourceToc"].astype(np.int64)
    v = int(np.nonzero(np.diff(stoc) >= 1)[0][0])
    w = int(np.nonzero(np.diff(stoc) >= 1)[0][1])
    o["bySourceData"][stoc[v]], o["bySourceData"][stoc[w]] = o["bySourceData"][stoc[w]], o["bySourceData"][stoc[v]]
    msg, _ = EB.oracle_find_rc_edges(d["toc"], d["rc"], o)
    assert msg.startswith("Assertion failed: edgeRc.source == v1Rc")
    if EB.have_ref():
        ref_msg, _ = EB.ref_find_rc_edges(d["toc"], d["rc"], o, threads=1)
        assert ref_msg.startswith("Assertion failed: edgeRc.source == v1Rc")


def test_header_struct_layout(tmp_path):
    """shb_marker_graph_edges_result in include/shb_marker_graph_edges.h against its ctypes mirror, as gcc lays it out."""
    from shasta_b200 import capi
    cls = capi.MarkerGraphEdgesResult
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "shb_marker_graph_edges.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(shb_marker_graph_edges_result));']
    lines += [f'printf("{f} %zu\\n", offsetof(shb_marker_graph_edges_result, {f}));' for f, _ in cls._fields_]
    lines += ['return 0; }']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(out.pop("size")) == C.sizeof(cls)
    assert {f: int(v) for f, v in out.items()} == {f: getattr(cls, f).offset for f, _ in cls._fields_}
