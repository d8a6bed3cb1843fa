"""createMarkerGraphEdges and findMarkerGraphReverseComplementEdges on the GPU (csrc/markergraph_edges.cu) against the C
restatement (oracle/markergraph_edges_oracle.c), which tests/test_oracle_markergraph_edges.py pins to the reference's own
code. Both give the reference's one-thread output, so the device's outputs must equal the restatement's exactly."""
import os

import numpy as np
import pytest

from oracle import markergraph_edges_bindings as EB
from support import PaddedSet, ctx, device_read_graph, need_memory, pack_ordinal_markers  # noqa: F401

from markergraph_edges_inputs import drop_interval, large_vertex_case, parallel_edge, rc_failure_inputs, vertex_cases
from reference_outputs import recorded, shrink

pytestmark = pytest.mark.gpu
CASES = vertex_cases()


def _upload(ctx, toc):
    ctx.set_markers(toc, pack_ordinal_markers(toc, np.zeros(int(toc[-1]), np.uint32)), np.zeros((len(toc) - 1) // 2, np.uint8))


def _device(ctx, d):
    from shasta_b200 import capi
    return capi.create_marker_graph_edges(ctx, capi.uint64_to_uint40(d["table"]), capi.uint64_to_uint40(d["vtoc"]), d["vdata"])


def _as_oracle_set(out):
    s = dict(out)
    s["bySourceData"] = EB.rows_from_uint40(out["bySourceData"])
    s["byTargetData"] = EB.rows_from_uint40(out["byTargetData"])
    return s


def _check(ctx, d, rc_too=True):
    from shasta_b200 import capi
    o = EB.oracle_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"])
    assert o["status"] == 0
    out, res = _device(ctx, d)
    s = _as_oracle_set(out)
    assert np.array_equal(out["edges"], o["edges"]), "edge records differ"
    for k in ("intervalsToc", "intervalsData", "bySourceToc", "bySourceData", "byTargetToc", "byTargetData"):
        assert np.array_equal(np.asarray(s[k]).reshape(-1), np.asarray(o[k]).reshape(-1)), k
    assert res.edgeCount == len(o["edges"]) and res.markerIntervalCount == len(o["intervalsData"])
    assert res.saturatedEdgeCount == o["saturated"] and res.vertexCount == len(d["vtoc"]) - 1
    rc = None
    if rc_too and d["rc"] is not None:
        msg, orc = EB.oracle_find_rc_edges(d["toc"], d["rc"], o)
        assert msg is None
        rc, rres = capi.find_marker_graph_reverse_complement_edges(ctx, d["rc"], out["edges"], out["intervalsToc"], out["intervalsData"],
                                                                   out["bySourceToc"], out["bySourceData"])
        assert np.array_equal(rc, orc)
        assert rres.edgeCount == res.edgeCount and rres.saturatedEdgeCount == res.saturatedEdgeCount
    return out, res, rc


@pytest.mark.parametrize("name", sorted(CASES))
def test_cases_against_oracle_and_reference(ctx, name):
    d = CASES[name]
    _upload(ctx, d["toc"])
    out, _, rc = _check(ctx, d)
    # The reference's recorded one-thread output (tests/test_oracle_markergraph_edges.py records it).
    ref = recorded("markergraph_edges", name, lambda: None)
    got = dict(fields=EB.named_fields(out["edges"]), itoc=out["intervalsToc"], idata=out["intervalsData"], stoc=out["bySourceToc"],
               sdata=EB.rows_from_uint40(out["bySourceData"]), ttoc=out["byTargetToc"], tdata=EB.rows_from_uint40(out["byTargetData"]))
    for k, v in got.items():
        assert np.array_equal(shrink(v, 4096).reshape(-1), np.asarray(ref[f"one/{k}"]).reshape(-1)), k
    if rc is not None:
        assert np.array_equal(shrink(rc, 4096).reshape(-1), np.asarray(ref["one/rc"]).reshape(-1))


def test_byte_identical_runs(ctx):
    d = CASES["deep/strand1"]
    _upload(ctx, d["toc"])
    first, _, _ = _check(ctx, d)
    second, _ = _device(ctx, d)
    for k in first:
        assert first[k].tobytes() == second[k].tobytes(), k


def test_chunk_seams(ctx, monkeypatch):
    """Vertex chunks of a few markers (1 MB budget: about 13 000 markers; the hook's unit), rc launches of a few edges."""
    for name in ("genome/cov2", "deep/strand1", "long_gap", "coverage_cap"):
        d = CASES[name]
        _upload(ctx, d["toc"])
        for budget, rc_chunk in [(1, 1), (1, 7), (2, 1000)]:
            monkeypatch.setenv("SHB_MARKERGRAPH_EDGES_BUDGET_MB", str(budget))
            monkeypatch.setenv("SHB_MARKERGRAPH_EDGES_RC_CHUNK", str(rc_chunk))
            _check(ctx, d)


def test_large_vertices(ctx):
    """Vertices of more than 32 and more than 4096 markers: the block sort and the radix sort."""
    d = large_vertex_case()
    _upload(ctx, d["toc"])
    sizes = np.diff(d["vtoc"].astype(np.int64))
    assert sizes.max() > 4096 and ((sizes > 32) & (sizes <= 4096)).any()
    _, res, _ = _check(ctx, d)
    assert res.saturatedEdgeCount > 0


def _pipeline():
    """LowHash0 -> computeAlignments -> createReadGraph2 -> flagCrossStrandReadGraphEdges1 -> flagChimericReads -> vertices
    -> rc vertices on the device."""
    from shasta_b200 import capi
    with device_read_graph(2) as (c, d, rec, ctoc, cdata, (edges, ctoc_g, cdata_g)):
        capi.flag_cross_strand_read_graph_edges1(c, 6, edges, ctoc_g, cdata_g, rec)
        flags = np.array(d["flags"], np.uint8)
        capi.flag_chimeric_reads(c, 2, edges, ctoc_g, cdata_g, flags, rec)
        table, vtoc, vdata, _, res = capi.create_marker_graph_vertices(c, capi.make_marker_graph_params(minCoverage=2), edges,
                                                                       ctoc, cdata, flags)
        rc = capi.find_marker_graph_reverse_complement_vertices(c, table, vtoc, vdata)
        return dict(toc=d["toc"], table=capi.uint40_to_uint64(table), vtoc=capi.uint40_to_uint64(vtoc), vdata=np.array(vdata),
                    rc=np.array(rc)), d


def test_on_the_device_pipeline(ctx):
    d, _ = _pipeline()
    assert len(d["vtoc"]) > 1000
    _upload(ctx, d["toc"])
    _, res, rc = _check(ctx, d)
    assert res.edgeCount > 1000 and rc is not None


def test_invalid_inputs(ctx):
    from shasta_b200 import capi
    d = CASES["genome/cov2"]
    _upload(ctx, d["toc"])
    t40, v40 = capi.uint64_to_uint40(d["table"]), capi.uint64_to_uint40(d["vtoc"])
    bad = []
    bad.append(("has", lambda: capi.create_marker_graph_edges(ctx, t40[:-5], v40, d["vdata"])))
    vt = d["vtoc"].copy()
    vt[3], vt[4] = vt[4], vt[3]
    bad.append(("decreases", lambda: capi.create_marker_graph_edges(ctx, t40, capi.uint64_to_uint40(vt), d["vdata"])))
    vd = d["vdata"].copy()
    vd[5] = int(d["toc"][-1]) + 3
    bad.append(("marker id out of range", lambda vd=vd: capi.create_marker_graph_edges(ctx, t40, v40, vd)))
    tb = d["table"].copy()
    tb[np.nonzero(tb != EB.INV40)[0][7]] = len(d["vtoc"]) + 10
    bad.append(("vertex id", lambda: capi.create_marker_graph_edges(ctx, capi.uint64_to_uint40(tb), v40, d["vdata"])))
    vd = d["vdata"].copy()
    k = int(np.nonzero(np.diff(d["vtoc"].astype(np.int64)) >= 2)[0][0])
    vd[d["vtoc"][k]], vd[d["vtoc"][k] + 1] = vd[d["vtoc"][k] + 1], vd[d["vtoc"][k]]
    bad.append(("increasing order", lambda vd=vd: capi.create_marker_graph_edges(ctx, t40, v40, vd)))
    for message, call in bad:
        with pytest.raises(capi.ShastaB200Error) as e:
            call()
        assert e.value.status == 1 and message in str(e.value), (message, str(e.value))
    # A call that succeeds after the failures.
    _check(ctx, d)


def test_rc_failures(ctx):
    """The reference's two messages and its assertion, each as the restatement gives it; then a call that succeeds."""
    from shasta_b200 import capi
    d = CASES["genome/cov2"]
    _upload(ctx, d["toc"])

    def device(s):
        return capi.find_marker_graph_reverse_complement_edges(ctx, d["rc"], s["edges"], s["intervalsToc"], s["intervalsData"],
                                                               s["bySourceToc"], capi.uint64_to_uint40(s["bySourceData"]))

    for name, _, s in rc_failure_inputs(d):
        msg, rc = EB.oracle_find_rc_edges(d["toc"], d["rc"], s)
        assert rc is None
        with pytest.raises(capi.ShastaB200Error) as e:
            device(s)
        assert e.value.status == 1 and str(e.value) == msg, name
    o = EB.oracle_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"])
    stoc = o["bySourceToc"].astype(np.int64)
    rows = np.nonzero(np.diff(stoc) >= 1)[0]
    s = {k: np.array(v) for k, v in o.items() if isinstance(v, np.ndarray)}
    s["bySourceData"][stoc[rows[0]]], s["bySourceData"][stoc[rows[1]]] = o["bySourceData"][stoc[rows[1]]], o["bySourceData"][stoc[rows[0]]]
    msg, _ = EB.oracle_find_rc_edges(d["toc"], d["rc"], s)
    with pytest.raises(capi.ShastaB200Error) as e:
        device(s)
    assert msg.startswith("Assertion failed: edgeRc.source == v1Rc") and str(e.value).startswith("Assertion failed: edgeRc.source == v1Rc")
    rv = d["rc"].copy()
    rv[0] = len(rv) + 4
    with pytest.raises(capi.ShastaB200Error) as e:
        capi.find_marker_graph_reverse_complement_edges(ctx, rv, o["edges"], o["intervalsToc"], o["intervalsData"], o["bySourceToc"],
                                                        capi.uint64_to_uint40(o["bySourceData"]))
    assert e.value.status == 1
    rc, _ = device(o)
    assert np.array_equal(rc, EB.oracle_find_rc_edges(d["toc"], d["rc"], o)[1])


def test_parallel_edges_first_match_in_stored_order(ctx):
    """Parallel edges whose intervals differ: the first match in stored row order, as the reference picks it."""
    from shasta_b200 import capi
    d = CASES["genome/cov2"]
    _upload(ctx, d["toc"])
    o = EB.oracle_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"])
    cov = np.diff(o["intervalsToc"].astype(np.int64))
    s = drop_interval(parallel_edge(o, int(np.nonzero(cov >= 2)[0][3])), len(o["edges"]))    # the copy loses an interval
    msg, orc = EB.oracle_find_rc_edges(d["toc"], d["rc"], s)
    rc = None
    try:
        rc, _ = capi.find_marker_graph_reverse_complement_edges(ctx, d["rc"], s["edges"], s["intervalsToc"], s["intervalsData"],
                                                                s["bySourceToc"], capi.uint64_to_uint40(s["bySourceData"]))
    except capi.ShastaB200Error as e:
        assert str(e) == msg
    if msg is None:
        assert np.array_equal(rc, orc)


def test_sharded_context_is_refused(ctx):
    from shasta_b200 import capi, synth
    d = CASES["genome/cov2"]
    toc = d["toc"]
    R = (len(toc) - 1) // 2
    half = toc[:R + 1] - toc[0]
    ctx.set_markers(half, synth.pack_markers(np.zeros(int(half[-1]), np.uint32), np.zeros(int(half[-1]), np.uint32)),
                    np.zeros(R, np.uint8), read_begin=0, read_end=R // 2, read_count_total=R)
    with pytest.raises(capi.ShastaB200Error) as e:
        _device(ctx, d)
    assert e.value.status == 4
    with pytest.raises(capi.ShastaB200Error) as e:
        capi.find_marker_graph_reverse_complement_edges(ctx, d["rc"], np.zeros((0, 14), np.uint8), np.zeros(1, np.uint64),
                                                        np.zeros((0, 3), np.uint32), np.zeros(len(d["rc"]) + 1, np.uint64),
                                                        np.zeros(0, np.uint8))
    assert e.value.status == 4


def test_facade_files(tmp_path, monkeypatch):
    """Assembler.createMarkerGraphEdges and findMarkerGraphReverseComplementEdges write files the reference's MemoryMapped
    code opens, with the restatement's contents."""
    from shasta_b200 import assembler as A, capi
    d = CASES["deep/strand1"]
    monkeypatch.chdir(tmp_path)
    prefix = str(tmp_path / "Data") + "/"
    os.makedirs(prefix)
    toc = d["toc"]
    M, R = int(toc[-1]), (len(toc) - 1) // 2
    A.mm_write_vector(prefix + "Markers.toc", toc)
    A.mm_write_vector(prefix + "Markers.data", pack_ordinal_markers(toc, np.zeros(M, np.uint32)), object_size=7)
    A.mm_write_vector(prefix + "ReadFlags", np.zeros(R, np.uint8))
    A.mm_write_vector(prefix + "MarkerGraphVertexTable", capi.uint64_to_uint40(d["table"]), object_size=5)
    A.mm_write_vector(prefix + "MarkerGraphVertices.toc", capi.uint64_to_uint40(d["vtoc"]), object_size=5)
    A.mm_write_vector(prefix + "MarkerGraphVertices.data", d["vdata"], object_size=8)
    A.mm_write_vector(prefix + "MarkerGraphReverseComplementeVertex", d["rc"], object_size=8)
    a = A.Assembler(largeDataFileNamePrefix=prefix)
    a.accessMarkers()
    a.createMarkerGraphEdges()
    b = A.Assembler(largeDataFileNamePrefix=prefix)
    b.accessMarkers()
    b.accessMarkerGraphEdges()
    b.findMarkerGraphReverseComplementEdges()
    b.accessMarkerGraphReverseComplementEdge()
    o = EB.oracle_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"])
    _, orc = EB.oracle_find_rc_edges(d["toc"], d["rc"], o)
    assert np.array_equal(b._marker_graph_rc_edge, orc)
    if EB.have_ref():
        f = EB.ref_open_marker_graph_edges(prefix)
        assert np.array_equal(f["edges"], o["edges"])
        for k in ("intervalsToc", "intervalsData", "bySourceToc", "bySourceData", "byTargetToc", "byTargetData"):
            assert np.array_equal(np.asarray(f[k]).reshape(-1), np.asarray(o[k]).reshape(-1)), k
        assert np.array_equal(f["rc"], orc)


def test_marker_ids_past_2_32(ctx):
    """Vertices on reads placed after 2^32 filler markers that carry no vertex."""
    import torch
    from shasta_b200 import capi
    need_memory(48)
    d = CASES["genome/cov2"]
    real = dict(toc=d["toc"], kmer=np.zeros(int(d["toc"][-1]), np.uint32), flags=np.zeros((len(d["toc"]) - 1) // 2, np.uint8))
    padded = PaddedSet(real, 10, 12345)
    padded.reals(5)
    padded.fill_to(((1 << 32) + 1000) & ~1)
    padded.reals(len(real["flags"]) - 5)
    padded.finish()
    rows = padded.real_rows()
    start = padded.toc[rows].astype(np.int64)
    lens = np.diff(d["toc"].astype(np.int64))
    mmap = np.concatenate([np.arange(s, s + n) for s, n in zip(start, lens)]).astype(np.int64)
    table = np.full(padded.M, EB.INV40, np.uint64)
    table[mmap] = d["table"]
    vdata = mmap[d["vdata"].astype(np.int64)].astype(np.uint64)
    gmap = padded.gmap.astype(np.int64)
    o = EB.oracle_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"])
    ids = padded.device_ids()
    c = capi.Context(0)
    try:
        c.set_markers_device(padded.toc, ids.data_ptr(), np.zeros(len(padded.flags), np.uint8), keepalive=ids)
        out, res = capi.create_marker_graph_edges(c, capi.uint64_to_uint40(table), capi.uint64_to_uint40(d["vtoc"]), vdata)
        assert np.array_equal(out["edges"], o["edges"]) and np.array_equal(out["intervalsToc"], o["intervalsToc"])
        iv = np.array(o["intervalsData"], np.int64)
        iv[:, 0] = 2 * gmap[iv[:, 0] >> 1] + (iv[:, 0] & 1)
        assert np.array_equal(np.asarray(out["intervalsData"], np.int64), iv)
        rc, _ = capi.find_marker_graph_reverse_complement_edges(c, d["rc"], out["edges"], out["intervalsToc"], out["intervalsData"],
                                                                out["bySourceToc"], out["bySourceData"])
        assert np.array_equal(rc, EB.oracle_find_rc_edges(d["toc"], d["rc"], o)[1])
        print(f"\n{padded.M} markers: {res.edgeCount} edges, {res.deviceMs:.0f} ms on the device, peak {res.peakDeviceBytes / 2**30:.1f} GiB")
    finally:
        c.close()
        del ids
        torch.cuda.empty_cache()
