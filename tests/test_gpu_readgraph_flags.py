"""flagCrossStrandReadGraphEdges1 and flagChimericReads on the GPU (csrc/readgraph_flags.cu) against the reference's own
ReadGraph code (oracle/_ref/libshasta_ref_readgraph_flags.so) where it is built, and otherwise against its outputs recorded in
tests/golden/reference_readgraph_flags.npz (readgraph_flags_inputs.expected), ties on markerCount included."""
import os

import numpy as np
import pytest

from oracle import readgraph_flags_bindings as F

from support import ctx, device_read_graph  # noqa: F401
from readgraph_flags_inputs import DISTANCES, bad_graphs, expected, families, hub

pytestmark = pytest.mark.gpu
FAM = families()




def _device_cross(ctx, g, d):
    from shasta_b200 import capi
    edges, rec = np.array(g["edges"], np.uint32), np.array(g["records"], np.uint32)
    res = capi.flag_cross_strand_read_graph_edges1(ctx, d, edges, g["toc"], g["data"], rec)
    return edges, rec, res


def _device_chimeric(ctx, g, d):
    from shasta_b200 import capi
    flags, rec = np.array(g["flags"], np.uint8), np.array(g["records"], np.uint32)
    res = capi.flag_chimeric_reads(ctx, d, g["edges"], g["toc"], g["data"], flags, rec)
    return flags, rec, res


def _check_cross(ctx, key, g, d):
    e = expected("cross", key, g, d)
    assert e["status"] == 0
    edges, rec, res = _device_cross(ctx, g, d)
    assert np.array_equal(edges, e["edges"]), f"{np.count_nonzero(edges != e['edges'])} edge words differ"
    assert np.array_equal(rec, e["records"])
    if d:
        assert (res["nearStrandJumpReportedCount"], res["regionCount"]) == (e["reported"], e["regions"])
    assert res["crossStrandEdgeCount"] == e["flagged"]
    return res


def _check_chimeric(ctx, key, g, d):
    e = expected("chimeric", key, g, d)
    assert e["status"] == 0
    flags, rec, res = _device_chimeric(ctx, g, d)
    assert np.array_equal(flags, e["flags"])
    assert np.array_equal(rec, e["records"])
    assert res["chimericReadCount"] == e["chimeric"]
    return res


@pytest.mark.parametrize("name", sorted(FAM))
@pytest.mark.parametrize("d", DISTANCES)
def test_families(ctx, name, d):
    _check_cross(ctx, name, FAM[name], d)
    _check_chimeric(ctx, name, FAM[name], d)


@pytest.mark.parametrize("capacity,batch", [(32, 1), (32, 3), (64, 2)])
def test_overflow_path_and_batch_seams(ctx, monkeypatch, capacity, batch):
    monkeypatch.setenv("SHB_READGRAPH_FLAGS_TABLE_CAPACITY", str(capacity))
    monkeypatch.setenv("SHB_READGRAPH_FLAGS_BATCH", str(batch))
    overflow = [0, 0]
    for key, g in (("hub300", hub(300, 7)), ("several_regions", FAM["several_regions"]), ("chimeric", FAM["chimeric"])):
        for d in (2, 6, 254):
            overflow[0] += _check_cross(ctx, key, g, d)["overflowReadCount"]
            overflow[1] += _check_chimeric(ctx, key, g, d)["overflowReadCount"]
    assert overflow[0] > 0 and overflow[1] > 0


def test_hub_overflows_at_default_capacity(ctx):
    g = hub(3000, 8)
    r = _check_chimeric(ctx, "hub3000", g, 3)
    assert r["overflowReadCount"] > 0
    r = _check_cross(ctx, "hub3000", g, 6)
    assert r["overflowReadCount"] > 0 and sum(r["ballSizeHistogram"]) == 3000


def test_repeated_calls_are_byte_identical(ctx):
    g = FAM["nested_jumps"]
    a = _device_cross(ctx, g, 6)
    b = _device_cross(ctx, g, 6)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    a = _device_chimeric(ctx, g, 2)
    b = _device_chimeric(ctx, g, 2)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# The reference's fifth region assertion, component0 != component0rc, cannot fail: every union joins (u, v) and
# (rc u, rc v) together, so the components stay closed under reverse complement, and an edge that would join a vertex to
# its reverse complement is flagged instead of united. No input reaches it.
@pytest.mark.parametrize("what", ["odd_region_size", "not_strand_pairs", "odd_edge_count", "pair_alignment_ids"])
def test_reference_assertions_are_refused(ctx, what):
    from shasta_b200 import capi
    g = bad_graphs()[what]
    assert expected("cross", what, g, 6)["status"] == 1
    edges, rec = np.array(g["edges"], np.uint32), np.array(g["records"], np.uint32)
    with pytest.raises(capi.ShastaB200Error):
        capi.flag_cross_strand_read_graph_edges1(ctx, 6, edges, g["toc"], g["data"], rec)
    assert np.array_equal(edges, g["edges"]) and np.array_equal(rec, g["records"])
    # a call on the same context after the failure
    _check_cross(ctx, "one_region", FAM["one_region"], 6)


def test_argument_refusals_leave_inputs_unchanged(ctx):
    from shasta_b200 import capi
    g = FAM["chimeric"]
    edges, rec, flags = np.array(g["edges"]), np.array(g["records"]), np.array(g["flags"])
    with pytest.raises(capi.ShastaB200Error):
        capi.flag_cross_strand_read_graph_edges1(ctx, -1, edges, g["toc"], g["data"], rec)
    with pytest.raises(capi.ShastaB200Error):
        capi.flag_chimeric_reads(ctx, 255, edges, g["toc"], g["data"], flags, rec)
    bad = np.array(g["data"])
    bad[0] = len(edges) + 5
    with pytest.raises(capi.ShastaB200Error):
        capi.flag_chimeric_reads(ctx, 2, edges, g["toc"], bad, flags, rec)
    assert np.array_equal(edges, g["edges"]) and np.array_equal(rec, g["records"]) and np.array_equal(flags, g["flags"])
    _check_chimeric(ctx, "chimeric", g, 2)


def test_end_to_end_into_marker_graph_vertices(ctx):
    """LowHash0 -> computeAlignments -> createReadGraph2 -> both flags -> createMarkerGraphVertices, all on the device."""
    from shasta_b200 import capi
    from oracle import markergraph_bindings as MB
    with device_read_graph(2) as (c, d, rec, ctoc, cdata, (edges, toc, data)):
        g = dict(edges=edges, toc=toc, data=data, records=rec.copy(), flags=np.array(d["flags"], np.uint8))
        _check_cross(ctx, "pipeline", g, 6)
        e1, r1, _ = _device_cross(c, g, 6)
        g2 = dict(g, edges=e1, records=r1)
        _check_chimeric(ctx, "pipeline", g2, 2)
        flags, r2, _ = _device_chimeric(c, g2, 2)
        table, vtoc, vdata, hist, res = capi.create_marker_graph_vertices(c, capi.make_marker_graph_params(**MB.DEFAULTS), e1,
                                                                          ctoc, cdata, flags)
        o = MB.oracle_create_marker_graph_vertices(d["toc"], d["kmer"], e1, ctoc, cdata, flags)
        assert o["status"] == 0
        assert np.array_equal(capi.uint40_to_uint64(table), o["table"]) and np.array_equal(vdata, o["vdata"])
        if MB.have_ref():
            # the reference's flags (built or recorded) followed by the reference's vertex code
            ref_e = expected("cross", "pipeline", g, 6)
            ref_f = expected("chimeric", "pipeline", dict(g, edges=ref_e["edges"], records=ref_e["records"]), 2)
            r = MB.ref_create_marker_graph_vertices(d["toc"], d["kmer"], ref_e["edges"], ctoc, cdata, ref_f["flags"])
            assert r["status"] == 0
            ref_form = MB.canonical(r["table"], r["vtoc"], r["vdata"])[:3]
            dev_form = MB.canonical(capi.uint40_to_uint64(table), capi.uint40_to_uint64(vtoc), vdata)[:3]
            assert all(np.array_equal(a, b) for a, b in zip(dev_form, ref_form))


def test_facade(tmp_path, monkeypatch, capsys):
    from shasta_b200 import assembler as A
    g = FAM["several_regions"]
    monkeypatch.chdir(tmp_path)
    prefix = str(tmp_path / "Data") + "/"
    os.makedirs(prefix)
    A.mm_write_vector(prefix + "ReadGraphEdges", g["edges"], object_size=16)
    A.mm_write_vector_of_vectors(prefix + "ReadGraphConnectivity", g["toc"], g["data"], data_object_size=4, toc_dtype=np.uint32)
    A.mm_write_vector(prefix + "AlignmentData", g["records"], object_size=64)
    A.mm_write_vector(prefix + "ReadFlags", g["flags"])
    a = A.Assembler(largeDataFileNamePrefix=prefix)
    a._alignment_data = np.array(g["records"])
    a.flagCrossStrandReadGraphEdges1(6)
    a.flagChimericReads(2)
    out = capsys.readouterr().out
    e = expected("cross", "several_regions", g, 6)
    c = expected("chimeric", "facade", dict(g, edges=e["edges"], records=e["records"]), 2)
    assert f"Found {e['regions']} strand jump regions." in out
    assert f"Marked {e['flagged']} read graph edges out of {len(g['edges'])} total as cross-strand." in out
    assert f"Flagged {c['chimeric']} reads as chimeric out of {len(g['flags'])} total." in out
    assert np.array_equal(A.mm_read_vector(prefix + "ReadGraphEdges", np.uint32, 16).reshape(-1, 4), e["edges"])
    assert np.array_equal(A.mm_read_vector(prefix + "AlignmentData", np.uint32, 64).reshape(-1, 16), c["records"])
    assert np.array_equal(A.mm_read_vector(prefix + "ReadFlags", np.uint8, 1), c["flags"])
    assert np.array_equal(a._read_graph_edges, e["edges"])
    if F.have_ref():
        # the files as the reference's MemoryMapped::Vector opens them
        from oracle import bindings as B
        edges, n = F.ref_open_read_graph_edges(prefix + "ReadGraphEdges", len(g["edges"]) + 1)
        assert n == len(g["edges"]) and np.array_equal(edges, e["edges"])
        assert B.ref_open_vector(prefix + "AlignmentData", 64) == (len(c["records"]), _fnv(c["records"].tobytes()))
        assert B.ref_open_vector(prefix + "ReadFlags", 1) == (len(c["flags"]), _fnv(c["flags"].tobytes()))


def _fnv(raw):
    h = 1469598103934665603
    for b in bytes(raw):
        h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h
