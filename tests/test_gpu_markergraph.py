"""createMarkerGraphVertices and findMarkerGraphReverseComplementVertices on the GPU (csrc/markergraph.cu) against the C
restatement (oracle/markergraph_oracle.c), which tests/test_oracle_markergraph.py pins to the reference's own components.
Both number vertices by their first marker, so the device's outputs must equal the oracle's exactly."""
import os

import numpy as np
import pytest

from oracle import markergraph_bindings as MB
from support import PaddedSet, ctx, device_read_graph, need_memory, pack_ordinal_markers  # noqa: F401

from markergraph_inputs import PARAMS, _finish, cases

pytestmark = pytest.mark.gpu
CASES = cases()
INV40 = (1 << 40) - 1


def _upload(ctx, d):
    toc = d["toc"]
    ctx.set_markers(toc, pack_ordinal_markers(toc, d["kmer"]), np.zeros((len(toc) - 1) // 2, np.uint8))


def _device(ctx, d, **params):
    from shasta_b200 import capi
    p = dict(MB.DEFAULTS)
    p.update(params)
    table, vtoc, vdata, hist, res = capi.create_marker_graph_vertices(ctx, capi.make_marker_graph_params(**p), d["edges"], d["ctoc"],
                                                                      d["cdata"], d["flags"])
    return table, vtoc, vdata, hist, res


def _check(ctx, d, **params):
    from shasta_b200 import capi
    o = MB.oracle_create_marker_graph_vertices(d["toc"], d["kmer"], d["edges"], d["ctoc"], d["cdata"], d["flags"], **params)
    assert o["status"] == 0
    table, vtoc, vdata, hist, res = _device(ctx, d, **params)
    for key in ("edgePairsUsed", "edgePairsSkipped", "alignedMarkerPairs", "disjointSetCount", "minCoverageUsed",
                "keptDisjointSetCount", "badDisjointSetCount", "vertexCount"):
        assert getattr(res, key) == o[key], key
    assert np.array_equal(hist, o["histogram"])
    t = capi.uint40_to_uint64(table)
    assert np.array_equal(t, o["table"]), f"{np.count_nonzero(t != o['table'])} table entries differ"
    assert np.array_equal(capi.uint40_to_uint64(vtoc), o["vtoc"])
    assert np.array_equal(vdata, o["vdata"])
    assert res.peakFinderFailed == o["peakFinderFailed"]
    assert res.peakFinderObservedAreaFraction == o["observedAreaFraction"]
    rc = capi.find_marker_graph_reverse_complement_vertices(ctx, table, vtoc, vdata)
    st, orc = MB.oracle_find_rc_vertices(d["toc"], o["table"], o["vtoc"], o["vdata"])
    assert st == 0 and np.array_equal(rc, orc)
    return (table, vtoc, vdata, hist), res


@pytest.mark.parametrize("name", sorted(CASES))
def test_cases_against_oracle(ctx, name):
    d = CASES[name]
    _upload(ctx, d)
    for pname in sorted(PARAMS):
        _check(ctx, d, **PARAMS[pname])


def test_byte_identical_runs(ctx):
    d = CASES["deep"]
    _upload(ctx, d)
    first, res = _check(ctx, d, **PARAMS["cov2"])
    second = _device(ctx, d, **PARAMS["cov2"])[:4]
    for a, b in zip(first, second):
        assert a.tobytes() == b.tobytes()
    assert res.peakDeviceBytes > 0 and res.kernelLaunches > 0


def test_rc_vertices_in_reference_numbering(ctx):
    """Vertex files renumbered by a random permutation, as the reference's own run numbers them."""
    from shasta_b200 import capi
    d = CASES["self_rc"]
    _upload(ctx, d)
    (table, vtoc, vdata, _), _ = _check(ctx, d, **PARAMS["cov2"])
    t = capi.uint40_to_uint64(table)
    toc = capi.uint40_to_uint64(vtoc).astype(np.int64)
    V = len(toc) - 1
    perm = np.random.default_rng(3).permutation(V)           # new id of vertex v
    inv = np.argsort(perm)
    parts = [vdata[toc[v]:toc[v + 1]] for v in inv]
    ntoc = np.zeros(V + 1, np.uint64)
    ntoc[1:] = np.cumsum([len(p) for p in parts])
    nt = t.copy()
    valid = t != INV40
    nt[valid] = perm[t[valid].astype(np.int64)]
    rc = capi.find_marker_graph_reverse_complement_vertices(ctx, capi.uint64_to_uint40(nt), capi.uint64_to_uint40(ntoc),
                                                            np.concatenate(parts))
    st, orc = MB.oracle_find_rc_vertices(d["toc"], nt, ntoc, np.concatenate(parts))
    assert st == 0 and np.array_equal(rc, orc)
    assert (rc[perm] == perm[MB.oracle_find_rc_vertices(d["toc"], t, capi.uint40_to_uint64(vtoc), vdata)[1].astype(np.int64)]).all()
    # A broken invariant: one marker of a vertex moved to another vertex's table entry.
    bad = nt.copy()
    m = int(np.concatenate(parts)[0])
    bad[m] = (int(bad[m]) + 1) % V
    with pytest.raises(capi.ShastaB200Error) as e:
        capi.find_marker_graph_reverse_complement_vertices(ctx, capi.uint64_to_uint40(bad), capi.uint64_to_uint40(ntoc), np.concatenate(parts))
    assert e.value.status == 1 and "reverse complement" in str(e.value)


def _mutated(d, what):
    from oracle import bindings as B
    d = {k: np.array(v) for k, v in d.items()}
    e = d["edges"]
    if what == "odd":
        d["edges"] = e[:-1]
    elif what == "not_rc":
        e[1, 0] ^= 2
    elif what == "unordered":
        e[0:2, 0:2] = e[0:2, [1, 0]]
    elif what == "alignment_id":
        e[0, 2] = len(d["ctoc"]) + 5
    elif what == "kmer":
        a = int(e[0, 2])
        first = B.oracle_decompress(d["cdata"][int(d["ctoc"][a]):int(d["ctoc"][a + 1])])[0, 0]
        d["kmer"][int(d["toc"][e[0, 0]]) + int(first)] = 1 << 21
    return d


@pytest.mark.parametrize("what,message", [("odd", "odd number"), ("not_rc", "not the reverse complement"),
                                          ("unordered", "orientedReadIds"), ("alignment_id", "alignmentId"),
                                          ("kmer", "k-mer ids")])
def test_invalid_inputs(ctx, what, message):
    from shasta_b200 import capi
    d = _mutated(CASES["genome_in_order"], what)
    _upload(ctx, d)
    with pytest.raises(capi.ShastaB200Error) as e:
        _device(ctx, d, **PARAMS["cov2"])
    assert e.value.status == 1 and message in str(e.value)


def test_counters_after_a_failed_call(ctx):
    """A call after one that failed on its k-mer check, on the same context, with no pair to unite: nothing of the failed
    call's counters may show."""
    from shasta_b200 import capi
    d = _mutated(CASES["genome_in_order"], "kmer")
    _upload(ctx, d)
    with pytest.raises(capi.ShastaB200Error):
        _device(ctx, d, **PARAMS["cov2"])
    for flag in (0, 1 << 30):
        e = {k: np.array(v) for k, v in d.items()}
        if flag:
            e["edges"][:, 3] |= flag                              # every pair skipped as crossesStrands
        else:
            e["edges"] = np.zeros((0, 4), np.uint32)
        _, res = _check(ctx, e, minCoverage=1, maxCoverage=100)
        assert res.alignedMarkerPairs == 0 and res.edgePairsUsed == 0


def test_sharded_context_is_refused(ctx):
    from shasta_b200 import capi
    d = CASES["genome"]
    R = (len(d["toc"]) - 1) // 2
    toc = d["toc"][:R + 1] - d["toc"][0]
    from shasta_b200 import synth
    ctx.set_markers(toc, synth.pack_markers(d["kmer"][:int(toc[-1])], np.zeros(int(toc[-1]), np.uint32)), np.zeros(R, np.uint8),
                    read_begin=0, read_end=R // 2, read_count_total=R)
    with pytest.raises(capi.ShastaB200Error) as e:
        _device(ctx, d, **PARAMS["cov2"])
    assert e.value.status == 4
    with pytest.raises(capi.ShastaB200Error) as e:
        capi.find_marker_graph_reverse_complement_vertices(ctx, np.zeros(5, np.uint8), np.zeros(10, np.uint8), np.zeros(1, np.uint64))
    assert e.value.status == 4


def test_chunk_seams(ctx, monkeypatch):
    """Tiny edge-pair batches (span uploads and gathers) and vertex-table chunks."""
    for name in ("genome", "genome_in_order", "formats"):
        d = CASES[name]
        _upload(ctx, d)
        for pairs, nbytes, chunk in [(1, 1, 7), (3, 200, 1000), (5, 1 << 20, 4096)]:
            monkeypatch.setenv("SHB_MARKERGRAPH_PAIR_BATCH", str(pairs))
            monkeypatch.setenv("SHB_MARKERGRAPH_BATCH_BYTES", str(nbytes))
            monkeypatch.setenv("SHB_MARKERGRAPH_TABLE_CHUNK", str(chunk))
            _check(ctx, d, **PARAMS["strand1"])


def test_zero_edges(ctx):
    from shasta_b200 import capi
    d = {k: np.array(v) for k, v in CASES["genome"].items()}
    d["edges"] = np.zeros((0, 4), np.uint32)
    _upload(ctx, d)
    (table, vtoc, vdata, hist), res = _check(ctx, d, minCoverage=1, maxCoverage=100)
    M = int(d["toc"][-1])
    assert res.vertexCount == M and np.array_equal(capi.uint40_to_uint64(table), np.arange(M)) and np.array_equal(vdata, np.arange(M))
    assert np.array_equal(hist, [0, M])


def test_large_sets(ctx):
    """Sets of more than 32 and more than 4096 markers (the block and radix sorts): every read aligned to read 0."""
    rng = np.random.default_rng(5)
    R = 4300
    lengths = [6] * R
    ords = np.stack([np.arange(6), np.arange(6)], 1).astype(np.uint32)
    alignments = [(0, 2 * r, ords[:5] if r % 2 else ords) for r in range(1, R)]
    alignments += [(0, 2 * r + 1, ords[:3]) for r in range(1, 80)]
    d = _finish(rng, lengths, alignments, [0] * len(alignments), np.zeros(0, np.int64))
    _upload(ctx, d)
    for params in (dict(minCoverage=1, maxCoverage=100000), dict(minCoverage=2, maxCoverage=100000, allowDuplicateMarkers=True)):
        _, res = _check(ctx, d, **params)
    assert res.vertexCount > 0


def _pipeline(method):
    with device_read_graph(method) as (_, d, _, ctoc, cdata, (edges, _, _)):
        flags = np.array(d["flags"], np.uint8)
        flags[::37] |= 2                                                    # a few chimeric reads
        return dict(toc=d["toc"], kmer=d["kmer"], edges=edges, ctoc=ctoc, cdata=cdata, flags=flags)


@pytest.mark.parametrize("method", [0, 2])
def test_on_the_device_pipeline(ctx, method):
    d = _pipeline(method)
    assert len(d["edges"]) > 500
    _upload(ctx, d)
    for pname in ("cov2", "auto", "strand1"):
        _, res = _check(ctx, d, **PARAMS[pname])
        assert res.alignedMarkerPairs > 10000


def test_facade_files(tmp_path, monkeypatch):
    """Assembler.createMarkerGraphVertices writes files the reference's MemoryMapped code opens, and the histogram CSV."""
    from oracle import bindings as B
    from shasta_b200 import assembler as A, capi
    d = _pipeline(2)
    monkeypatch.chdir(tmp_path)
    prefix = str(tmp_path / "Data") + "/"
    os.makedirs(prefix)
    R = (len(d["toc"]) - 1) // 2
    A.mm_write_vector(prefix + "Markers.toc", d["toc"])
    A.mm_write_vector(prefix + "Markers.data", pack_ordinal_markers(d["toc"], d["kmer"]), object_size=7)
    A.mm_write_vector(prefix + "ReadFlags", np.zeros(R, np.uint8))
    A.mm_write_vector(prefix + "ReadGraphEdges", d["edges"], object_size=16)
    A.mm_write_vector_of_vectors(prefix + "CompressedAlignments", d["ctoc"], d["cdata"], data_object_size=1)
    A.mm_write_vector(prefix + "ReadFlags", d["flags"])                     # as flagChimericReads leaves it
    a = A.Assembler(largeDataFileNamePrefix=prefix)
    a.accessMarkers()
    a.accessReadGraph()
    a.accessCompressedAlignments()
    a.createMarkerGraphVertices(0, 100, 0, False, 0.08, 2)
    b = A.Assembler(largeDataFileNamePrefix=prefix)
    b.accessMarkers()
    b.accessMarkerGraphVertices()
    b.findMarkerGraphReverseComplementVertices()
    o = MB.oracle_create_marker_graph_vertices(d["toc"], d["kmer"], d["edges"], d["ctoc"], d["cdata"], d["flags"], minCoverage=0)
    if MB.have_ref():
        # Object sizes 5 / 5 / 8 / 8, opened by the reference's MemoryMapped::Vector.
        for name, expected in [("MarkerGraphVertexTable", o["table"]), ("MarkerGraphVertices.toc", o["vtoc"])]:
            n, values = MB.ref_open_vector40(prefix + name)
            assert n == len(expected) and np.array_equal(values, expected), name
        for name, count in [("MarkerGraphVertices.data", len(o["vdata"])), ("MarkerGraphReverseComplementeVertex", o["vertexCount"])]:
            assert B.ref_open_vector(prefix + name, 8)[0] == count, name
    assert np.array_equal(capi.uint40_to_uint64(A.mm_read_vector(prefix + "MarkerGraphVertexTable", np.uint8, 5)), o["table"])
    assert np.array_equal(A.mm_read_vector(prefix + "MarkerGraphVertices.data", np.uint64, 8), o["vdata"])
    expected = "Coverage,Frequency\n" + "".join(f"{c},{f}\n" for c, f in enumerate(o["histogram"].tolist()) if f)
    assert open("DisjointSetsHistogram.csv").read() == expected
    if MB.have_ref():
        r = MB.ref_create_marker_graph_vertices(d["toc"], d["kmer"], d["edges"], d["ctoc"], d["cdata"], d["flags"], minCoverage=0)
        assert np.array_equal(r["histogram"], o["histogram"])


def test_marker_ids_past_2_32(ctx):
    """A read graph on real reads placed after 2^32 filler markers (filler reads are singletons, dropped by minCoverage 2)."""
    import torch
    from shasta_b200 import capi
    need_memory(64)
    d = _pipeline(0)
    real = dict(toc=d["toc"], kmer=d["kmer"], flags=np.zeros((len(d["toc"]) - 1) // 2, np.uint8))
    padded = PaddedSet(real, 10, 12345)
    padded.reals(5)
    padded.fill_to(((1 << 32) + 1000) & ~1)
    padded.reals(len(real["flags"]) - 5)
    padded.finish()
    gmap = padded.gmap.astype(np.int64)
    edges = d["edges"].copy()
    edges[:, :2] = 2 * gmap[edges[:, :2] >> 1] + (edges[:, :2] & 1)
    flags = np.zeros(len(padded.flags), np.uint8)
    flags[gmap] = d["flags"]
    o = MB.oracle_create_marker_graph_vertices(d["toc"], d["kmer"], d["edges"], d["ctoc"], d["cdata"], d["flags"], **PARAMS["cov2"])
    # real marker id -> padded marker id
    rows = padded.real_rows()
    start = padded.toc[rows].astype(np.int64)
    lens = np.diff(d["toc"].astype(np.int64))
    mmap = np.concatenate([np.arange(s, s + n) for s, n in zip(start, lens)]).astype(np.uint64)
    ids = padded.device_ids()
    c = capi.Context(0)
    try:
        c.set_markers_device(padded.toc, ids.data_ptr(), flags, keepalive=ids)
        table, vtoc, vdata, hist, res = capi.create_marker_graph_vertices(c, capi.make_marker_graph_params(**PARAMS["cov2"]), edges,
                                                                          d["ctoc"], d["cdata"], flags)
        assert res.vertexCount == o["vertexCount"] and vdata.max() >= 1 << 32
        assert np.array_equal(capi.uint40_to_uint64(vtoc), o["vtoc"]) and np.array_equal(vdata, mmap[o["vdata"].astype(np.int64)])
        t = table.reshape(-1, 5)
        assert np.array_equal(capi.uint40_to_uint64(t[mmap.astype(np.int64)]), o["table"])
        filler = np.ones(padded.M, bool)
        filler[mmap.astype(np.int64)] = False
        for b in range(0, padded.M, 1 << 28):
            chunk = t[b:b + (1 << 28)][filler[b:b + (1 << 28)]]
            assert (chunk == 0xff).all()
        assert hist[1] == o["histogram"][1] + padded.M - len(mmap)
        rc = capi.find_marker_graph_reverse_complement_vertices(c, table, vtoc, vdata)
        assert np.array_equal(rc, MB.oracle_find_rc_vertices(d["toc"], o["table"], o["vtoc"], o["vdata"])[1])
        print(f"\n{padded.M} markers: {res.vertexCount} vertices, {res.deviceMs:.0f} ms on the device, "
              f"peak {res.peakDeviceBytes / 2**30:.1f} GiB")
    finally:
        c.close()
        del ids
        torch.cuda.empty_cache()
