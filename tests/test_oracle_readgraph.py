"""The read graph oracle (oracle/readgraph_oracle.c: createReadGraph and createReadGraph2, ReadGraph.creationMethod 0 and 2)
and the oracle's alignment and candidate tables (oracle/align_oracle.c), against:
  * a direct statement of src/AssemblerReadGraph.cpp:35-175 (per read, the maxAlignmentCount largest (markerCount,
    alignmentId) pairs; edges in alignment order; every connectivity row in DECREASING edge index, the order in which
    MemoryMapped::VectorOfVectors::store leaves the rows, src/MemoryMappedVectorOfVectors.hpp:384-387);
  * the reference's own code: oracle/ref_glue/ref_readgraph.cpp follows the members over the reference's containers,
    AlignmentData, OrientedReadId, Histogram2 and std::nth_element. Its outputs are recorded in
    tests/golden/reference_readgraph.npz (tests/golden/reference_outputs.py), large ones as SHA-256 digests.
The input families are in tests/golden/readgraph_inputs.py, shared with tests/test_gpu_readgraph_reference.py."""
import numpy as np

from oracle import bindings as B
from support import assert_same, outcome, table_summary

from readgraph_inputs import (quality_records, read_graph2_families, read_graph_families, records, scale_family, unordered2_cases,
                              unordered_cases)
from reference_outputs import recorded


def _direct(rec, reads, k):
    n = len(rec)
    keep = np.zeros(n, np.uint8)
    for r in range(reads):
        ids = [a for a in range(n) if rec[a, 0] == r or rec[a, 1] == r]
        best = sorted(((int(rec[a, 9]), a) for a in ids), reverse=True)[:k]
        for _, a in best:
            keep[a] = 1
    edges = []
    for a in range(n):
        if keep[a]:
            o0, o1 = 2 * int(rec[a, 0]), 2 * int(rec[a, 1]) + (0 if rec[a, 2] else 1)
            edges.append((o0, o1, a, 0))
            edges.append((o0 ^ 1, o1 ^ 1, a, 0))
    conn = [[] for _ in range(2 * reads)]
    for i, e in enumerate(edges):
        conn[e[0]].insert(0, i)         # each row in decreasing edge index
        conn[e[1]].insert(0, i)
    toc = np.zeros(2 * reads + 1, np.uint32)
    toc[1:] = np.cumsum([len(c) for c in conn])
    data = np.array([i for c in conn for i in c], np.uint32)
    return keep, np.array(edges, np.uint32).reshape(-1, 4), toc, data


def test_against_direct_statement_rows_in_decreasing_edge_order():
    rng = np.random.default_rng(3)
    for n, reads, k in [(0, 5, 3), (1, 4, 6), (60, 12, 3), (300, 25, 6), (300, 25, 1), (200, 10, 0), (150, 8, 1000)]:
        rec = records(rng, n, reads)
        out, keep, edges, toc, data = B.oracle_create_read_graph(rec, reads, k)
        dkeep, dedges, dtoc, ddata = _direct(rec, reads, k)
        assert np.array_equal(keep, dkeep), (n, reads, k)
        assert np.array_equal(edges, dedges) and np.array_equal(toc, dtoc) and np.array_equal(data, ddata)
        assert np.array_equal(out[:, 15] & 1, keep) and np.array_equal(out[:, :15], rec[:, :15])
        # an edge joins (r0, 0) with (r1, 0 / 1) and is ordered (src/AssemblerReadGraph.cpp:129,137)
        assert np.all(edges[:, 0] < edges[:, 1]) if len(edges) else True


def test_histogram2_and_indicators_against_the_reference_classes():
    """Against the reference's own Histogram2 and AlignmentInfo accessors (recorded in tests/golden/reference_readgraph.npz)."""
    fractions = (0.015, 0.12, 0.5, 0.88, 0.985, 1.0)
    rng = np.random.default_rng(5)
    for (start, stop, bins) in [(0, 1, 100), (0, 3000, 300), (0, 100, 100)]:
        for trial in range(20):
            n = int(rng.integers(0, 400))
            # in range, exactly on the upper edge, and well beyond it (the dynamic-bounds growth path)
            x = rng.uniform(start, stop * rng.choice([0.5, 1.0, 1.7]), n)
            if n and trial % 3 == 0:
                x[rng.integers(0, n)] = stop
            x = np.round(x, 2) if stop > 1 else x
            wants = recorded("readgraph", f"histogram2_{start}_{stop}_{bins}_{trial}",
                             lambda: np.array([B.ref_histogram2_threshold(x, start, stop, bins, f) for f in fractions]))
            for fraction, want in zip(fractions, wants):
                got = B.oracle_histogram2_threshold(x, start, stop, bins, fraction)
                assert want == got or (np.isnan(want) and np.isnan(got)), (start, stop, bins, trial, fraction)
    rec = quality_records(rng, 200, 30)
    indicators = recorded("readgraph", "alignment_indicators", lambda: np.stack([B.ref_alignment_indicators(r) for r in rec]))
    for r, want in zip(rec, indicators):
        d0, d1 = r[3:6].astype(np.int64), r[6:9].astype(np.int64)
        frac = min(r[9] / (d0[2] + 1 - d0[1]), r[9] / (d1[2] + 1 - d1[1]))
        trim = max(min(d0[1], d1[1]), min(d0[0] - 1 - d0[2], d1[0] - 1 - d1[2]))
        assert np.array_equal(want, np.array([frac, r[9], r[14], r[13], trim], np.float64))


def test_creation_method_2_against_direct_statement():
    rng = np.random.default_rng(8)
    pc = (0.015, 0.12, 0.12, 0.12, 0.015)      # ReadGraph.*Percentile defaults (src/AssemblerOptions.cpp)
    for n, reads, k in [(0, 4, 6), (400, 30, 6), (3000, 120, 6), (3000, 120, 2)]:
        rec = quality_records(rng, n, reads)
        crit, out, keep, edges, toc, data = B.oracle_create_read_graph2(rec, reads, k, pc)
        ok = np.zeros(n, bool)
        for a in range(n):
            r = rec[a]
            d0, d1 = r[3:6].astype(np.int64), r[6:9].astype(np.int64)
            frac = min(r[9] / (d0[2] + 1 - d0[1]), r[9] / (d1[2] + 1 - d1[1]))
            trim = max(min(d0[1], d1[1]), min(d0[0] - 1 - d0[2], d1[0] - 1 - d1[2]))
            ok[a] = not (frac < crit["minAlignedFraction"] or r[9] < crit["minAlignedMarkerCount"] or r[14] > crit["maxDrift"]
                         or r[13] > crit["maxSkip"] or trim > crit["maxTrim"])
        if n:
            assert 0 < ok.sum() < n
        # the selection of method 0 restricted to the alignments that pass: compare through the sub-table
        sub = rec[ok]
        _, skeep, _, _, _ = B.oracle_create_read_graph(sub, reads, k)
        want = np.zeros(n, np.uint8)
        want[np.flatnonzero(ok)[skeep.astype(bool)]] = 1
        assert np.array_equal(keep, want)
        dkeep, dedges, dtoc, ddata = _direct(rec[:, :], reads, 0)      # edges / connectivity from the keep flags
        kept = np.flatnonzero(keep)
        assert np.array_equal(edges[0::2, 2], kept) and np.array_equal(edges[1::2, 2], kept)
        assert np.array_equal(out[:, 15] & 1, keep)


# ---------------------------------------------------------------------------------------------------------------------------
# Against the reference's own code.


def test_read_graph_against_the_reference():
    for name, rec, reads, ks in read_graph_families():
        for k in ks:
            want = recorded("readgraph", f"rg0_{name}_{k}", outcome, B.ref_create_read_graph, rec, reads, k)
            got = outcome(B.oracle_create_read_graph, rec, reads, k)
            assert_same(want, got, (name, k))
            out = B.oracle_create_read_graph(rec, reads, k)[0]
            assert np.array_equal(out[:, :15], rec[:, :15]) and np.array_equal(out[:, 15] >> 1, rec[:, 15] >> 1)


def test_read_graph_connectivity_rows_are_in_decreasing_edge_order():
    """The reference's own rows, recorded: three kept alignments of read 0 give row 0 = [4, 2, 0]."""
    rec = np.zeros((3, 16), np.uint32)
    rec[:, 1] = [1, 2, 3]
    rec[:, 2] = 1
    rec[:, 9] = 9
    want = recorded("readgraph", "rg0_three_edges_of_read0", outcome, B.ref_create_read_graph, rec, 4, 10)
    assert list(want["data"][want["toc"][0]:want["toc"][1]]) == [4, 2, 0]
    assert_same(want, outcome(B.oracle_create_read_graph, rec, 4, 10), "three edges")


def test_read_graph2_against_the_reference():
    for name, rec, reads, ks, pc in read_graph2_families():
        for k in ks:
            want = recorded("readgraph", f"rg2_{name}_{k}", outcome, B.ref_create_read_graph2, rec, reads, k, pc)
            got = outcome(B.oracle_create_read_graph2, rec, reads, k, pc)
            assert_same(want, got, (name, k))
            if name == "percentiles0":          # every alignment passes: the graph of creationMethod 0
                assert_same({x: want[x] for x in ("keep", "word15", "edges", "toc", "data")},
                            outcome(B.oracle_create_read_graph, rec, reads, k), (name, k))
            if name == "percentiles1":          # none passes
                assert not np.any(want["keep"]) and len(want["edges"]) == 0


def test_unordered_edges_against_the_reference():
    for name, rec, reads, k, refused in unordered_cases():
        want = recorded("readgraph", f"unordered_{name}", outcome, B.ref_create_read_graph, rec, reads, k)
        assert (want == "refused") == refused, name
        assert_same(want, outcome(B.oracle_create_read_graph, rec, reads, k), name)
    for name, rec, reads, k, refused in unordered2_cases():
        want = recorded("readgraph", f"unordered2_{name}", outcome, B.ref_create_read_graph2, rec, reads, k, (0.0,) * 5)
        assert (want == "refused") == refused, name
        assert_same(want, outcome(B.oracle_create_read_graph2, rec, reads, k, (0.0,) * 5), name)


def test_tables_against_the_reference():
    for name, rec, reads, _ in read_graph_families() + [c[:3] + (None,) for c in unordered_cases()[::2]]:
        want = recorded("readgraph", f"alignment_table_{name}", lambda: table_summary(*B.ref_compute_alignment_table(rec, reads)))
        assert_same(want, table_summary(*B.oracle_compute_alignment_table(rec, reads)), name)
        cand = np.ascontiguousarray(rec[:, :3])
        want = recorded("readgraph", f"candidate_table_{name}", lambda: table_summary(*B.ref_compute_candidate_table(cand, reads)))
        assert_same(want, table_summary(*B.oracle_compute_candidate_table(cand, reads)), name)


def test_scale_against_the_reference():
    rec, reads, ks = scale_family()
    for k in ks:
        want = recorded("readgraph", f"rg0_scale_{k}", outcome, B.ref_create_read_graph, rec, reads, k)
        assert_same(want, outcome(B.oracle_create_read_graph, rec, reads, k), k)
