"""The read graph oracle (oracle/readgraph_oracle.c: createReadGraph and createReadGraph2, ReadGraph.creationMethod 0 and 2)
and the oracle's alignment and candidate tables (oracle/align_oracle.c), against:
  * a direct statement of src/AssemblerReadGraph.cpp:35-175 (per read, the maxAlignmentCount largest (markerCount,
    alignmentId) pairs; edges in alignment order; every connectivity row in DECREASING edge index, the order in which
    MemoryMapped::VectorOfVectors::store leaves the rows, src/MemoryMappedVectorOfVectors.hpp:384-387);
  * the reference's own code: oracle/ref_glue/ref_readgraph.cpp follows the members over the reference's containers,
    AlignmentData, OrientedReadId, Histogram2 and std::nth_element. Its outputs are recorded in
    tests/golden/reference_readgraph.npz (tests/golden/reference_outputs.py), large ones as SHA-256 digests.
The input families (read_graph_families, read_graph2_families) are shared with tests/test_gpu_readgraph_reference.py."""
import hashlib
import os
import sys

import numpy as np

from oracle import bindings as B

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from reference_outputs import recorded  # noqa: E402


def _records(rng, n, reads):
    rec = np.zeros((n, 16), np.uint32)
    a = rng.integers(0, reads, n)
    b = rng.integers(0, reads, n)
    same = a == b
    b[same] = (a[same] + 1) % reads
    rec[:, 0] = np.minimum(a, b)
    rec[:, 1] = np.maximum(a, b)
    rec[:, 2] = rng.integers(0, 2, n)
    rec[:, 9] = rng.integers(10, 14, n)         # few distinct marker counts: ties are decided by the alignment id
    rec[:, 15] = rng.integers(0, 2, n)          # stale flags must be overwritten
    return rec


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
        rec = _records(rng, n, reads)
        out, keep, edges, toc, data = B.oracle_create_read_graph(rec, reads, k)
        dkeep, dedges, dtoc, ddata = _direct(rec, reads, k)
        assert np.array_equal(keep, dkeep), (n, reads, k)
        assert np.array_equal(edges, dedges) and np.array_equal(toc, dtoc) and np.array_equal(data, ddata)
        assert np.array_equal(out[:, 15] & 1, keep) and np.array_equal(out[:, :15], rec[:, :15])
        # an edge joins (r0, 0) with (r1, 0 / 1) and is ordered (src/AssemblerReadGraph.cpp:129,137)
        assert np.all(edges[:, 0] < edges[:, 1]) if len(edges) else True


def _quality_records(rng, n, reads):
    """AlignmentData with plausible AlignmentInfo words: Data{markerCount, firstOrdinal, lastOrdinal} x 2, markerCount, offsets,
    maxSkip, maxDrift."""
    rec = _records(rng, n, reads)
    for side in (0, 1):
        total = rng.integers(200, 5000, n)
        first = rng.integers(0, 150, n)
        last = total - 1 - rng.integers(0, 150, n)
        rec[:, 3 + 3 * side] = total
        rec[:, 4 + 3 * side] = first
        rec[:, 5 + 3 * side] = np.maximum(last, first)
    span = np.minimum(rec[:, 5] - rec[:, 4], rec[:, 8] - rec[:, 7]) + 1
    rec[:, 9] = np.maximum(1, (span * rng.uniform(0.2, 1.0, n)).astype(np.uint32))       # markerCount: up to ~4800 (beyond 3000)
    rec[:, 13] = rng.integers(0, 140, n)        # maxSkip: some beyond the histogram's 100
    rec[:, 14] = rng.integers(0, 120, n)        # maxDrift
    return rec


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
    rec = _quality_records(rng, 200, 30)
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
        rec = _quality_records(rng, n, reads)
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
U32_MAX = 2**32 - 1
DEFAULT_PERCENTILES = (0.015, 0.12, 0.12, 0.12, 0.015)      # ReadGraph.*Percentile defaults (src/AssemblerOptions.cpp)
DIGEST_ABOVE = 4096         # outputs with more elements are recorded as SHA-256 digests


def _hub_records(rng, hub, reads, n_hub, n_other):
    """Read `hub` in n_hub alignments (several with the same partner), the other reads in n_other alignments among themselves
    with better marker counts, so that the hub's alignments are mostly kept or dropped by the hub's own row."""
    rec = _records(rng, n_hub + n_other, reads)
    leaf = rng.integers(0, reads - 1, n_hub)
    leaf[leaf >= hub] += 1
    rec[:n_hub, 0] = np.minimum(leaf, hub)
    rec[:n_hub, 1] = np.maximum(leaf, hub)
    rec[:n_hub, 9] = rng.integers(10, 14, n_hub)
    rec[n_hub:, 9] = rng.integers(20, 24, n_other)
    return rec[rng.permutation(len(rec))]


def _sparse_records(rng, n, reads):
    """Read ids drawn from a subset with gaps at the start (0-4), in the middle (20-29) and at the end (>= reads - 14):
    reads without alignments, and a read count above the largest read id."""
    ids = np.array([r for r in range(5, reads - 14) if not 20 <= r < 30])
    rec = _records(rng, n, len(ids))
    rec[:, 0], rec[:, 1] = ids[rec[:, 0]], ids[rec[:, 1]]
    return rec


def _repeated_pair_records(rng, pairs, reads):
    """Several alignments of one read pair (1-6 each, same or different marker counts and strands), out of read order."""
    base = _records(rng, pairs, reads)
    rec = np.repeat(base, rng.integers(1, 7, pairs), axis=0)
    rec[:, 9] = rng.integers(10, 13, len(rec))
    rec[:, 2] = rng.integers(0, 2, len(rec))
    return rec[rng.permutation(len(rec))]


def _add_junk(rng, rec):
    """Junk in the three padding bytes after isSameStrand and in bits 1-31 of word 15 (the bits after isInReadGraph)."""
    n = len(rec)
    rec[:, 2] |= rng.integers(0, 1 << 24, n, dtype=np.uint32) << 8
    rec[:, 15] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    return rec


def read_graph_families():
    """(name, records, readCount, maxAlignmentCounts) for creationMethod 0 and the tables. Every family is legal for the
    reference: a kept alignment always has readIds[0] < readIds[1]."""
    out = []
    for i, (n, reads) in enumerate([(60, 12), (300, 25), (5000, 300)]):
        out.append((f"records{i}", _records(np.random.default_rng(100 + i), n, reads), reads, (0, 1, 3, 6, 1000)))
    out.append(("quality", _quality_records(np.random.default_rng(110), 3000, 120), 120, (2, 6)))
    rec = _records(np.random.default_rng(111), 2000, 80)
    rec[:, 9] = 7                                       # ties everywhere: decided by the alignment id
    out.append(("equal_counts", rec, 80, (1, 2, 5)))
    rng = np.random.default_rng(112)
    rec = _records(rng, 2000, 80)
    rec[:, 9] = rng.choice(np.array([0, 1, U32_MAX - 1, U32_MAX], np.uint32), 2000)
    out.append(("extreme_counts", rec, 80, (1, 3)))
    rec = _hub_records(np.random.default_rng(113), 17, 3000, 30000, 6000)
    degree = int(np.count_nonzero((rec[:, 0] == 17) | (rec[:, 1] == 17)))
    out.append(("hub", rec, 3000, (0, 1, degree - 1, degree, degree + 1, U32_MAX)))
    out.append(("sparse_reads", _sparse_records(np.random.default_rng(114), 600, 64), 64, (1, 3)))
    out.append(("repeated_pairs", _repeated_pair_records(np.random.default_rng(115), 150, 40), 40, (1, 2, 4)))
    out.append(("junk", _add_junk(np.random.default_rng(116), _records(np.random.default_rng(117), 1500, 70)), 70, (1, 3, 6)))
    return out


def _growth_records(rng, n, reads):
    """Quality records whose indicators go past each histogram's upper bound (markerCount 3000, alignedFraction 1, maxDrift,
    maxSkip and trim 100), early and late in alignment order: the order-dependent growth path of Histogram2."""
    rec = _quality_records(rng, n, reads)
    for j in list(range(0, 40, 4)) + list(range(n - 40, n, 4)):
        span = 3200 + j
        rec[j, 3:9] = [span + 10, 5, span + 4, span + 10, 5, span + 4]       # aligned fraction exactly 1, trim 5
        rec[j, 9] = span
    rec[1::97, 13] = 100 + np.arange(len(rec[1::97])) % 30
    rec[2::89, 14] = 100 + np.arange(len(rec[2::89])) % 30
    rec[3::83, 4] = 100 + np.arange(len(rec[3::83])) % 30                   # left trim past 100 on both sides
    rec[3::83, 7] = 100 + np.arange(len(rec[3::83])) % 30
    return rec


def _all_eligible_records(rng, n, reads):
    """With percentiles 0 every alignment passes: indicators inside every histogram, markerCount above 5."""
    rec = _quality_records(rng, n, reads)
    rec[:, 9] = np.maximum(rec[:, 9], 10)
    rec[:, 13] = np.minimum(rec[:, 13], 90)
    rec[:, 14] = np.minimum(rec[:, 14], 90)
    return rec


def read_graph2_families():
    """(name, records, readCount, maxAlignmentCounts, percentiles) for creationMethod 2."""
    return [
        ("default", _quality_records(np.random.default_rng(120), 3000, 120), 120, (2, 6), DEFAULT_PERCENTILES),
        ("percentiles0", _all_eligible_records(np.random.default_rng(121), 2000, 100), 100, (1, 4), (0.0,) * 5),
        ("percentiles1", _quality_records(np.random.default_rng(122), 2000, 100), 100, (1, 4), (1.0,) * 5),
        ("growth", _growth_records(np.random.default_rng(123), 3000, 120), 120, (2, 6), DEFAULT_PERCENTILES),
        ("junk", _add_junk(np.random.default_rng(124), _quality_records(np.random.default_rng(125), 1500, 70)), 70, (1, 3),
         DEFAULT_PERCENTILES),
    ]


def unordered_cases():
    """(name, records, readCount, maxAlignmentCount, refused): alignments whose edge or reverse-complement edge is not
    ordered, kept (the reference asserts) and not kept (legal: only kept alignments make edges)."""
    rng = np.random.default_rng(130)
    base = _records(rng, 400, 30)
    base[:, 9] = rng.integers(50, 60, 400)
    out = []
    for name, (r0, r1, same) in [("swapped", (9, 4, 1)), ("self_opposite", (6, 6, 0)), ("self_same", (6, 6, 1))]:
        for kept in (True, False):
            rec = base.copy()
            rec[200, :3] = (r0, r1, same)
            rec[200, 9] = U32_MAX if kept else 0        # best of its reads, or the worst of reads that have 3 better ones
            out.append((f"{name}_{'kept' if kept else 'dropped'}", rec, 30, 3, kept))
    return out


def unordered2_cases():
    """The same for creationMethod 2, with percentiles 0: every alignment passes but the one with 1 marker."""
    base = _all_eligible_records(np.random.default_rng(131), 400, 30)
    out = []
    for name, (r0, r1, same) in [("swapped", (9, 4, 1)), ("self_opposite", (6, 6, 0)), ("self_same", (6, 6, 1))]:
        for kept in (True, False):
            rec = base.copy()
            rec[200, :3] = (r0, r1, same)
            if not kept:
                rec[200, 9] = 1                         # below minAlignedMarkerCount (5)
            out.append((f"{name}_{'kept' if kept else 'dropped'}", rec, 30, 1000, kept))
    return out


def _digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(a.dtype.str.encode() + str(a.shape).encode() + a.tobytes()).hexdigest()


def summary(rec, keep, edges, toc, data, criteria=None):
    """What the comparisons look at: keep flags, word 15 (isInReadGraph and the bits after it), edges, connectivity, and the
    creationMethod 2 criteria; arrays above DIGEST_ABOVE elements as digests."""
    d = dict(keep=keep, word15=np.ascontiguousarray(rec[:, 15]), edges=edges, toc=toc, data=data)
    if criteria is not None:
        d["criteria_fraction"] = np.float64(criteria["minAlignedFraction"])
        d["criteria_counts"] = np.array([criteria[k] for k in ("minAlignedMarkerCount", "maxDrift", "maxSkip", "maxTrim")], np.uint64)
    return {k: (_digest(v) if np.size(v) > DIGEST_ABOVE else np.asarray(v)) for k, v in d.items()}


def table_summary(toc, data):
    return {k: (_digest(v) if np.size(v) > DIGEST_ABOVE else np.asarray(v)) for k, v in dict(toc=toc, data=data).items()}


def outcome(fn, *args):
    """summary() of a read graph call, or "refused" where it raises UnorderedReadGraphEdge."""
    try:
        out = fn(*args)
    except B.UnorderedReadGraphEdge:
        return "refused"
    return summary(*out[1:], criteria=out[0]) if isinstance(out[0], dict) else summary(*out)


def assert_same(want, got, what):
    if isinstance(want, str) or isinstance(got, str):
        assert want == got, what
        return
    assert sorted(want) == sorted(got), what
    for k in want:
        w, g = want[k], got[k]
        if isinstance(w, str) or isinstance(g, str):
            assert w == g, (what, k)
        else:
            assert np.array_equal(np.asarray(w), np.asarray(g)) and np.asarray(w).shape == np.asarray(g).shape, (what, k)


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


def scale_family():
    """A few million alignments over about 100 k reads: both device radix sorts run over many tiles."""
    return _records(np.random.default_rng(140), 3_000_000, 100_000), 100_000, (1, 6)


def test_scale_against_the_reference():
    rec, reads, ks = scale_family()
    for k in ks:
        want = recorded("readgraph", f"rg0_scale_{k}", outcome, B.ref_create_read_graph, rec, reads, k)
        assert_same(want, outcome(B.oracle_create_read_graph, rec, reads, k), k)
