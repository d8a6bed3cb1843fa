"""Inputs of the read graph tests (tests/test_oracle_readgraph.py, tests/test_gpu_readgraph.py,
tests/test_gpu_readgraph_reference.py): AlignmentData records built from fixed seeds, and the input families compared with
the reference's own createReadGraph, createReadGraph2 and tables."""
import numpy as np

U32_MAX = 2**32 - 1
DEFAULT_PERCENTILES = (0.015, 0.12, 0.12, 0.12, 0.015)      # ReadGraph.*Percentile defaults (src/AssemblerOptions.cpp)


def records(rng, n, reads):
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


def quality_records(rng, n, reads):
    """AlignmentData with plausible AlignmentInfo words: Data{markerCount, firstOrdinal, lastOrdinal} x 2, markerCount, offsets,
    maxSkip, maxDrift."""
    rec = records(rng, n, reads)
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


def _hub_records(rng, hub, reads, n_hub, n_other):
    """Read `hub` in n_hub alignments (several with the same partner), the other reads in n_other alignments among themselves
    with better marker counts, so that the hub's alignments are mostly kept or dropped by the hub's own row."""
    rec = records(rng, n_hub + n_other, reads)
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
    rec = records(rng, n, len(ids))
    rec[:, 0], rec[:, 1] = ids[rec[:, 0]], ids[rec[:, 1]]
    return rec


def _repeated_pair_records(rng, pairs, reads):
    """Several alignments of one read pair (1-6 each, same or different marker counts and strands), out of read order."""
    base = records(rng, pairs, reads)
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
        out.append((f"records{i}", records(np.random.default_rng(100 + i), n, reads), reads, (0, 1, 3, 6, 1000)))
    out.append(("quality", quality_records(np.random.default_rng(110), 3000, 120), 120, (2, 6)))
    rec = records(np.random.default_rng(111), 2000, 80)
    rec[:, 9] = 7                                       # ties everywhere: decided by the alignment id
    out.append(("equal_counts", rec, 80, (1, 2, 5)))
    rng = np.random.default_rng(112)
    rec = records(rng, 2000, 80)
    rec[:, 9] = rng.choice(np.array([0, 1, U32_MAX - 1, U32_MAX], np.uint32), 2000)
    out.append(("extreme_counts", rec, 80, (1, 3)))
    rec = _hub_records(np.random.default_rng(113), 17, 3000, 30000, 6000)
    degree = int(np.count_nonzero((rec[:, 0] == 17) | (rec[:, 1] == 17)))
    out.append(("hub", rec, 3000, (0, 1, degree - 1, degree, degree + 1, U32_MAX)))
    out.append(("sparse_reads", _sparse_records(np.random.default_rng(114), 600, 64), 64, (1, 3)))
    out.append(("repeated_pairs", _repeated_pair_records(np.random.default_rng(115), 150, 40), 40, (1, 2, 4)))
    out.append(("junk", _add_junk(np.random.default_rng(116), records(np.random.default_rng(117), 1500, 70)), 70, (1, 3, 6)))
    return out


def _growth_records(rng, n, reads):
    """Quality records whose indicators go past each histogram's upper bound (markerCount 3000, alignedFraction 1, maxDrift,
    maxSkip and trim 100), early and late in alignment order: the order-dependent growth path of Histogram2."""
    rec = quality_records(rng, n, reads)
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
    rec = quality_records(rng, n, reads)
    rec[:, 9] = np.maximum(rec[:, 9], 10)
    rec[:, 13] = np.minimum(rec[:, 13], 90)
    rec[:, 14] = np.minimum(rec[:, 14], 90)
    return rec


def read_graph2_families():
    """(name, records, readCount, maxAlignmentCounts, percentiles) for creationMethod 2."""
    return [
        ("default", quality_records(np.random.default_rng(120), 3000, 120), 120, (2, 6), DEFAULT_PERCENTILES),
        ("percentiles0", _all_eligible_records(np.random.default_rng(121), 2000, 100), 100, (1, 4), (0.0,) * 5),
        ("percentiles1", quality_records(np.random.default_rng(122), 2000, 100), 100, (1, 4), (1.0,) * 5),
        ("growth", _growth_records(np.random.default_rng(123), 3000, 120), 120, (2, 6), DEFAULT_PERCENTILES),
        ("junk", _add_junk(np.random.default_rng(124), quality_records(np.random.default_rng(125), 1500, 70)), 70, (1, 3),
         DEFAULT_PERCENTILES),
    ]


def unordered_cases():
    """(name, records, readCount, maxAlignmentCount, refused): alignments whose edge or reverse-complement edge is not
    ordered, kept (the reference asserts) and not kept (legal: only kept alignments make edges)."""
    rng = np.random.default_rng(130)
    base = records(rng, 400, 30)
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


def scale_family():
    """A few million alignments over about 100 k reads: both device radix sorts run over many tiles."""
    return records(np.random.default_rng(140), 3_000_000, 100_000), 100_000, (1, 6)
