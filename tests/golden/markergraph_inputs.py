"""Inputs of the createMarkerGraphVertices tests (tests/test_oracle_markergraph.py, tests/test_gpu_markergraph.py): markers,
read-graph edge pairs and compressed alignments built from fixed seeds. The k-mer ids are chosen after the alignments so that
every aligned pair the reference unites has equal k-mer ids (one id per connected component of the unions)."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from oracle import bindings as B

CROSSES, INCONSISTENT = 1 << 30, 1 << 31        # bits 62, 63 of the edge's second word, in its fourth uint32


def _toc(lengths):
    toc = np.zeros(2 * len(lengths) + 1, np.uint64)
    toc[1:] = np.cumsum(np.repeat(np.asarray(lengths, np.int64), 2))
    return toc


def _rc(toc, o, ordinal):
    return int(toc[o ^ 1]) + int(toc[o + 1] - toc[o]) - 1 - ordinal


def _finish(rng, lengths, alignments, flags_of_pair, chimeric, perm=True, corrupt=None):
    """alignments: list of (o0, o1, ordinals uint32[n,2]). Returns dict(toc, kmer, edges, ctoc, cdata, flags)."""
    toc = _toc(lengths)
    M = int(toc[-1])
    R = len(lengths)
    order = rng.permutation(len(alignments)) if perm else np.arange(len(alignments))
    blobs = [B.oracle_compress(alignments[a][2]) for a in order]     # alignment ids: positions in this order
    ctoc = np.zeros(len(blobs) + 1, np.uint64)
    ctoc[1:] = np.cumsum([len(b) for b in blobs])
    cdata = np.concatenate(blobs) if blobs else np.zeros(0, np.uint8)
    aid = np.empty(len(alignments), np.int64)
    aid[order] = np.arange(len(alignments))
    flags = np.zeros(R, np.uint8)
    flags[chimeric] |= 2
    flags[rng.random(R) < 0.1] |= 1                                # palindromic bit: not a filter here
    edges, src, dst = [], [], []
    for i, (o0, o1, ords) in enumerate(alignments):
        f = flags_of_pair[i]
        edges.append([o0, o1, aid[i], f])
        edges.append([o0 ^ 1, o1 ^ 1, aid[i], f])
        if f or (flags[o0 >> 1] | flags[o1 >> 1]) & 2:
            continue
        for a, b in ords.tolist():
            src += [int(toc[o0]) + a, _rc(toc, o0, a)]
            dst += [int(toc[o1]) + b, _rc(toc, o1, b)]
    g = coo_matrix((np.ones(len(src)), (np.array(src, np.int64), np.array(dst, np.int64))), shape=(M, M)) if M else None
    labels = connected_components(g, directed=False)[1] if M else np.zeros(0, np.int64)
    kmer = rng.integers(0, 1 << 20, max(M, 1), dtype=np.uint32)[labels] if M else np.zeros(0, np.uint32)
    out = dict(toc=toc, kmer=kmer.astype(np.uint32), edges=np.array(edges, np.uint32).reshape(-1, 4), ctoc=ctoc, cdata=cdata,
               flags=flags)
    return out


def genome_case(seed, reads=80, genome=3000, mean_len=400, drop=0.05, pairs_per_read=4, flag_rate=0.05, chimeric_rate=0.05,
                self_rc=0, perm=True, shift_rate=0.0):
    """Reads as windows of a marker genome on either strand, with dropped markers; alignments between overlapping reads
    pair the ordinals of shared genome positions. With shift_rate, that fraction of the alignments is off by one marker
    from a random point on, which merges neighbouring positions: sets with two markers of one read."""
    rng = np.random.default_rng(seed)
    starts = rng.integers(0, genome - 50, reads)
    lens = np.minimum(rng.integers(mean_len // 3, 2 * mean_len, reads), genome - starts)
    rev = rng.random(reads) < 0.5
    pos = []
    for r in range(reads):
        p = np.arange(starts[r], starts[r] + lens[r])
        p = p[rng.random(len(p)) >= drop]
        pos.append(p if not rev[r] else p[::-1])
    lengths = [len(p) for p in pos]
    alignments = []
    for r0 in range(reads):
        for r1 in rng.choice(reads, pairs_per_read, replace=False):
            r1 = int(r1)
            if r1 <= r0 or not lengths[r0] or not lengths[r1]:
                continue
            fwd0 = pos[r0] if not rev[r0] else pos[r0][::-1]
            fwd1 = pos[r1] if not rev[r1] else pos[r1][::-1]
            common, i0, i1 = np.intersect1d(fwd0, fwd1, return_indices=True)
            if len(common) < 2:
                continue
            keep = rng.random(len(common)) >= 0.02
            i0, i1 = i0[keep], i1[keep]
            # oriented reads whose strand 0/1 runs forward along the genome: ordinal in that oriented read
            o0, a0 = (2 * r0, i0) if not rev[r0] else (2 * r0 + 1, i0)
            o1, a1 = (2 * r1, i1) if not rev[r1] else (2 * r1 + 1, i1)
            if o0 & 1:                                               # keep orientedReadIds[0] on strand 0
                o0, o1 = o0 ^ 1, o1 ^ 1
                a0, a1 = lengths[r0] - 1 - a0[::-1], lengths[r1] - 1 - a1[::-1]
            if rng.random() < shift_rate and len(a1) > 2 and a1[-1] + 1 < lengths[r1]:
                a1 = a1.copy()
                a1[int(rng.integers(len(a1))):] += 1
            alignments.append((o0, o1, np.stack([a0, a1], 1).astype(np.uint32)))
    for _ in range(self_rc):                                         # palindrome-like: a read against its own reverse complement
        r = int(rng.integers(reads))
        n = lengths[r]
        if n < 4:
            continue
        a = np.sort(rng.choice(n, min(n, 30), replace=False))
        alignments.append((2 * r, 2 * r + 1, np.stack([a, a], 1).astype(np.uint32)))
    flags = [int(rng.choice([CROSSES, INCONSISTENT, CROSSES | INCONSISTENT])) if rng.random() < flag_rate else 0
             for _ in alignments]
    chimeric = np.nonzero(rng.random(reads) < chimeric_rate)[0]
    return _finish(rng, lengths, alignments, flags, chimeric, perm=perm)


def formats_case(seed=7):
    """Streaks in all five compressed formats: skips past 2^3, 2^9, 2^19 and streaks longer than 8, 32, 512 pairs."""
    rng = np.random.default_rng(seed)
    lengths = [600_000, 600_000, 3000, 3000]
    ords = []
    a = b = 0
    for skip0, skip1, n in [(0, 0, 5), (2, 1, 8), (6, -3, 20), (100, 200, 300), (-400, 300, 400), (3000, 2000, 600),
                            (530_000, 2, 3), (1, 3, 2000), (5, 5, 40), (-20, 7, 30)]:
        a += skip0 if ords else 0
        b += skip1 if ords else 0
        for i in range(n):
            ords.append((a + i, b + i))
        a += n - 1
        b += n - 1
    ords = np.array(ords, np.int64)
    ords = ords[(ords[:, 0] >= 0) & (ords[:, 1] >= 0)]
    _, first = np.unique(ords[:, 0], return_index=True)
    ords = ords[np.sort(first)]
    ords = ords[np.concatenate([[True], (np.diff(ords[:, 0]) > 0) & (np.diff(ords[:, 1]) > 0)])]
    small = np.stack([np.arange(0, 2900, 3), np.arange(50, 2950, 3)], 1)
    alignments = [(0, 2, ords.astype(np.uint32)), (4, 7, small.astype(np.uint32)), (2, 5, small[::2].astype(np.uint32))]
    return _finish(rng, lengths, alignments, [0, 0, 0], np.zeros(0, np.int64), perm=False)


def cases():
    return {
        "genome": genome_case(1),
        "genome_in_order": genome_case(2, perm=False, flag_rate=0.0, chimeric_rate=0.0),
        "deep": genome_case(3, reads=200, genome=2000, mean_len=300, pairs_per_read=8, shift_rate=0.2),
        "self_rc": genome_case(4, reads=30, self_rc=12),
        "empty_reads": genome_case(5, reads=40, mean_len=30, drop=0.5),
        "formats": formats_case(),
    }


PARAMS = {
    "cov2": dict(minCoverage=2, maxCoverage=100, minCoveragePerStrand=0, allowDuplicateMarkers=False),
    "dup_ok_cut6": dict(minCoverage=1, maxCoverage=6, minCoveragePerStrand=1, allowDuplicateMarkers=True),
    "strand2": dict(minCoverage=1, maxCoverage=1000, minCoveragePerStrand=2, allowDuplicateMarkers=False),
    "strand1": dict(minCoverage=1, maxCoverage=1000, minCoveragePerStrand=1, allowDuplicateMarkers=False),
    "auto": dict(minCoverage=0, maxCoverage=100, minCoveragePerStrand=0, allowDuplicateMarkers=False),
}


def histograms():
    """Histograms for PeakFinder: plateaus and ties, one peak, a small second peak, startIndex past the end, coverage-like."""
    rng = np.random.default_rng(11)
    out = {}
    for i in range(120):
        n = int(rng.integers(1, 40))
        out[f"random{i}"] = rng.integers(0, 6 if i % 2 else 1000, n).astype(np.uint64)
    for i in range(60):
        n = int(rng.integers(2, 30))
        y = rng.integers(0, 3, n).astype(np.uint64)                      # many ties and plateaus
        y[rng.integers(n)] = 5
        out[f"ties{i}"] = y
    for i in range(60):
        cov = int(rng.integers(5, 60))
        x = np.arange(0, 3 * cov)
        y = (rng.integers(1000, 100000) * np.exp(-0.5 * ((x - cov) / (0.25 * cov)) ** 2)).astype(np.int64)
        y += (rng.integers(1000, 1_000_000) * np.exp(-x / rng.uniform(0.5, 3))).astype(np.int64)
        y[0] = 0
        out[f"coverage{i}"] = np.maximum(y, 0).astype(np.uint64)
    out["one_peak"] = np.array([0, 10, 7, 3, 1], np.uint64)
    out["flat"] = np.array([4, 4, 4, 4], np.uint64)
    out["single"] = np.array([0], np.uint64)
    out["tiny_second"] = np.array([0, 1000, 10, 1, 2, 1, 0], np.uint64)
    out["start_past_end"] = np.array([0, 50, 10, 30, 5], np.uint64)
    return out


START_INDEX = {"start_past_end": 9}
