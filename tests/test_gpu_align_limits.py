"""GPU parity tests (run on an H100 with -m gpu), against the CPU oracle, for the alignment paths that long reads and
single-pair calls take: the 32 000-marker limit of the stage-1 forward kernel (16-bit packed ordinal offsets), the widest
band classes (8 192 and 16 384 offsets, one warp per block) of both DP kernels, the skip of candidates too wide for any
class (tooWideCount, a documented deviation from the reference), the Align.maxBand limit, and the single-pair entry point
shb_align_oriented_reads with explicit orientations and its host-side decoder.

Every test first checks on the host that its input reaches the path it is for (marker and downsampled row counts, band
widths), from the markers and from how the reads were cut from their genome."""
import numpy as np
import pytest

from oracle import bindings as B
from shasta_b200 import synth

pytestmark = pytest.mark.gpu

K = 10
FORWARD_MAX_MARKERS = 32000     # kStage1ForwardMaxMarkers (csrc/align_kernels.cuh)
FORWARD_MAX_ROWS = 512          # kStage1ForwardMaxRows
MAX_BAND_WIDTH = 16384          # widest band class (kMaxBandWidth, csrc/align.cu)
PERMISSIVE = dict(k=K, maxSkip=100000, maxDrift=100000, maxTrim=100000, minAlignedMarkerCount=1, minAlignedFraction=0.0)


@pytest.fixture(scope="module")
def ctx():
    from shasta_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


# ---- host model ----------------------------------------------------------------------------------------------------
def downsampling_hash(kmer, k):
    """kmerDownsamplingHash (csrc/align_kernels.cuh): MurmurHash2 of kmer + reverse complement, seed 13477, vectorised."""
    n = np.asarray(kmer, np.uint64) + synth.reverse_complement_kmer(kmer, k).astype(np.uint64)
    m = np.uint32(0x5bd1e995)
    with np.errstate(over="ignore"):
        h = np.full(n.shape, np.uint32(13477 ^ 8), np.uint32)
        for word in (n.astype(np.uint32), (n >> np.uint64(32)).astype(np.uint32)):
            w = word * m
            w ^= w >> np.uint32(24)
            w *= m
            h *= m
            h ^= w
        h ^= h >> np.uint32(13)
        h *= m
        h ^= h >> np.uint32(15)
    return h


def downsampled_count(row, factor):
    return int((downsampling_hash(row, K) < np.uint32(int(factor * 4294967295.0))).sum())


def padded_width(W):
    """Padded width of a band of W offsets (dpBandShape): W + 2 rounded up to 16 or 64 lanes' sub-chunks; the classes
    above 1 024 offsets all run on whole warps."""
    need = W + 2
    return (need + 63) & ~63 if need > 128 else (need + 15) & ~15


class Genome:
    """A random marker genome; reads are cut from it with marker drop-outs and insertions (the marker-level image of
    sequencing errors). Every row comes with the genome index of each of its markers (-1 for inserted markers)."""

    def __init__(self, markers, seed, drop=0.04, ins=0.02):
        self.rng = np.random.default_rng(seed)
        self.kmer = self.rng.integers(0, 1 << (2 * K), markers).astype(np.uint32)
        self.drop, self.ins = drop, ins

    def read(self, start, length, keep=None):
        """Row of genome markers [start, start + length); keep = ("head", n) or ("tail", n) keeps n markers of it."""
        g = np.arange(start, start + length)
        g = g[self.rng.random(length) >= self.drop]
        idx = np.insert(g, np.flatnonzero(self.rng.random(len(g)) < self.ins) + 1, -1)
        row = np.where(idx >= 0, self.kmer[np.maximum(idx, 0)], self.rng.integers(0, 1 << (2 * K), len(idx))).astype(np.uint32)
        if keep is not None:
            sl = slice(0, keep[1]) if keep[0] == "head" else slice(len(row) - keep[1], len(row))
            row, idx = row[sl], idx[sl]
            assert len(row) == keep[1]
        return row, idx


def assemble(rows0):
    lengths = np.array([len(r) for r in rows0], np.int64)
    toc = np.zeros(2 * len(rows0) + 1, np.uint64)
    toc[1:] = np.cumsum(np.repeat(lengths, 2)).astype(np.uint64)
    parts = []
    for r in rows0:
        parts += [r, synth.reverse_complement_kmer(r[::-1], K)]
    kmer = np.concatenate(parts).astype(np.uint32)
    pos = (np.arange(len(kmer)) % (1 << 24)).astype(np.uint32)
    return dict(toc=toc, kmer=kmer, data=synth.pack_markers(kmer, pos), flags=np.zeros(len(rows0), np.uint8))


def true_offsets(origin, r0, r1):
    """Ordinal offsets (ordinal0 - ordinal1) of the markers the two strand-0 rows share in the genome."""
    a, b = origin[r0], origin[r1]
    _, ia, ib = np.intersect1d(a[a >= 0], b[b >= 0], return_indices=True)
    ia = np.flatnonzero(a >= 0)[ia]
    ib = np.flatnonzero(b >= 0)[ib]
    return ia.astype(np.int64) - ib.astype(np.int64)


def oracle_options(opts):
    return B.make_align_options(**{k: v for k, v in opts.items() if k in B.ALIGN_DEFAULTS})


def compare(ctx, d, cand, expected_skips=(), **opts):
    """GPU records, compressed toc and bytes equal the oracle's on every candidate except the expected skips."""
    from shasta_b200 import capi
    cand = np.asarray(cand, np.uint32).reshape(-1, 3)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    rec, ctoc, cdata, res = capi.compute_alignments(ctx, cand, capi.make_align_options(**opts))
    keep = np.ones(len(cand), bool)
    keep[list(expected_skips)] = False
    orec, otoc, odata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], cand[keep], oracle_options(opts), threads=8)
    assert res.tooWideCount == len(expected_skips)
    assert rec.shape == orec.shape, (rec.shape, orec.shape)
    assert np.array_equal(rec, orec)
    assert np.array_equal(ctoc, otoc)
    assert np.array_equal(cdata, odata)
    return rec, res


# ---- B. the 32 000-marker edge of the stage-1 forward kernel -------------------------------------------------------
def edge_dataset():
    # Per long read X of 31 999, 32 000 or 32 001 markers: a partner Y whose head overlaps X's last ~300 markers (ordinal
    # offsets near +32 000) and a partner Z of 32 000 markers whose tail overlaps X's first ~300 (offsets near -32 000).
    genome = Genome(240000, seed=4)
    rows, origin, triples = [], [], []
    for i, L in enumerate((31999, 32000, 32001)):
        start = 40000 + 75000 * i
        x = genome.read(start, 36000, ("head", L))
        y = genome.read(int(x[1].max()) - 300, 3000)
        z = genome.read(start + 300 - 36000, 36000, ("tail", 32000))
        triples.append((len(rows), len(rows) + 1, len(rows) + 2))
        for r, idx in (x, y, z):
            rows.append(r)
            origin.append(idx)
    return assemble(rows), rows, origin, triples


@pytest.mark.parametrize("method", [3, 4])
def test_forward_kernel_marker_limit_edge(ctx, method):
    d, rows, origin, triples = edge_dataset()
    factor = 0.012
    cand = []
    for x, y, z in triples:
        cand += [(x, y, 1), (x, z, 1), (x, y, 0), (x, z, 0)]
    longest = [max(len(rows[a]), len(rows[b])) for a, b, _ in cand]
    assert {31999, 32000, 32001} <= set(longest)
    assert max(downsampled_count(r, factor) for r in rows) <= FORWARD_MAX_ROWS      # the marker count alone routes
    for x, y, z in triples:
        assert true_offsets(origin, x, y).max() > FORWARD_MAX_MARKERS - 600
        assert true_offsets(origin, x, z).min() < -(FORWARD_MAX_MARKERS - 600)
    opts = dict(PERMISSIVE, alignMethod=method, downsamplingFactor=factor, bandExtend=10, maxBand=1000)
    if method == 4:
        opts.update(align4DeltaX=200, align4DeltaY=10, align4MinEntryCountPerCell=2, align4MaxDistanceFromBoundary=400)
    rec, _ = compare(ctx, d, cand, **opts)
    offsets = rec[:, 10:12].view(np.int32)
    assert len(rec) >= 6 and offsets[:, 1].max() > FORWARD_MAX_MARKERS - 600 and offsets[:, 0].min() < -(FORWARD_MAX_MARKERS - 600)


# ---- B. the widest band classes and the too-wide skip --------------------------------------------------------------
def wide_dataset():
    lengths = (2700, 3200, 4300, 4400, 7900, 8600, 9600)
    starts = (0, 500, 1000, 1500, 800, 300, 100)
    genome = Genome(20000, seed=9, drop=0.03, ins=0.01)
    rows, origin = zip(*(genome.read(s, L) for s, L in zip(starts, lengths)))
    cand = np.array([(i, j, 1) for i in range(len(rows)) for j in range(i + 1, len(rows))], np.uint32)
    return assemble(rows), rows, origin, cand


def _class_of(W):
    need = padded_width(W)
    return None if need > MAX_BAND_WIDTH else (8192 if need > 4096 and need <= 8192 else 16384 if need > 8192 else 0)


def test_widest_stage1_classes_and_skip(ctx):
    d, rows, _, cand = wide_dataset()
    factor = 0.97
    ds = [downsampled_count(r, factor) for r in rows]
    assert min(ds) > FORWARD_MAX_ROWS                                    # every stage 1 takes the traced kernel
    widths = [ds[a] + ds[b] + 1 for a, b, _ in cand]                     # unbanded: offsets -ny ... nx
    classes = [_class_of(W) for W in widths]
    skips = [i for i, c in enumerate(classes) if c is None]
    assert classes.count(8192) >= 2 and classes.count(16384) >= 2 and len(skips) >= 2
    compare(ctx, d, cand, skips, alignMethod=3, downsamplingFactor=factor, bandExtend=10, maxBand=1000,
            **{k: v for k, v in PERMISSIVE.items() if k != "minAlignedMarkerCount"}, minAlignedMarkerCount=10)


def test_widest_method1_classes_and_skip(ctx):
    d, rows, _, cand = wide_dataset()
    widths = [len(rows[a]) + len(rows[b]) + 1 for a, b, _ in cand]       # method 1: one unbanded DP on the full rows
    classes = [_class_of(W) for W in widths]
    skips = [i for i, c in enumerate(classes) if c is None]
    assert classes.count(8192) >= 2 and classes.count(16384) >= 2 and len(skips) >= 2
    compare(ctx, d, cand, skips, alignMethod=1, **PERMISSIVE)


def test_widest_stage2_class_at_max_band(ctx):
    d, rows, origin, cand = wide_dataset()
    band_extend, max_band = 4200, 16317
    wide = 0
    for a, b, _ in cand:
        off = true_offsets(origin, a, b)
        lo, hi = off.min() - band_extend, off.max() + band_extend
        W = min(hi, len(rows[a])) - max(lo, -len(rows[b])) + 1
        wide += int(hi - lo <= max_band - 100 and padded_width(W) > 8192 + 128)
    assert wide >= 3
    compare(ctx, d, cand, alignMethod=3, downsamplingFactor=0.1, bandExtend=band_extend, maxBand=max_band, **PERMISSIVE)


def test_max_band_limit(ctx):
    from shasta_b200 import capi
    d, _, _, cand = wide_dataset()
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    capi.compute_alignments(ctx, cand[:1], capi.make_align_options(k=K, maxBand=16317))
    with pytest.raises(capi.ShastaB200Error, match="limit 16317"):
        capi.compute_alignments(ctx, cand[:1], capi.make_align_options(k=K, maxBand=16318))


# ---- C. the single-pair entry point --------------------------------------------------------------------------------
def pair_dataset():
    d = synth.generate(synth.SynthParams(reads=40, k=K, genome_markers=6000, n50_bases=8000, min_bases=3000, seed=71))
    lp = B.LowHashParams(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=2, maxBucketSize=30, minFrequency=2)
    cand, _, _ = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], lp)
    return d, cand


def row(d, o):
    toc = d["toc"].astype(np.int64)
    return d["kmer"][toc[o]:toc[o + 1]]


def single_pair_options(method):
    opts = dict(PERMISSIVE, alignMethod=method)
    if method == 3:
        opts.update(downsamplingFactor=0.1, bandExtend=10, maxBand=1000)
    elif method == 4:
        opts.update(align4DeltaX=200, align4DeltaY=10, align4MinEntryCountPerCell=2, align4MaxDistanceFromBoundary=200, maxBand=1000)
    return opts


def expected_single_pair(row0, row1, opts):
    """The oracle's stored alignment of row0 against row1 (record, ordinals), or None, from a two-read marker set whose
    reads are the two rows on strand 0."""
    two = assemble([row0, row1])
    orec, otoc, odata, _ = B.oracle_compute_alignments(two["toc"], two["kmer"], np.array([[0, 1, 1]], np.uint32),
                                                       oracle_options(opts), threads=1)
    if len(orec) == 0:
        return None
    return orec[0], B.oracle_decompress(odata[int(otoc[0]):int(otoc[1])])


@pytest.mark.parametrize("method", [1, 3, 4])
def test_align_oriented_reads(ctx, method):
    from shasta_b200 import capi
    d, cand = pair_dataset()
    opts = single_pair_options(method)
    go = capi.make_align_options(**opts)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    pairs = []
    for r0, r1, _ in cand[:6]:
        for s0 in (0, 1):
            for s1 in (0, 1):
                pairs += [(2 * r0 + s0, 2 * r1 + s1), (2 * r1 + s1, 2 * r0 + s0)]
    pairs += [(2 * r, 2 * r + 1) for r in (0, 5, 17)] + [(2 * r + 1, 2 * r) for r in (3, 11)]
    assert any(o0 >> 1 > o1 >> 1 for o0, o1 in pairs) and any(o0 & 1 for o0, _ in pairs)
    stored = 0
    for o0, o1 in pairs:
        ords, info = capi.align_oriented_reads(ctx, o0, o1, go)
        exp = expected_single_pair(row(d, o0), row(d, o1), opts)
        if method in (3, 4):
            _, pair_ords, _ = B.oracle_align_pair(row(d, o0), row(d, o1), oracle_options(opts))
            if len(ords):
                assert np.array_equal(ords, pair_ords), (o0, o1)
        if exp is None:
            assert len(ords) == 0 and not info.any(), (o0, o1)
            continue
        stored += 1
        assert np.array_equal(info, exp[0][3:16]), (o0, o1)
        assert np.array_equal(ords, exp[1]), (o0, o1)
    assert stored >= 12
    # Strand-0-first candidates with readId0 < readId1 give what computeAlignments gives on the same candidate.
    rec, ctoc, cdata, _ = capi.compute_alignments(ctx, cand[:6], go)
    same = {(int(r0), int(r1)): int(s) for r0, r1, s in cand[:6]}
    assert len(rec) >= 3
    for i in range(len(rec)):
        r0, r1 = int(rec[i, 0]), int(rec[i, 1])
        ords, info = capi.align_oriented_reads(ctx, 2 * r0, 2 * r1 + (0 if same[r0, r1] else 1), go)
        assert np.array_equal(info, rec[i, 3:16])
        assert np.array_equal(ords, B.oracle_decompress(cdata[int(ctoc[i]):int(ctoc[i + 1])]))


def test_align_oriented_reads_refusals(ctx):
    from shasta_b200 import capi
    d, _ = pair_dataset()
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    go = capi.make_align_options(**single_pair_options(3))
    with pytest.raises(capi.ShastaB200Error, match="two different oriented reads"):
        capi.align_oriented_reads(ctx, 7, 7, go)
    with pytest.raises(capi.ShastaB200Error, match="Invalid oriented read pair"):
        capi.align_oriented_reads(ctx, 2, 2 * len(d["flags"]), go)
