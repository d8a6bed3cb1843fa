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
from support import (FORWARD_MAX_MARKERS, FORWARD_MAX_ROWS, K, PERMISSIVE, Genome, assemble, candidate_set,  # noqa: F401
                     compare_alignments, ctx, downsampled, expected_single_pair, oracle_options, padded_width, row,
                     single_pair_options, wide_band_class)

pytestmark = pytest.mark.gpu


def true_offsets(origin, r0, r1):
    """Ordinal offsets (ordinal0 - ordinal1) of the markers the two strand-0 rows share in the genome."""
    a, b = origin[r0], origin[r1]
    _, ia, ib = np.intersect1d(a[a >= 0], b[b >= 0], return_indices=True)
    ia = np.flatnonzero(a >= 0)[ia]
    ib = np.flatnonzero(b >= 0)[ib]
    return ia.astype(np.int64) - ib.astype(np.int64)


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
    return assemble(rows, K), rows, origin, triples


@pytest.mark.parametrize("method", [3, 4])
def test_forward_kernel_marker_limit_edge(ctx, method):
    d, rows, origin, triples = edge_dataset()
    factor = 0.012
    cand = []
    for x, y, z in triples:
        cand += [(x, y, 1), (x, z, 1), (x, y, 0), (x, z, 0)]
    longest = [max(len(rows[a]), len(rows[b])) for a, b, _ in cand]
    assert {31999, 32000, 32001} <= set(longest)
    assert max(len(downsampled(r, factor)[0]) for r in rows) <= FORWARD_MAX_ROWS      # the marker count alone routes
    for x, y, z in triples:
        assert true_offsets(origin, x, y).max() > FORWARD_MAX_MARKERS - 600
        assert true_offsets(origin, x, z).min() < -(FORWARD_MAX_MARKERS - 600)
    opts = dict(PERMISSIVE, alignMethod=method, downsamplingFactor=factor, bandExtend=10, maxBand=1000)
    if method == 4:
        opts.update(align4DeltaX=200, align4DeltaY=10, align4MinEntryCountPerCell=2, align4MaxDistanceFromBoundary=400)
    rec = compare_alignments(ctx, d, cand, **opts)[0]
    offsets = rec[:, 10:12].view(np.int32)
    assert len(rec) >= 6 and offsets[:, 1].max() > FORWARD_MAX_MARKERS - 600 and offsets[:, 0].min() < -(FORWARD_MAX_MARKERS - 600)


# ---- B. the widest band classes and the too-wide skip --------------------------------------------------------------
def wide_dataset():
    lengths = (2700, 3200, 4300, 4400, 7900, 8600, 9600)
    starts = (0, 500, 1000, 1500, 800, 300, 100)
    genome = Genome(20000, seed=9, drop=0.03, ins=0.01)
    rows, origin = zip(*(genome.read(s, L) for s, L in zip(starts, lengths)))
    cand = np.array([(i, j, 1) for i in range(len(rows)) for j in range(i + 1, len(rows))], np.uint32)
    return assemble(rows, K), rows, origin, cand


def test_widest_stage1_classes_and_skip(ctx):
    d, rows, _, cand = wide_dataset()
    factor = 0.97
    ds = [len(downsampled(r, factor)[0]) for r in rows]
    assert min(ds) > FORWARD_MAX_ROWS                                    # every stage 1 takes the traced kernel
    widths = [ds[a] + ds[b] + 1 for a, b, _ in cand]                     # unbanded: offsets -ny ... nx
    classes = [wide_band_class(W) for W in widths]
    skips = [i for i, c in enumerate(classes) if c is None]
    assert classes.count(8192) >= 2 and classes.count(16384) >= 2 and len(skips) >= 2
    compare_alignments(ctx, d, cand, skips, alignMethod=3, downsamplingFactor=factor, bandExtend=10, maxBand=1000,
                       **{k: v for k, v in PERMISSIVE.items() if k != "minAlignedMarkerCount"}, minAlignedMarkerCount=10)


def test_widest_method1_classes_and_skip(ctx):
    d, rows, _, cand = wide_dataset()
    widths = [len(rows[a]) + len(rows[b]) + 1 for a, b, _ in cand]       # method 1: one unbanded DP on the full rows
    classes = [wide_band_class(W) for W in widths]
    skips = [i for i, c in enumerate(classes) if c is None]
    assert classes.count(8192) >= 2 and classes.count(16384) >= 2 and len(skips) >= 2
    compare_alignments(ctx, d, cand, skips, alignMethod=1, **PERMISSIVE)


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
    compare_alignments(ctx, d, cand, alignMethod=3, downsamplingFactor=0.1, bandExtend=band_extend, maxBand=max_band, **PERMISSIVE)


def test_max_band_limit(ctx):
    from shasta_b200 import capi
    d, _, _, cand = wide_dataset()
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    capi.compute_alignments(ctx, cand[:1], capi.make_align_options(k=K, maxBand=16317))
    with pytest.raises(capi.ShastaB200Error, match="limit 16317"):
        capi.compute_alignments(ctx, cand[:1], capi.make_align_options(k=K, maxBand=16318))


# ---- C. the single-pair entry point --------------------------------------------------------------------------------
def pair_dataset():
    return candidate_set(40, K, 71, genome_markers=6000, n50=8000, min_bases=3000)


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
