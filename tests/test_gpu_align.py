"""GPU parity tests for Assembler::computeAlignments (method 3) through the C ABI, against the CPU oracle
(oracle/align_oracle.c) on the same seeded inputs. Bar: bit-exact AlignmentData records and compressed bytes.
The DP tie-break rule itself is 'parity unpinned' with respect to SeqAn (see oracle/align_oracle.c)."""
import numpy as np
import pytest

from oracle import bindings as B
from support import candidate_set, compare_alignments, ctx  # noqa: F401

pytestmark = pytest.mark.gpu


def test_method3_nanopore_like(ctx):
    d, cand = candidate_set(300, 10, 5)
    rec, _, _, res = compare_alignments(ctx, d, cand[:1500], alignMethod=3, k=10, maxSkip=30, maxDrift=30, maxTrim=30,
                                        minAlignedMarkerCount=100, minAlignedFraction=0.4, downsamplingFactor=0.1,
                                        bandExtend=10, maxBand=1000)
    assert len(rec) > 100 and res.dpCells > 0


def test_method3_may2022_options(ctx):
    d, cand = candidate_set(250, 14, 9)
    rec = compare_alignments(ctx, d, cand[:1200], alignMethod=3, k=14, maxSkip=100, maxDrift=100, maxTrim=100,
                             minAlignedMarkerCount=10, minAlignedFraction=0.1, downsamplingFactor=0.05, bandExtend=10,
                             maxBand=1000)[0]
    assert len(rec) > 100


def test_method3_strict_filters_and_containments(ctx):
    d, cand = candidate_set(250, 14, 13, drop=0.02, ins=0.01)
    compare_alignments(ctx, d, cand[:1000], alignMethod=3, k=14, maxSkip=6, maxDrift=4, maxTrim=2, minAlignedMarkerCount=200,
                       minAlignedFraction=0.97, downsamplingFactor=0.05, bandExtend=10, maxBand=1000)
    compare_alignments(ctx, d, cand[:1000], alignMethod=3, k=14, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=50,
                       minAlignedFraction=0.3, downsamplingFactor=0.1, bandExtend=5, maxBand=40, suppressContainments=1)


def test_method3_random_pairs_and_scores(ctx):
    # Unrelated read pairs (mostly empty / rejected alignments) and non-default scores.
    d, _ = candidate_set(120, 10, 21)
    rng = np.random.default_rng(3)
    a = rng.integers(0, 119, 600)
    b = rng.integers(0, 119, 600)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    ok = lo < hi
    cand = np.stack([lo[ok], hi[ok], rng.integers(0, 2, ok.sum())], 1).astype(np.uint32)
    compare_alignments(ctx, d, cand, alignMethod=3, k=10, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=5,
                       minAlignedFraction=0.05, downsamplingFactor=0.2, bandExtend=10, maxBand=1000)
    compare_alignments(ctx, d, cand, alignMethod=3, k=10, maxSkip=50, maxDrift=50, maxTrim=1000, minAlignedMarkerCount=3,
                       minAlignedFraction=0.0, matchScore=3, mismatchScore=-2, gapScore=-1, downsamplingFactor=0.3,
                       bandExtend=3, maxBand=200)


def test_method1_unbanded_all_markers(ctx):
    # Align.alignMethod 1 (src/AssemblerAlign1.cpp:129-148): one unbanded DP on all markers; the bands are as wide as
    # nx + ny + 1, i.e. the widest wavefront classes and the scan kernel.
    d, cand = candidate_set(60, 10, 7, genome_markers=4000, n50=6000, min_bases=4000)
    rec = compare_alignments(ctx, d, cand[:150], alignMethod=1, k=10, maxSkip=30, maxDrift=30, maxTrim=30,
                             minAlignedMarkerCount=50, minAlignedFraction=0.3)[0]
    assert len(rec) > 10


def test_alignment_properties(ctx):
    # Size-independent properties of the stored alignments: ordinals strictly increasing, codec round trip.
    from shasta_b200 import capi
    d, cand = candidate_set(200, 10, 33)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    rec, ctoc, cdata, _ = capi.compute_alignments(ctx, cand[:800], capi.make_align_options(k=10, minAlignedMarkerCount=50))
    assert len(rec)
    for i in range(len(rec)):
        ords = B.oracle_decompress(cdata[int(ctoc[i]):int(ctoc[i + 1])])
        assert len(ords) == rec[i, 9]
        assert (np.diff(ords[:, 0].astype(np.int64)) > 0).all() and (np.diff(ords[:, 1].astype(np.int64)) > 0).all()
        assert ords[0, 0] == rec[i, 4] and ords[-1, 0] == rec[i, 5] and ords[0, 1] == rec[i, 7] and ords[-1, 1] == rec[i, 8]
        off = ords[:, 0].astype(np.int64) - ords[:, 1].astype(np.int64)
        assert off.min() == np.int32(rec[i, 10]) and off.max() == np.int32(rec[i, 11])


def test_method4_default_cells(ctx):
    # Align4 (north_star's method): deltaX 200, deltaY 10, minEntryCountPerCell 10, maxDistanceFromBoundary 100
    # (src/AssemblerOptions.cpp:471-489); May2022-style filter values.
    d, cand = candidate_set(300, 10, 5)
    rec, _, _, res = compare_alignments(ctx, d, cand[:1200], alignMethod=4, k=10, maxSkip=100, maxDrift=100, maxTrim=100,
                                        minAlignedMarkerCount=10, minAlignedFraction=0.1, maxBand=1000)
    assert len(rec) > 100 and res.dpCells > 0


def test_method4_small_cells_strict_and_containments(ctx):
    d, cand = candidate_set(250, 14, 9)
    compare_alignments(ctx, d, cand[:800], alignMethod=4, k=14, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=60,
                       minAlignedFraction=0.4, align4DeltaX=100, align4DeltaY=5, align4MinEntryCountPerCell=4,
                       align4MaxDistanceFromBoundary=50, maxBand=300)
    compare_alignments(ctx, d, cand[:800], alignMethod=4, k=14, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10,
                       minAlignedFraction=0.1, align4DeltaX=50, align4DeltaY=20, align4MinEntryCountPerCell=1,
                       align4MaxDistanceFromBoundary=1000, maxBand=100, suppressContainments=1)


@pytest.mark.parametrize("smem_cells", ["1", "6"])
def test_method4_front_end_global_path(ctx, monkeypatch, smem_cells):
    """The Align4 front end keeps a candidate's existing cells in shared memory when they fit; candidates with more
    cells take the global-memory path. A tiny limit sends (nearly) every candidate through that path."""
    monkeypatch.setenv("SHB_ALIGN4_SMEM_CELLS", smem_cells)
    d, cand = candidate_set(250, 14, 9)
    compare_alignments(ctx, d, cand[:600], alignMethod=4, k=14, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10,
                       minAlignedFraction=0.1, align4DeltaX=50, align4DeltaY=20, align4MinEntryCountPerCell=1,
                       align4MaxDistanceFromBoundary=1000, maxBand=100)
    compare_alignments(ctx, d, cand[:600], alignMethod=4, k=14, maxSkip=100, maxDrift=100, maxTrim=100,
                       minAlignedMarkerCount=10, minAlignedFraction=0.1, maxBand=1000)


def test_method4_random_pairs(ctx):
    d, _ = candidate_set(120, 10, 21)
    rng = np.random.default_rng(5)
    a = rng.integers(0, 119, 500)
    b = rng.integers(0, 119, 500)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    ok = lo < hi
    cand = np.stack([lo[ok], hi[ok], rng.integers(0, 2, ok.sum())], 1).astype(np.uint32)
    compare_alignments(ctx, d, cand, alignMethod=4, k=10, maxSkip=100, maxDrift=100, maxTrim=1000, minAlignedMarkerCount=5,
                       minAlignedFraction=0.05, align4MinEntryCountPerCell=2, maxBand=2000)


def test_alignment_table(ctx):
    from shasta_b200 import capi
    d, cand = candidate_set(200, 10, 33)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    rec, _, _, _ = capi.compute_alignments(ctx, cand[:900], capi.make_align_options(k=10, minAlignedMarkerCount=50))
    toc, table = capi.compute_alignment_table(ctx, rec, 200)
    otoc, otable = B.oracle_compute_alignment_table(rec, 200)
    assert len(rec) > 50
    assert np.array_equal(toc, otoc) and np.array_equal(table, otable)
    # every alignment appears exactly 4 times
    assert np.array_equal(np.bincount(table, minlength=len(rec)), np.full(len(rec), 4))
    toc0, table0 = capi.compute_alignment_table(ctx, rec[:0], 200)
    assert toc0.sum() == 0 and len(table0) == 0


def test_candidate_table(ctx):
    from shasta_b200 import capi
    d, cand = candidate_set(200, 10, 33)
    toc, table = capi.compute_candidate_table(ctx, cand, 200)
    otoc, otable = B.oracle_compute_candidate_table(cand, 200)
    assert len(cand) > 500
    assert toc.dtype == np.uint64 and table.dtype == np.uint64
    assert np.array_equal(toc, otoc) and np.array_equal(table, otable)
    assert np.array_equal(np.bincount(table.astype(np.int64), minlength=len(cand)), np.full(len(cand), 4))
    toc0, table0 = capi.compute_candidate_table(ctx, cand[:0], 200)
    assert toc0.sum() == 0 and len(table0) == 0


@pytest.mark.parametrize("band_extend,max_band", [(40, 1000), (90, 1000), (150, 1000), (230, 1000), (350, 2000), (480, 2000),
                                                  (700, 3000), (1500, 6000)])
def test_all_band_classes(ctx, band_extend, max_band):
    # bandExtend widens the stage-2 band so that every kernel class is exercised: the register-resident wavefront kernel
    # with C = 2, 3, 4, 6, 8, 12, 16 sub-chunk widths, and the shared-memory scan kernel for bands wider than 1024.
    d, cand = candidate_set(150, 10, 45)
    compare_alignments(ctx, d, cand[:250], alignMethod=3, k=10, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=50,
                       minAlignedFraction=0.3, downsamplingFactor=0.1, bandExtend=band_extend, maxBand=max_band)


def test_long_reads_wide_stage1(ctx):
    # Ultra-long-like reads: stage 1 runs on ~700 downsampled markers per read (band classes C = 12/16 and the scan kernel).
    d, cand = candidate_set(24, 10, 3, genome_markers=9000, n50=90000, min_bases=60000, sigma=0.2)
    assert len(cand) > 20
    compare_alignments(ctx, d, cand[:60], alignMethod=3, k=10, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10,
                       minAlignedFraction=0.1, downsamplingFactor=0.15, bandExtend=10, maxBand=1000)
    compare_alignments(ctx, d, cand[:60], alignMethod=4, k=10, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10,
                       minAlignedFraction=0.1, maxBand=1000)
