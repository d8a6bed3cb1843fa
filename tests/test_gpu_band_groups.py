"""GPU parity tests, against the CPU oracle, for the DP kernels that run several jobs per warp: stage-2 bands of up to
126 offsets on groups of 8 lanes, and the stage-1 forward kernel on groups of 8 and 16 lanes. They cover the edges of
the band and row classes, groups left without a job at the end of a launch, and short or off-diagonal bands."""
import numpy as np
import pytest

from support import candidate_set, compare_alignments, ctx  # noqa: F401

pytestmark = pytest.mark.gpu


def _random_pairs(reads, count, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, reads, count)
    b = rng.integers(0, reads, count)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    ok = lo < hi
    return np.stack([lo[ok], hi[ok], rng.integers(0, 2, ok.sum())], 1).astype(np.uint32)


# Stage-2 band width W = (largest - smallest matching offset of the stage-1 path) + 2 * bandExtend + 1, before clipping to
# the matrix. A sweep of bandExtend puts bands on both sides of every 16-offset class edge of the 8-lane groups
# (W + 2 = 16C and 16C + 1) and of the 126 / 128 edge to the whole-warp classes; small maxBand values drop the bands just
# above them.
@pytest.mark.parametrize("band_extend,max_band", [(0, 1000), (2, 1000), (5, 1000), (7, 13), (9, 1000), (13, 29), (15, 1000),
                                                  (21, 45), (23, 1000), (29, 61), (31, 1000), (37, 77), (45, 93), (53, 109),
                                                  (60, 125), (61, 126), (62, 127), (63, 1000), (64, 1000), (66, 1000)])
def test_stage2_group_class_edges(ctx, band_extend, max_band):
    d, cand = candidate_set(150, 10, 45)
    compare_alignments(ctx, d, cand[:250], alignMethod=3, k=10, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=20,
                       minAlignedFraction=0.2, downsamplingFactor=0.1, bandExtend=band_extend, maxBand=max_band)


def test_short_reads_and_off_diagonal_bands(ctx):
    # Reads of a few markers (fewer than 8: a group has more lanes than rows), unrelated pairs, and Align4 bands that lie
    # entirely above or below the main diagonal (lo > 0 or hi < 0).
    d, _ = candidate_set(120, 10, 17, min_bases=40, n50=3000, sigma=1.2)
    lengths = np.diff(d["toc"].astype(np.int64))
    assert (lengths < 8).any()
    cand = _random_pairs(119, 800, 11)
    compare_alignments(ctx, d, cand, alignMethod=3, k=10, maxSkip=50, maxDrift=50, maxTrim=1000, minAlignedMarkerCount=1,
                       minAlignedFraction=0.0, downsamplingFactor=0.5, bandExtend=3, maxBand=100)
    compare_alignments(ctx, d, cand, alignMethod=4, k=10, maxSkip=100, maxDrift=100, maxTrim=1000, minAlignedMarkerCount=1,
                       minAlignedFraction=0.0, align4DeltaX=20, align4DeltaY=4, align4MinEntryCountPerCell=1,
                       align4MaxDistanceFromBoundary=1000, maxBand=60)


# Stage 1 on the forward kernel: downsampled reads of 8 .. 512 markers. The downsampling factors move the row counts
# across the class edges G * R / G * R + 1 of both group sizes, including 128 / 129 (8 -> 16 lanes) and 256 / 257
# (16 lanes -> whole warps).
@pytest.mark.parametrize("factor", [0.02, 0.05, 0.08, 0.12, 0.18, 0.25, 0.4])
def test_stage1_forward_row_classes(ctx, factor):
    d, _ = candidate_set(120, 10, 29, n50=20000, min_bases=2000, sigma=0.8)
    cand = _random_pairs(119, 500, 7)
    compare_alignments(ctx, d, cand, alignMethod=3, k=10, maxSkip=50, maxDrift=50, maxTrim=1000, minAlignedMarkerCount=5,
                       minAlignedFraction=0.05, downsamplingFactor=factor, bandExtend=10, maxBand=1000)


@pytest.mark.parametrize("chunk", ["1", "3", "5", "13"])
def test_partly_filled_warps(ctx, monkeypatch, chunk):
    # Launches of a few jobs: the last warp of every launch has groups without a job.
    monkeypatch.setenv("SHB_ALIGN_BATCH", "97")
    monkeypatch.setenv("SHB_ALIGN_CHUNK", chunk)
    d, cand = candidate_set(150, 10, 45)
    compare_alignments(ctx, d, cand[:300], alignMethod=3, k=10, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=20,
                       minAlignedFraction=0.2, downsamplingFactor=0.1, bandExtend=20, maxBand=1000)
