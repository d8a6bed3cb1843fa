"""GPU tests of the batching / chunking / multi-stream machinery of shb_compute_alignments.

The production sizes (262 144 candidates per batch, 32 768 jobs per chunk) need inputs far larger than the oracle can check in
seconds, so the library's test hooks SHB_ALIGN_BATCH / SHB_ALIGN_CHUNK shrink them: a few thousand candidates then run through
many batches, many chunks per band class on all streams, and the result must still be bit-identical to the oracle's and to a
second run of the same call."""
import numpy as np
import pytest

from oracle import bindings as B
from support import candidate_set, ctx, oracle_options  # noqa: F401

pytestmark = pytest.mark.gpu

OPTS = dict(alignMethod=3, k=14, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10, minAlignedFraction=0.1,
            downsamplingFactor=0.05, bandExtend=10, maxBand=1000)


@pytest.fixture(scope="module")
def dataset():
    d, cand = candidate_set(500, 14, 77, genome_markers=30000)
    assert len(cand) > 2500
    return d, cand[:3000]


def _run(ctx, d, cand, **opts):
    from shasta_b200 import capi
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    rec, ctoc, cdata, res = capi.compute_alignments(ctx, cand, capi.make_align_options(**opts))
    return rec.copy(), ctoc.copy(), cdata.copy(), res


@pytest.mark.parametrize("batch,chunk", [(700, 64), (257, 1000000), (4096, 33)])
def test_small_batches_and_chunks_match_oracle(ctx, dataset, monkeypatch, batch, chunk):
    d, cand = dataset
    orec, otoc, odata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], cand, oracle_options(OPTS), threads=8)
    monkeypatch.setenv("SHB_ALIGN_BATCH", str(batch))
    monkeypatch.setenv("SHB_ALIGN_CHUNK", str(chunk))
    rec, ctoc, cdata, res = _run(ctx, d, cand, **OPTS)
    assert res.candidateCount == len(cand)
    assert len(orec) > 300
    assert np.array_equal(rec, orec) and np.array_equal(ctoc, otoc) and np.array_equal(cdata, odata)


@pytest.mark.parametrize("workers", [1, 2, 3])
def test_worker_threads_match_oracle(ctx, dataset, monkeypatch, workers):
    # The batches of one call are spread over host worker threads, each with its own streams and scratch; the kept
    # alignments land in a shared arena in completion order and are put back into candidate order at the end.
    d, cand = dataset
    orec, otoc, odata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], cand, oracle_options(OPTS), threads=8)
    monkeypatch.setenv("SHB_ALIGN_BATCH", "211")
    monkeypatch.setenv("SHB_ALIGN_CHUNK", "70")
    monkeypatch.setenv("SHB_ALIGN_WORKERS", str(workers))
    for _ in range(2):
        rec, ctoc, cdata, res = _run(ctx, d, cand, **OPTS)
        assert res.workers == workers
        assert np.array_equal(rec, orec) and np.array_equal(ctoc, otoc) and np.array_equal(cdata, odata)


def test_method4_small_batches_match_oracle(ctx, dataset, monkeypatch):
    d, cand = dataset
    opts = dict(OPTS, alignMethod=4)
    orec, otoc, odata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], cand[:1200], oracle_options(opts), threads=8)
    monkeypatch.setenv("SHB_ALIGN_BATCH", "300")
    monkeypatch.setenv("SHB_ALIGN_CHUNK", "50")
    rec, ctoc, cdata, _ = _run(ctx, d, cand[:1200], **opts)
    assert np.array_equal(rec, orec) and np.array_equal(ctoc, otoc) and np.array_equal(cdata, odata)


def test_repeated_calls_are_identical(ctx, dataset, monkeypatch):
    # The chunks of a batch run on several streams; a missing dependency would show up as run-to-run differences.
    d, cand = dataset
    monkeypatch.setenv("SHB_ALIGN_BATCH", "1500")
    monkeypatch.setenv("SHB_ALIGN_CHUNK", "100")
    first = _run(ctx, d, cand, **OPTS)
    for _ in range(3):
        again = _run(ctx, d, cand, **OPTS)
        assert all(np.array_equal(x, y) for x, y in zip(first[:3], again[:3]))
    # ... and the production sizes give the same answer as the shrunken ones
    monkeypatch.delenv("SHB_ALIGN_BATCH")
    monkeypatch.delenv("SHB_ALIGN_CHUNK")
    full = _run(ctx, d, cand, **OPTS)
    assert all(np.array_equal(x, y) for x, y in zip(first[:3], full[:3]))
