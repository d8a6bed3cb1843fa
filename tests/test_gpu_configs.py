"""GPU parity on the parameter sets of the five BASELINE.json configurations, at sizes the oracle finishes in seconds:
both entry points (LowHash0 then computeAlignments) through the C ABI, bit-exact against the CPU oracle.
  C1 conf/Nanopore-Dec2019.conf      (k 10, MinHash 5/30/5, Align defaults + minAlignedFraction 0.4, method 3)
  C2 conf/Nanopore-May2022.conf      (k 14, MinHash 5/30/5, method 3, ds 0.05, skip/drift/trim 100, minMarkers 10, minFrac 0.1)
  C3 = C2 sharded (tests/test_gpu_distributed.py at world 1, tests/run_distributed_gpu.py on 2+ GPUs)
  C4 conf/Nanopore-UL-May2022.conf   (long reads, MinHash 10/50/5, method 3 and --Align.alignMethod 4)
  C5 conf/HiFi-Oct2021.conf          (low error, hashFraction 0.05, 100 iterations, 10/60/3, skip 6, drift 4, trim 2, 200, 0.97)
MinHash defaults: m 4, hashFraction 0.01, 10 iterations (src/AssemblerOptions.cpp:327-378)."""
import numpy as np
import pytest

from oracle import bindings as B
from shasta_b200 import synth

pytestmark = pytest.mark.gpu

CONFIGS = {
    "C1-Nanopore-Dec2019": dict(
        synth=dict(reads=500, k=10, genome_markers=35000, n50_bases=20000, min_bases=10000, drop=0.12, ins=0.05, seed=101),
        minhash=dict(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=5, maxBucketSize=30, minFrequency=5),
        align=dict(alignMethod=3, k=10, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=100, minAlignedFraction=0.4,
                   downsamplingFactor=0.1, bandExtend=10, maxBand=1000)),
    "C2-Nanopore-May2022": dict(
        synth=dict(reads=400, k=14, genome_markers=40000, n50_bases=30000, min_bases=10000, drop=0.12, ins=0.05, seed=102),
        minhash=dict(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=5, maxBucketSize=30, minFrequency=5),
        align=dict(alignMethod=3, k=14, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10, minAlignedFraction=0.1,
                   downsamplingFactor=0.05, bandExtend=10, maxBand=1000)),
    "C4-Nanopore-UL-May2022-method3": dict(
        synth=dict(reads=120, k=14, genome_markers=40000, n50_bases=100000, min_bases=50000, sigma=0.3, drop=0.12, ins=0.05, seed=104),
        minhash=dict(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=10, maxBucketSize=50, minFrequency=5),
        align=dict(alignMethod=3, k=14, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10, minAlignedFraction=0.1,
                   downsamplingFactor=0.05, bandExtend=10, maxBand=1000)),
    "C4-Nanopore-UL-May2022-method4": dict(
        synth=dict(reads=120, k=14, genome_markers=40000, n50_bases=100000, min_bases=50000, sigma=0.3, drop=0.12, ins=0.05, seed=104),
        minhash=dict(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=10, maxBucketSize=50, minFrequency=5),
        align=dict(alignMethod=4, k=14, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10, minAlignedFraction=0.1,
                   maxBand=1000, align4DeltaX=200, align4DeltaY=10, align4MinEntryCountPerCell=10, align4MaxDistanceFromBoundary=100)),
    "C5-HiFi-Oct2021": dict(
        synth=dict(reads=500, k=14, genome_markers=40000, n50_bases=15000, min_bases=8000, drop=0.004, ins=0.002, seed=105),
        minhash=dict(m=4, hashFraction=0.05, minHashIterationCount=100, minBucketSize=10, maxBucketSize=60, minFrequency=3),
        align=dict(alignMethod=3, k=14, maxSkip=6, maxDrift=4, maxTrim=2, minAlignedMarkerCount=200, minAlignedFraction=0.97,
                   downsamplingFactor=0.05, bandExtend=10, maxBand=1000)),
}


@pytest.fixture(scope="module")
def ctx():
    from shasta_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("name", list(CONFIGS))
def test_config_parity(ctx, name):
    from shasta_b200 import capi
    cfg = CONFIGS[name]
    d = synth.generate(synth.SynthParams(**cfg["synth"]))
    cand, stats, res = ctx.find_alignment_candidates_lowhash0(d["toc"], d["data"], d["flags"], capi.make_lowhash_params(**cfg["minhash"]))
    oc, os_, osum = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], B.LowHashParams(**cfg["minhash"]))
    assert np.array_equal(cand, oc) and np.array_equal(stats, os_)
    assert res.iterations == cfg["minhash"]["minHashIterationCount"] == len(osum)
    assert len(cand) > 50, "the synthetic set should produce candidates for this configuration"
    sub = cand[:600]
    rec, ctoc, cdata, ares = capi.compute_alignments(ctx, sub, capi.make_align_options(**cfg["align"]))
    oo = B.make_align_options(**{k: v for k, v in cfg["align"].items() if k in B.ALIGN_DEFAULTS})
    orec, otoc, odata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], sub, oo, threads=8)
    assert np.array_equal(rec, orec) and np.array_equal(ctoc, otoc) and np.array_equal(cdata, odata)
    assert len(rec) > 10, "the synthetic set should produce stored alignments for this configuration"
