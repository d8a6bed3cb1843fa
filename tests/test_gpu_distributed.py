"""GPU test of the library's sharded path (csrc/dist.cu) as a world of 1 (NCCL). tests/run_distributed_gpu.py is the same
check under torchrun for 2+ GPUs (usage in its docstring)."""
import numpy as np
import pytest

# The library takes libnccl.so.2 from the process (csrc/dist.cu). Torch is imported first, as a host that uses torch would,
# so that the process holds torch's NCCL build: the tests that import torch after this one fail to load it otherwise.
import torch  # noqa: F401

pytestmark = pytest.mark.gpu


def test_c_abi_sharded_path_world1_matches_oracle():
    """The library's own NCCL orchestration (csrc/dist.cu: shb_dist_init / shb_lowhash0_sharded /
    shb_compute_alignments_sharded) as a world of one: same calls as on 8 GPUs, NCCL send/recv to self."""
    from oracle import bindings as B
    from shasta_b200 import capi, synth

    d = synth.generate(synth.SynthParams(reads=400, k=14, genome_markers=30000, n50_bases=12000, min_bases=6000, seed=61,
                                         palindromic_every=40))
    params = dict(m=4, hashFraction=0.01, minHashIterationCount=10, alignmentCandidatesPerRead=20.0, log2MinHashBucketCount=0,
                  minBucketSize=2, maxBucketSize=30, minFrequency=2)
    ctx = capi.Context(0)
    try:
        ctx.dist_init(1, 0, capi.dist_unique_id())
        ctx.set_markers(d["toc"], d["data"], d["flags"])
        lp = capi.make_lowhash_params(**params)
        cand, stats, res = ctx.lowhash0_sharded(lp)
        oc, os_, _ = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], B.LowHashParams(**params))
        assert np.array_equal(cand, oc) and np.array_equal(stats, os_)
        assert res.candidateDigest == capi.digest_candidates(oc) and res.iterations == 10
        opts = dict(alignMethod=3, k=14, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10, minAlignedFraction=0.1,
                    downsamplingFactor=0.05, bandExtend=10, maxBand=1000)
        for _ in range(2):          # the second call reuses the gathered markers
            rec, ctoc, cdata, ares = capi.compute_alignments_sharded(ctx, cand[:1500], capi.make_align_options(**opts))
            orec, otoc, odata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], oc[:1500],
                                                               B.make_align_options(**{k: v for k, v in opts.items() if k in B.ALIGN_DEFAULTS}), threads=8)
            assert np.array_equal(rec, orec) and np.array_equal(ctoc, otoc) and np.array_equal(cdata, odata)
        # new markers -> gathered again
        ctx.set_markers(d["toc"], d["data"], d["flags"])
        cand2, _, _ = ctx.lowhash0_sharded(lp)
        assert np.array_equal(cand2, oc)
        rec2, _, _, _ = capi.compute_alignments_sharded(ctx, cand[:300], capi.make_align_options(**opts))
        assert np.array_equal(rec2, orec[:len(rec2)])
        t = ctx.dist_timing()
        assert t.entriesReceived > 0 and t.totalSeconds > 0
        # the candidate-driven stopping rule needs a per-iteration merge over the ranks: refused, with the reason
        with pytest.raises(capi.ShastaB200Error, match="fixed MinHash.minHashIterationCount"):
            ctx.lowhash0_sharded(capi.make_lowhash_params(**dict(params, minHashIterationCount=0)))
    finally:
        ctx.dist_finalize()
        ctx.close()
