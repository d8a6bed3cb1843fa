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
from support import CONFIGS, compare_alignments, ctx  # noqa: F401

pytestmark = pytest.mark.gpu


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
    rec = compare_alignments(ctx, d, cand[:600], **cfg["align"])[0]
    assert len(rec) > 10, "the synthetic set should produce stored alignments for this configuration"
