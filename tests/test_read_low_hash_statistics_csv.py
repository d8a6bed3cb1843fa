"""ReadLowHashStatistics.csv written by the facade against the file the reference's own LowHash0 leaves in its working directory
(src/LowHash0.cpp:220-243), recorded in tests/golden/reference_csv.npz."""
from oracle import bindings as B
from shasta_b200 import assembler as A
from shasta_b200 import synth

import support  # noqa: F401  (puts tests/golden on sys.path)
from reference_outputs import recorded


def _reference_csv(d, p):
    B.ref_lowhash0(d["toc"], d["data"], d["flags"], p, threads=2)
    return open("ReadLowHashStatistics.csv").read()


def test_csv_is_byte_identical_to_the_reference(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("SHB_REF_KEEP_CSV", str(tmp_path))
    d = synth.generate(synth.SynthParams(reads=300, k=10, genome_markers=30000, n50_bases=12000, min_bases=6000, seed=17,
                                         palindromic_every=23))
    for m, min_bucket, max_bucket in ((4, 2, 30), (3, 5, 8)):
        p = B.LowHashParams(m=m, hashFraction=0.02, minHashIterationCount=6, minBucketSize=min_bucket, maxBucketSize=max_bucket,
                            minFrequency=2)
        want = recorded("csv", f"m{m}_bucket{min_bucket}_{max_bucket}", _reference_csv, d, p)
        _, stats, _ = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], p)
        A.write_read_low_hash_statistics_csv("ours.csv", stats, d["toc"], d["flags"], m)
        got = open("ours.csv").read()
        assert got == want
        assert want.count("\n") == 301 and ",Yes," in want
