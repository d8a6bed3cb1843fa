"""GPU parity tests (run on an H100 with -m gpu): the CUDA LowHash0 path, called through the
C ABI, against the reference's golden vectors and against the CPU oracle on the same seeded inputs.
Bar: bit-exact candidates (order included) and ReadLowHashStatistics."""
import json
import os

import numpy as np
import pytest

from oracle import bindings as B
from shasta_b200 import synth
from support import LOWHASH, TILE, ctx, feature_hashes, hash_threshold  # noqa: F401

import make_golden as MG

pytestmark = pytest.mark.gpu


def _params(capi, params, **extra):
    kw = dict(params)
    kw.update(extra)
    return capi.make_lowhash_params(**kw)


@pytest.mark.parametrize("name", list(MG.LOWHASH_CASES))
def test_golden_deferred_merge(ctx, name, golden_dir):
    from shasta_b200 import capi
    # With the candidate-driven iteration count (minHashIterationCount 0) the library merges after every iteration by
    # itself: the default call must still give the reference's candidates, statistics and number of iterations.
    spec, params = MG.LOWHASH_CASES[name]
    d = MG.load_input(spec)
    g = np.load(os.path.join(golden_dir, "lowhash_golden.npz"))
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    cand, stats, _, res = ctx.lowhash0(_params(capi, params))
    assert np.array_equal(cand, g[name + "/candidates"])
    assert np.array_equal(stats, g[name + "/stats"])
    assert res.iterations == len(g[name + "/summary"])
    assert res.kernelLaunches > 0


@pytest.mark.parametrize("limit", [1, 5000])
def test_golden_with_forced_intermediate_reductions(ctx, golden_dir, monkeypatch, limit):
    """The pair hits of the iterations are buffered raw and reduced (sorted, counted) in one go; a tiny buffer limit
    forces a reduction + merge after every iteration or every few, which must give the same candidates."""
    from shasta_b200 import capi
    g = np.load(os.path.join(golden_dir, "lowhash_golden.npz"))
    monkeypatch.setenv("SHB_LOWHASH_RAW_LIMIT", str(limit))
    for name, (spec, params) in MG.LOWHASH_CASES.items():
        if params.get("minHashIterationCount", 10) == 0:
            continue
        d = MG.load_input(spec)
        ctx.set_markers(d["toc"], d["data"], d["flags"])
        cand, stats, _, res = ctx.lowhash0(_params(capi, params))
        assert np.array_equal(cand, g[name + "/candidates"]), name
        assert np.array_equal(stats, g[name + "/stats"]), name


@pytest.mark.parametrize("aggregate", ["0", "1", "overflow"])
def test_golden_with_and_without_per_read_aggregation(ctx, golden_dir, monkeypatch, aggregate):
    """Pair hits are either buffered raw (Nanopore-like hashFraction) or counted per read in shared memory first (HiFi-like);
    both organisations must give the reference's candidates and statistics on every golden case, including the
    candidate-driven iteration count."""
    from shasta_b200 import capi
    g = np.load(os.path.join(golden_dir, "lowhash_golden.npz"))
    monkeypatch.setenv("SHB_LOWHASH_AGGREGATE", "0" if aggregate == "0" else "1")
    if aggregate == "overflow":         # one probe only: every collision in the per-read table takes the single-hit path
        monkeypatch.setenv("SHB_LOWHASH_TABLE_PROBES", "1")
    for name, (spec, params) in MG.LOWHASH_CASES.items():
        d = MG.load_input(spec)
        ctx.set_markers(d["toc"], d["data"], d["flags"])
        cand, stats, _, res = ctx.lowhash0(_params(capi, params))
        assert np.array_equal(cand, g[name + "/candidates"]), name
        assert np.array_equal(stats, g[name + "/stats"]), name


@pytest.mark.parametrize("name", list(MG.LOWHASH_CASES))
def test_golden_per_iteration_merge(ctx, name, golden_dir):
    from shasta_b200 import capi
    spec, params = MG.LOWHASH_CASES[name]
    d = MG.load_input(spec)
    g = np.load(os.path.join(golden_dir, "lowhash_golden.npz"))
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    cand, stats, summ, res = ctx.lowhash0(_params(capi, params, perIterationMerge=1), max_iter_summary=256)
    assert np.array_equal(cand, g[name + "/candidates"])
    assert np.array_equal(stats, g[name + "/stats"])
    assert np.array_equal(summ, g[name + "/summary"])


def test_tinytest_pin_through_host_call(ctx, golden_dir):
    # The reference-facing call with host buffers; SURVEY.md Appendix D pin.
    from shasta_b200 import capi
    z = np.load(os.path.join(golden_dir, "tinytest_markers.npz"))
    cand, stats, res = ctx.find_alignment_candidates_lowhash0(
        z["toc"], z["data"], z["flags"],
        capi.make_lowhash_params(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=0, maxBucketSize=10, minFrequency=2))
    assert len(cand) == 186 and B.candidate_digest(cand) == 0x3fc2c96e354f8733
    assert res.log2BucketCount == 16


@pytest.mark.parametrize("m", [1, 2, 3, 6, 7, 8, 9, 12, 13, 16, 31, 32])
def test_feature_lengths_against_oracle(ctx, m):
    from shasta_b200 import capi
    d = synth.generate(synth.SynthParams(reads=120, k=10, genome_markers=15000, n50_bases=12000, min_bases=6000, seed=40 + m))
    kw = dict(m=m, hashFraction=0.02, minHashIterationCount=5, minBucketSize=0, maxBucketSize=20, minFrequency=1)
    if m > 8:
        # Generic kernel (m > 8): some low hash of the launch starts at the last position of a full tile, so that its
        # feature reads m - 1 words of the halo that follows the tile (at m = 32, up to its last word).
        M = int(d["toc"][-1])
        local = np.arange(TILE - m + 1, TILE)
        positions = (np.arange(1, M // TILE)[:, None] * TILE + local[None, :] - TILE).ravel()
        h = feature_hashes(d["kmer"], m, [37 * s for s in range(5)], positions=positions)
        halo = (h < np.uint64(hash_threshold(0.02))).any(0)
        assert (positions[halo] % TILE == TILE - 1).any()
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    cand, stats, _, _ = ctx.lowhash0(capi.make_lowhash_params(**kw))
    oc, os_, _ = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], B.LowHashParams(**kw))
    assert np.array_equal(cand, oc)
    assert np.array_equal(stats, os_)


def test_feature_length_33_is_refused(ctx):
    from shasta_b200 import capi
    d = synth.generate(synth.SynthParams(reads=20, k=10, genome_markers=6000, n50_bases=9000, min_bases=4000, seed=3))
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    with pytest.raises(capi.ShastaB200Error, match="MinHash.m must be between 1 and 32"):
        ctx.lowhash0(capi.make_lowhash_params(m=33))


def test_edge_cases_against_oracle(ctx):
    from shasta_b200 import capi
    d = synth.generate(synth.SynthParams(reads=60, k=10, genome_markers=8000, n50_bases=9000, min_bases=4000, seed=77,
                                         palindromic_every=3))
    toc = d["toc"].astype(np.int64)
    # Ragged input: empty reads and reads shorter than m markers.
    kmer, pos = synth.unpack_markers(d["data"])
    keep_rows = []
    newtoc = [0]
    for r in range(60):
        a, b, c = toc[2 * r], toc[2 * r + 1], toc[2 * r + 2]
        n = 0 if r % 7 == 0 else (2 if r % 7 == 1 else b - a)
        keep_rows.append(np.arange(a, a + n))
        newtoc.append(newtoc[-1] + n)
        keep_rows.append(np.arange(c - n, c))
        newtoc.append(newtoc[-1] + n)
    idx = np.concatenate(keep_rows).astype(np.int64)
    data = synth.pack_markers(kmer[idx], pos[idx])
    newtoc = np.array(newtoc, np.uint64)
    for kw in (dict(m=4, hashFraction=0.05, minHashIterationCount=3, minBucketSize=0, maxBucketSize=6, minFrequency=1),
               dict(m=4, hashFraction=0.9, minHashIterationCount=2, minBucketSize=3, maxBucketSize=50, minFrequency=2),
               dict(m=4, hashFraction=0.01, minHashIterationCount=17, minBucketSize=0, maxBucketSize=1000000, minFrequency=1),
               dict(m=4, hashFraction=0.03, minHashIterationCount=0, alignmentCandidatesPerRead=1.2, minBucketSize=0, maxBucketSize=10, minFrequency=2)):
        ctx.set_markers(newtoc, data, d["flags"])
        cand, stats, _, res = ctx.lowhash0(capi.make_lowhash_params(**kw))
        oc, os_, osum = B.oracle_lowhash0(newtoc, data, d["flags"], B.LowHashParams(**kw))
        assert np.array_equal(cand, oc), kw
        assert np.array_equal(stats, os_), kw
        assert res.iterations == len(osum)


def test_empty_input_and_errors(ctx):
    from shasta_b200 import capi
    # All reads empty.
    toc = np.zeros(2 * 5 + 1, np.uint64)
    ctx.set_markers(toc, np.zeros(0, np.uint8), np.zeros(5, np.uint8))
    cand, stats, _, _ = ctx.lowhash0(capi.make_lowhash_params())
    assert len(cand) == 0 and stats.sum() == 0
    # The reference throws "log2MinHashBucketCount is unreasonably small." (src/LowHash0.cpp:86)
    d = synth.generate(synth.SynthParams(reads=40, k=10, genome_markers=6000, n50_bases=9000, min_bases=4000, seed=2))
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    with pytest.raises(capi.ShastaB200Error, match="unreasonably small"):
        ctx.lowhash0(capi.make_lowhash_params(log2MinHashBucketCount=3))


def test_uint16_frequency_wraps(ctx):
    # src/LowHash0.hpp:116 / LowHash0.cpp:521: the pair frequency is a uint16 that wraps. Two reads
    # sharing one repeated feature 300 times give 300*300 = 90000 hits per iteration = 24464 mod 65536.
    from shasta_b200 import capi
    motif = np.array([5, 9, 2, 7], np.uint32)
    row = np.tile(motif, 300)
    rc = synth.reverse_complement_kmer(row[::-1], 10)
    kmer = np.concatenate([row, rc, row, rc])
    pos = np.arange(len(kmer), dtype=np.uint32) % 60000
    toc = np.array([0, 1200, 2400, 3600, 4800], np.uint64)
    data = synth.pack_markers(kmer, pos)
    flags = np.zeros(2, np.uint8)
    # ~716k hits = ~61k mod 65536: kept at minFrequency 60000, dropped at 62000 (a non-wrapping sum keeps both).
    for minFrequency, expected in ((60000, 1), (62000, 0)):
        kw = dict(m=4, hashFraction=0.999, minHashIterationCount=1, minBucketSize=0, maxBucketSize=100000, minFrequency=minFrequency)
        ctx.set_markers(toc, data, flags)
        cand, stats, _, _ = ctx.lowhash0(capi.make_lowhash_params(**kw))
        oc, os_, _ = B.oracle_lowhash0(toc, data, flags, B.LowHashParams(**kw))
        assert len(oc) == expected
        assert np.array_equal(cand, oc) and np.array_equal(stats, os_)


def test_larger_synthetic_properties_and_oracle(ctx):
    # A larger case (10k-read class is exercised by bench.py); here 3000 reads against the oracle, plus
    # size-independent properties of the output.
    from shasta_b200 import capi
    d = synth.generate(synth.SynthParams(reads=3000, k=14, genome_markers=250000, n50_bases=20000, seed=21))
    kw = dict(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=5, maxBucketSize=30, minFrequency=5)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    cand, stats, _, res = ctx.lowhash0(capi.make_lowhash_params(**kw))
    assert (cand[:, 0] < cand[:, 1]).all()
    key = (cand[:, 0].astype(np.uint64) << np.uint64(33)) | (cand[:, 1].astype(np.uint64) << np.uint64(1)) | (1 - cand[:, 2]).astype(np.uint64)
    assert (np.diff(key.astype(np.int64)) > 0).all()           # strictly increasing (readId0, readId1, strand)
    assert int(stats.sum()) == res.lowHashCount
    oc, os_, _ = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], B.LowHashParams(**kw))
    assert np.array_equal(cand, oc) and np.array_equal(stats, os_)
    # Idempotence: a second run on the same context gives the same bytes.
    cand2, stats2, _, _ = ctx.lowhash0(capi.make_lowhash_params(**kw))
    assert np.array_equal(cand, cand2) and np.array_equal(stats, stats2)


def test_device_generator_matches_numpy(ctx):
    # The bench's on-device generator (csrc/synth.cu) must reproduce shasta_b200.synth.generate bit for bit.
    from shasta_b200 import capi
    p = synth.SynthParams(reads=400, k=14, genome_markers=40000, n50_bases=15000, min_bases=5000, seed=123, palindromic_every=50)
    d = synth.generate(p)
    dm = capi.synth_generate_device(ctx, p, want_data7=True)
    assert np.array_equal(dm.toc, d["toc"])
    assert np.array_equal(dm.kmer_ids_to_host(), d["kmer"])
    assert np.array_equal(dm.data7_to_host(), d["data"])
    assert np.array_equal(dm.flags, d["flags"])
    # Device-resident path gives the same candidates as the host-upload path.
    ctx.set_markers_device(dm.toc, dm.kmer_ptr, dm.flags, keepalive=dm)
    c1, s1, _, _ = ctx.lowhash0(capi.make_lowhash_params(**LOWHASH))
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    c2, s2, _, _ = ctx.lowhash0(capi.make_lowhash_params(**LOWHASH))
    assert np.array_equal(c1, c2) and np.array_equal(s1, s2) and len(c1) > 0
    dm.free()
