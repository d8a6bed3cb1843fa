"""flagPalindromicReads on the GPU (csrc/palindromic.cu, shb_flag_palindromic_reads) against the C restatement
(oracle/palindromic_oracle.c), which tests/test_oracle_palindromic.py pins to the reference build."""
import os

import numpy as np
import pytest

from oracle import palindromic_bindings as B
from support import LOWHASH, ctx, pack_ordinal_markers  # noqa: F401

from palindromic_inputs import cases, killer_case, oriented, palindrome, reverse_complement, rows_to_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = cases()


def _upload(ctx, toc, ids, flags=None):
    R = (len(toc) - 1) // 2
    ctx.set_markers(toc, pack_ordinal_markers(toc, ids), np.zeros(R, np.uint8) if flags is None else flags)


def _params(p):
    from shasta_b200 import capi
    d = dict(B.PALINDROMIC_DEFAULTS)
    d.update(p)
    return capi.make_palindromic_params(**d)


def _compare(ctx, toc, ids, params, paths=True):
    from shasta_b200 import capi
    R = (len(toc) - 1) // 2
    _upload(ctx, toc, ids)
    o = B.oracle_flag_palindromic(toc, ids, **params)
    flags = np.full(R, 0xfe, np.uint8)
    aligned, near, res = capi.flag_palindromic_reads(ctx, _params(params), read_flags=flags)
    assert np.array_equal(flags & 1, o["flags"]) and np.all(flags & 0xfe == 0xfe)
    assert np.array_equal(aligned, o["aligned"]) and np.array_equal(near, o["nearDiagonal"])
    assert res.readCount == R and res.palindromicReadCount == int(o["flags"].sum())
    assert res.exactReadCount == int(o["survives"].sum()) == o["counters"]["exactReads"]
    assert res.vertexCount == o["counters"]["vertices"] and res.edgeCount == o["counters"]["edges"]
    assert res.heapPushCount == o["counters"]["heapPushes"]
    if paths:
        for r in np.flatnonzero(o["survives"]):
            want = B.oracle_flag_palindromic(toc, ids, path_read=int(r), **params)["path"]
            assert np.array_equal(capi.palindromic_read_alignment(ctx, int(r), _params(params)), want), f"read {r}"
    return o, res


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_equals_oracle(ctx, name):
    toc, ids, params = CASES[name]
    _compare(ctx, toc, ids, params)


@pytest.mark.gpu
def test_heapsort_fallback_and_small_batches(ctx, monkeypatch):
    toc, ids, params = killer_case(B.oracle_sort_killer_keys(3000))
    # Zero thresholds send every read to the exact phase, where the device sorts its rows as the oracle does.
    params = dict(params, alignedFractionThreshold=0.0, nearDiagonalFractionThreshold=0.0)
    o, res = _compare(ctx, toc, ids, params)
    assert res.heapsortFallbackCount == o["counters"]["heapsortFallbacks"] > 0
    # One read per phase-B batch and a few reads per phase-A sort chunk give the same result.
    monkeypatch.setenv("SHB_PALINDROMIC_BUDGET_MB", "1")
    monkeypatch.setenv("SHB_PALINDROMIC_SORT_CHUNK", "1000")
    toc, ids, params = CASES["noisy_palindromes"]
    _compare(ctx, toc, ids, params, paths=False)


@pytest.mark.gpu
def test_null_outputs_and_context_flags(ctx):
    from shasta_b200 import capi
    toc, ids, params = CASES["noisy_palindromes"]
    R = (len(toc) - 1) // 2
    flags = (np.arange(R) * 37 % 256).astype(np.uint8) | 1
    _upload(ctx, toc, ids, flags)
    o = B.oracle_flag_palindromic(toc, ids, **params)
    _, _, res = capi.flag_palindromic_reads(ctx, _params(params), read_flags=None, want_counts=False)
    assert res.palindromicReadCount == int(o["flags"].sum())
    # Bits 1-7 of the caller's array are kept whatever bit 0 was.
    out = flags.copy()
    capi.flag_palindromic_reads(ctx, _params(params), read_flags=out)
    assert np.array_equal(out, (flags & 0xfe) | o["flags"])


@pytest.mark.gpu
def test_lowhash0_sees_new_flags(ctx):
    """A synthetic read set with injected palindromic reads: LowHash0 after the call equals LowHash0 on markers uploaded
    with the oracle's flags."""
    from shasta_b200 import capi, synth
    d = synth.generate(synth.SynthParams(reads=300, k=10, genome_markers=30000, n50_bases=12000, min_bases=6000, seed=11))
    toc, kmer, flags0 = d["toc"], d["kmer"].copy(), d["flags"].copy()
    R = len(flags0)
    for r in range(0, R, 50):
        b, m, e = int(toc[2 * r]), int(toc[2 * r + 1]), int(toc[2 * r + 2])
        s0 = kmer[b:m].copy()
        h = len(s0) // 2
        s0[len(s0) - h:] = reverse_complement(s0[:h][::-1], 10)
        kmer[b:m] = s0
        kmer[m:e] = reverse_complement(s0[::-1], 10)
    params = dict(B.PALINDROMIC_DEFAULTS)
    o = B.oracle_flag_palindromic(toc, kmer, **params)
    assert o["flags"].sum() >= R // 50
    data7 = synth.pack_markers(kmer, d["pos"])
    lp = capi.make_lowhash_params(**LOWHASH)
    ctx.set_markers(toc, data7, flags0)
    flags = flags0.copy()
    capi.flag_palindromic_reads(ctx, _params(params), read_flags=flags)
    assert np.array_equal(flags, (flags0 & 0xfe) | o["flags"])
    cand, stats, _, _ = ctx.lowhash0(lp)
    ctx.set_markers(toc, data7, (flags0 & 0xfe) | o["flags"])
    cand2, stats2, _, _ = ctx.lowhash0(lp)
    assert np.array_equal(cand, cand2) and np.array_equal(stats, stats2)
    # LowHash0 skips palindromic reads (src/LowHash0.cpp:325): none of the flagged reads is in a candidate pair.
    flagged = np.flatnonzero(o["flags"])
    assert len(cand) and not np.isin(cand[:, :2], flagged).any()


@pytest.mark.gpu
def test_markers_from_find_markers(ctx):
    from shasta_b200 import capi
    r = np.load(os.path.join(ROOT, "tests", "golden", "tinytest_reads.npz"))
    m = np.load(os.path.join(ROOT, "tests", "golden", "tinytest_markers.npz"))
    toc, data, _ = ctx.find_markers(10, r["word_offsets"], r["words"], r["base_counts"], m["flags"], is_marker_bitmap=r["is_marker_bitmap"])
    ids = np.ascontiguousarray(np.asarray(data, np.uint8).reshape(-1, 7)[:, :4]).view(np.uint32).reshape(-1)
    for params in (dict(), dict(alignedFractionThreshold=0.0, nearDiagonalFractionThreshold=0.0)):
        o = B.oracle_flag_palindromic(toc, ids, **params)
        aligned, near, res = capi.flag_palindromic_reads(ctx, _params(params))
        assert np.array_equal(aligned, o["aligned"]) and np.array_equal(near, o["nearDiagonal"])
        assert res.palindromicReadCount == int(o["flags"].sum())


@pytest.mark.gpu
def test_sharded_context_refused(ctx):
    from shasta_b200 import capi
    toc, ids, params = CASES["random"]
    R = (len(toc) - 1) // 2
    half = R // 2
    local = toc[:2 * half + 1]
    ctx.set_markers(local, pack_ordinal_markers(local, ids[:int(local[-1])]), np.zeros(R, np.uint8), read_begin=0, read_end=half,
                    read_count_total=R, total_marker_count=int(toc[-1]))
    with pytest.raises(capi.ShastaB200Error) as e:
        capi.flag_palindromic_reads(ctx, _params(params))
    assert e.value.status == 4          # SHB_ERR_STATE


@pytest.mark.gpu
def test_ul_length_palindrome(ctx):
    """A UL-length palindromic read (7 500 markers per strand) next to ordinary reads."""
    rng = np.random.default_rng(99)
    reads = [oriented(palindrome(rng, 7500, noise=0.03)), oriented(rng.integers(0, 1 << 28, 3000))]
    toc, ids, params = rows_to_case(reads)
    o, res = _compare(ctx, toc, ids, params)
    assert o["flags"][0] == 1 and res.exactReadCount >= 1


@pytest.mark.gpu
def test_facade_writes_read_flags(tmp_path):
    from shasta_b200.assembler import Assembler, mm_read_vector, mm_write_vector
    toc, ids, params = CASES["noisy_palindromes"]
    R = (len(toc) - 1) // 2
    prefix = str(tmp_path / "Data") + "/"
    os.makedirs(prefix)
    flags = (np.arange(R) * 5 % 256).astype(np.uint8)
    mm_write_vector(prefix + "Markers.toc", np.asarray(toc, np.uint64))
    mm_write_vector(prefix + "Markers.data", pack_ordinal_markers(toc, ids), object_size=7)
    mm_write_vector(prefix + "ReadFlags", flags)
    a = Assembler(prefix)
    a.accessMarkers()
    a.flagPalindromicReads(100, 100, 10, 0.1, 0.1, 100)
    o = B.oracle_flag_palindromic(toc, ids)
    out = np.asarray(mm_read_vector(prefix + "ReadFlags", np.uint8, object_size=1))
    assert np.array_equal(out, (flags & 0xfe) | o["flags"])
