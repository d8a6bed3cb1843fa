"""GPU parity tests (run on an H100 with -m gpu) for the LowHash0 sweep paths that the synthetic workload does not reach:
the inline path taken when a tile's shared-memory queue is full, the global binary search for tiles that span more than
kSweepTileReads oriented reads, slab regrowth, and full tiles loaded from a k-mer id array that is not 16-byte aligned.
Bar: bit-exact candidates (order included) and ReadLowHashStatistics against the CPU oracle or the reference goldens.

Every test first checks on the host that its input reaches the path it is for (queued hits per tile, reads per tile, low
hashes per iteration), with a numpy MurmurHash64A that is itself checked against the oracle's."""
import os

import numpy as np
import pytest

from oracle import bindings as B
from shasta_b200 import synth
from support import LOWHASH, TILE, assemble, ctx, feature_hashes, hash_threshold, strand0_rows  # noqa: F401

import make_golden as MG

pytestmark = pytest.mark.gpu

U64 = np.uint64
TILE_READS = 32                 # kSweepTileReads
QUEUE_MIN, QUEUE_MAX = 256, 6144
UNROLLED_GROUPS = (16, 10, 8, 4, 2, 1)

HIFI = dict(m=4, hashFraction=0.05, minHashIterationCount=20, minBucketSize=10, maxBucketSize=60, minFrequency=3)


# ---- host model of the sweep ---------------------------------------------------------------------------------------
def sweep_groups(params):
    """Iterations fused into one sweep launch, in order (lowhash0 in csrc/lowhash.cu); None when the candidate count decides
    the number of iterations (groups of one)."""
    n = params.get("minHashIterationCount", 10)
    if n == 0 or params.get("perIterationMerge", 0):
        return None
    groups, left = [], n
    while left:
        g = next(g for g in UNROLLED_GROUPS if g <= left)
        groups.append(g)
        left -= g
    return groups


def queue_capacity(group, hash_fraction):
    # Restates the queue sizing of lowhashSweep (csrc/lowhash.cu): 1.5 x the expected 2048 * group * hashFraction + 64.
    return int(min(QUEUE_MAX, max(QUEUE_MIN, 1.5 * TILE * group * hash_fraction + 64.)))


def queued_per_tile(kmer, m, hash_fraction, first_iteration, group):
    """Hits the hot loop queues in every tile for one launch: (position, seed) pairs whose hash passes the high-word test.
    The high 32 bits of MurmurHash64A before its final h ^= h >> 47 are those of the finished hash."""
    seeds = [37 * (first_iteration + s) for s in range(group)]
    h = feature_hashes(kmer, m, seeds)
    hit = (h >> U64(32)) <= U64(hash_threshold(hash_fraction) >> 32)
    per_position = hit.sum(0)
    tiles = (len(kmer) + TILE - 1) // TILE
    return np.bincount(np.arange(len(per_position)) // TILE, weights=per_position, minlength=tiles).astype(np.int64), per_position


def valid_feature_mask(toc, flags, m):
    """Positions whose feature lies inside one oriented read of a non-palindromic read (src/LowHash0.cpp:325-344)."""
    toc = np.asarray(toc, np.int64)
    M = int(toc[-1])
    row = np.repeat(np.arange(len(toc) - 1), np.diff(toc))
    ok = (np.arange(M) + m <= toc[row + 1]) & (np.asarray(flags)[row >> 1] & 1 == 0)
    return ok[:max(M - m + 1, 0)]


def compare_with_oracle(ctx, d, params):
    from shasta_b200 import capi
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    cand, stats, _, res = ctx.lowhash0(capi.make_lowhash_params(**params))
    oc, os_, osum = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], B.LowHashParams(**params))
    assert np.array_equal(cand, oc)
    assert np.array_equal(stats, os_)
    assert res.iterations == len(osum)
    return cand, res


def test_numpy_murmur_matches_oracle():
    rng = np.random.default_rng(1)
    lib = B.oracle_lib()
    for m in (1, 2, 3, 4, 5, 13, 16, 31, 32):
        kmer = rng.integers(0, 1 << 32, 3 * m, dtype=np.uint64).astype(np.uint32)
        h = feature_hashes(kmer, m, [0, 37, 37 * 19])
        for i, seed in enumerate((0, 37, 37 * 19)):
            for p in range(2 * m + 1):
                assert int(h[i, p]) == lib.orc_murmurhash64a(kmer[p:].ctypes.data, 4 * m, seed)


# ---- A. tandem repeats: tiles whose queue overflows -----------------------------------------------------------------
def tandem_repeat_dataset():
    k = 10
    base = synth.generate(synth.SynthParams(reads=160, k=k, genome_markers=40000, n50_bases=16000, min_bases=6000, seed=91,
                                            palindromic_every=23))
    rng = np.random.default_rng(91)
    rows = strand0_rows(base)
    repeat = []
    periods = (1, 4, 12, 30)
    for i, r in enumerate(range(0, len(rows), 3)):
        period = periods[i % len(periods)]
        unit = rng.integers(0, 1 << (2 * k), period).astype(np.uint32)
        length = int(rng.integers(500, 3001))
        block = np.resize(unit, length)
        at = int(rng.integers(0, len(rows[r]) + 1))
        rows[r] = np.concatenate([rows[r][:at], block, rows[r][at:]])
        repeat.append((r, at, length))
    d = assemble(rows, k, base["flags"])
    in_repeat = np.zeros(int(d["toc"][-1]), bool)       # strand-0 repeat blocks and their reverse complements
    toc = d["toc"].astype(np.int64)
    for r, at, length in repeat:
        in_repeat[toc[2 * r] + at:toc[2 * r] + at + length] = True
        end1 = toc[2 * r + 2]
        in_repeat[end1 - at - length:end1 - at] = True
    return d, in_repeat


@pytest.mark.parametrize("aggregate", ["0", "1"])
@pytest.mark.parametrize("config", ["nanopore", "hifi"])
def test_tandem_repeats_overflow_the_sweep_queue(ctx, monkeypatch, aggregate, config):
    params = LOWHASH if config == "nanopore" else HIFI
    d, in_repeat = tandem_repeat_dataset()
    overflowing, ordinary_spill = 0, 0
    first = 0
    for group in sweep_groups(params):
        per_tile, per_position = queued_per_tile(d["kmer"], params["m"], params["hashFraction"], first, group)
        over = np.nonzero(per_tile > queue_capacity(group, params["hashFraction"]))[0]
        overflowing += len(over)
        for t in over:
            sl = slice(t * TILE, min((t + 1) * TILE, len(per_position)))
            ordinary_spill += int(per_position[sl][~in_repeat[sl]].sum() > 0)
        first += group
    assert overflowing >= 5 and ordinary_spill >= 3, (overflowing, ordinary_spill)
    monkeypatch.setenv("SHB_LOWHASH_AGGREGATE", aggregate)
    cand, _ = compare_with_oracle(ctx, d, params)
    assert len(cand) > 100


# ---- A. queue of one entry: every golden case through the inline path ----------------------------------------------
@pytest.mark.parametrize("aggregate", ["0", "1"])
def test_golden_cases_through_the_inline_path(ctx, golden_dir, monkeypatch, aggregate):
    from shasta_b200 import capi
    g = np.load(os.path.join(golden_dir, "lowhash_golden.npz"))
    monkeypatch.setenv("SHB_LOWHASH_AGGREGATE", aggregate)
    monkeypatch.setenv("SHB_LOWHASH_QUEUE_CAPACITY", "1")
    for name, (spec, params) in MG.LOWHASH_CASES.items():
        d = MG.load_input(spec)
        kmer, _ = synth.unpack_markers(d["data"])
        groups = sweep_groups(params) or [1]
        per_tile, _ = queued_per_tile(kmer[:TILE + 64], params["m"], params["hashFraction"], 0, groups[0])
        assert per_tile[0] > 1, name           # the first tile alone queues more than one hit
        ctx.set_markers(d["toc"], d["data"], d["flags"])
        cand, stats, _, res = ctx.lowhash0(capi.make_lowhash_params(**params))
        assert np.array_equal(cand, g[name + "/candidates"]), name
        assert np.array_equal(stats, g[name + "/stats"]), name
        assert res.iterations == len(g[name + "/summary"]), name


def test_queue_capacity_hook_is_clamped(ctx, monkeypatch):
    # Values beyond kSweepQueueMax are clamped (the dynamic shared memory stays within what the kernel allows).
    d = MG.load_input(MG.LOWHASH_CASES["synth600"][0])
    monkeypatch.setenv("SHB_LOWHASH_QUEUE_CAPACITY", "1000000")
    compare_with_oracle(ctx, d, MG.LOWHASH_CASES["synth600"][1])


# ---- A. many short reads per tile ----------------------------------------------------------------------------------
def short_reads_dataset():
    """Reads of 0 - 40 markers cut from a small genome (random strand), runs of 45 empty reads, palindromic flags; one read
    starts exactly at a tile boundary and is followed by rows whose 32nd boundary is exactly the tile's end."""
    k = 10
    rng = np.random.default_rng(5)
    genome = rng.integers(0, 1 << (2 * k), 6000).astype(np.uint32)
    lengths = []

    def random_reads(count):
        i = 0
        while i < count:
            if rng.random() < 0.01:
                lengths.extend([0] * 45)
                i += 45
            else:
                lengths.append(int(rng.integers(0, 41)))
                i += 1

    random_reads(1500)
    # Pad to the next tile boundary but one with reads of at most 40 markers (rows come in pairs of equal length).
    cum = 2 * sum(lengths)
    target = (cum // TILE + 2) * TILE
    while target - cum > 80:
        lengths.append(int(rng.integers(1, 41)))
        cum += 2 * lengths[-1]
    lengths.append((target - cum) // 2)
    boundary_read = len(lengths)
    lengths.append(1000)                                # rows at [target, target + 2000)
    lengths.extend([2] * 9 + [1] * 6)                   # 30 more rows: the tile's 32 rows end at target + 2048
    random_reads(1500)
    rows = []
    for L in lengths:
        s = int(rng.integers(0, len(genome) - L))
        r = genome[s:s + L]
        rows.append(synth.reverse_complement_kmer(r[::-1], k) if rng.random() < 0.5 else r)
    flags = np.zeros(len(lengths), np.uint8)
    flags[6::7] = 1
    flags[boundary_read] = 0
    return assemble(rows, k, flags), boundary_read


def test_tiles_with_many_short_reads(ctx):
    params = dict(m=4, hashFraction=0.05, minHashIterationCount=10, minBucketSize=0, maxBucketSize=30, minFrequency=1)
    d, boundary_read = short_reads_dataset()
    toc = d["toc"].astype(np.int64)
    M = int(toc[-1])
    lengths = np.diff(toc)
    # The input: empty runs of 40+, palindromic reads, a read starting at a tile boundary whose tile's 32 staged rows end
    # exactly at the tile's end.
    zero_run = np.diff(np.flatnonzero(np.diff(np.r_[1, lengths[::2], 1] == 0)))
    assert zero_run.max() >= 40 and d["flags"].sum() > 100
    b = toc[2 * boundary_read]
    assert b % TILE == 0 and lengths[2 * boundary_read] > 0 and toc[2 * boundary_read + TILE_READS] == b + TILE
    # Hits (exact test) that lie beyond the 32 staged rows of their tile take the global search; one lies exactly at the
    # first position beyond them.
    tiles = (M + TILE - 1) // TILE
    first_read = np.searchsorted(toc[:-1], np.arange(tiles) * TILE, side="right") - 1     # sweepTileReadsKernel
    staged_end = toc[np.minimum(first_read + TILE_READS, len(toc) - 1)]
    h = feature_hashes(d["kmer"], params["m"], [37 * s for s in range(10)])
    p = np.arange(h.shape[1])
    hit = (h < U64(hash_threshold(params["hashFraction"]))).any(0)
    beyond = hit & (p >= staged_end[p // TILE])
    assert np.unique(p[beyond] // TILE).size >= 10
    assert (hit & (p == staged_end[p // TILE])).any()
    cand, _ = compare_with_oracle(ctx, d, params)
    assert len(cand) > 1000
    compare_with_oracle(ctx, d, dict(params, m=1, minHashIterationCount=3))


# ---- A. slab regrowth ----------------------------------------------------------------------------------------------
def test_slab_regrowth(ctx):
    params = dict(LOWHASH)
    k, m, hf = 10, params["m"], params["hashFraction"]
    base = synth.generate(synth.SynthParams(reads=30, k=k, genome_markers=20000, n50_bases=12000, min_bases=6000, seed=13))
    # A k-mer whose feature (the k-mer m times) is a low hash in some iteration of the (only) group.
    th = U64(hash_threshold(hf))
    candidates = np.arange(1, 5000, dtype=np.uint32)
    h = feature_hashes(np.repeat(candidates, m), m, [37 * s for s in range(10)], positions=np.arange(len(candidates)) * m)
    kmer = int(candidates[(h < th).any(0)][0])
    rows = strand0_rows(base)
    rows.append(np.full(80000, kmer, np.uint32))
    d = assemble(rows, k, np.zeros(len(rows), np.uint8))
    M = int(d["toc"][-1])
    capacity = min(int(1.25 * hf * M) + 65536, M + 1)
    low = (feature_hashes(d["kmer"], m, [37 * s for s in range(10)]) < th) & valid_feature_mask(d["toc"], d["flags"], m)
    assert sweep_groups(params) == [10] and low.sum(1).max() > capacity
    cand, res = compare_with_oracle(ctx, d, params)
    assert res.sweepLaunches > 1 and len(cand) > 10


# ---- A. k-mer ids that are not 16-byte aligned ---------------------------------------------------------------------
@pytest.mark.parametrize("offset", [1, 2, 3])
def test_misaligned_kmer_ids(ctx, offset):
    import torch
    from shasta_b200 import capi
    d = synth.generate(synth.SynthParams(reads=200, k=10, genome_markers=25000, n50_bases=12000, min_bases=6000, seed=8))
    params = LOWHASH
    M = int(d["toc"][-1])
    buf = torch.zeros(M + 8, dtype=torch.int32, device="cuda")
    buf[offset:offset + M] = torch.from_numpy(d["kmer"].view(np.int32)).cuda()
    torch.cuda.synchronize()
    ptr = buf.data_ptr() + 4 * offset
    assert ptr % 16 != 0 and M >= 4 * TILE
    ctx.set_markers_device(d["toc"], ptr, d["flags"], keepalive=buf)
    c1, s1, _, _ = ctx.lowhash0(capi.make_lowhash_params(**params))
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    c2, s2, _, _ = ctx.lowhash0(capi.make_lowhash_params(**params))
    assert len(c1) > 100 and np.array_equal(c1, c2) and np.array_equal(s1, s2)
    del buf
