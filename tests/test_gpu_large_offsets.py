"""GPU parity tests (run on an H100 with -m gpu) for marker-set sizes and type limits that the other tests never reach:
  * the chunk seams of the marker upload (staging chunks of 32 Mi markers), of the downsampled CSR (chunks of 2^27 markers)
    and of the Align4 sorted markers (row chunks of at most 2^28 markers), crossed at small sizes through the
    SHB_MARKER_UPLOAD_CHUNK / SHB_DOWNSAMPLE_CHUNK / SHB_ALIGN4_SORT_CHUNK test hooks;
  * marker offsets past 2^31 and 2^32 at the production chunk sizes: real reads between filler reads of one constant k-mer
    id, in a marker set built directly in device memory;
  * the 8- and 16-byte streak formats of the compressed alignments (skips of 2^19 or more, a streak longer than 2^21);
  * k = 16 (the high word of the downsampling hash, the k == 16 reverse complement) and the 24-bit position limit of the
    marker finder.
Bar: bit-exact candidates, ReadLowHashStatistics, AlignmentData, compressed toc and bytes against the CPU oracle.

Every test first checks on the host that its input reaches the path it is for (seams inside rows and on row boundaries,
offsets covered by real rows, the streak formats in the oracle's bytes, downsampled sets that differ without the hash's
high word)."""
import ctypes as C
import time

import numpy as np
import pytest

from oracle import bindings as B
from shasta_b200 import synth
from support import (LOWHASH, K, Genome, PaddedSet, assemble, compare_alignments, ctx, downsampled,  # noqa: F401
                     downsampling_hash, downsampling_threshold, feature_hashes, hash_threshold, murmur2_u64, need_memory,
                     oracle_options, strand0_rows)

pytestmark = pytest.mark.gpu

HOOKS = ("SHB_MARKER_UPLOAD_CHUNK", "SHB_DOWNSAMPLE_CHUNK", "SHB_ALIGN4_SORT_CHUNK")
SEAM_CHUNKS = (1000, 1001, 1024, 4097)
DOWNSAMPLE_CHUNK = 1 << 27          # buildDownsampled (csrc/align.cu)
SORT_CHUNK = 1 << 28                # buildSortedMarkers
ALIGN3 = dict(alignMethod=3, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=50, minAlignedFraction=0.3,
              downsamplingFactor=0.1, bandExtend=10, maxBand=1000)
ALIGN4 = dict(alignMethod=4, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10, minAlignedFraction=0.1,
              align4DeltaX=200, align4DeltaY=10, align4MinEntryCountPerCell=2, align4MaxDistanceFromBoundary=100, maxBand=1000)


def sort_chunks(toc, limit):
    """The row chunks of buildSortedMarkers: (rowBegin, rowEnd) pairs."""
    toc = [int(x) for x in toc]
    rows, out, begin = len(toc) - 1, [], 0
    while begin < rows:
        end = begin + 1
        while end < rows and toc[end + 1] - toc[begin] <= limit:
            end += 1
        out.append((begin, end))
        begin = end
    return out


def resident_kmer_ids(ctx):
    """The context's resident k-mer ids, read back through shb_markers_device + shb_copy_device_to_host."""
    from shasta_b200 import capi
    ptr, n = C.c_void_p(), C.c_uint64()
    capi._check(capi.lib().shb_markers_device(ctx._h, C.byref(ptr), C.byref(n)))
    out = np.empty(n.value, np.uint32)
    capi._check(capi.lib().shb_copy_device_to_host(out.ctypes.data, ptr, out.nbytes))
    return out


def streak_tags(cdata, ctoc):
    """Low bits of the first byte of every streak: 0 (1 byte), 1 (2), 3 (4), 5 (8), 7 (16) (src/compressAlignment.hpp)."""
    tags = set()
    for i in range(len(ctoc) - 1):
        pos, end = int(ctoc[i]), int(ctoc[i + 1])
        while pos < end:
            c0 = int(cdata[pos])
            tag = 0 if c0 & 1 == 0 else c0 & 7
            tags.add(tag)
            pos += {0: 1, 1: 2, 3: 4, 5: 8, 7: 16}[tag]
        assert pos == end
    return tags


# ---- 1. chunk seams at small sizes (test hooks) -------------------------------------------------------------------
def seam_dataset(k):
    """Synthetic reads, with some lengths set so that for every chunk size c of SEAM_CHUNKS one row starts exactly on a
    multiple of c after a strand-0 row and one after a strand-1 row; the marker count is 2 mod 4, so that the last upload
    chunk has a byte count that is not a multiple of 4."""
    d = synth.generate(synth.SynthParams(reads=400, k=k, genome_markers=60000, n50_bases=14000, min_bases=5000, seed=60 + k))
    rows = strand0_rows(d)
    rng = np.random.default_rng(k)

    def set_length(i, L):
        r = rows[i]
        rows[i] = r[:L] if L <= len(r) else np.concatenate([r, rng.integers(0, 4 ** k, L - len(r)).astype(np.uint32)])

    for j, c in enumerate(SEAM_CHUNKS):
        for strand in (0, 1):
            i = 20 + 60 * j + 30 * strand
            start = 2 * sum(len(r) for r in rows[:i])
            set_length(i, next(L for L in range(300, 300 + 2 * c) if (start + (strand + 1) * L) % c == 0))
    if sum(len(r) for r in rows) % 2 == 0:
        set_length(len(rows) - 1, len(rows[-1]) - 1)
    return assemble(rows, k)


def check_seams(toc, c):
    """The input reaches the seams of chunk size c (hook value) of all three chunking loops."""
    toc = toc.astype(np.int64)
    M = int(toc[-1])
    upload = (c + 1023) & ~1023
    assert M // upload >= 100 and (M % upload) * 7 % 4 != 0           # last chunk: byte count not a multiple of 4
    seams = np.arange(c, M, c)
    assert len(np.setdiff1d(seams, toc)) >= 100                          # seams inside rows
    on_seam = np.flatnonzero((toc[:-1] % c == 0) & (toc[:-1] > 0) & (toc[:-1] < M))
    assert (on_seam % 2 == 0).any() and (on_seam % 2 == 1).any()         # rows starting on a seam, after either strand
    chunks = sort_chunks(toc, c)
    assert len(chunks) >= 100
    assert any(e - b >= 2 for b, e in chunks)                            # chunks of several rows
    if c <= 1024:                                                        # oversize rows that are their own chunk
        assert sum(e - b == 1 and toc[e] - toc[b] > c for b, e in chunks) >= 100


@pytest.mark.parametrize("k", [10, 14])
def test_chunk_seams(ctx, monkeypatch, k):
    from shasta_b200 import capi
    d = seam_dataset(k)
    for c in SEAM_CHUNKS:
        check_seams(d["toc"], c)
    for name in HOOKS:
        monkeypatch.delenv(name, raising=False)
    lp = capi.make_lowhash_params(**LOWHASH)
    a3, a4 = dict(ALIGN3, k=k), dict(ALIGN4, k=k)
    # Default chunk sizes against the oracle.
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    cand, stats, _, _ = ctx.lowhash0(lp)
    oc, os_, _ = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], B.LowHashParams(**LOWHASH))
    assert np.array_equal(cand, oc) and np.array_equal(stats, os_) and len(cand) > 300
    base3 = compare_alignments(ctx, d, cand, **a3)
    base4 = compare_alignments(ctx, d, cand[:400], **a4)
    assert len(base3[0]) > 100 and len(base4[0]) > 100
    # Every hooked chunk size gives the same bytes. The derived marker caches are rebuilt by set_markers.
    for c in SEAM_CHUNKS:
        for name in HOOKS:
            monkeypatch.setenv(name, str(c))
        ctx.set_markers(d["toc"], d["data"], d["flags"])
        assert np.array_equal(resident_kmer_ids(ctx), d["kmer"]), c
        cand_c, stats_c, _, _ = ctx.lowhash0(lp)
        assert np.array_equal(cand_c, cand) and np.array_equal(stats_c, stats), c
        for got, base in ((capi.compute_alignments(ctx, cand, capi.make_align_options(**a3)), base3),
                          (capi.compute_alignments(ctx, cand[:400], capi.make_align_options(**a4)), base4)):
            assert all(np.array_equal(x, y) for x, y in zip(got[:3], base[:3])), c


# ---- 2. offsets past 2^31 and 2^32 at the production chunk sizes --------------------------------------------------
def choose_filler(k, m, seeds, hash_fraction, factor=None):
    """A k-mer id f whose features f...f and rc(f)...rc(f) have a hash with a high word above threshold >> 32 for every
    iteration seed (no low hash, no sweep-queue entry) and, given a downsampling factor, that is not downsampled."""
    hi = np.uint64(hash_threshold(hash_fraction) >> 32)
    for f in range(12345, 12345 + 10000):
        rc = int(synth.reverse_complement_kmer(np.array([f], np.uint32), k)[0])
        h = np.concatenate([feature_hashes(np.full(m, x, np.uint32), m, seeds)[:, 0] for x in (f, rc)])
        kept = factor is not None and downsampling_hash([f], k)[0] < downsampling_threshold(factor)
        if ((h >> np.uint64(32)) > hi).all() and not kept:
            return f
    raise AssertionError("no filler k-mer id")


def real_set():
    return synth.generate(synth.SynthParams(reads=300, k=14, genome_markers=40000, n50_bases=12000, min_bases=6000, seed=231))


def expected_lowhash(real, padded, log2_buckets):
    """The oracle's candidates on the real reads alone, and what the padded set must give: read ids mapped to the padded
    set (a monotone map, so the order is kept) and zero statistics for the filler reads."""
    oc, os_, _ = B.oracle_lowhash0(real["toc"], real["data"], real["flags"],
                                   B.LowHashParams(**LOWHASH, log2MinHashBucketCount=log2_buckets))
    cand = oc.copy()
    cand[:, :2] = padded.gmap[oc[:, :2]]
    stats = np.zeros((len(padded.flags), 3), np.uint64)
    stats[padded.gmap] = os_
    return oc, cand, stats


def run_padded_case(monkeypatch, padded, real, expected, opts, log2_buckets, aggregates, single_pairs):
    """LowHash0, computeAlignments and single-pair alignments on the padded set against the oracle on the real reads."""
    import torch
    from shasta_b200 import capi
    oc, cand, stats = expected
    orec, otoc, odata, _ = B.oracle_compute_alignments(real["toc"], real["kmer"], oc, oracle_options(opts), threads=8)
    mapped = orec.copy()
    mapped[:, :2] = padded.gmap[orec[:, :2]]
    same = {(int(a), int(b)): int(s) for a, b, s in oc}
    t0 = time.time()
    ids = padded.device_ids()
    c = capi.Context(0)
    try:
        c.set_markers_device(padded.toc, ids.data_ptr(), padded.flags, keepalive=ids)
        lp = capi.make_lowhash_params(**LOWHASH, log2MinHashBucketCount=log2_buckets)
        for aggregate in aggregates:
            monkeypatch.setenv("SHB_LOWHASH_AGGREGATE", aggregate)
            got, gstats, _, res = c.lowhash0(lp)
            assert res.log2BucketCount == log2_buckets
            assert np.array_equal(got, cand), aggregate
            assert np.array_equal(gstats, stats), aggregate
        rec, ctoc, cdata, res = capi.compute_alignments(c, cand, capi.make_align_options(**opts))
        assert res.tooWideCount == 0
        assert np.array_equal(rec, mapped) and np.array_equal(ctoc, otoc) and np.array_equal(cdata, odata)
        go = capi.make_align_options(**opts)
        for i in single_pairs(mapped):
            r0, r1 = int(orec[i, 0]), int(orec[i, 1])
            g0, g1 = int(mapped[i, 0]), int(mapped[i, 1])
            ords, info = capi.align_oriented_reads(c, 2 * g0, 2 * g1 + (0 if same[r0, r1] else 1), go)
            assert np.array_equal(info, orec[i, 3:16])
            assert np.array_equal(ords, B.oracle_decompress(odata[int(otoc[i]):int(otoc[i + 1])]))
        print(f"padded set of {padded.M} markers: {len(cand)} candidates, {len(rec)} alignments, "
              f"{time.time() - t0:.1f} s from the device set-up to the last check")
    finally:
        c.close()
        del ids
        torch.cuda.empty_cache()


def test_offsets_past_2_31_and_2_32_method3(monkeypatch):
    need_memory(32)
    real = real_set()
    k, log2_buckets = 14, 26
    seeds = [37 * i for i in range(LOWHASH["minHashIterationCount"])]
    s = PaddedSet(real, k, choose_filler(k, LOWHASH["m"], seeds, LOWHASH["hashFraction"], ALIGN3["downsamplingFactor"]))
    s.reals(128)                                    # reads below 2^31
    s.fill_to(3 * DOWNSAMPLE_CHUNK)
    s.reals(1)                                      # starts exactly on a downsampling chunk seam
    s.fill_to(5 * DOWNSAMPLE_CHUNK - 2 * s.real_length(s.next_real))
    s.reals(1)                                      # its strand-1 row ends exactly on one
    s.fill_to((1 << 31) - 2 * (s.real_length(s.next_real) // 4))
    s.reals(1)                                      # strand-0 row over 2^31 - 1 and 2^31
    s.fill_to((1 << 32) - 2 * (s.real_length(s.next_real) // 4))
    s.reals(len(real["flags"]) - s.next_real)       # strand-0 row over 2^32 - 1 and 2^32, then the reads above 2^32
    s.finish()
    toc = s.toc.astype(np.int64)
    rows = s.real_rows()
    assert (1 << 32) < s.M < (1 << 32) + (1 << 21)
    for x in (1 << 31, 1 << 32):
        assert ((toc[rows] <= x - 1) & (toc[rows + 1] > x)).sum() == 1, x
    assert ((toc[rows] > 0) & (toc[rows] % DOWNSAMPLE_CHUNK == 0)).any()
    assert (toc[rows + 1] % DOWNSAMPLE_CHUNK == 0).any()
    assert log2_buckets >= int(LOWHASH["hashFraction"] * s.M).bit_length()
    expected = expected_lowhash(real, s, log2_buckets)
    cand = expected[1].astype(np.int64)
    low, high = toc[2 * cand[:, 0] + 2] <= (1 << 31), toc[2 * cand[:, 1]] >= (1 << 32)
    assert (low & high).sum() >= 50

    def spanning(mapped):
        g = mapped[:, :2].astype(np.int64)
        picked = np.flatnonzero((toc[2 * g[:, 0] + 2] <= (1 << 31)) & (toc[2 * g[:, 1]] >= (1 << 32)))[:4]
        assert len(picked) == 4
        return picked

    run_padded_case(monkeypatch, s, real, expected, dict(ALIGN3, k=k), log2_buckets, ("0", "1"), spanning)


def test_align4_sort_chunks_past_2_29_method4(monkeypatch):
    need_memory(16)
    real = real_set()
    k, log2_buckets = 14, 26
    seeds = [37 * i for i in range(LOWHASH["minHashIterationCount"])]
    s = PaddedSet(real, k, choose_filler(k, LOWHASH["m"], seeds, LOWHASH["hashFraction"]))
    s.reals(100)
    s.fill_to(SORT_CHUNK)                           # the next real read is the first row of a chunk
    s.reals(100)
    s.fill_to(2 * SORT_CHUNK)
    s.reals(len(real["flags"]) - s.next_real)
    s.finish()
    toc = s.toc.astype(np.int64)
    rows = set(s.real_rows().tolist())
    chunks = sort_chunks(toc, SORT_CHUNK)
    assert (1 << 29) < s.M < (1 << 29) + (1 << 21) and len(chunks) >= 3
    assert all(any(r in rows for r in range(b, e)) for b, e in chunks)        # real reads in every chunk
    assert sum(b in rows for b, _ in chunks[1:]) >= 2                          # ... and as the first row of a chunk
    chunk_of = np.zeros(len(toc) - 1, np.int64)
    for i, (b, e) in enumerate(chunks):
        chunk_of[b:e] = i
    expected = expected_lowhash(real, s, log2_buckets)
    cand = expected[1].astype(np.int64)
    assert (chunk_of[2 * cand[:, 0]] != chunk_of[2 * cand[:, 1]]).sum() >= 50
    run_padded_case(monkeypatch, s, real, expected, dict(ALIGN4, k=k), log2_buckets, ("0",), lambda mapped: [])


# ---- 3. compressed streak formats and very long alignments --------------------------------------------------------
def streak_dataset():
    g = Genome(2_900_000, seed=17, drop=0.04, ins=0.02)
    rng = np.random.default_rng(18)
    rows, cand = [], []

    def pair(a, b):
        cand.append((len(rows), len(rows) + 1, 1))
        rows.extend([a, b])

    x = g.kmer[0:600_000].copy()
    pair(x, g.read(550_000, 50_000)[0])                                # X and its last 50 000 markers, with errors
    dup = g.kmer[700_000:2_810_000].copy()
    pair(dup, dup.copy())                                              # one streak of 2 110 000 markers
    exact = g.kmer[2_830_000:2_831_000]
    pair(*(np.concatenate([g.read(2_820_000, 10_000)[0], exact, g.read(2_831_000, 10_000)[0]]) for _ in range(2)))
    pair(*(np.concatenate([g.read(2_840_000, 20_000)[0], rng.integers(0, 1 << 20, 600).astype(np.uint32),
                           g.read(2_860_000, 20_000)[0]]) for _ in range(2)))   # 600 unmatched markers in both reads
    ordinary = [g.read(s, 20_000)[0] for s in (2_860_000, 2_868_000, 2_875_000)]
    base = len(rows)
    rows.extend(ordinary)
    cand += [(base, base + 1, 1), (base, base + 2, 1), (base + 1, base + 2, 1)]
    return assemble(rows, K), rows, np.array(cand, np.uint32)


def test_compressed_streak_formats(ctx):
    d, rows, cand = streak_dataset()
    factor = 0.0037
    ds = [len(downsampled(r, factor)[0]) for r in rows]
    assert max(ds[a] + ds[b] for a, b, _ in cand) <= 16381             # every unbanded stage fits a band class
    assert len(rows[2]) >= 2_100_000 and np.array_equal(rows[2], rows[3])
    opts = dict(k=K, alignMethod=3, downsamplingFactor=factor, bandExtend=100, maxBand=16000, maxSkip=1_000_000,
                maxDrift=1_000_000, maxTrim=1_000_000, minAlignedMarkerCount=1, minAlignedFraction=0.0)
    orec, otoc, odata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], cand, oracle_options(opts), threads=8)
    assert len(orec) == len(cand)                                      # records in candidate order

    def record(i):
        return odata[int(otoc[i]):int(otoc[i + 1])]

    assert streak_tags(odata, otoc) == {0, 1, 3, 5, 7}
    first = B.oracle_decompress(record(0))[0]
    assert first[0] >= 1 << 19 and record(0)[0] & 7 == 7                  # 16 bytes by skip: X ordinal beyond 524 287
    assert len(record(1)) == 16 and record(1)[0] & 7 == 7                  # 16 bytes by length: one streak
    assert len(B.oracle_decompress(record(1), cap=1 << 22)) == len(rows[2]) > 1 << 21
    for i in (2, 3):                                                       # 8 bytes by length, by skip
        assert 5 in streak_tags(record(i), [0, len(record(i))]), i
    compare_alignments(ctx, d, cand, **opts)


# ---- 4. k = 16 and the 24-bit position limit ----------------------------------------------------------------------
@pytest.mark.parametrize("method", [3, 4])
def test_k16_alignments(ctx, method):
    from shasta_b200 import capi
    d = synth.generate(synth.SynthParams(reads=200, k=16, genome_markers=20000, n50_bases=10000, min_bases=5000, seed=16))
    n = d["kmer"].astype(np.uint64) + synth.reverse_complement_kmer(d["kmer"], 16).astype(np.uint64)
    assert (n >> np.uint64(32) != 0).mean() > 0.3
    if method == 3:
        thr = downsampling_threshold(ALIGN3["downsamplingFactor"])
        full = downsampling_hash(d["kmer"], 16) < thr
        low_word_only = murmur2_u64(n & np.uint64(0xffffffff)) < thr
        assert (full != low_word_only).sum() > 1000
    opts = dict(ALIGN3 if method == 3 else ALIGN4, k=16)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    cand, stats, _, _ = ctx.lowhash0(capi.make_lowhash_params(**LOWHASH))
    oc, os_, _ = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], B.LowHashParams(**LOWHASH))
    assert np.array_equal(cand, oc) and np.array_equal(stats, os_) and len(cand) > 300
    assert len(compare_alignments(ctx, d, cand, **opts)[0]) > 100


def pack_reads(reads):
    """LongBaseSequences layout (src/LongBaseSequence.hpp:33-41) of base arrays (values 0..3), vectorised."""
    offsets, words = [0], []
    for b in reads:
        blocks = (len(b) + 63) // 64
        pad = np.zeros(blocks * 64, np.uint8)
        pad[:len(b)] = b
        planes = [np.packbits((pad >> s) & 1, bitorder="big").view(">u8").astype(np.uint64) for s in (0, 1)]
        words.append(np.stack(planes, 1).reshape(-1))
        offsets.append(offsets[-1] + 2 * blocks)
    words = np.concatenate(words) if words else np.zeros(0, np.uint64)
    return np.array(offsets, np.uint64), words, np.array([len(b) for b in reads], np.uint64)


def kmer_ids_of(b, k):
    """k-mer id at every position of a read: (high bit plane << k) | low bit plane, first base most significant."""
    P_ = len(b) - k + 1
    lo = np.zeros(P_, np.uint64)
    hi = np.zeros(P_, np.uint64)
    for j in range(k):
        w = b[j:j + P_].astype(np.uint64)
        lo = (lo << np.uint64(1)) | (w & np.uint64(1))
        hi = (hi << np.uint64(1)) | (w >> np.uint64(1))
    return ((hi << np.uint64(k)) | lo).astype(np.uint32)


def numpy_marker_finder(reads, k, is_marker):
    """MarkerFinder (src/MarkerFinder.cpp:16-127): strand 0 in position order; strand 1 reversed, reverse-complemented,
    position baseCount - k - position. Returns (toc, 7-byte records)."""
    toc, kmers, positions = [0], [], []
    for b in reads:
        n = len(b)
        if n < k:
            toc += [toc[-1], toc[-1]]
            continue
        ids = kmer_ids_of(b, k)
        p0 = np.flatnonzero(is_marker(ids))
        k0 = ids[p0]
        kmers += [k0, synth.reverse_complement_kmer(k0[::-1], k)]
        positions += [p0, n - k - p0[::-1]]
        toc += [toc[-1] + len(p0), toc[-1] + 2 * len(p0)]
    kmer = np.concatenate(kmers).astype(np.uint32)
    pos = np.concatenate(positions).astype(np.uint32)
    return np.array(toc, np.uint64), synth.pack_markers(kmer, pos), pos


def test_marker_finder_k16_and_24_bit_positions(ctx):
    from shasta_b200 import capi
    k = 16
    rng = np.random.default_rng(24)
    lengths = [0, 15, 16, 17, 63, 64, 65, 129, 5000, (1 << 24) - 1, 3000]
    reads = [rng.integers(0, 4, n).astype(np.uint8) for n in lengths]
    bitmap = np.zeros(1 << 27, np.uint32)                                   # 4^16 bits
    for b in reads:
        if len(b) >= k:
            ids = kmer_ids_of(b, k)
            chosen = ids[rng.random(len(ids)) < 0.1]
            if len(b) == (1 << 24) - 1:
                chosen = np.concatenate([chosen, ids[-40:][::3], ids[-1:]])    # markers in the last 64-base block
            np.bitwise_or.at(bitmap, (chosen >> 5).astype(np.int64), np.left_shift(np.uint32(1), chosen & np.uint32(31)))
    np.bitwise_or.at(bitmap, rng.integers(0, 1 << 27, 100000), np.uint32(1) << rng.integers(0, 32, 100000).astype(np.uint32))

    def is_marker(ids):
        return (bitmap[(ids >> 5).astype(np.int64)] >> (ids & np.uint32(31))) & np.uint32(1) == 1

    etoc, edata, epos = numpy_marker_finder(reads, k, is_marker)
    long_read = lengths.index((1 << 24) - 1)
    a, b_, c = (int(x) for x in etoc[2 * long_read:2 * long_read + 3])
    assert epos[b_ - 1] == (1 << 24) - 1 - k and epos[b_] == 0                # strand 0 ends at 2^24 - 1 - k, strand 1 starts at 0
    assert (epos[a:b_] >= (1 << 24) - 64).sum() >= 10
    wo, w, bc = pack_reads(reads)
    toc, data, res = ctx.find_markers(k, wo, w, bc, np.zeros(len(reads), np.uint8), is_marker_bitmap=bitmap)
    assert res.markerCount == int(etoc[-1]) > 300000
    assert np.array_equal(toc, etoc)
    assert np.array_equal(data, edata)
    # A read of 2^24 bases is refused: marker positions are 24 bits.
    wo, w, bc = pack_reads([rng.integers(0, 4, 1 << 24).astype(np.uint8)])
    with pytest.raises(capi.ShastaB200Error, match="2\\^24 or more bases"):
        ctx.find_markers(k, wo, w, bc, np.zeros(1, np.uint8), is_marker_bitmap=bitmap)


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5])
def test_marker_finder_small_k_against_oracle(ctx, k):
    rng = np.random.default_rng(100 + k)
    is_marker = (rng.random(4 ** k) < 0.4).astype(np.uint8)
    lengths = [0, 1, k - 1, k, k + 1, 63, 64, 65, 127, 128, 129, 1000, 5000, 0, 2]
    reads = [rng.integers(0, 4, n).astype(np.uint8) for n in lengths]
    wo, w, bc = pack_reads(reads)
    otoc, odata = B.oracle_find_markers(wo, w, bc, is_marker, k)
    etoc, edata, _ = numpy_marker_finder(reads, k, lambda ids: is_marker[ids] == 1)
    assert np.array_equal(otoc, etoc) and np.array_equal(odata, edata)
    bitmap = np.packbits(np.concatenate([is_marker, np.zeros(32, np.uint8)])[:max(32, 4 ** k)], bitorder="little").view(np.uint32)
    toc, data, res = ctx.find_markers(k, wo, w, bc, np.zeros(len(reads), np.uint8), is_marker_bitmap=bitmap)
    assert res.markerCount == int(otoc[-1]) > 1000
    assert np.array_equal(toc, otoc) and np.array_equal(data, odata)
