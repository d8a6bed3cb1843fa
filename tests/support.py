"""Helpers that several test modules share: the per-module context fixture, marker-set builders, numpy models of the
device's hashes and band classes, and the comparisons against the oracle and the reference's recorded outputs.

Importing this module puts tests/golden on sys.path, so that the input and recording modules there can be imported after
it. Pytest does not collect it: its name does not start with test_."""
import contextlib
import hashlib
import os
import sys

import numpy as np
import pytest

from oracle import bindings as B
from shasta_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)

from readgraph_inputs import DEFAULT_PERCENTILES  # noqa: E402
from reference_outputs import recorded  # noqa: E402


@pytest.fixture(scope="module")
def ctx():
    """A context per test module: a module leaves its markers and hook settings behind on its own context only."""
    from shasta_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


# ---- parameters ------------------------------------------------------------------------------------------------------
K = 10
LOWHASH = dict(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=2, maxBucketSize=30, minFrequency=2)
PERMISSIVE = dict(k=K, maxSkip=100000, maxDrift=100000, maxTrim=100000, minAlignedMarkerCount=1, minAlignedFraction=0.0)
FORWARD_MAX_MARKERS = 32000     # kStage1ForwardMaxMarkers (csrc/align_kernels.cuh)
FORWARD_MAX_ROWS = 512          # kStage1ForwardMaxRows
MAX_BAND_WIDTH = 16384          # widest band class (kMaxBandWidth, csrc/align.cu)
TILE = 2048                     # kSweepTile (csrc/lowhash_kernels.cuh)

# The parameter sets of the five BASELINE.json configurations, at sizes the oracle finishes in seconds.
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


# ---- marker sets -----------------------------------------------------------------------------------------------------
def assemble(rows0, k, flags=None):
    """Marker set of reads whose strand-0 rows are rows0; each strand-1 row is its strand-0 row reversed and
    reverse-complemented. Positions count markers modulo 2^24; flags default to zero."""
    lengths = np.array([len(r) for r in rows0], np.int64)
    toc = np.zeros(2 * len(rows0) + 1, np.uint64)
    toc[1:] = np.cumsum(np.repeat(lengths, 2)).astype(np.uint64)
    rows0 = [np.asarray(r, np.uint32) for r in rows0]
    parts = [x for r in rows0 for x in (r, synth.reverse_complement_kmer(r[::-1], k))]
    kmer = np.concatenate(parts).astype(np.uint32) if parts else np.zeros(0, np.uint32)
    pos = (np.arange(len(kmer)) % (1 << 24)).astype(np.uint32)
    flags = np.zeros(len(rows0), np.uint8) if flags is None else np.asarray(flags, np.uint8)
    return dict(toc=toc, kmer=kmer, data=synth.pack_markers(kmer, pos), flags=flags)


def strand0_rows(d):
    toc = d["toc"].astype(np.int64)
    return [d["kmer"][toc[2 * i]:toc[2 * i + 1]].copy() for i in range(len(d["flags"]))]


def row(d, o):
    toc = d["toc"].astype(np.int64)
    return d["kmer"][toc[o]:toc[o + 1]]


def pack_ordinal_markers(toc, kmer):
    """7-byte marker records of the k-mer ids, each marker's position being its ordinal in its row."""
    pos = np.concatenate([np.arange(toc[i + 1] - toc[i], dtype=np.uint32) for i in range(len(toc) - 1)] or [np.zeros(0, np.uint32)])
    return synth.pack_markers(np.asarray(kmer, np.uint32), pos)


def candidate_set(reads, k, seed, **kw):
    """A synthetic read set and the oracle's LowHash0 candidates (LOWHASH) on it. Unless kw says otherwise the genome has
    20 000 markers, the read N50 is 15 000 bases and reads have at least 8 000."""
    p = synth.SynthParams(reads=reads, k=k, genome_markers=kw.pop("genome_markers", 20000), n50_bases=kw.pop("n50", 15000),
                          min_bases=kw.pop("min_bases", 8000), seed=seed, **kw)
    d = synth.generate(p)
    cand, _, _ = B.oracle_lowhash0(d["toc"], d["data"], d["flags"], B.LowHashParams(**LOWHASH))
    return d, cand


class Genome:
    """A random marker genome; reads are cut from it with marker drop-outs and insertions (the marker-level image of
    sequencing errors). Every row comes with the genome index of each of its markers (-1 for inserted markers)."""

    def __init__(self, markers, seed, drop=0.04, ins=0.02):
        self.rng = np.random.default_rng(seed)
        self.kmer = self.rng.integers(0, 1 << (2 * K), markers).astype(np.uint32)
        self.drop, self.ins = drop, ins

    def read(self, start, length, keep=None):
        """Row of genome markers [start, start + length); keep = ("head", n) or ("tail", n) keeps n markers of it."""
        g = np.arange(start, start + length)
        g = g[self.rng.random(length) >= self.drop]
        idx = np.insert(g, np.flatnonzero(self.rng.random(len(g)) < self.ins) + 1, -1)
        row = np.where(idx >= 0, self.kmer[np.maximum(idx, 0)], self.rng.integers(0, 1 << (2 * K), len(idx))).astype(np.uint32)
        if keep is not None:
            sl = slice(0, keep[1]) if keep[0] == "head" else slice(len(row) - keep[1], len(row))
            row, idx = row[sl], idx[sl]
            assert len(row) == keep[1]
        return row, idx


FILLER_ROW_MAX = 1 << 27            # filler rows stay below the 2^28-marker row limit of computeAlignments


class PaddedSet:
    """Real reads (both strands, in their order) placed at chosen marker offsets between filler reads of one constant
    k-mer id f (strand 1: rc(f))."""

    def __init__(self, real, k, f):
        self.real, self.k, self.f = real, k, int(f)
        self.rtoc = real["toc"].astype(np.int64)
        self.items = []         # ("real", real read id, offset) or ("fill", row length, offset)
        self.end = 0
        self.next_real = 0

    def real_length(self, i):
        return int(self.rtoc[2 * i + 1] - self.rtoc[2 * i])

    def reals(self, n):
        for _ in range(n):
            self.items.append(("real", self.next_real, self.end))
            self.end += 2 * self.real_length(self.next_real)
            self.next_real += 1

    def fill_to(self, target):
        gap = target - self.end
        assert gap >= 0 and gap % 2 == 0, (gap, target)
        while gap:
            L = min(gap // 2, FILLER_ROW_MAX)
            self.items.append(("fill", L, self.end))
            self.end += 2 * L
            gap -= 2 * L

    def finish(self):
        assert self.next_real == len(self.real["flags"])
        lengths = [self.real_length(a) if kind == "real" else a for kind, a, _ in self.items]
        self.toc = np.zeros(2 * len(lengths) + 1, np.uint64)
        self.toc[1:] = np.cumsum(np.repeat(np.array(lengths, np.int64), 2)).astype(np.uint64)
        self.M = int(self.toc[-1])
        self.gmap = np.array([g for g, (kind, _, _) in enumerate(self.items) if kind == "real"], np.uint32)
        self.flags = np.zeros(len(lengths), np.uint8)
        return self

    def device_ids(self):
        """The k-mer ids as a CUDA tensor (M + 64 entries; the tail is zero)."""
        import torch
        ids = torch.zeros(self.M + 64, dtype=torch.int32, device="cuda")
        fv = int(np.uint32(self.f).view(np.int32))
        rv = int(synth.reverse_complement_kmer(np.array([self.f], np.uint32), self.k).view(np.int32)[0])
        for kind, a, off in self.items:
            if kind == "fill":
                ids[off:off + a] = fv
                ids[off + a:off + 2 * a] = rv
            else:
                src = self.real["kmer"][self.rtoc[2 * a]:self.rtoc[2 * a + 2]].view(np.int32)
                ids[off:off + len(src)] = torch.from_numpy(src).to("cuda")
        torch.cuda.synchronize()        # the library works on streams of its own that do not wait for torch's
        return ids

    def real_rows(self):
        """Global row index of every real row."""
        return np.sort(np.concatenate([2 * self.gmap, 2 * self.gmap + 1])).astype(np.int64)


def need_memory(gb):
    import torch
    free, _ = torch.cuda.mem_get_info()
    print(f"\nfree device memory before the case: {free / 2**30:.1f} GB")
    if free < gb * 2**30:
        pytest.skip(f"needs {gb} GB of free device memory, {free / 2**30:.1f} GB free")


# ---- host models -----------------------------------------------------------------------------------------------------
def murmur2_u64(n):
    """MurmurHash2 (src/MurmurHash2.cpp:37-88) of the 8 bytes of each uint64 n, seed 13477, vectorised."""
    n = np.asarray(n, np.uint64)
    m = np.uint32(0x5bd1e995)
    with np.errstate(over="ignore"):
        h = np.full(n.shape, np.uint32(13477 ^ 8), np.uint32)
        for word in (n.astype(np.uint32), (n >> np.uint64(32)).astype(np.uint32)):
            w = word * m
            w ^= w >> np.uint32(24)
            w *= m
            h *= m
            h ^= w
        h ^= h >> np.uint32(13)
        h *= m
        h ^= h >> np.uint32(15)
    return h


def downsampling_hash(kmer, k):
    """kmerDownsamplingHash (csrc/align_kernels.cuh): MurmurHash2 of kmer + reverse complement."""
    return murmur2_u64(np.asarray(kmer, np.uint64) + synth.reverse_complement_kmer(kmer, k).astype(np.uint64))


def downsampling_threshold(factor):
    return np.uint32(int(factor * 4294967295.0))             # uint32_t(factor * double(UINT32_MAX))


def downsampled(row, factor):
    """(k-mers, ordinals) that method 3's stage 1 keeps of a row of k = K markers."""
    keep = np.flatnonzero(downsampling_hash(row, K) < downsampling_threshold(factor))
    return row[keep], keep.astype(np.int64)


def padded_width(W):
    """Padded width of a band of W offsets (dpBandShape): W + 2 rounded up to 16 or 64 lanes' sub-chunks; the classes
    above 1 024 offsets all run on whole warps."""
    need = W + 2
    return (need + 63) & ~63 if need > 128 else (need + 15) & ~15


def wide_band_class(W):
    """8192 or 16384 for a band of W offsets on one of the two widest classes, 0 on a narrower one, None when too wide."""
    need = padded_width(W)
    return None if need > MAX_BAND_WIDTH else (8192 if need > 4096 and need <= 8192 else 16384 if need > 8192 else 0)


MURMUR_M = np.uint64(0xc6a4a7935bd1e995)


def feature_hashes(kmer, m, seeds, positions=None):
    """MurmurHash64A of the 4*m bytes of k-mer ids starting at each position (all p with p + m <= len(kmer) by default),
    for every seed: uint64[len(seeds), len(positions)]."""
    U64 = np.uint64
    kmer = np.asarray(kmer, np.uint32)
    if positions is None:
        positions = np.arange(max(len(kmer) - m + 1, 0), dtype=np.int64)
    positions = np.asarray(positions, np.int64)
    with np.errstate(over="ignore"):
        mixed = []
        for b in range(m // 2):
            k = kmer[positions + 2 * b].astype(U64) | (kmer[positions + 2 * b + 1].astype(U64) << U64(32))
            k *= MURMUR_M
            k ^= k >> U64(47)
            k *= MURMUR_M
            mixed.append(k)
        tail = kmer[positions + m - 1].astype(U64) if m & 1 else None
        out = np.empty((len(seeds), len(positions)), U64)
        for i, seed in enumerate(seeds):
            h = np.full(len(positions), U64(seed) ^ (U64(4 * m) * MURMUR_M), U64)
            for k in mixed:
                h ^= k
                h *= MURMUR_M
            if tail is not None:
                h ^= tail
                h *= MURMUR_M
            h ^= h >> U64(47)
            h *= MURMUR_M
            h ^= h >> U64(47)
            out[i] = h
    return out


def hash_threshold(hash_fraction):
    return int(hash_fraction * 18446744073709551616.0)         # uint64_t(hashFraction * double(UINT64_MAX))


# ---- alignments against the oracle -----------------------------------------------------------------------------------
def oracle_options(opts):
    return B.make_align_options(**{k: v for k, v in opts.items() if k in B.ALIGN_DEFAULTS})


def compare_alignments(ctx, d, cand, expected_skips=(), **opts):
    """computeAlignments on ctx, with the markers d uploaded, equals the oracle on every candidate except the expected
    skips (too wide for any band class): records, compressed toc and bytes, the device digests of those bytes, and the
    result counters. Returns what compute_alignments returned."""
    from shasta_b200 import capi
    cand = np.asarray(cand, np.uint32).reshape(-1, 3)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    rec, ctoc, cdata, res = capi.compute_alignments(ctx, cand, capi.make_align_options(**opts))
    keep = np.ones(len(cand), bool)
    keep[list(expected_skips)] = False
    orec, otoc, odata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], cand[keep], oracle_options(opts), threads=8)
    assert res.candidateCount == len(cand)
    assert res.tooWideCount == len(expected_skips)
    assert rec.shape == orec.shape, (rec.shape, orec.shape)
    assert np.array_equal(rec, orec)
    assert np.array_equal(ctoc, otoc)
    assert np.array_equal(cdata, odata)
    # the device-side digests carried by every bench line are those of exactly these bytes
    assert res.alignmentDataDigest == capi.digest_records(orec, 16)
    assert res.compressedDigest == capi.digest_compressed(orec, otoc, odata)
    assert res.dpUsefulCells <= res.dpCells
    return rec, ctoc, cdata, res


def single_pair_options(method):
    opts = dict(PERMISSIVE, alignMethod=method)
    if method == 3:
        opts.update(downsamplingFactor=0.1, bandExtend=10, maxBand=1000)
    elif method == 4:
        opts.update(align4DeltaX=200, align4DeltaY=10, align4MinEntryCountPerCell=2, align4MaxDistanceFromBoundary=200, maxBand=1000)
    return opts


def expected_single_pair(row0, row1, opts):
    """The oracle's stored alignment of row0 against row1 (record, ordinals), or None, from a two-read marker set whose
    reads are the two rows on strand 0."""
    two = assemble([row0, row1], K)
    orec, otoc, odata, _ = B.oracle_compute_alignments(two["toc"], two["kmer"], np.array([[0, 1, 1]], np.uint32),
                                                       oracle_options(opts), threads=1)
    if len(orec) == 0:
        return None
    return orec[0], B.oracle_decompress(odata[int(otoc[0]):int(otoc[1])])


# ---- the device chain up to the read graph ---------------------------------------------------------------------------
READ_GRAPH_SET = dict(reads=400, k=10, genome_markers=40000, n50_bases=12000, min_bases=6000, seed=9)
READ_GRAPH_ALIGN = dict(alignMethod=3, k=10, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=50, minAlignedFraction=0.3,
                        downsamplingFactor=0.1, bandExtend=10, maxBand=1000)


def device_alignments(ctx):
    """The read set of the read-graph tests, then LowHash0 and computeAlignments on ctx: (markers, candidates,
    AlignmentData records, compressed toc, compressed bytes)."""
    from shasta_b200 import capi
    d = synth.generate(synth.SynthParams(**READ_GRAPH_SET))
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    cand, _, _, _ = ctx.lowhash0(capi.make_lowhash_params(**LOWHASH))
    rec, ctoc, cdata, _ = capi.compute_alignments(ctx, cand, capi.make_align_options(**READ_GRAPH_ALIGN))
    return d, cand, np.array(rec, np.uint32), np.array(ctoc), np.array(cdata)


@contextlib.contextmanager
def device_read_graph(method):
    """device_alignments on a context of its own, then createReadGraph (method 0) or createReadGraph2 (method 2, default
    percentiles) with maxAlignmentCount 6. Yields (context, markers, records, compressed toc, compressed bytes,
    (edges, connectivity toc, connectivity data)); the context is closed on exit."""
    from shasta_b200 import capi
    c = capi.Context(0)
    try:
        d, _, rec, ctoc, cdata = device_alignments(c)
        reads = READ_GRAPH_SET["reads"]
        if method == 0:
            graph = capi.create_read_graph(c, rec, reads, 6)
        else:
            graph = capi.create_read_graph2(c, rec, reads, 6, *DEFAULT_PERCENTILES)
        yield c, d, rec, ctoc, cdata, tuple(np.array(x) for x in graph[-3:])
    finally:
        c.close()


# ---- read graph outputs against the reference --------------------------------------------------------------------------
DIGEST_ABOVE = 4096         # outputs with more elements are recorded as SHA-256 digests


def _digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(a.dtype.str.encode() + str(a.shape).encode() + a.tobytes()).hexdigest()


def summary(rec, keep, edges, toc, data, criteria=None):
    """What the comparisons look at: keep flags, word 15 (isInReadGraph and the bits after it), edges, connectivity, and the
    creationMethod 2 criteria; arrays above DIGEST_ABOVE elements as digests."""
    d = dict(keep=keep, word15=np.ascontiguousarray(rec[:, 15]), edges=edges, toc=toc, data=data)
    if criteria is not None:
        d["criteria_fraction"] = np.float64(criteria["minAlignedFraction"])
        d["criteria_counts"] = np.array([criteria[k] for k in ("minAlignedMarkerCount", "maxDrift", "maxSkip", "maxTrim")], np.uint64)
    return {k: (_digest(v) if np.size(v) > DIGEST_ABOVE else np.asarray(v)) for k, v in d.items()}


def table_summary(toc, data):
    return {k: (_digest(v) if np.size(v) > DIGEST_ABOVE else np.asarray(v)) for k, v in dict(toc=toc, data=data).items()}


def outcome(fn, *args):
    """summary() of a read graph call, or "refused" where it raises UnorderedReadGraphEdge."""
    try:
        out = fn(*args)
    except B.UnorderedReadGraphEdge:
        return "refused"
    return summary(*out[1:], criteria=out[0]) if isinstance(out[0], dict) else summary(*out)


def assert_same(want, got, what):
    if isinstance(want, str) or isinstance(got, str):
        assert want == got, what
        return
    assert sorted(want) == sorted(got), what
    for k in want:
        w, g = want[k], got[k]
        if isinstance(w, str) or isinstance(g, str):
            assert w == g, (what, k)
        else:
            assert np.array_equal(np.asarray(w), np.asarray(g)) and np.asarray(w).shape == np.asarray(g).shape, (what, k)


# ---- markers from the reference's ReadLoader and MarkerFinder ----------------------------------------------------------
def write_synthetic_fasta(path, reads=40, seed=3):
    rng = np.random.default_rng(seed)
    with open(path, "w") as f:
        for i in range(reads):
            n = int(rng.integers(10000, 14000))
            # homopolymer runs of random length so that the run-length encoding has something to do
            bases = np.repeat(rng.integers(0, 4, n), rng.integers(1, 4, n))[:n]
            f.write(f">read{i}\n" + "".join("ACGT"[b] for b in bases) + "\n")


def _reference_markers(path, reads, seed, k):
    write_synthetic_fasta(path, reads=reads, seed=seed)
    r = B.ref_reads_from_fasta(path, k=k, min_read_length=1000)
    m = B.ref_markers_from_fasta(path, k=k, min_read_length=1000)
    # The marker table is stored as the marker k-mers that occur (both strands): k-mers absent from the reads cannot change
    # the output, and the whole table is 4^k entries. The 7-byte records are stored as their SHA-256.
    kmers = np.ascontiguousarray(m["data"].reshape(-1, 7)[:, :4]).view("<u4").reshape(-1)
    return dict(word_offsets=r["word_offsets"], words=r["words"], base_counts=r["base_counts"], marker_kmers=np.unique(kmers),
                toc=m["toc"], flags=m["flags"], data_sha256=hashlib.sha256(m["data"].tobytes()).hexdigest())


def reference_markers(tmp_path, reads, seed, k):
    """What the reference's ReadLoader and MarkerFinder make of write_synthetic_fasta(reads, seed) with k-mer length k."""
    return recorded("markers", f"reads{reads}_seed{seed}_k{k}", _reference_markers, str(tmp_path / f"synthetic_{seed}.fasta"),
                    reads, seed, k)
