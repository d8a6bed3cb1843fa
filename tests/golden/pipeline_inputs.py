"""Reads in base space and the shipped configurations they are run at, for the whole-pipeline tests
(tests/test_oracle_shipped_pipeline.py, tests/test_gpu_shipped_pipeline.py).

A genome is random bases with no two equal neighbours (the run-length representation the reference stores), with tandem
arrays of short units spliced in, so that marker k-mers repeat inside a read as they do on real genomes. Reads are windows
on either strand with substitution, insertion and deletion errors, run-length compressed again afterwards. A few reads are
injected: palindromic reads (a window followed by its reverse complement), chimeric reads (two distant windows joined),
empty reads and reads shorter than k. The marker set takes each reverse-complement pair {x, rc x} with probability p, and
each palindromic k-mer (x = rc x, even k only) on its own with probability p. Everything comes from fixed seeds."""
import functools

import numpy as np

# Error rates per base of the run-length representation (homopolymer length errors do not show there).
NANOPORE = dict(sub=0.012, ins=0.008, dele=0.01)
NANOPORE_Q20 = dict(sub=0.005, ins=0.003, dele=0.004)       # the 2022 chemistry the May2022 and Oct2021 files target
HIFI = dict(sub=0.0005, ins=0.0003, dele=0.0003)
CHIMERIC = 16           # injected chimeric reads per configuration

# Reference defaults (src/AssemblerOptions.cpp) for what a configuration file does not set.
PALINDROMIC = dict(maxSkip=100, maxDrift=100, maxMarkerFrequency=10, alignedFractionThreshold=0.1,
                   nearDiagonalFractionThreshold=0.1, deltaThreshold=100)
MINHASH = dict(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=0, maxBucketSize=10, minFrequency=2)
ALIGN = dict(alignMethod=3, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=100, minAlignedFraction=0.0,
             matchScore=6, mismatchScore=-1, gapScore=-1, downsamplingFactor=0.1, bandExtend=10, maxBand=1000,
             align4DeltaX=200, align4DeltaY=10, align4MinEntryCountPerCell=10, align4MaxDistanceFromBoundary=100)
READGRAPH = dict(creationMethod=0, maxAlignmentCount=6, strandSeparationMethod=1, crossStrandMaxDistance=6,
                 maxChimericReadDistance=2, percentiles=(0.015, 0.12, 0.12, 0.12, 0.015))
MARKERGRAPH = dict(minCoverage=10, maxCoverage=100, minCoveragePerStrand=0, allowDuplicateMarkers=False,
                   peakFinderMinAreaFraction=0.08, peakFinderAreaStartIndex=2)

# Substitutions, where the device has no counterpart of what a file asks for:
# - strandSeparationMethod 2 runs flagCrossStrandReadGraphEdges2 after flagChimericReads; the device has no version of it,
#   so those configurations go from flagChimericReads straight to the marker graph (and skip flagCrossStrandReadGraphEdges1,
#   as the reference does for method 2).
# - Align.sameChannelReadAlignment.suppressDeltaThreshold (candidate suppression) needs read names: not applied.
# - Every file here that sets Align.alignMethod sets 3; the one that does not (PacBio-CCS-Dec2019) gets the default, 3.
#   "-align4" entries run the same file with --Align.alignMethod 4 and the default Align4 values.


def _config(conf, k, probability, reads, minhash=None, align=None, readgraph=None, markergraph=None):
    c = dict(conf=conf, k=k, probability=probability, reads=reads, palindromic=dict(PALINDROMIC))
    c["minhash"] = dict(MINHASH, **(minhash or {}))
    c["align"] = dict(ALIGN, k=k, **(align or {}))
    c["readgraph"] = dict(READGRAPH, **(readgraph or {}))
    c["markergraph"] = dict(MARKERGRAPH, **(markergraph or {}))
    return c


_NANOPORE_ALIGN = dict(downsamplingFactor=0.05, maxSkip=100, maxDrift=100, maxTrim=100, minAlignedMarkerCount=10,
                       minAlignedFraction=0.1)
# genome: bases before the tandem arrays; arrays: (unit length, copies); n50 / sigma / min: read lengths in bases.
_ONT = dict(errors=NANOPORE, genome=100_000, arrays=[(60, 12), (45, 20), (80, 30), (30, 16), (120, 10)], coverage=25,
            n50=9000, sigma=0.4, min=3000)
_UL = dict(errors=NANOPORE, genome=300_000, arrays=[(60, 12), (45, 20), (80, 30), (300, 30), (120, 10)], coverage=22,
           n50=30000, sigma=0.3, min=12000)

CONFIGS = {
    # conf/Nanopore-Phased-Jan2022.conf
    "Nanopore-Phased-Jan2022": _config(
        "Nanopore-Phased-Jan2022.conf", 8, 0.07, dict(_ONT, seed=11),
        minhash=dict(minBucketSize=5, maxBucketSize=30, minFrequency=5), align=_NANOPORE_ALIGN,
        readgraph=dict(creationMethod=2, strandSeparationMethod=2, maxAlignmentCount=6),
        markergraph=dict(minCoverage=6, minCoveragePerStrand=1)),
    # conf/Nanopore-UL-Phased-Jan2022.conf
    "Nanopore-UL-Phased-Jan2022": _config(
        "Nanopore-UL-Phased-Jan2022.conf", 8, 0.07, dict(_UL, seed=12),
        minhash=dict(minBucketSize=10, maxBucketSize=50, minFrequency=5), align=_NANOPORE_ALIGN,
        readgraph=dict(creationMethod=2, strandSeparationMethod=2, maxAlignmentCount=12),
        markergraph=dict(minCoverage=6, minCoveragePerStrand=1)),
    # conf/Nanopore-UL-Phased-Jan2022.conf with --Align.alignMethod 4
    "Nanopore-UL-Phased-Jan2022-align4": _config(
        "Nanopore-UL-Phased-Jan2022.conf", 8, 0.07, dict(_UL, seed=12),
        minhash=dict(minBucketSize=10, maxBucketSize=50, minFrequency=5), align=dict(_NANOPORE_ALIGN, alignMethod=4),
        readgraph=dict(creationMethod=2, strandSeparationMethod=2, maxAlignmentCount=12),
        markergraph=dict(minCoverage=6, minCoveragePerStrand=1)),
    # conf/Nanopore-UL-iterative-Sep2020.conf
    "Nanopore-UL-iterative-Sep2020": _config(
        "Nanopore-UL-iterative-Sep2020.conf", 10, 0.1, dict(_UL, seed=16),
        minhash=dict(minBucketSize=10, maxBucketSize=40, minFrequency=5),
        align=dict(_NANOPORE_ALIGN, gapScore=-3), readgraph=dict(creationMethod=2, maxAlignmentCount=12),
        markergraph=dict(minCoveragePerStrand=3)),
    # conf/Nanopore-Human-SingleFlowcell-May2022.conf
    "Nanopore-Human-SingleFlowcell-May2022": _config(
        "Nanopore-Human-SingleFlowcell-May2022.conf", 14, 0.1, dict(_ONT, errors=NANOPORE_Q20, seed=14),
        minhash=dict(minBucketSize=5, maxBucketSize=30, minHashIterationCount=100, minFrequency=5),
        align=dict(downsamplingFactor=0.05, maxSkip=30, maxDrift=15, maxTrim=30, minAlignedMarkerCount=200, minAlignedFraction=0.6),
        readgraph=dict(creationMethod=0, maxAlignmentCount=12), markergraph=dict(minCoverage=0)),
    # conf/Nanopore-UL-Phased-Oct2021.conf
    "Nanopore-UL-Phased-Oct2021": _config(
        "Nanopore-UL-Phased-Oct2021.conf", 14, 0.1, dict(_UL, errors=NANOPORE_Q20, seed=15),
        minhash=dict(minBucketSize=10, maxBucketSize=60, minFrequency=5),
        align=dict(downsamplingFactor=0.05, minAlignedMarkerCount=400, minAlignedFraction=0.6, maxDrift=20, maxSkip=50, maxTrim=50),
        readgraph=dict(creationMethod=0, maxAlignmentCount=12, strandSeparationMethod=2),
        markergraph=dict(minCoverage=8, minCoveragePerStrand=1)),
    # conf/HiFi-Oct2021.conf
    "HiFi-Oct2021": _config(
        "HiFi-Oct2021.conf", 14, 0.1,
        dict(errors=HIFI, genome=120_000, arrays=[(60, 12), (45, 20), (80, 30), (120, 10)], coverage=25, n50=12000, sigma=0.25,
             min=6000, seed=17),
        minhash=dict(hashFraction=0.05, minHashIterationCount=100, minFrequency=3, minBucketSize=10, maxBucketSize=60),
        align=dict(downsamplingFactor=0.05, minAlignedFraction=0.97, minAlignedMarkerCount=200, maxSkip=6, maxDrift=4, maxTrim=2),
        readgraph=dict(maxAlignmentCount=30, maxChimericReadDistance=2), markergraph=dict(minCoverage=6)),
    # conf/Nanopore-May2022.conf (bench.py's configuration)
    "Nanopore-May2022": _config(
        "Nanopore-May2022.conf", 14, 0.1, dict(_ONT, seed=18),
        minhash=dict(minBucketSize=5, maxBucketSize=30, minFrequency=5), align=_NANOPORE_ALIGN,
        readgraph=dict(creationMethod=2), markergraph=dict(minCoverage=0)),
    # conf/PacBio-CCS-Dec2019.conf
    "PacBio-CCS-Dec2019": _config(
        "PacBio-CCS-Dec2019.conf", 15, 0.02,
        dict(errors=HIFI, genome=150_000, arrays=[(60, 12), (45, 20), (80, 30), (120, 10)], coverage=25, n50=12000, sigma=0.25,
             min=6000, chimeric_half=8000, seed=13),
        minhash=dict(m=12, minBucketSize=20, maxBucketSize=100, minHashIterationCount=25, minFrequency=10),
        readgraph=dict(maxAlignmentCount=20)),
}


# ---- k-mers ------------------------------------------------------------------------------------------------------------
def _plane_table(k):
    """T[v] = the k-bit reversal of the complement of plane v: rc(x) = T[x >> k] << k | T[x & (2^k - 1)]."""
    mask = (1 << k) - 1
    v = ~np.arange(1 << k, dtype=np.uint32) & np.uint32(mask)
    out = np.zeros(1 << k, np.uint32)
    for i in range(k):
        out |= ((v >> np.uint32(i)) & np.uint32(1)) << np.uint32(k - 1 - i)
    return out


def reverse_complement_kmer(x, k):
    """Bit-plane reverse complement of k-mer ids (src/ShortBaseSequence.hpp:109-118)."""
    t = _plane_table(k)
    x = np.asarray(x, np.uint32)
    return (t[x >> np.uint32(k)] << np.uint32(k)) | t[x & np.uint32((1 << k) - 1)]


def _fmix32(h):
    h = h ^ (h >> np.uint32(16))
    h = h * np.uint32(0x85EBCA6B)
    h = h ^ (h >> np.uint32(13))
    h = h * np.uint32(0xC2B2AE35)
    return h ^ (h >> np.uint32(16))


@functools.lru_cache(maxsize=1)
def marker_set(k, probability, seed=231):
    """(is_marker uint8[4^k], bitmap uint32[max(1, 4^k / 32)]): x is a marker when hash(min(x, rc x)) < p. The set is
    closed under reverse complement, and a palindromic k-mer is drawn on its own. One set is kept (1 GiB at k = 15)."""
    n = 1 << (2 * k)
    t = _plane_table(k)
    mask = np.uint32((1 << k) - 1)
    threshold = np.uint64(int(probability * 2.0 ** 32))
    is_marker = np.empty(n, np.uint8)
    step = 1 << 24
    with np.errstate(over="ignore"):
        for b in range(0, n, step):
            x = np.arange(b, min(n, b + step), dtype=np.uint32)
            rc = (t[x >> np.uint32(k)] << np.uint32(k)) | t[x & mask]
            h = _fmix32(np.minimum(x, rc) ^ np.uint32(seed * 0x9E3779B1 & 0xFFFFFFFF))
            is_marker[b:b + len(x)] = h.astype(np.uint64) < threshold
    bitmap = np.packbits(np.concatenate([is_marker, np.zeros(max(0, 32 - n), np.uint8)]), bitorder="little").view(np.uint32)
    return is_marker, bitmap


# ---- bases -------------------------------------------------------------------------------------------------------------
def _rle_bases(rng, n):
    """n random bases, no two equal neighbours."""
    return (np.cumsum(rng.integers(1, 4, n)) % 4).astype(np.uint8) if n else np.zeros(0, np.uint8)


def collapse(b):
    """Run-length compression: one base per run."""
    b = np.asarray(b, np.uint8)
    return b[np.r_[True, b[1:] != b[:-1]]] if len(b) else b


def reverse_complement(b):
    return (np.uint8(3) - np.asarray(b, np.uint8))[::-1]


def genome(rng, length, arrays):
    """Random bases with the tandem arrays (unit length, copies) spliced in at evenly spaced places."""
    parts, at = [], np.linspace(0, length, len(arrays) + 2).astype(np.int64)[1:-1]
    g = _rle_bases(rng, length)
    prev = 0
    for (unit, copies), a in zip(arrays, at):
        u = _rle_bases(rng, unit)
        parts += [g[prev:a], np.tile(u, copies)]
        prev = a
    parts.append(g[prev:])
    return collapse(np.concatenate(parts)), at


def sequencing_errors(rng, b, errors):
    """Each base deleted, substituted, or followed by an inserted base at the given rates; then run-length compressed."""
    n = len(b)
    u = rng.random(n)
    dele = u < errors["dele"]
    sub = (u >= errors["dele"]) & (u < errors["dele"] + errors["sub"])
    out = b.copy()
    out[sub] = (out[sub] + rng.integers(1, 4, int(sub.sum()))) % 4
    ins = np.nonzero(rng.random(n) < errors["ins"])[0]
    keep = np.nonzero(~dele)[0]
    keys = np.concatenate([2 * keep, 2 * ins + 1])
    values = np.concatenate([out[keep], rng.integers(0, 4, len(ins)).astype(np.uint8)])
    return collapse(values[np.argsort(keys, kind="stable")])


def reads(cfg):
    """dict(reads list of uint8 base arrays, palindromic / chimeric / short index arrays, genome)."""
    p = cfg["reads"]
    rng = np.random.default_rng(p["seed"])
    g, array_at = genome(rng, p["genome"], p["arrays"])
    G = len(g)
    mu = np.log(p["n50"]) - p["sigma"] ** 2
    out, total = [], 0
    while total < p["coverage"] * G:
        n = int(np.clip(np.exp(mu + p["sigma"] * rng.standard_normal()), p["min"], G // 2))
        s = int(rng.integers(0, G - n))
        w = g[s:s + n]
        if rng.integers(0, 2):
            w = reverse_complement(w)
        out.append(sequencing_errors(rng, w, p["errors"]))
        total += n
    injected = {"palindromic": [], "chimeric": [], "short": []}
    # Palindromic reads: a window, often over a tandem array, followed by its reverse complement.
    for i in range(6):
        n = int(p["min"] // 2 + rng.integers(0, p["min"]))
        s = int(np.clip(array_at[i % len(array_at)] - n // 3, 0, G - n)) if i % 2 == 0 else int(rng.integers(0, G - n))
        w = g[s:s + n]
        injected["palindromic"].append(sequencing_errors(rng, np.concatenate([w, reverse_complement(w)]), p["errors"]))
    # Chimeric reads: two windows half a genome apart, each on a random strand. Each half must hold more markers than
    # minAlignedMarkerCount to align on its own (chimeric_half, in bases; a third of n50 by default).
    for _ in range(CHIMERIC):
        n = int(p.get("chimeric_half", p["n50"] // 3))
        s0 = int(rng.integers(0, G // 2 - n))
        halves = [g[s:s + n] if rng.integers(0, 2) else reverse_complement(g[s:s + n]) for s in (s0, s0 + G // 2)]
        injected["chimeric"].append(sequencing_errors(rng, np.concatenate(halves), p["errors"]))
    # Empty reads and reads shorter than k (no markers).
    injected["short"] = [np.zeros(0, np.uint8), _rle_bases(rng, 1), _rle_bases(rng, cfg["k"] - 1), np.zeros(0, np.uint8),
                         _rle_bases(rng, cfg["k"] // 2)]
    allreads = out + injected["palindromic"] + injected["chimeric"] + injected["short"]
    kinds = np.array([""] * len(out) + ["palindromic"] * 6 + ["chimeric"] * CHIMERIC + ["short"] * 5, object)
    order = rng.permutation(len(allreads))
    kinds = kinds[order]
    return dict(reads=[allreads[i] for i in order], genome=g,
                **{kind: np.nonzero(kinds == kind)[0] for kind in ("palindromic", "chimeric", "short")})


def pack(reads):
    """LongBaseSequences layout (src/LongBaseSequence.hpp:33-41): per read, blocks of 64 bases as two words (low bit
    plane, high bit plane), base j of a block at bit 63 - j. Returns (word_offsets uint64[R+1], words uint64[], base_counts
    uint64[R])."""
    counts = np.array([len(r) for r in reads], np.int64)
    blocks = (counts + 63) // 64
    offsets = np.zeros(len(reads) + 1, np.uint64)
    offsets[1:] = np.cumsum(2 * blocks)
    total = int(blocks.sum())
    buf = np.zeros(64 * total, np.uint8)
    if total:
        cat = np.concatenate([np.asarray(r, np.uint8) for r in reads])
        first = np.cumsum(counts) - counts
        dest = np.repeat(64 * (np.cumsum(blocks) - blocks) - first, counts) + np.arange(len(cat))
        buf[dest] = cat
    bits = buf.reshape(total, 64)
    words = np.empty(2 * total, np.uint64)
    words[0::2] = np.packbits(bits & 1, axis=1).view(">u8").reshape(-1)
    words[1::2] = np.packbits(bits >> 1, axis=1).view(">u8").reshape(-1)
    return offsets, words, counts.astype(np.uint64)


@functools.lru_cache(maxsize=2)
def inputs(name):
    """The reads of configuration `name`, packed. dict(word_offsets, words, base_counts, palindromic, chimeric, short, k)."""
    cfg = CONFIGS[name]
    r = reads(cfg)
    wo, w, bc = pack(r["reads"])
    return dict(word_offsets=wo, words=w, base_counts=bc, palindromic=r["palindromic"], chimeric=r["chimeric"],
                short=r["short"], k=cfg["k"])


def kmer_ids(data7):
    return np.ascontiguousarray(np.asarray(data7, np.uint8).reshape(-1, 7)[:, :4]).view(np.uint32).reshape(-1)
