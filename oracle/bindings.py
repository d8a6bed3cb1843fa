"""TEST INFRASTRUCTURE — ctypes bindings to the CPU oracle (oracle/_build/liboracle.so) and,
when present, to the unmodified reference build (oracle/_ref/libshasta_ref.so), both built by oracle/Makefile.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module. The product (shasta_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle._load import have, load, take

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "_build", "liboracle.so")
REF_SO = os.path.join(_HERE, "_ref", "libshasta_ref.so")


def build(quiet=True):
    """Compile the oracle (always) and every reference library (only where the Makefile's SHASTA_REF_SRC tree exists)."""
    subprocess.check_call(["make", "-C", _HERE, "-j8", "all"], stdout=subprocess.DEVNULL if quiet else None)


class AlignOptions(C.Structure):
    """orc_align_options: AlignOptions of src/AssemblerOptions.hpp:177-199 as used on the path."""
    _fields_ = [("alignMethod", C.c_uint32), ("k", C.c_uint32),
                ("maxSkip", C.c_uint64), ("maxDrift", C.c_uint64), ("maxTrim", C.c_uint64),
                ("minAlignedMarkerCount", C.c_uint64), ("minAlignedFraction", C.c_double),
                ("matchScore", C.c_int32), ("mismatchScore", C.c_int32), ("gapScore", C.c_int32),
                ("downsamplingFactor", C.c_double), ("bandExtend", C.c_int32), ("maxBand", C.c_int32),
                ("suppressContainments", C.c_uint32),
                ("align4DeltaX", C.c_uint64), ("align4DeltaY", C.c_uint64),
                ("align4MinEntryCountPerCell", C.c_uint64), ("align4MaxDistanceFromBoundary", C.c_uint64)]


class _Alignment(C.Structure):
    _fields_ = [("ord", C.c_void_p), ("n", C.c_uint64), ("cap", C.c_uint64)]


_TABLE = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]
_READ_GRAPH = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
_READ_GRAPH2 = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32] + [C.c_void_p] * 7
_HISTOGRAM2 = [C.c_void_p, C.c_uint64, C.c_double, C.c_double, C.c_uint64, C.c_double]

_ORACLE_PROTOS = {
    "orc_murmurhash64a": (C.c_uint64, [C.c_void_p, C.c_int, C.c_uint64]),
    "orc_murmurhash2": (C.c_uint32, [C.c_void_p, C.c_int, C.c_uint32]),
    "orc_reverse_complement_kmer": (C.c_uint32, [C.c_uint32, C.c_uint32]),
    "orc_kmer_downsampling_hash": (C.c_uint32, [C.c_uint32, C.c_uint32]),
    "orc_lowhash0": (C.c_int, [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_uint64, C.c_double, C.c_uint64, C.c_double, C.c_uint64,
                               C.c_uint64, C.c_uint64, C.c_uint64,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "orc_free": (None, [C.c_void_p]),
    "orc_find_markers": (C.c_int, [C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    "orc_overlap_align": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_int64, C.c_int64, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]),
    "orc_compress_alignment": (C.c_uint64, [C.c_void_p, C.c_uint64, C.c_void_p]),
    "orc_decompress_alignment": (C.c_uint64, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]),
    "orc_alignment_info": (None, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p]),
    "orc_align_method3": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(AlignOptions), C.c_void_p]),
    "orc_align_method4": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(AlignOptions), C.c_void_p,
                                    C.POINTER(C.c_int)]),
    "orc_compute_alignments": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(AlignOptions), C.c_uint32,
                                         C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_void_p),
                                         C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    "orc_compute_alignment_table": (None, _TABLE),
    "orc_compute_candidate_table": (None, _TABLE),
    "orc_create_read_graph": (C.c_int, _READ_GRAPH),
    "orc_create_read_graph2": (C.c_int, _READ_GRAPH2),
    "orc_histogram2_threshold": (C.c_double, _HISTOGRAM2),
    "orc_set_dp_policy": (None, [C.c_int]),
    "orc_get_dp_policy": (C.c_int, []),
    "orc_reset_tie_flags": (None, []),
    "orc_get_tie_flags": (C.c_int, []),
    "orc_release_thread_scratch": (None, []),
}

_REF_PROTOS = {
    "ref_lowhash0": (C.c_int, [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_uint64, C.c_double, C.c_uint64, C.c_double, C.c_uint64,
                               C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                               C.c_void_p, C.c_uint64, C.c_void_p]),
    "ref_markers_from_fasta": (C.c_int, [C.c_char_p, C.c_uint64, C.c_double, C.c_int, C.c_uint64, C.c_uint64,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ref_reads_from_fasta": (C.c_int, [C.c_char_p, C.c_uint64, C.c_double, C.c_int, C.c_uint64, C.c_uint64,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ref_murmurhash64a": (C.c_uint64, [C.c_void_p, C.c_int, C.c_uint64]),
    "ref_murmurhash2": (C.c_uint32, [C.c_void_p, C.c_int, C.c_uint32]),
    "ref_free": (None, [C.c_void_p]),
    "ref_write_data_dir": (C.c_int, [C.c_char_p, C.c_char_p, C.c_uint64, C.c_double, C.c_int, C.c_uint64, C.c_uint64]),
    "ref_open_vector": (C.c_int, [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "ref_align4": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                             C.c_uint64, C.c_double, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                             C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]),
    "ref_alignment_info": (None, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p]),
    "ref_compress_alignment": (C.c_uint64, [C.c_void_p, C.c_uint64, C.c_void_p]),
    "ref_decompress_alignment": (C.c_uint64, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]),
    "ref_test_alignment_compression": (C.c_int, []),
    "ref_histogram2_threshold": (C.c_double, _HISTOGRAM2),
    "ref_alignment_indicators": (None, [C.c_void_p, C.c_void_p]),
    "ref_compute_alignment_table": (C.c_int, _TABLE),
    "ref_compute_candidate_table": (C.c_int, _TABLE),
    "ref_create_read_graph": (C.c_int, _READ_GRAPH),
    "ref_create_read_graph2": (C.c_int, _READ_GRAPH2),
}


def oracle_lib(protos=None):
    """liboracle.so, built first if it is missing, with this module's prototypes and, when given, those of protos: the table
    of the binding module that wraps the restatements it calls."""
    if not os.path.exists(ORACLE_SO):
        build()
    lib = load(ORACLE_SO, _ORACLE_PROTOS)
    return load(ORACLE_SO, protos) if protos else lib


def have_ref():
    return have(REF_SO)


def have_ref_readgraph():
    """The reference build is present AND has the read graph glue (ref_glue/ref_readgraph.cpp's table and read graph entry
    points). A prebuilt oracle/_ref from before that glue lacks them: the tests then use the recorded outputs instead."""
    if not have_ref():
        return False
    lib = ref_lib()
    return all(hasattr(lib, name) for name in ("ref_compute_alignment_table", "ref_compute_candidate_table",
                                               "ref_create_read_graph", "ref_create_read_graph2"))


def ref_lib():
    return load(REF_SO, _REF_PROTOS)


class LowHashParams(dict):
    """m, hashFraction, minHashIterationCount, alignmentCandidatesPerRead, log2MinHashBucketCount,
    minBucketSize, maxBucketSize, minFrequency  (src/Assembler.hpp:688-699)."""

    DEFAULTS = dict(m=4, hashFraction=0.01, minHashIterationCount=10, alignmentCandidatesPerRead=20.0,
                    log2MinHashBucketCount=0, minBucketSize=0, maxBucketSize=10, minFrequency=2)

    def __init__(self, **kw):
        d = dict(self.DEFAULTS)
        d.update(kw)
        super().__init__(d)


def _common(toc, data, flags):
    toc = np.ascontiguousarray(toc, dtype=np.uint64)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    flags = np.ascontiguousarray(flags, dtype=np.uint8)
    R = (len(toc) - 1) // 2
    # 8 bytes of slack: the 7-byte records are read with 4-byte loads.
    pad = np.zeros(len(data) + 8, np.uint8)
    pad[:len(data)] = data
    return R, toc, pad, flags


def oracle_lowhash0(toc, data, flags, p: LowHashParams, max_iters=4096):
    """Returns (candidates uint32[n,3], stats uint64[R,3], iterSummary uint64[iters,2])."""
    lib = oracle_lib()
    R, toc, data, flags = _common(toc, data, flags)
    cand = C.c_void_p()
    n = C.c_uint64()
    iters = C.c_uint64()
    stats = np.zeros((R, 3), np.uint64)
    summ = np.zeros((max_iters, 2), np.uint64)
    rc = lib.orc_lowhash0(R, toc.ctypes.data, data.ctypes.data, flags.ctypes.data,
                          p["m"], p["hashFraction"], p["minHashIterationCount"],
                          p["alignmentCandidatesPerRead"], p["log2MinHashBucketCount"],
                          p["minBucketSize"], p["maxBucketSize"], p["minFrequency"],
                          C.byref(cand), C.byref(n), stats.ctypes.data, summ.ctypes.data, max_iters,
                          C.byref(iters))
    if rc == 2:
        raise RuntimeError("alignmentCandidatesPerRead was not reached within max_iters iterations")
    if rc != 0:
        raise RuntimeError("log2MinHashBucketCount is unreasonably small.")
    return take(cand, 3 * n.value, np.uint32, lib.orc_free).reshape(-1, 3), stats, summ[:iters.value].copy()


def ref_lowhash0(toc, data, flags, p: LowHashParams, threads=0, max_iters=4096, quiet=True):
    """Same, through the unmodified reference LowHash0. Also returns the constructor's wall seconds."""
    lib = ref_lib()
    R, toc, data, flags = _common(toc, data, flags)
    cand = C.c_void_p()
    n = C.c_uint64()
    iters = C.c_uint64()
    sec = C.c_double()
    stats = np.zeros((R, 3), np.uint64)
    summ = np.zeros((max_iters, 2), np.uint64)
    rc = lib.ref_lowhash0(R, toc.ctypes.data, data.ctypes.data, flags.ctypes.data,
                          p["m"], p["hashFraction"], p["minHashIterationCount"],
                          p["alignmentCandidatesPerRead"], p["log2MinHashBucketCount"],
                          p["minBucketSize"], p["maxBucketSize"], p["minFrequency"], threads,
                          C.byref(cand), C.byref(n), stats.ctypes.data, C.byref(sec), 1 if quiet else 0,
                          summ.ctypes.data, max_iters, C.byref(iters))
    if rc != 0:
        raise RuntimeError("reference LowHash0 failed")
    return take(cand, 3 * n.value, np.uint32, lib.ref_free).reshape(-1, 3), stats, summ[:iters.value].copy(), sec.value


def ref_markers_from_fasta(path, k=10, probability=0.1, seed=231, min_read_length=10000, threads=4, want_hash=False):
    lib = ref_lib()
    R = C.c_uint64()
    toc = C.c_void_p()
    data = C.c_void_p()
    flags = C.c_void_p()
    kh = C.c_void_p()
    rc = lib.ref_markers_from_fasta(path.encode(), k, probability, seed, min_read_length, threads,
                                    C.byref(R), C.byref(toc), C.byref(data), C.byref(flags),
                                    C.byref(kh) if want_hash else None)
    if rc != 0:
        raise RuntimeError("reference marker finding failed")
    R = R.value
    tocn = take(toc, 2 * R + 1, np.uint64, lib.ref_free)
    out = dict(toc=tocn, data=take(data, 7 * int(tocn[-1]), np.uint8, lib.ref_free), flags=take(flags, R, np.uint8, lib.ref_free),
               k=k)
    if want_hash:
        out["kmerHash"] = take(kh, 1 << (2 * k), np.uint32, lib.ref_free)
    return out


def ref_reads_from_fasta(path, k=10, probability=0.1, seed=231, min_read_length=10000, threads=4):
    """The inputs of the reference's MarkerFinder as the reference stores them: dict(word_offsets uint64[R+1], words uint64[],
    base_counts uint64[R], is_marker uint8[4^k]) — RLE reads in LongBaseSequences layout + kmerTable[].isMarker."""
    lib = ref_lib()
    R = C.c_uint64()
    off, words, bc, im = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
    rc = lib.ref_reads_from_fasta(path.encode(), k, probability, seed, min_read_length, threads,
                                  C.byref(R), C.byref(off), C.byref(words), C.byref(bc), C.byref(im))
    if rc != 0:
        raise RuntimeError("reference read loading failed")
    R = R.value
    offn = take(off, R + 1, np.uint64, lib.ref_free)
    return dict(word_offsets=offn, words=take(words, int(offn[-1]), np.uint64, lib.ref_free),
                base_counts=take(bc, R, np.uint64, lib.ref_free), is_marker=take(im, 1 << (2 * k), np.uint8, lib.ref_free), k=k)


def oracle_find_markers(word_offsets, words, base_counts, is_marker, k):
    """CPU restatement of MarkerFinder (oracle/markers_oracle.c). Returns (toc uint64[2R+1], data uint8[7M])."""
    lib = oracle_lib()
    wo = np.ascontiguousarray(word_offsets, np.uint64)
    w = np.ascontiguousarray(words, np.uint64)
    bc = np.ascontiguousarray(base_counts, np.uint64)
    im = np.ascontiguousarray(is_marker, np.uint8)
    R = len(bc)
    toc, data = C.c_void_p(), C.c_void_p()
    lib.orc_find_markers(R, k, wo.ctypes.data, w.ctypes.data, bc.ctypes.data, im.ctypes.data, C.byref(toc), C.byref(data))
    tocn = take(toc, 2 * R + 1, np.uint64, lib.orc_free)
    return tocn, take(data, 7 * int(tocn[-1]), np.uint8, lib.orc_free)


def candidate_digest(c):
    """FNV-1a style digest over (readId0, readId1, isSameStrand) rows (SURVEY.md Appendix D)."""
    h = 1469598103934665603
    for a, b, s in np.asarray(c).tolist():
        for v in (a, b, s):
            h = ((h ^ v) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


# ---------------------------------------------------------------------------------------------------
# Alignment half
ALIGN_DEFAULTS = dict(alignMethod=3, k=10, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=100,
                      minAlignedFraction=0.4, matchScore=6, mismatchScore=-1, gapScore=-1, downsamplingFactor=0.1,
                      bandExtend=10, maxBand=1000, suppressContainments=0, align4DeltaX=200, align4DeltaY=10,
                      align4MinEntryCountPerCell=10, align4MaxDistanceFromBoundary=100)


def make_align_options(**kw):
    d = dict(ALIGN_DEFAULTS)
    d.update(kw)
    return AlignOptions(**d)


def overlap_align(a, b, match=6, mismatch=-1, gap=-1, band=None):
    """The oracle's DP. Returns (score, path uint32[n,2]) — diagonal steps in path order; score None on failure."""
    lib = oracle_lib()
    a = np.ascontiguousarray(a, np.uint32)
    b = np.ascontiguousarray(b, np.uint32)
    p = C.c_void_p()
    n = C.c_uint64()
    lo, hi = band if band is not None else (0, 0)
    s = lib.orc_overlap_align(a.ctypes.data, len(a), b.ctypes.data, len(b), match, mismatch, gap,
                              1 if band is not None else 0, lo, hi, C.byref(p), C.byref(n))
    if s == -2**31:
        return None, np.zeros((0, 2), np.uint32)
    return s, take(p, 2 * n.value, np.uint32, lib.orc_free).reshape(-1, 2)


def oracle_align_pair(a, b, opts: AlignOptions):
    """Single pair through method 3 or 4. Returns (status, ordinals uint32[n,2], tie flag)."""
    lib = oracle_lib()
    a = np.ascontiguousarray(a, np.uint32)
    b = np.ascontiguousarray(b, np.uint32)
    al = _Alignment(None, 0, 0)
    tie = C.c_int(0)
    if opts.alignMethod == 4:
        st = lib.orc_align_method4(a.ctypes.data, len(a), b.ctypes.data, len(b), C.byref(opts), C.byref(al), C.byref(tie))
    else:
        st = lib.orc_align_method3(a.ctypes.data, len(a), b.ctypes.data, len(b), C.byref(opts), C.byref(al))
    return st, take(al.ord, 2 * al.n, np.uint32, lib.orc_free).reshape(-1, 2), tie.value


def oracle_alignment_info(ordinals, nx, ny):
    lib = oracle_lib()
    o = np.ascontiguousarray(ordinals, np.uint32).reshape(-1)
    out = np.zeros(12, np.uint32)
    lib.orc_alignment_info(o.ctypes.data, len(o) // 2, nx, ny, out.ctypes.data)
    return out


def oracle_compress(ordinals):
    lib = oracle_lib()
    o = np.ascontiguousarray(ordinals, np.uint32).reshape(-1)
    buf = np.zeros(8 * len(o) + 16, np.uint8)
    n = lib.orc_compress_alignment(o.ctypes.data, len(o) // 2, buf.ctypes.data)
    return buf[:n].copy()


def oracle_decompress(data, cap=1 << 20):
    lib = oracle_lib()
    d = np.ascontiguousarray(data, np.uint8)
    out = np.zeros((cap, 2), np.uint32)
    n = lib.orc_decompress_alignment(d.ctypes.data, len(d), out.ctypes.data, cap)
    return out[:n].copy()


def oracle_compute_alignments(toc, kmer_ids, candidates, opts: AlignOptions, threads=1):
    """Returns (records uint32[count,16], compressedToc uint64[count+1], compressedData uint8[], ties uint8[n])."""
    lib = oracle_lib()
    toc = np.ascontiguousarray(toc, np.uint64)
    kmer_ids = np.ascontiguousarray(kmer_ids, np.uint32)
    cand = np.ascontiguousarray(candidates, np.uint32).reshape(-1, 3)
    rec = C.c_void_p()
    cnt = C.c_uint64()
    ctoc = C.c_void_p()
    cdata = C.c_void_p()
    ties = C.c_void_p()
    lib.orc_compute_alignments(toc.ctypes.data, kmer_ids.ctypes.data, cand.ctypes.data, len(cand), C.byref(opts), threads,
                               C.byref(rec), C.byref(cnt), C.byref(ctoc), C.byref(cdata), C.byref(ties))
    n = cnt.value
    records = take(rec, 16 * n, np.uint32, lib.orc_free).reshape(-1, 16)
    ctocn = take(ctoc, n + 1, np.uint64, lib.orc_free)
    return records, ctocn, take(cdata, int(ctocn[-1]), np.uint8, lib.orc_free), take(ties, len(cand), np.uint8, lib.orc_free)


# ---- reference side (unmodified Align4.cpp / Alignment.cpp / compressAlignment.cpp) ----
def ref_align4(a, b, opts: AlignOptions):
    lib = ref_lib()
    a = np.ascontiguousarray(a, np.uint32)
    b = np.ascontiguousarray(b, np.uint32)
    p = C.c_void_p()
    n = C.c_uint64()
    rc = lib.ref_align4(a.ctypes.data, len(a), b.ctypes.data, len(b), opts.align4DeltaX, opts.align4DeltaY,
                        opts.align4MinEntryCountPerCell, opts.align4MaxDistanceFromBoundary, opts.minAlignedMarkerCount,
                        opts.minAlignedFraction, opts.maxSkip, opts.maxDrift, opts.maxTrim, opts.maxBand, C.byref(p), C.byref(n))
    if rc:
        raise RuntimeError("reference Align4 failed")
    return take(p, 2 * n.value, np.uint32, lib.ref_free).reshape(-1, 2)


def ref_alignment_info(ordinals, nx, ny):
    lib = ref_lib()
    o = np.ascontiguousarray(ordinals, np.uint32).reshape(-1)
    out = np.zeros(12, np.uint32)
    lib.ref_alignment_info(o.ctypes.data, len(o) // 2, nx, ny, out.ctypes.data)
    return out


def ref_compress(ordinals):
    lib = ref_lib()
    o = np.ascontiguousarray(ordinals, np.uint32).reshape(-1)
    buf = np.zeros(8 * len(o) + 16, np.uint8)
    n = lib.ref_compress_alignment(o.ctypes.data, len(o) // 2, buf.ctypes.data)
    return buf[:n].copy()


def oracle_compute_alignment_table(records, read_count):
    """Returns (toc uint32[2R+1], table uint32[4n]) — src/AssemblerAlign.cpp:509-571."""
    lib = oracle_lib()
    rec = np.ascontiguousarray(records, np.uint32).reshape(-1, 16)
    toc = np.zeros(2 * read_count + 1, np.uint32)
    table = np.zeros(4 * len(rec) + 1, np.uint32)
    lib.orc_compute_alignment_table(rec.ctypes.data, len(rec), read_count, toc.ctypes.data, table.ctypes.data)
    return toc, table[:4 * len(rec)].copy()


def oracle_compute_candidate_table(candidates, read_count):
    """Returns (toc uint64[2R+1], table uint64[4n]) — src/AssemblerAlignmentCandidates.cpp:379-448."""
    lib = oracle_lib()
    cand = np.ascontiguousarray(candidates, np.uint32).reshape(-1, 3)
    toc = np.zeros(2 * read_count + 1, np.uint64)
    table = np.zeros(4 * len(cand) + 1, np.uint64)
    lib.orc_compute_candidate_table(cand.ctypes.data, len(cand), read_count, toc.ctypes.data, table.ctypes.data)
    return toc, table[:4 * len(cand)].copy()


class UnorderedReadGraphEdge(ValueError):
    """A kept alignment gives a read graph edge, or a reverse-complement edge, whose oriented reads are not in increasing
    order: the SHASTA_ASSERT of src/AssemblerReadGraph.cpp:134,140."""


def _read_graph_buffers(records, read_count):
    rec = np.ascontiguousarray(records, np.uint32).reshape(-1, 16).copy()
    n = len(rec)
    return rec, np.zeros(n + 1, np.uint8), np.zeros((2 * n + 1, 4), np.uint32), np.zeros(2 * read_count + 1, np.uint32), \
        np.zeros(4 * n + 1, np.uint32)


def _criteria(crit):
    return dict(minAlignedFraction=float(crit[:1].view(np.float64)[0]), minAlignedMarkerCount=int(crit[1]), maxDrift=int(crit[2]),
                maxSkip=int(crit[3]), maxTrim=int(crit[4]))


def oracle_create_read_graph(records, read_count, max_alignment_count):
    """Assembler::createReadGraph, creationMethod 0 (src/AssemblerReadGraph.cpp:35-175). records uint32[n,16] is NOT modified.
    Returns (records with isInReadGraph set, keep uint8[n], edges uint32[E,4], connectivityToc uint32[2R+1], connectivityData uint32[2E]);
    each connectivity row lists its edges in decreasing edge index, as the reference's VectorOfVectors::store leaves them.
    Raises UnorderedReadGraphEdge where the reference's assertion fails."""
    lib = oracle_lib()
    rec, keep, edges, toc, data = _read_graph_buffers(records, read_count)
    n = len(rec)
    e = C.c_uint64()
    if lib.orc_create_read_graph(rec.ctypes.data, n, read_count, int(max_alignment_count), keep.ctypes.data, edges.ctypes.data,
                                 C.byref(e), toc.ctypes.data, data.ctypes.data):
        raise UnorderedReadGraphEdge("a kept alignment gives an unordered read graph edge")
    e = e.value
    return rec, keep[:n].copy(), edges[:e].copy(), toc, data[:2 * e].copy()


def oracle_create_read_graph2(records, read_count, max_alignment_count, percentiles):
    """Assembler::createReadGraph2, creationMethod 2 (src/AssemblerReadGraph2.cpp:69-248). percentiles = (markerCount,
    alignedFraction, maxSkip, maxDrift, maxTrim). Returns (criteria dict, records, keep, edges, connectivityToc, connectivityData),
    the last five as in oracle_create_read_graph."""
    lib = oracle_lib()
    rec, keep, edges, toc, data = _read_graph_buffers(records, read_count)
    n = len(rec)
    pc = np.array(percentiles, np.float64)
    crit = np.zeros(5, np.uint64)
    e = C.c_uint64()
    if lib.orc_create_read_graph2(rec.ctypes.data, n, read_count, int(max_alignment_count), pc.ctypes.data, crit.ctypes.data,
                                  keep.ctypes.data, edges.ctypes.data, C.byref(e), toc.ctypes.data, data.ctypes.data):
        raise UnorderedReadGraphEdge("a kept alignment gives an unordered read graph edge")
    e = e.value
    return _criteria(crit), rec, keep[:n].copy(), edges[:e].copy(), toc, data[:2 * e].copy()


def ref_create_read_graph(records, read_count, max_alignment_count):
    """The reference's createReadGraph and createReadGraphUsingSelectedAlignments over its own containers
    (oracle/ref_glue/ref_readgraph.cpp). Same arguments, returns and refusal as oracle_create_read_graph."""
    lib = ref_lib()
    rec, keep, edges, toc, data = _read_graph_buffers(records, read_count)
    n = len(rec)
    e = C.c_uint64()
    if lib.ref_create_read_graph(rec.ctypes.data, n, read_count, int(max_alignment_count), keep.ctypes.data, edges.ctypes.data,
                                 C.byref(e), toc.ctypes.data, data.ctypes.data):
        raise UnorderedReadGraphEdge("the reference refused the read graph")
    e = e.value
    return rec, keep[:n].copy(), edges[:e].copy(), toc, data[:2 * e].copy()


def ref_create_read_graph2(records, read_count, max_alignment_count, percentiles):
    """The reference's createReadGraph2 (Histogram2 criteria, then the selection of createReadGraph) over its own containers.
    Same arguments, returns and refusal as oracle_create_read_graph2."""
    lib = ref_lib()
    rec, keep, edges, toc, data = _read_graph_buffers(records, read_count)
    n = len(rec)
    pc = np.array(percentiles, np.float64)
    crit = np.zeros(5, np.uint64)
    e = C.c_uint64()
    if lib.ref_create_read_graph2(rec.ctypes.data, n, read_count, int(max_alignment_count), pc.ctypes.data, crit.ctypes.data,
                                  keep.ctypes.data, edges.ctypes.data, C.byref(e), toc.ctypes.data, data.ctypes.data):
        raise UnorderedReadGraphEdge("the reference refused the read graph")
    e = e.value
    return _criteria(crit), rec, keep[:n].copy(), edges[:e].copy(), toc, data[:2 * e].copy()


def ref_compute_alignment_table(records, read_count):
    """The reference's computeAlignmentTable over its own VectorOfVectors. Returns (toc uint32[2R+1], table uint32[4n])."""
    lib = ref_lib()
    rec = np.ascontiguousarray(records, np.uint32).reshape(-1, 16)
    toc = np.zeros(2 * read_count + 1, np.uint32)
    table = np.zeros(4 * len(rec) + 1, np.uint32)
    if lib.ref_compute_alignment_table(rec.ctypes.data, len(rec), read_count, toc.ctypes.data, table.ctypes.data):
        raise RuntimeError("reference computeAlignmentTable failed")
    return toc, table[:4 * len(rec)].copy()


def ref_compute_candidate_table(candidates, read_count):
    """The reference's computeCandidateTable over its own VectorOfVectors. Returns (toc uint64[2R+1], table uint64[4n])."""
    lib = ref_lib()
    cand = np.ascontiguousarray(candidates, np.uint32).reshape(-1, 3)
    toc = np.zeros(2 * read_count + 1, np.uint64)
    table = np.zeros(4 * len(cand) + 1, np.uint64)
    if lib.ref_compute_candidate_table(cand.ctypes.data, len(cand), read_count, toc.ctypes.data, table.ctypes.data):
        raise RuntimeError("reference computeCandidateTable failed")
    return toc, table[:4 * len(cand)].copy()


def oracle_histogram2_threshold(x, start, stop, bin_count, fraction):
    x = np.ascontiguousarray(x, np.float64)
    return oracle_lib().orc_histogram2_threshold(x.ctypes.data, len(x), start, stop, bin_count, fraction)


def ref_histogram2_threshold(x, start, stop, bin_count, fraction):
    """The reference's own Histogram2 (dynamic bounds), compiled unmodified (oracle/_ref)."""
    x = np.ascontiguousarray(x, np.float64)
    return ref_lib().ref_histogram2_threshold(x.ctypes.data, len(x), start, stop, bin_count, fraction)


def ref_alignment_indicators(record16):
    """(minAlignedFraction, markerCount, maxDrift, maxSkip, trim) by the reference's AlignmentInfo accessors."""
    rec = np.ascontiguousarray(record16, np.uint32).reshape(16)
    out = np.zeros(5, np.float64)
    ref_lib().ref_alignment_indicators(rec.ctypes.data, out.ctypes.data)
    return out


def set_dp_policy(bits):
    """Tie-break policy of the oracle's DP at run time (include/shb_dp_policy.h: bit 0 diagonal wins ties, bit 1 vertical
    before horizontal, bit 2 first maximum is the end cell). Returns the previous policy."""
    lib = oracle_lib()
    old = lib.orc_get_dp_policy()
    lib.orc_set_dp_policy(int(bits))
    return old


def default_dp_policy():
    return oracle_lib().orc_get_dp_policy()


def ref_write_data_dir(fasta, prefix, k=10, probability=0.1, seed=231, min_read_length=10000, threads=4):
    if ref_lib().ref_write_data_dir(fasta.encode(), prefix.encode(), k, probability, seed, min_read_length, threads):
        raise RuntimeError("reference failed to write the Data directory")


def ref_open_vector(path, object_size):
    """(count, fnv checksum) of a MemoryMapped::Vector file as seen by the reference's own accessExistingReadOnly."""
    n, h = C.c_uint64(), C.c_uint64()
    if ref_lib().ref_open_vector(path.encode(), object_size, C.byref(n), C.byref(h)):
        raise RuntimeError(f"the reference could not open {path}")
    return n.value, h.value
