"""TEST INFRASTRUCTURE — ctypes bindings for flagPalindromicReads (src/AssemblerAlign.cpp:652-770): the CPU restatement in
oracle/palindromic_oracle.c (part of oracle/_build/liboracle.so) and, when present, the unmodified reference's
AlignmentGraph.cpp in oracle/_ref/libshasta_ref_palindromic.so (built by oracle/Makefile).

Only tests/ and bench_palindromic.py may import this module. The product (shasta_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import bindings
from oracle._load import have, load, take

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "_ref", "libshasta_ref_palindromic.so")


class PalindromicCounters(C.Structure):
    _fields_ = [("heapsortFallbacks", C.c_uint64), ("vertices", C.c_uint64), ("edges", C.c_uint64),
                ("heapPushes", C.c_uint64), ("exactReads", C.c_uint64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


_PAL = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, C.c_double, C.c_uint32]
_ORACLE_PROTOS = {
    "orc_flag_palindromic": (C.c_int, _PAL + [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64),
                                              C.POINTER(PalindromicCounters)]),
    "orc_std_sort_markers": (C.c_uint64, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "orc_sort_killer_keys": (None, [C.c_uint32, C.c_void_p]),
}
_REF_PROTOS = {
    "ref_flag_palindromic": (C.c_int, _PAL + [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p),
                                              C.POINTER(C.c_uint64)]),
    "ref_free_palindromic": (None, [C.c_void_p]),
}


def oracle_lib():
    return bindings.oracle_lib(_ORACLE_PROTOS)


def have_ref():
    return have(REF_SO)


def ref_lib():
    return load(REF_SO, _REF_PROTOS)


PALINDROMIC_DEFAULTS = dict(maxSkip=100, maxDrift=100, maxMarkerFrequency=10, alignedFractionThreshold=0.1,
                            nearDiagonalFractionThreshold=0.1, deltaThreshold=100)


def _pal_args(p):
    d = dict(PALINDROMIC_DEFAULTS)
    d.update(p)
    return (int(d["maxSkip"]), int(d["maxDrift"]), int(d["maxMarkerFrequency"]), float(d["alignedFractionThreshold"]),
            float(d["nearDiagonalFractionThreshold"]), int(d["deltaThreshold"]))


def oracle_flag_palindromic(toc, kmer_ids, exact_all=False, path_read=None, **params):
    """The C restatement (oracle/palindromic_oracle.c). Returns dict(flags, aligned, nearDiagonal, vBound, vNearBound,
    survives, counters[, path]). With exact_all=False the reads the prefilter rejects carry their bounds as counts."""
    lib = oracle_lib()
    toc = np.ascontiguousarray(toc, np.uint64)
    kmer_ids = np.ascontiguousarray(kmer_ids, np.uint32)
    R = (len(toc) - 1) // 2
    out = dict(flags=np.zeros(R, np.uint8), aligned=np.zeros(R, np.uint32), nearDiagonal=np.zeros(R, np.uint32),
               vBound=np.zeros(R, np.uint64), vNearBound=np.zeros(R, np.uint64), survives=np.zeros(R, np.uint8))
    p, n, k = C.c_void_p(), C.c_uint64(), PalindromicCounters()
    lib.orc_flag_palindromic(R, toc.ctypes.data, kmer_ids.ctypes.data, *_pal_args(params), 1 if exact_all else 0,
                             out["flags"].ctypes.data, out["aligned"].ctypes.data, out["nearDiagonal"].ctypes.data,
                             out["vBound"].ctypes.data, out["vNearBound"].ctypes.data, out["survives"].ctypes.data,
                             2**64 - 1 if path_read is None else int(path_read), C.byref(p), C.byref(n), C.byref(k))
    out["counters"] = k.asdict()
    if path_read is not None:
        out["path"] = take(p, 2 * n.value, np.uint32, lib.orc_free).reshape(-1, 2)
    return out


def ref_flag_palindromic(toc, kmer_ids, path_read=None, **params):
    """The reference build: shasta::align of each read against its reverse complement, compiled unmodified, and the two
    thresholds. Returns dict(flags, aligned, nearDiagonal[, path])."""
    lib = ref_lib()
    toc = np.ascontiguousarray(toc, np.uint64)
    kmer_ids = np.ascontiguousarray(kmer_ids, np.uint32)
    R = (len(toc) - 1) // 2
    out = dict(flags=np.zeros(R, np.uint8), aligned=np.zeros(R, np.uint32), nearDiagonal=np.zeros(R, np.uint32))
    p, n = C.c_void_p(), C.c_uint64()
    if lib.ref_flag_palindromic(R, toc.ctypes.data, kmer_ids.ctypes.data, *_pal_args(params), out["flags"].ctypes.data,
                                out["aligned"].ctypes.data, out["nearDiagonal"].ctypes.data,
                                2**64 - 1 if path_read is None else int(path_read), C.byref(p), C.byref(n)):
        raise RuntimeError("reference flagPalindromicReads failed")
    if path_read is not None:
        out["path"] = take(p, 2 * n.value, np.uint32, lib.ref_free_palindromic).reshape(-1, 2)
    return out


def oracle_std_sort_markers(kmer_ids, ordinals):
    """std::sort of MarkerWithOrdinal by kmerId as restated in the oracle. Returns (kmerIds, ordinals, heapsort fallbacks)."""
    k = np.ascontiguousarray(kmer_ids, np.uint32).copy()
    o = np.ascontiguousarray(ordinals, np.uint32).copy()
    fb = oracle_lib().orc_std_sort_markers(k.ctypes.data, o.ctypes.data, len(k))
    return k, o, int(fb)


def oracle_sort_killer_keys(n):
    """n keys on which the restated std::sort uses up its introsort depth limit (McIlroy's adversary)."""
    out = np.zeros(n, np.uint32)
    oracle_lib().orc_sort_killer_keys(n, out.ctypes.data)
    return out
