"""TEST INFRASTRUCTURE — ctypes bindings for flagPalindromicReads (src/AssemblerAlign.cpp:652-770): the CPU restatement in
oracle/palindromic_oracle.c (part of oracle/_build/liboracle.so) and, when present, the unmodified reference's
AlignmentGraph.cpp in oracle/_ref/libshasta_ref_palindromic.so (built by oracle/palindromic.mk).

Only tests/ and bench_palindromic.py may import this module. The product (shasta_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.bindings import oracle_lib

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_PALINDROMIC_SO = os.path.join(_HERE, "_ref", "libshasta_ref_palindromic.so")
_ref = None


def build(quiet=True):
    """Compile the reference's AlignmentGraph build (only where palindromic.mk's SHASTA_REF_SRC tree exists)."""
    subprocess.check_call(["make", "-C", _HERE, "-f", "palindromic.mk", "-j4", "ref"], stdout=subprocess.DEVNULL if quiet else None)


def have_ref():
    return os.path.exists(REF_PALINDROMIC_SO)


def ref_lib():
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_PALINDROMIC_SO)
        _ref.ref_free_palindromic.argtypes = [C.c_void_p]
    return _ref


class PalindromicCounters(C.Structure):
    _fields_ = [("heapsortFallbacks", C.c_uint64), ("vertices", C.c_uint64), ("edges", C.c_uint64),
                ("heapPushes", C.c_uint64), ("exactReads", C.c_uint64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


PALINDROMIC_DEFAULTS = dict(maxSkip=100, maxDrift=100, maxMarkerFrequency=10, alignedFractionThreshold=0.1,
                            nearDiagonalFractionThreshold=0.1, deltaThreshold=100)


def _pal_args(p):
    d = dict(PALINDROMIC_DEFAULTS)
    d.update(p)
    return (int(d["maxSkip"]), int(d["maxDrift"]), int(d["maxMarkerFrequency"]), float(d["alignedFractionThreshold"]),
            float(d["nearDiagonalFractionThreshold"]), int(d["deltaThreshold"]))


def _pal_path(lib_free, p, n):
    out = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint32)), (n, 2)).copy() if n else np.zeros((0, 2), np.uint32)
    if p:
        lib_free(p)
    return out


def oracle_flag_palindromic(toc, kmer_ids, exact_all=False, path_read=None, **params):
    """The C restatement (oracle/palindromic_oracle.c). Returns dict(flags, aligned, nearDiagonal, vBound, vNearBound,
    survives, counters[, path]). With exact_all=False the reads the prefilter rejects carry their bounds as counts."""
    lib = oracle_lib()
    f = lib.orc_flag_palindromic
    f.restype = C.c_int
    f.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, C.c_double, C.c_uint32,
                  C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(PalindromicCounters)]
    toc = np.ascontiguousarray(toc, np.uint64)
    kmer_ids = np.ascontiguousarray(kmer_ids, np.uint32)
    R = (len(toc) - 1) // 2
    out = dict(flags=np.zeros(R, np.uint8), aligned=np.zeros(R, np.uint32), nearDiagonal=np.zeros(R, np.uint32),
               vBound=np.zeros(R, np.uint64), vNearBound=np.zeros(R, np.uint64), survives=np.zeros(R, np.uint8))
    p, n, k = C.c_void_p(), C.c_uint64(), PalindromicCounters()
    f(R, toc.ctypes.data, kmer_ids.ctypes.data, *_pal_args(params), 1 if exact_all else 0,
      out["flags"].ctypes.data, out["aligned"].ctypes.data, out["nearDiagonal"].ctypes.data, out["vBound"].ctypes.data,
      out["vNearBound"].ctypes.data, out["survives"].ctypes.data, 2**64 - 1 if path_read is None else int(path_read),
      C.byref(p), C.byref(n), C.byref(k))
    out["counters"] = k.asdict()
    if path_read is not None:
        out["path"] = _pal_path(lib.orc_free, p, n.value)
    return out


def ref_flag_palindromic(toc, kmer_ids, path_read=None, **params):
    """The reference build: shasta::align of each read against its reverse complement, compiled unmodified, and the two
    thresholds. Returns dict(flags, aligned, nearDiagonal[, path])."""
    lib = ref_lib()
    f = lib.ref_flag_palindromic
    f.restype = C.c_int
    f.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, C.c_double, C.c_uint32,
                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    toc = np.ascontiguousarray(toc, np.uint64)
    kmer_ids = np.ascontiguousarray(kmer_ids, np.uint32)
    R = (len(toc) - 1) // 2
    out = dict(flags=np.zeros(R, np.uint8), aligned=np.zeros(R, np.uint32), nearDiagonal=np.zeros(R, np.uint32))
    p, n = C.c_void_p(), C.c_uint64()
    if f(R, toc.ctypes.data, kmer_ids.ctypes.data, *_pal_args(params), out["flags"].ctypes.data, out["aligned"].ctypes.data,
         out["nearDiagonal"].ctypes.data, 2**64 - 1 if path_read is None else int(path_read), C.byref(p), C.byref(n)):
        raise RuntimeError("reference flagPalindromicReads failed")
    if path_read is not None:
        out["path"] = _pal_path(lib.ref_free_palindromic, p, n.value)
    return out


def oracle_std_sort_markers(kmer_ids, ordinals):
    """std::sort of MarkerWithOrdinal by kmerId as restated in the oracle. Returns (kmerIds, ordinals, heapsort fallbacks)."""
    lib = oracle_lib()
    lib.orc_std_sort_markers.restype = C.c_uint64
    lib.orc_std_sort_markers.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    k = np.ascontiguousarray(kmer_ids, np.uint32).copy()
    o = np.ascontiguousarray(ordinals, np.uint32).copy()
    fb = lib.orc_std_sort_markers(k.ctypes.data, o.ctypes.data, len(k))
    return k, o, int(fb)


def oracle_sort_killer_keys(n):
    """n keys on which the restated std::sort uses up its introsort depth limit (McIlroy's adversary)."""
    lib = oracle_lib()
    lib.orc_sort_killer_keys.argtypes = [C.c_uint32, C.c_void_p]
    out = np.zeros(n, np.uint32)
    lib.orc_sort_killer_keys(n, out.ctypes.data)
    return out
