"""TEST INFRASTRUCTURE — ctypes bindings for createMarkerGraphVertices / findMarkerGraphReverseComplementVertices
(src/AssemblerMarkerGraph.cpp): the C restatement in oracle/markergraph_oracle.c (part of oracle/_build/liboracle.so) and,
when present, the reference's own DisjointSets, decompress and PeakFinder behind ref_glue/ref_markergraph.cpp in
oracle/_ref/libshasta_ref_markergraph.so (built by oracle/markergraph.mk).

Only tests/ and bench_markergraph.py may import this module. The product (shasta_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle.bindings import oracle_lib

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_MARKERGRAPH_SO = os.path.join(_HERE, "_ref", "libshasta_ref_markergraph.so")
_ref = None

DEFAULTS = dict(minCoverage=10, maxCoverage=100, minCoveragePerStrand=0, allowDuplicateMarkers=False,
                peakFinderMinAreaFraction=0.08, peakFinderAreaStartIndex=2)


def have_ref():
    return os.path.exists(REF_MARKERGRAPH_SO)


def ref_lib():
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_MARKERGRAPH_SO)
        _ref.ref_free_markergraph.argtypes = [C.c_void_p]
    return _ref


def _take(lib_free, p, n):
    out = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint64)), (n,)).copy() if n else np.zeros(0, np.uint64)
    lib_free(p)
    return out


_PROTO = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
          C.c_double] + [C.POINTER(C.c_void_p)] * 4 + [C.c_void_p]


def _run(f, lib_free, toc, kmer, edges, ctoc, cdata, flags, threads, **params):
    d = dict(DEFAULTS)
    d.update(params)
    toc = np.ascontiguousarray(toc, np.uint64)
    kmer = np.ascontiguousarray(kmer, np.uint32)
    edges = np.ascontiguousarray(edges, np.uint32).reshape(-1, 4)
    ctoc = np.ascontiguousarray(ctoc, np.uint64)
    cdata = np.ascontiguousarray(cdata, np.uint8)
    flags = np.ascontiguousarray(flags, np.uint8)
    R = (len(toc) - 1) // 2
    pv = np.array([d["minCoverage"], d["maxCoverage"], d["minCoveragePerStrand"], int(bool(d["allowDuplicateMarkers"])),
                   d["peakFinderAreaStartIndex"], threads], np.uint64)
    counts = np.zeros(12, np.uint64)
    t, vt, vd, h = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
    f.restype = C.c_int
    f.argtypes = _PROTO
    status = f(toc.ctypes.data, R, kmer.ctypes.data, edges.ctypes.data, len(edges), ctoc.ctypes.data, cdata.ctypes.data,
               len(ctoc) - 1, flags.ctypes.data, pv.ctypes.data, float(d["peakFinderMinAreaFraction"]), C.byref(t), C.byref(vt),
               C.byref(vd), C.byref(h), counts.ctypes.data)
    if status:
        return dict(status=int(status))
    M, V = int(toc[-1]), int(counts[8])
    return dict(status=0, table=_take(lib_free, t, M), vtoc=_take(lib_free, vt, V + 1), vdata=_take(lib_free, vd, int(counts[10])),
                histogram=_take(lib_free, h, int(counts[9])), minCoverageUsed=int(counts[0]), peakFinderFailed=int(counts[1]),
                disjointSetCount=int(counts[5]), keptDisjointSetCount=int(counts[6]), badDisjointSetCount=int(counts[7]),
                vertexCount=V, observedAreaFraction=float(counts[11:12].view(np.float64)[0]),
                edgePairsUsed=int(counts[2]), edgePairsSkipped=int(counts[3]), alignedMarkerPairs=int(counts[4]))


def oracle_create_marker_graph_vertices(toc, kmer, edges, ctoc, cdata, flags, **params):
    """The C restatement. Returns dict(status, table uint64[M], vtoc, vdata, histogram, counts...); status != 0 is the
    reference assertion it stands for (see markergraph_oracle.c)."""
    lib = oracle_lib()
    return _run(lib.orc_create_marker_graph_vertices, lib.orc_free, toc, kmer, edges, ctoc, cdata, flags, 0, **params)


def ref_create_marker_graph_vertices(toc, kmer, edges, ctoc, cdata, flags, threads=1, **params):
    """The reference's components in the member's control flow. Vertex numbering is the reference's (by representative)."""
    lib = ref_lib()
    return _run(lib.ref_create_marker_graph_vertices, lib.ref_free_markergraph, toc, kmer, edges, ctoc, cdata, flags, threads, **params)


def _rc(f, toc, table, vtoc, vdata):
    toc = np.ascontiguousarray(toc, np.uint64)
    table = np.ascontiguousarray(table, np.uint64)
    vtoc = np.ascontiguousarray(vtoc, np.uint64)
    vdata = np.ascontiguousarray(vdata, np.uint64)
    V = len(vtoc) - 1
    rc = np.zeros(V + 1, np.uint64)
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    status = f(toc.ctypes.data, (len(toc) - 1) // 2, table.ctypes.data, vtoc.ctypes.data, vdata.ctypes.data, V, rc.ctypes.data)
    return int(status), rc[:V].copy()


def oracle_find_rc_vertices(toc, table, vtoc, vdata):
    return _rc(oracle_lib().orc_find_rc_vertices, toc, table, vtoc, vdata)


def ref_find_rc_vertices(toc, table, vtoc, vdata):
    return _rc(ref_lib().ref_find_rc_vertices, toc, table, vtoc, vdata)


def ref_open_vector40(path):
    """(count, values uint64[count]) of a MemoryMapped::Vector<Uint40> file, opened by the reference's own code."""
    lib = ref_lib()
    f = lib.ref_open_vector40
    f.restype = C.c_int
    f.argtypes = [C.c_char_p, C.POINTER(C.c_uint64), C.POINTER(C.c_void_p)]
    n, p = C.c_uint64(), C.c_void_p()
    if f(path.encode(), C.byref(n), C.byref(p)):
        raise RuntimeError(f"the reference could not open {path}")
    return n.value, _take(lib.ref_free_markergraph, p, n.value)


def _cutoff(f, y, min_area_fraction, start_index):
    y = np.ascontiguousarray(y, np.uint64)
    cutoff, observed = C.c_uint64(0), C.c_double(0)
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_uint64, C.c_double, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double)]
    threw = f(y.ctypes.data, len(y), float(min_area_fraction), int(start_index), C.byref(cutoff), C.byref(observed))
    return int(threw), int(cutoff.value), float(observed.value)


def oracle_peak_finder_cutoff(y, min_area_fraction=0.08, start_index=2):
    """(threw, cutoff, observedPercentArea) of the restated PeakFinder."""
    return _cutoff(oracle_lib().orc_peak_finder_cutoff, y, min_area_fraction, start_index)


def ref_peak_finder_cutoff(y, min_area_fraction=0.08, start_index=2):
    """(threw, cutoff, observedPercentArea) of the reference's PeakFinder (not for an empty histogram: undefined there)."""
    return _cutoff(ref_lib().ref_peak_finder_cutoff, y, min_area_fraction, start_index)


def canonical(table, vtoc, vdata):
    """Vertices sorted by first marker; the table mapped through each vertex's first marker (2^40-1 stays). Returns
    (table of first markers or 2^40-1, vtoc, vdata, order) where order[v] = the canonical index of vertex v."""
    vtoc = np.asarray(vtoc, np.int64)
    vdata = np.asarray(vdata, np.uint64)
    V = len(vtoc) - 1
    first = vdata[vtoc[:-1]] if V else np.zeros(0, np.uint64)
    order_new = np.argsort(first, kind="stable")
    rank = np.empty(V, np.int64)
    rank[order_new] = np.arange(V)
    sizes = np.diff(vtoc)[order_new]
    ntoc = np.zeros(V + 1, np.uint64)
    ntoc[1:] = np.cumsum(sizes)
    parts = [vdata[vtoc[v]:vtoc[v + 1]] for v in order_new]
    ndata = np.concatenate(parts) if parts else np.zeros(0, np.uint64)
    table = np.asarray(table, np.uint64)
    inv = np.uint64((1 << 40) - 1)
    valid = table != inv
    ct = np.full(len(table), inv, np.uint64)
    ct[valid] = first[table[valid].astype(np.int64)]
    return ct, ntoc, ndata, rank
