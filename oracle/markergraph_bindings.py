"""TEST INFRASTRUCTURE — ctypes bindings for createMarkerGraphVertices / findMarkerGraphReverseComplementVertices
(src/AssemblerMarkerGraph.cpp): the C restatement in oracle/markergraph_oracle.c (part of oracle/_build/liboracle.so) and,
when present, the reference's own DisjointSets, decompress and PeakFinder behind ref_glue/ref_markergraph.cpp in
oracle/_ref/libshasta_ref_markergraph.so (built by oracle/Makefile).

Only tests/ and bench_markergraph.py may import this module. The product (shasta_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import bindings
from oracle._load import have, load, take

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "_ref", "libshasta_ref_markergraph.so")

DEFAULTS = dict(minCoverage=10, maxCoverage=100, minCoveragePerStrand=0, allowDuplicateMarkers=False,
                peakFinderMinAreaFraction=0.08, peakFinderAreaStartIndex=2)


_VERTICES = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
             C.c_void_p, C.c_double] + [C.POINTER(C.c_void_p)] * 4 + [C.c_void_p]
_RC = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
_CUTOFF = [C.c_void_p, C.c_uint64, C.c_double, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double)]
_ORACLE_PROTOS = {
    "orc_create_marker_graph_vertices": (C.c_int, _VERTICES),
    "orc_find_rc_vertices": (C.c_int, _RC),
    "orc_peak_finder_cutoff": (C.c_int, _CUTOFF),
}
_REF_PROTOS = {
    "ref_create_marker_graph_vertices": (C.c_int, _VERTICES),
    "ref_find_rc_vertices": (C.c_int, _RC),
    "ref_peak_finder_cutoff": (C.c_int, _CUTOFF),
    "ref_open_vector40": (C.c_int, [C.c_char_p, C.POINTER(C.c_uint64), C.POINTER(C.c_void_p)]),
    "ref_free_markergraph": (None, [C.c_void_p]),
}


def oracle_lib():
    return bindings.oracle_lib(_ORACLE_PROTOS)


def have_ref():
    return have(REF_SO)


def ref_lib():
    return load(REF_SO, _REF_PROTOS)


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
    status = f(toc.ctypes.data, R, kmer.ctypes.data, edges.ctypes.data, len(edges), ctoc.ctypes.data, cdata.ctypes.data,
               len(ctoc) - 1, flags.ctypes.data, pv.ctypes.data, float(d["peakFinderMinAreaFraction"]), C.byref(t), C.byref(vt),
               C.byref(vd), C.byref(h), counts.ctypes.data)
    if status:
        return dict(status=int(status))
    M, V = int(toc[-1]), int(counts[8])
    return dict(status=0, table=take(t, M, np.uint64, lib_free), vtoc=take(vt, V + 1, np.uint64, lib_free),
                vdata=take(vd, int(counts[10]), np.uint64, lib_free), histogram=take(h, int(counts[9]), np.uint64, lib_free),
                minCoverageUsed=int(counts[0]), peakFinderFailed=int(counts[1]),
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
    status = f(toc.ctypes.data, (len(toc) - 1) // 2, table.ctypes.data, vtoc.ctypes.data, vdata.ctypes.data, V, rc.ctypes.data)
    return int(status), rc[:V].copy()


def oracle_find_rc_vertices(toc, table, vtoc, vdata):
    return _rc(oracle_lib().orc_find_rc_vertices, toc, table, vtoc, vdata)


def ref_find_rc_vertices(toc, table, vtoc, vdata):
    return _rc(ref_lib().ref_find_rc_vertices, toc, table, vtoc, vdata)


def ref_open_vector40(path):
    """(count, values uint64[count]) of a MemoryMapped::Vector<Uint40> file, opened by the reference's own code."""
    lib = ref_lib()
    n, p = C.c_uint64(), C.c_void_p()
    if lib.ref_open_vector40(path.encode(), C.byref(n), C.byref(p)):
        raise RuntimeError(f"the reference could not open {path}")
    return n.value, take(p, n.value, np.uint64, lib.ref_free_markergraph)


def _cutoff(f, y, min_area_fraction, start_index):
    y = np.ascontiguousarray(y, np.uint64)
    cutoff, observed = C.c_uint64(0), C.c_double(0)
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
