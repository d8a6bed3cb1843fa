"""TEST INFRASTRUCTURE — ctypes bindings for createMarkerGraphEdges / findMarkerGraphReverseComplementEdges
(src/AssemblerMarkerGraph.cpp): the C restatement in oracle/markergraph_edges_oracle.c (part of oracle/_build/liboracle.so)
and, when present, the reference's own MarkerGraph, MultithreadedObject and MemoryMapped containers behind
ref_glue/ref_markergraph_edges.cpp in oracle/_ref/libshasta_ref_markergraph_edges.so (built by oracle/Makefile).

Edge sets are dicts: edges uint8[E,14], intervalsToc uint64[E+1], intervalsData uint32[I,3], bySourceToc / byTargetToc
uint64[V+1], bySourceData / byTargetData uint64[E]. Only tests/ and bench_markergraph_edges.py import this module.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import bindings
from oracle._load import have, load, take

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "_ref", "libshasta_ref_markergraph_edges.so")
INV40 = (1 << 40) - 1

_EDGES = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
_RC_EDGES = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64] + [C.c_void_p] * 4
_ORACLE_PROTOS = {
    "orc_create_marker_graph_edges": (C.c_int, _EDGES + [C.POINTER(C.c_void_p)] * 7 + [C.c_void_p]),
    "orc_find_rc_edges": (C.c_int, _RC_EDGES + [C.c_void_p] * 2),
}
_REF_PROTOS = {
    "ref_create_marker_graph_edges": (C.c_int, _EDGES + [C.c_uint64] + [C.POINTER(C.c_void_p)] * 7 + [C.c_void_p]),
    "ref_find_rc_edges": (C.c_int, _RC_EDGES + [C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64]),
    "ref_open_marker_graph_edges": (C.c_int, [C.c_char_p] * 5 + [C.POINTER(C.c_void_p)] * 8 + [C.c_void_p]),
    "ref_free_markergraph_edges": (None, [C.c_void_p]),
}


def oracle_lib():
    return bindings.oracle_lib(_ORACLE_PROTOS)


def have_ref():
    return have(REF_SO)


def ref_lib():
    return load(REF_SO, _REF_PROTOS)


def _edge_set(free, ptrs, E, I, V):
    return dict(edges=take(ptrs[0], 14 * E, np.uint8, free).reshape(-1, 14), intervalsToc=take(ptrs[1], E + 1, np.uint64, free),
                intervalsData=take(ptrs[2], 3 * I, np.uint32, free).reshape(-1, 3), bySourceToc=take(ptrs[3], V + 1, np.uint64, free),
                bySourceData=take(ptrs[4], E, np.uint64, free), byTargetToc=take(ptrs[5], V + 1, np.uint64, free),
                byTargetData=take(ptrs[6], E, np.uint64, free))


def _u64(a):
    return np.ascontiguousarray(a, np.uint64)


def oracle_create_marker_graph_edges(toc, table, vtoc, vdata):
    """The C restatement (one thread's output). table, vtoc: uint64. Returns dict(status, the edge set, saturated)."""
    lib = oracle_lib()
    toc, table, vtoc, vdata = _u64(toc), _u64(table), _u64(vtoc), _u64(vdata)
    V = len(vtoc) - 1
    ptrs = [C.c_void_p() for _ in range(7)]
    counts = np.zeros(3, np.uint64)
    status = lib.orc_create_marker_graph_edges(toc.ctypes.data, (len(toc) - 1) // 2, table.ctypes.data, vtoc.ctypes.data,
                                               vdata.ctypes.data, V, *[C.byref(p) for p in ptrs], counts.ctypes.data)
    if status:
        return dict(status=int(status))
    out = _edge_set(lib.orc_free, ptrs, int(counts[0]), int(counts[1]), V)
    out.update(status=0, saturated=int(counts[2]))
    return out


def ref_create_marker_graph_edges(toc, table, vtoc, vdata, threads=1):
    """The reference's objects in the members' control flow. threads=0: all cores."""
    lib = ref_lib()
    toc, table, vtoc, vdata = _u64(toc), _u64(table), _u64(vtoc), _u64(vdata)
    V = len(vtoc) - 1
    ptrs = [C.c_void_p() for _ in range(7)]
    counts = np.zeros(2, np.uint64)
    status = lib.ref_create_marker_graph_edges(toc.ctypes.data, (len(toc) - 1) // 2, table.ctypes.data, vtoc.ctypes.data,
                                               vdata.ctypes.data, V, threads, *[C.byref(p) for p in ptrs], counts.ctypes.data)
    if status:
        return dict(status=int(status))
    out = _edge_set(lib.ref_free_markergraph_edges, ptrs, int(counts[0]), int(counts[1]), V)
    out.update(status=0)
    return out


_RC_MESSAGES = {1: "Unable to locate reverse complement of marker graph edge {0} {1}->{2}",
                2: "Reverse complement edge check failed at edge {0}: {1} {2}",
                3: "Assertion failed: edgeRc.source == v1Rc"}


def oracle_find_rc_edges(toc, rc_vertex, s):
    """(message or None, rc uint64[E]) of the C restatement on edge set s. The messages are the reference's (the assertion's
    without its location)."""
    f = oracle_lib().orc_find_rc_edges
    toc, rv = _u64(toc), _u64(rc_vertex)
    e = np.ascontiguousarray(s["edges"], np.uint8)
    E = len(e)
    rc = np.zeros(E + 1, np.uint64)
    info = np.zeros(3, np.uint64)
    iv = np.ascontiguousarray(s["intervalsData"], np.uint32)
    status = f(toc.ctypes.data, (len(toc) - 1) // 2, rv.ctypes.data, len(rv), e.ctypes.data, E, _u64(s["intervalsToc"]).ctypes.data,
               iv.ctypes.data, _u64(s["bySourceToc"]).ctypes.data, _u64(s["bySourceData"]).ctypes.data, rc.ctypes.data, info.ctypes.data)
    if status:
        return _RC_MESSAGES[status].format(*info.tolist()), None
    return None, rc[:E]


def ref_find_rc_edges(toc, rc_vertex, s, threads=1):
    """(message or None, rc uint64[E]) of the reference's member on edge set s."""
    f = ref_lib().ref_find_rc_edges
    toc, rv = _u64(toc), _u64(rc_vertex)
    e = np.ascontiguousarray(s["edges"], np.uint8)
    E = len(e)
    rc = np.zeros(E + 1, np.uint64)
    msg = C.create_string_buffer(1024)
    iv = np.ascontiguousarray(s["intervalsData"], np.uint32)
    status = f(toc.ctypes.data, (len(toc) - 1) // 2, rv.ctypes.data, len(rv), e.ctypes.data, E, _u64(s["intervalsToc"]).ctypes.data,
               iv.ctypes.data, _u64(s["bySourceToc"]).ctypes.data, _u64(s["bySourceData"]).ctypes.data, threads, rc.ctypes.data, msg, 1024)
    if status:
        return msg.value.decode(), None
    return None, rc[:E]


def ref_open_marker_graph_edges(prefix, with_rc=True):
    """The five file sets the facade writes under prefix (Data/), opened by the reference's own MemoryMapped code."""
    lib = ref_lib()
    ptrs = [C.c_void_p() for _ in range(8)]
    counts = np.zeros(4, np.uint64)
    names = [prefix + n for n in ("GlobalMarkerGraphEdges", "GlobalMarkerGraphEdgeMarkerIntervals", "GlobalMarkerGraphEdgesBySource",
                                  "GlobalMarkerGraphEdgesByTarget")]
    rc_path = (prefix + "MarkerGraphReverseComplementeEdge").encode() if with_rc else None
    if lib.ref_open_marker_graph_edges(*[n.encode() for n in names], rc_path, *[C.byref(p) for p in ptrs], counts.ctypes.data):
        raise RuntimeError(f"the reference could not open the marker graph edges under {prefix}")
    E, I, V = int(counts[0]), int(counts[1]), int(counts[2])
    assert int(counts[3]) == V
    out = _edge_set(lib.ref_free_markergraph_edges, ptrs[:7], E, I, V)
    if with_rc:
        out["rc"] = take(ptrs[7], E, np.uint64, lib.ref_free_markergraph_edges)
    return out


def named_fields(edges):
    """uint64[E,10]: bytes 0-10 of each Edge and its named flag bits (wasRemovedByTransitiveReduction ... wasAssembled, isSecondary,
    wasRemovedWhileSplittingSecondaryEdges, flag6); the other bits of bytes 11 and 13 are never set by the members."""
    e = np.asarray(edges, np.uint8).reshape(-1, 14).astype(np.uint64)
    src = sum(e[:, k] << np.uint64(8 * k) for k in range(5))
    tgt = sum(e[:, 5 + k] << np.uint64(8 * k) for k in range(5))
    cols = [src, tgt, e[:, 10], e[:, 11] & np.uint64(0x1f), e[:, 12], e[:, 13] & np.uint64(3)]
    return np.stack(cols, 1) if len(e) else np.zeros((0, 6), np.uint64)


def rows_from_uint40(data):
    b = np.asarray(data, np.uint8).reshape(-1, 5)
    out = np.zeros((len(b), 8), np.uint8)
    out[:, :5] = b
    return out.view(np.uint64).reshape(-1)


def canonical(s, rc=None):
    """Edge set s renumbered in increasing (source, target) order (ties, from parallel edges, by intervals), rows as sorted
    sets, rc renumbered through the same permutation. Returns (fields uint64[E,6], itoc, idata, stoc, sorted sdata, ttoc,
    sorted tdata, rc or None)."""
    f = named_fields(s["edges"])
    itoc = np.asarray(s["intervalsToc"], np.int64)
    idata = np.asarray(s["intervalsData"], np.uint32).reshape(-1, 3)
    E = len(f)
    order = np.lexsort((f[:, 1], f[:, 0])) if E else np.zeros(0, np.int64)
    if E and not (np.diff(f[order, 0].astype(np.int64)) | np.diff(f[order, 1].astype(np.int64))).all():
        keys = [tuple(f[e, :2].tolist()) + tuple(idata[itoc[e]:itoc[e + 1]].reshape(-1).tolist()) for e in range(E)]
        order = np.array(sorted(range(E), key=lambda e: keys[e]), np.int64)
    rank = np.empty(E, np.int64)
    rank[order] = np.arange(E)
    sizes = np.diff(itoc)[order] if E else np.zeros(0, np.int64)
    ntoc = np.zeros(E + 1, np.int64)
    ntoc[1:] = np.cumsum(sizes)
    gather = np.repeat(itoc[:-1][order] - ntoc[:-1], sizes) + np.arange(ntoc[-1]) if E else np.zeros(0, np.int64)
    nd = idata[gather]

    def rows(toc, data):
        toc = np.asarray(toc, np.int64)
        d = rank[np.asarray(data, np.int64)] if E else np.zeros(0, np.int64)
        row = np.repeat(np.arange(len(toc) - 1), np.diff(toc))
        return toc.astype(np.uint64), d[np.lexsort((d, row))]

    stoc, sd = rows(s["bySourceToc"], s["bySourceData"])
    ttoc, td = rows(s["byTargetToc"], s["byTargetData"])
    nrc = None
    if rc is not None:
        nrc = np.empty(E, np.int64)
        nrc[rank] = rank[np.asarray(rc, np.int64)]
    return f[order], ntoc.astype(np.uint64), nd.reshape(-1, 3), stoc, sd, ttoc, td, nrc
