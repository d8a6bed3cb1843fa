"""TEST INFRASTRUCTURE — flagCrossStrandReadGraphEdges1 and flagChimericReads (src/AssemblerReadGraph.cpp:355-583, 775-1041):
a plain restatement in Python (breadth-first searches over the read graph, the regions processed with a STABLE sort) and,
when present, the reference's own ReadGraph behind ref_glue/ref_readgraph_flags.cpp in
oracle/_ref/libshasta_ref_readgraph_flags.so (built by oracle/Makefile).

The restatement of the region step equals the reference whenever no two edge pairs of a region tie on markerCount (the
reference's two std::sort calls are unstable); region_ties() says whether an input has such a tie. Everything else is a
property of sets and is exact.

Only tests/ and bench_readgraph_flags.py may import this module. The product (shasta_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os
from collections import deque

import numpy as np

from oracle._load import have, load

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "_ref", "libshasta_ref_readgraph_flags.so")
CROSS = np.uint32(1 << 30)          # crossesStrands: bit 62 of the second 64-bit word = bit 30 of word 3

_REF_PROTOS = {
    "ref_flag_cross_strand_read_graph_edges1": (C.c_int, [C.c_int64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
                                                          C.c_void_p, C.c_uint64, C.c_void_p]),
    "ref_flag_chimeric_reads": (C.c_int, [C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                          C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]),
    "ref_open_read_graph_edges": (C.c_int, [C.c_char_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
}


def have_ref():
    return have(REF_SO)


def ref_lib():
    return load(REF_SO, _REF_PROTOS)


def _inputs(g):
    return (np.array(g["edges"], np.uint32, copy=True).reshape(-1, 4), np.ascontiguousarray(g["toc"], np.uint32),
            np.ascontiguousarray(g["data"], np.uint32), np.array(g["records"], np.uint32, copy=True).reshape(-1, 16),
            np.array(g["flags"], np.uint8, copy=True))


def ref_cross_strand(g, max_distance, threads=1):
    """dict(status, edges, records, reported, regions, flagged) from the reference's code."""
    edges, toc, data, rec, _ = _inputs(g)
    counts = np.zeros(3, np.uint64)
    st = ref_lib().ref_flag_cross_strand_read_graph_edges1(int(max_distance), edges.ctypes.data, len(edges), toc.ctypes.data,
                                                           data.ctypes.data, (len(toc) - 1) // 2, rec.ctypes.data, threads,
                                                           counts.ctypes.data)
    if st:
        return dict(status=int(st))
    return dict(status=0, edges=edges, records=rec, reported=int(counts[0]), regions=int(counts[1]), flagged=int(counts[2]))


def ref_chimeric(g, max_distance, threads=1):
    """dict(status, flags, records, chimeric) from the reference's code."""
    edges, toc, data, rec, flags = _inputs(g)
    n = np.zeros(1, np.uint64)
    st = ref_lib().ref_flag_chimeric_reads(int(max_distance), edges.ctypes.data, len(edges), toc.ctypes.data, data.ctypes.data,
                                           (len(toc) - 1) // 2, flags.ctypes.data, rec.ctypes.data, len(rec), threads, n.ctypes.data)
    if st:
        return dict(status=int(st))
    return dict(status=0, flags=flags, records=rec, chimeric=int(n[0]))


def ref_open_read_graph_edges(path, capacity):
    """uint32[n, 4] of a Data/ReadGraphEdges file, opened by the reference's MemoryMapped::Vector<ReadGraphEdge>."""
    out = np.zeros((capacity, 4), np.uint32)
    n = C.c_uint64()
    if ref_lib().ref_open_read_graph_edges(path.encode(), out.ctypes.data, capacity, C.byref(n)):
        raise RuntimeError(f"the reference could not open {path}")
    return out[:min(n.value, capacity)], n.value


# ---- the restatement ---------------------------------------------------------------------------------------------------

def _rows(g):
    toc, data = np.asarray(g["toc"]), np.asarray(g["data"])
    return [data[toc[v]:toc[v + 1]].tolist() for v in range(len(toc) - 1)]


def _ball(rows, ends, cross, start, d, skip_cross):
    """{vertex: distance} for every vertex within distance d of start."""
    dist = {start: 0}
    q = deque([start])
    while q:
        v = q.popleft()
        if dist[v] >= d:
            continue
        for e in rows[v]:
            if skip_cross and cross[e]:
                continue
            a, b = ends[e]
            u = b if a == v else a
            if u not in dist:
                dist[u] = dist[v] + 1
                q.append(u)
    return dist


class _UF:
    def __init__(self):
        self.p = {}

    def find(self, x):
        self.p.setdefault(x, x)
        while self.p[x] != x:
            self.p[x] = self.p[self.p[x]]
            x = self.p[x]
        return x

    def union(self, a, b):
        a, b = self.find(a), self.find(b)
        if a != b:
            self.p[max(a, b)] = min(a, b)


def _alignment_id(w):
    return int(w[2]) | ((int(w[3]) & 0x3FFFFFFF) << 32)


def near_reads(g, max_distance):
    edges = np.asarray(g["edges"]).reshape(-1, 4)
    rows = _rows(g)
    ends = [(int(a), int(b)) for a, b in edges[:, :2]]
    R = len(rows) // 2
    return [max_distance > 0 and (2 * x + 1) in _ball(rows, ends, None, 2 * x, max_distance, False) for x in range(R)]


def _regions(g, near):
    edges = np.asarray(g["edges"]).reshape(-1, 4)
    uf = _UF()
    for a, b in edges[:, :2].tolist():
        if near[a >> 1] and near[b >> 1]:
            uf.union(a, b)
    groups = {}
    for v in range(2 * len(near)):
        if near[v >> 1]:
            groups.setdefault(uf.find(v), []).append(v)
    return [vs for vs in groups.values() if len(vs) >= 2]


def _region_pairs(g, vertices):
    """The region's edge pairs in gathering order (None when a reference assertion trips on the way)."""
    edges = np.asarray(g["edges"]).reshape(-1, 4)
    rows = _rows(g)
    vs = set(vertices)
    if len(vertices) % 2 or any(vertices[i] >> 1 != vertices[i + 1] >> 1 or vertices[i] & 1 or not vertices[i + 1] & 1
                                for i in range(0, len(vertices), 2)):
        return None
    ids = []
    for v0 in vertices:
        for e in rows[v0]:
            a, b = int(edges[e, 0]), int(edges[e, 1])
            if (b if a == v0 else a) in vs and a == v0:
                ids.append((e, _alignment_id(edges[e])))
    if len(ids) % 2:
        return None
    ids.sort(key=lambda p: p[1])
    if any(ids[i][1] != ids[i + 1][1] for i in range(0, len(ids), 2)):
        return None
    return [(ids[i][0], ids[i + 1][0], ids[i][1]) for i in range(0, len(ids), 2)]


def region_ties(g, max_distance):
    """True when two edge pairs of one strand jump region have the same markerCount (where only the reference decides)."""
    rec = np.asarray(g["records"]).reshape(-1, 16)
    for vertices in _regions(g, near_reads(g, max_distance)):
        pairs = _region_pairs(g, vertices) or []
        counts = [int(rec[a, 9]) for _, _, a in pairs]
        if len(counts) != len(set(counts)):
            return True
    return False


def py_cross_strand(g, max_distance):
    edges, _, _, rec, _ = _inputs(g)
    if max_distance < 0:
        return dict(status=1)
    edges[:, 3] &= ~CROSS
    if max_distance == 0:
        return dict(status=0, edges=edges, records=rec, reported=0, regions=0, flagged=0)
    near = near_reads(g, max_distance)
    R = len(near)
    reported = sum(1 for v in range(R) if near[v >> 1])
    regions = _regions(g, near)
    flagged = []
    for vertices in regions:
        pairs = _region_pairs(g, vertices)
        if pairs is None:
            return dict(status=1)
        pairs = sorted(pairs, key=lambda p: -int(rec[p[2], 9]))       # stable
        uf = _UF()
        for e0, e1, _ in pairs:
            for e in (e0, e1):
                a, b = int(edges[e, 0]), int(edges[e, 1])
                c0, c1, c0rc, c1rc = uf.find(a), uf.find(b), uf.find(a ^ 1), uf.find(b ^ 1)
                if c0 == c0rc or c1 == c1rc:
                    return dict(status=1)
                if c0 == c1rc or c1 == c0rc:
                    flagged.append(e)
                else:
                    uf.union(a, b)
                    uf.union(a ^ 1, b ^ 1)
    for e in flagged:
        edges[e, 3] |= CROSS
        rec[_alignment_id(edges[e]), 15] &= ~np.uint32(1)
    return dict(status=0, edges=edges, records=rec, reported=reported, regions=len(regions), flagged=len(flagged))


def py_chimeric(g, max_distance):
    edges, _, _, rec, flags = _inputs(g)
    if max_distance >= 255:
        return dict(status=1)
    rows = _rows(g)
    R = len(rows) // 2
    flags &= ~np.uint8(2)
    if max_distance == 0:
        return dict(status=0, flags=flags, records=rec, chimeric=0)
    ends = [(int(a), int(b)) for a, b in edges[:, :2]]
    cross = ((edges[:, 3] & CROSS) != 0).tolist()
    chim = np.zeros(R, bool)
    for x in range(R):
        dist = _ball(rows, ends, cross, 2 * x, max_distance, True)
        uf = _UF()
        for v in dist:
            if v >> 1 == x:
                continue
            for e in rows[v]:
                if cross[e]:
                    continue
                a, b = ends[e]
                u = b if a == v else a
                if u >> 1 != x and u in dist:
                    uf.union(v, u)
        roots = {uf.find(v) for v, d in dist.items() if d == max_distance and v >> 1 != x}
        chim[x] = len(roots) >= 2
    flags[chim] |= np.uint8(2)
    if chim.any():
        hit = chim[rec[:, 0]] | chim[rec[:, 1]]
        rec[hit, 15] &= ~np.uint32(1)
    return dict(status=0, flags=flags, records=rec, chimeric=int(chim.sum()))
