"""Inputs of the createMarkerGraphEdges tests (tests/test_oracle_markergraph_edges.py, tests/test_gpu_markergraph_edges.py):
marker graph vertices, each as (toc, table uint64[M], vtoc uint64[V+1], vdata uint64[], rc uint64[V]). The vertices of every
createMarkerGraphVertices case and parameter set come from the vertex restatement; the others are built here from groups of
markers closed under reverse complement, from fixed seeds."""
import hashlib

import numpy as np

from oracle import markergraph_bindings as MB
from oracle import markergraph_edges_bindings as EB

from markergraph_inputs import PARAMS, cases

INV40 = (1 << 40) - 1


def _toc(lengths):
    toc = np.zeros(2 * len(lengths) + 1, np.uint64)
    toc[1:] = np.cumsum(np.repeat(np.asarray(lengths, np.int64), 2))
    return toc


def _rc_marker(toc, m):
    o = int(np.searchsorted(toc, m, side="right")) - 1
    return int(toc[o ^ 1]) + int(toc[o + 1] - toc[o]) - 1 - (m - int(toc[o]))


def from_groups(toc, groups):
    """Vertices from groups of marker ids: each group and its reverse complement (once when they are equal), numbered by
    first marker. A marker in two groups stays in the first."""
    M = int(toc[-1])
    table = np.full(M, INV40, np.uint64)
    sets = []
    for g in groups:
        g = sorted(set(int(m) for m in g if table[int(m)] == INV40))
        if not g:
            continue
        r = sorted(_rc_marker(toc, m) for m in g)
        if any(table[m] != INV40 for m in r) and r != g:
            continue
        for s in ([g] if r == g else [g, r]):
            for m in s:
                table[m] = len(sets)
            sets.append(s)
    order = sorted(range(len(sets)), key=lambda k: sets[k][0])
    rank = {k: i for i, k in enumerate(order)}
    sets = [sets[k] for k in order]
    table = np.array([INV40 if t == INV40 else rank[int(t)] for t in table.tolist()], np.uint64)
    vtoc = np.zeros(len(sets) + 1, np.uint64)
    vtoc[1:] = np.cumsum([len(s) for s in sets])
    vdata = np.array([m for s in sets for m in s], np.uint64)
    rc = np.array([table[_rc_marker(toc, s[0])] for s in sets], np.uint64)
    return dict(toc=toc, table=table, vtoc=vtoc, vdata=vdata, rc=rc)


def permuted(d, seed):
    """The same vertices under a random numbering, as the reference's schedule-dependent numbering gives them."""
    rng = np.random.default_rng(seed)
    V = len(d["vtoc"]) - 1
    perm = rng.permutation(V)                       # new id of old vertex v
    inv = np.argsort(perm)
    sizes = np.diff(d["vtoc"].astype(np.int64))[inv]
    vtoc = np.zeros(V + 1, np.uint64)
    vtoc[1:] = np.cumsum(sizes)
    vdata = np.concatenate([d["vdata"][d["vtoc"][v]:d["vtoc"][v + 1]] for v in inv]) if V else np.zeros(0, np.uint64)
    table = np.asarray(d["table"], np.uint64).copy()
    valid = table != INV40
    table[valid] = perm[table[valid].astype(np.int64)]
    rc = perm[np.asarray(d["rc"], np.int64)[inv]].astype(np.uint64)
    return dict(toc=d["toc"], table=table, vtoc=vtoc, vdata=vdata.astype(np.uint64), rc=rc)


def vertex_cases():
    out = {}
    for name, d in cases().items():
        for pname, p in PARAMS.items():
            o = MB.oracle_create_marker_graph_vertices(d["toc"], d["kmer"], d["edges"], d["ctoc"], d["cdata"], d["flags"], **p)
            st, rc = MB.oracle_find_rc_vertices(d["toc"], o["table"], o["vtoc"], o["vdata"])
            if st:                               # duplicate markers can leave a set without a consistent reverse complement
                rc = None
            out[f"{name}/{pname}"] = dict(toc=d["toc"], table=o["table"], vtoc=o["vtoc"], vdata=o["vdata"], rc=rc)
    rng = np.random.default_rng(21)
    # Two markers of one oriented read in one vertex (allowDuplicateMarkers): self-loops v -> v.
    toc = _toc([12] * 20)
    groups = [[int(toc[2 * r]) + a for r in range(20)] + [int(toc[2 * r]) + a + 1 for r in range(0, 20, 3)] for a in range(0, 11, 2)]
    out["duplicates"] = from_groups(toc, groups)
    # One vertex pair joined by 300 intervals: coverage 255.
    toc = _toc([4] * 300)
    out["coverage_cap"] = from_groups(toc, [[int(toc[2 * r]) + a for r in range(300)] for a in range(2)])
    # Reads with vertices only at their ends, about 30000 markers apart.
    toc = _toc([30000, 30001, 29999, 50])
    ends = [[int(toc[2 * r]) for r in range(4)], [int(toc[2 * r + 1]) - 1 for r in range(3)], [int(toc[6]) + 20]]
    out["long_gap"] = from_groups(toc, ends)
    # Reads with no vertex marker or with one.
    lengths = rng.integers(0, 40, 200).tolist()
    toc = _toc(lengths)
    groups = []
    for _ in range(150):
        rs = rng.choice(200, int(rng.integers(1, 6)), replace=False)
        g = [int(toc[2 * r]) + int(rng.integers(lengths[r])) for r in rs if lengths[r] and r % 4]
        groups.append(g)
    groups += [[int(toc[2 * r]) + lengths[r] // 2] for r in range(3, 200, 4) if lengths[r]]       # one vertex marker per read
    out["sparse"] = from_groups(toc, groups)
    out["zero"] = from_groups(_toc([5, 7, 3]), [])
    out["permuted"] = permuted(out["genome/cov2"], 3)
    out["permuted_deep"] = permuted(out["deep/strand1"], 4)
    return out


def large_vertex_case(reads=4400, length=6):
    """Vertices of more than 32 and more than 4096 markers: ordinal a of every read forms one vertex."""
    toc = _toc([length] * reads)
    groups = [[int(toc[2 * r]) + a for r in range(reads if a % 2 else 40 + 30 * a)] for a in range(length)]
    return from_groups(toc, groups)


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def parallel_edge(s, e):
    """Edge e duplicated at the end of the edge list, with its intervals, and listed in its source's row: parallel edges."""
    s = {k: np.array(v) for k, v in s.items() if isinstance(v, np.ndarray)}
    E = len(s["edges"])
    itoc = s["intervalsToc"].astype(np.int64)
    s["edges"] = np.concatenate([s["edges"], s["edges"][e:e + 1]])
    s["intervalsData"] = np.concatenate([s["intervalsData"], s["intervalsData"][itoc[e]:itoc[e + 1]]])
    s["intervalsToc"] = np.append(s["intervalsToc"], s["intervalsToc"][-1] + (itoc[e + 1] - itoc[e])).astype(np.uint64)
    src = int(EB.named_fields(s["edges"][e:e + 1])[0, 0])
    stoc = s["bySourceToc"].astype(np.int64)
    data = list(s["bySourceData"].tolist())
    data.insert(stoc[src], E)                            # the new id first: rows are in decreasing edge id
    s["bySourceData"] = np.array(data, np.uint64)
    s["bySourceToc"][src + 1:] += 1
    return s


def drop_interval(s, e):
    """Edge e without its last interval."""
    s = {k: np.array(v) for k, v in s.items() if isinstance(v, np.ndarray)}
    itoc = s["intervalsToc"].astype(np.int64)
    s["intervalsData"] = np.delete(s["intervalsData"], itoc[e + 1] - 1, axis=0)
    s["intervalsToc"][e + 1:] -= 1
    return s


def rc_failure_inputs(d):
    """(name, vertices d, edge set) for the two failures the reference reports, on the edges of the vertices d."""
    o = EB.oracle_create_marker_graph_edges(d["toc"], d["table"], d["vtoc"], d["vdata"])
    cov = np.diff(o["intervalsToc"].astype(np.int64))
    e = int(np.nonzero(cov >= 2)[0][3])
    return [("missing_interval", d, drop_interval(o, e)), ("parallel", d, parallel_edge(o, e))]
