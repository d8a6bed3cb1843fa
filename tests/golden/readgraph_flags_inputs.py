"""Read graphs for the flagCrossStrandReadGraphEdges1 / flagChimericReads tests, built directly as (edges, connectivity,
AlignmentData, ReadFlags) from fixed seeds. Every alignment (r0 < r1) becomes an edge and its reverse complement, edges
2i and 2i+1, as createReadGraph writes them; each connectivity row lists its edges in decreasing index."""
import numpy as np


def build(R, alignments, seed=0, cross_fraction=0.0):
    """alignments: list of (r0, r1, sameStrand, markerCount) with r0 < r1 (any order)."""
    rng = np.random.default_rng(seed)
    n = len(alignments)
    rec = np.zeros((n, 16), np.uint32)
    edges = np.zeros((2 * n, 4), np.uint32)
    for i, (r0, r1, same, mc) in enumerate(alignments):
        rec[i, 0], rec[i, 1], rec[i, 2], rec[i, 9] = r0, r1, 1 if same else 0, mc
        rec[i, 15] = 1 | (int(rng.integers(0, 1 << 8)) << 8)        # isInReadGraph, and other bytes that must survive
        o0, o1 = 2 * r0, 2 * r1 + (0 if same else 1)
        edges[2 * i] = (o0, o1, i, 0)
        edges[2 * i + 1] = (o0 ^ 1, o1 ^ 1, i, 0)
    if cross_fraction:
        edges[rng.random(2 * n) < cross_fraction, 3] |= np.uint32(1 << 30)
    rows = [[] for _ in range(2 * R)]
    for e in range(2 * n - 1, -1, -1):
        rows[edges[e, 0]].append(e)
        rows[edges[e, 1]].append(e)
    toc = np.zeros(2 * R + 1, np.uint32)
    toc[1:] = np.cumsum([len(r) for r in rows])
    data = np.array([e for r in rows for e in r], np.uint32)
    flags = rng.integers(0, 256, R).astype(np.uint8)
    return dict(edges=edges, toc=toc, data=data, records=rec, flags=flags)


def _chain(reads, rng, reach=3, same=True, mc=(50, 500)):
    out = []
    for i, r in enumerate(reads):
        for j in range(1, reach + 1):
            if i + j < len(reads):
                a, b = sorted((r, reads[i + j]))
                out.append((a, b, same, int(rng.integers(*mc))))
    return out


def random_graph(R, n, seed, mc=(1, 1000)):
    rng = np.random.default_rng(seed)
    al = set()
    while len(al) < n:
        a, b = sorted(int(x) for x in rng.integers(0, R, 2))
        if a != b:
            al.add((a, b, bool(rng.integers(0, 2))))
    return build(R, [(a, b, s, int(rng.integers(*mc))) for a, b, s in sorted(al)], seed)


def strand_jump(R, jumps, seed, reach=3, mc=(50, 500)):
    """A chain of reads 0..R-1 on one strand; each jump (i, j) adds an opposite-strand alignment between reads i and j."""
    rng = np.random.default_rng(seed)
    al = _chain(list(range(R)), rng, reach, True, mc)
    al += [(min(i, j), max(i, j), False, int(rng.integers(*mc))) for i, j in jumps]
    return build(R, al, seed)


def bridged(R, seed, bridge=None, reach=2):
    """Two chains, reads [0, R/2) and [R/2, R), joined only through read `bridge` (a chimeric read); bridge None: joined by
    an ordinary overlap of the two chain ends (a near-chimeric control)."""
    rng = np.random.default_rng(seed)
    h = R // 2
    left, right = [r for r in range(h) if r != bridge], [r for r in range(h, R) if r != bridge]
    al = _chain(left, rng, reach) + _chain(right, rng, reach)
    if bridge is None:
        al += [(left[-1], right[0], True, 300), (left[-2], right[0], True, 300), (left[-1], right[1], True, 300)]
    else:
        al += [(min(bridge, r), max(bridge, r), True, 300) for r in (left[-1], left[-2], right[0], right[1])]
    return build(R, al, seed)


def hub(R, seed):
    """Read 0 aligned to every other read, plus a chain: every ball is large."""
    rng = np.random.default_rng(seed)
    al = [(0, r, bool(rng.integers(0, 2)), int(rng.integers(1, 1000))) for r in range(1, R)]
    al += _chain(list(range(1, R)), rng, 1)
    return build(R, sorted(set(al)), seed)


def families():
    """name -> graph."""
    f = {}
    f["empty"] = build(0, [])
    f["isolated"] = build(7, [])
    f["isolated_and_pair"] = build(5, [(1, 3, True, 10)])
    for s in range(3):
        f[f"random{s}"] = random_graph(60, 150, 10 + s)
    f["random_sparse"] = random_graph(200, 180, 20)
    f["one_region"] = strand_jump(40, [(18, 21)], 30)
    f["several_regions"] = strand_jump(120, [(10, 13), (50, 52), (95, 99)], 31)
    f["nested_jumps"] = strand_jump(60, [(20, 30), (23, 27), (24, 26)], 32)
    f["ties"] = strand_jump(60, [(20, 24), (40, 42)], 33, mc=(100, 102))
    f["all_tied"] = strand_jump(40, [(15, 19)], 34, mc=(7, 8))
    f["chimeric"] = bridged(40, 40, bridge=20)
    f["near_chimeric"] = bridged(40, 41)
    f["hub"] = hub(80, 50)
    flagged = random_graph(60, 150, 60)
    flagged_in = build(60, [(int(r[0]), int(r[1]), bool(r[2]), int(r[9])) for r in flagged["records"]], 60, cross_fraction=0.3)
    f["flagged_on_input"] = flagged_in
    f["jump_flagged_on_input"] = build(40, [(int(r[0]), int(r[1]), bool(r[2]), int(r[9]))
                                            for r in strand_jump(40, [(18, 21)], 61)["records"]], 61, cross_fraction=0.2)
    return f


DISTANCES = [0, 1, 2, 6, 7, 254]


def raw(R, ends, seed=0):
    """A read graph from an explicit edge list (o0, o1), edge i on alignment i, with no reverse-complement pairing: inputs
    that trip the reference's region assertions."""
    rng = np.random.default_rng(seed)
    rec = np.zeros((len(ends), 16), np.uint32)
    edges = np.zeros((len(ends), 4), np.uint32)
    for i, (a, b) in enumerate(ends):
        rec[i, 0], rec[i, 1], rec[i, 9], rec[i, 15] = a >> 1, b >> 1, 100 + i, 1
        edges[i] = (a, b, i, 0)
    rows = [[] for _ in range(2 * R)]
    for e in range(len(ends) - 1, -1, -1):
        rows[edges[e, 0]].append(e)
        rows[edges[e, 1]].append(e)
    toc = np.zeros(2 * R + 1, np.uint32)
    toc[1:] = np.cumsum([len(r) for r in rows])
    return dict(edges=edges, toc=toc, data=np.array([e for r in rows for e in r], np.uint32), records=rec,
                flags=rng.integers(0, 256, R).astype(np.uint8))


def bad_graphs():
    """name -> a read graph on which flagCrossStrandReadGraphEdges1(6) trips one of the reference's region assertions."""
    out = {}
    # Reads x = 0, y = 1, z = 2 (oriented reads 0..5). x-0 and x-1 meet through z-0, so x is near a strand jump.
    # odd_region_size: y-0 - y-1 directly; the region {x-0, y-0, y-1} has three vertices.
    out["odd_region_size"] = raw(3, [(0, 4), (1, 4), (2, 3), (0, 2)])
    # not_strand_pairs: y-0 and y-1 meet through z-0 too; the region {x-0, y-0} is not made of the two strands of its reads.
    out["not_strand_pairs"] = raw(3, [(0, 4), (1, 4), (2, 4), (3, 4), (0, 2)])
    g = strand_jump(30, [(12, 15)], 3)
    jump = int(np.nonzero(g["records"][:, 2] == 0)[0][0])
    # odd_edge_count: the jump's edge without its reverse complement.
    al = [(int(r[0]), int(r[1]), bool(r[2]), int(r[9])) for r in g["records"]]
    b = build(30, al, 3)
    keep = np.ones(len(b["edges"]), bool)
    keep[2 * jump + 1] = False
    remap = np.cumsum(keep) - 1
    rows = [[int(remap[e]) for e in b["data"][b["toc"][v]:b["toc"][v + 1]] if keep[e]] for v in range(60)]
    out["odd_edge_count"] = dict(b, edges=b["edges"][keep], toc=np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.uint32),
                                 data=np.array([e for r in rows for e in r], np.uint32))
    # pair_alignment_ids: the jump's reverse complement edge names another alignment.
    e = np.array(g["edges"])
    e[2 * jump + 1, 2] = len(g["records"]) - 1 if jump != len(g["records"]) - 1 else 0
    out["pair_alignment_ids"] = dict(g, edges=e)
    return out


def _digest(g):
    import hashlib
    h = hashlib.sha256()
    for k, t in (("edges", np.uint32), ("toc", np.uint32), ("data", np.uint32), ("records", np.uint32), ("flags", np.uint8)):
        h.update(np.ascontiguousarray(g[k], t).tobytes())
    return h.hexdigest()


def expected(kind, key, g, d):
    """The reference's output for flagCrossStrandReadGraphEdges1 (kind "cross") or flagChimericReads ("chimeric") on g at
    distance d: from the reference build oracle/_ref/libshasta_ref_readgraph_flags.so where it exists, else as recorded from
    it in tests/golden/reference_readgraph_flags.npz under `key` (SHB_RECORD_REFERENCE=1 rewrites the recordings). The
    recording carries a digest of its input, which must be this input."""
    from oracle import readgraph_flags_bindings as F
    from reference_outputs import RECORD, recorded
    fn = F.ref_cross_strand if kind == "cross" else F.ref_chimeric

    def run(g, d):
        return dict(fn(g, d), input_sha256=_digest(g))

    if F.have_ref() and not RECORD:
        return fn(g, d)
    out = dict(recorded("readgraph_flags", f"{kind}/{key}/{d}", run, g, d))
    assert out.pop("input_sha256") == _digest(g), f"the recording {kind}/{key}/{d} was made for another input"
    return out
