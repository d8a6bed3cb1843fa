"""Digests of each pipeline stage's outputs, and the reference's outputs at each stage, for the whole-pipeline tests
(tests/test_oracle_shipped_pipeline.py records and checks them, tests/test_gpu_shipped_pipeline.py checks the device's
chain against them). Outputs are stored in tests/golden/reference_pipeline.npz as SHA-256 digests, raw where small.

Every digest function takes the outputs of one stage, whoever computed them (oracle, reference or device), so the same
call digests all three."""
import numpy as np

from oracle import bindings as B
from oracle import markergraph_bindings as MB
from oracle import markergraph_edges_bindings as EB
from oracle import palindromic_bindings as PB
from oracle import readgraph_flags_bindings as F
from reference_outputs import recorded, shrink, stored

STAGES = ("palindromic", "lowhash", "alignments", "readgraph", "cross", "chimeric", "vertices", "edges")


RAW = ("flaggedEdges",)         # stored as they are: the chain downstream of the reference is rebuilt from them


def digest(outputs):
    return {k: shrink(v, 4096) if isinstance(v, np.ndarray) and k not in RAW else v for k, v in outputs.items()}


def same(got, ref, what):
    """got: dict of arrays and scalars; ref: a digest with the same keys."""
    for k, v in got.items():
        if isinstance(v, np.ndarray):
            assert np.array_equal(shrink(v, 4096).reshape(-1), np.asarray(ref[k]).reshape(-1)), f"{what}: {k}"
        else:
            assert v == ref[k], f"{what}: {k} {v} != {ref[k]}"


# ---- the outputs of each stage ---------------------------------------------------------------------------------------
def palindromic_outputs(flags, aligned, near, exact):
    """The counts of the reads aligned exactly (the others carry the prefilter's bounds on the device and in the oracle,
    and exact counts in the reference), zero elsewhere."""
    exact = np.asarray(exact, bool)
    return dict(flags=np.asarray(flags, np.uint8) & 1, aligned=np.where(exact, np.asarray(aligned, np.uint32), 0).astype(np.uint32),
                nearDiagonal=np.where(exact, np.asarray(near, np.uint32), 0).astype(np.uint32))


def lowhash_outputs(cand, stats):
    return dict(candidates=np.asarray(cand, np.uint32).reshape(-1, 3), stats=np.asarray(stats, np.uint64))


def alignment_outputs(info, ctoc, cdata):
    return dict(info=np.asarray(info, np.uint32).reshape(-1, 12), ctoc=np.asarray(ctoc, np.uint64), cdata=np.asarray(cdata, np.uint8))


def readgraph_outputs(records, keep, edges, toc, data):
    return dict(records=np.asarray(records, np.uint32), keep=np.asarray(keep, np.uint8), edges=np.asarray(edges, np.uint32),
                toc=np.asarray(toc, np.uint32), data=np.asarray(data, np.uint32))


VERTEX_COUNTS = ("minCoverageUsed", "peakFinderFailed", "disjointSetCount", "keptDisjointSetCount", "badDisjointSetCount",
                 "vertexCount")


def vertices_outputs(table, vtoc, vdata, rc, histogram, **counts):
    """Vertices in canonical form (by first marker): the oracle's and the device's numbering, and the reference's renumbered."""
    table, vtoc, vdata, rank = MB.canonical(table, vtoc, vdata)
    crc = np.zeros(len(rc), np.int64)
    crc[rank] = rank[np.asarray(rc, np.int64)]
    return dict(table=table, vtoc=vtoc, vdata=vdata, rc=crc.astype(np.uint64), histogram=np.asarray(histogram, np.uint64), **counts)


def edges_outputs(s, rc):
    """s: an edge set with bySourceData / byTargetData as uint64."""
    return dict(fields=EB.named_fields(s["edges"]), itoc=np.asarray(s["intervalsToc"], np.uint64),
                idata=np.asarray(s["intervalsData"], np.uint32), stoc=np.asarray(s["bySourceToc"], np.uint64),
                sdata=np.asarray(s["bySourceData"], np.uint64), ttoc=np.asarray(s["byTargetToc"], np.uint64),
                tdata=np.asarray(s["byTargetData"], np.uint64), rc=np.asarray(rc, np.uint64))


# ---- the reference at each stage -------------------------------------------------------------------------------------
def ref_palindromic(toc, kmer, params, exact):
    r = PB.ref_flag_palindromic(toc, kmer, **params)
    return palindromic_outputs(r["flags"], r["aligned"], r["nearDiagonal"], exact)


def ref_lowhash(toc, data, flags, params):
    cand, stats, _, _ = B.ref_lowhash0(toc, data, flags, B.LowHashParams(**params), threads=0)
    return lowhash_outputs(cand, stats)


def ref_alignments(toc, records, ctoc, cdata):
    """The reference's AlignmentInfo and compressAlignment of each stored alignment's ordinals."""
    info, comp, rtoc = [], [], [0]
    for i, r in enumerate(np.asarray(records, np.uint32).reshape(-1, 16)):
        ords = B.oracle_decompress(cdata[int(ctoc[i]):int(ctoc[i + 1])])
        o0, o1 = 2 * int(r[0]), 2 * int(r[1]) + (0 if r[2] else 1)
        info.append(B.ref_alignment_info(ords, int(toc[o0 + 1] - toc[o0]), int(toc[o1 + 1] - toc[o1])))
        comp.append(B.ref_compress(ords))
        rtoc.append(rtoc[-1] + len(comp[-1]))
    return alignment_outputs(np.array(info, np.uint32), np.array(rtoc, np.uint64),
                             np.concatenate(comp) if comp else np.zeros(0, np.uint8))


def ref_readgraph(records, R, rg):
    if rg["creationMethod"] == 0:
        return readgraph_outputs(*B.ref_create_read_graph(records, R, rg["maxAlignmentCount"]))
    crit, *out = B.ref_create_read_graph2(records, R, rg["maxAlignmentCount"], rg["percentiles"])
    return dict(readgraph_outputs(*out), **crit)


def ref_cross(g, d):
    r = F.ref_cross_strand(g, d, threads=4)
    assert r["status"] == 0
    return dict(edges=r["edges"], records=r["records"], reported=r["reported"], regions=r["regions"], flagged=r["flagged"],
                flaggedEdges=np.nonzero(r["edges"][:, 3] & F.CROSS)[0].astype(np.uint32))


def cross_outputs(g, flagged_edges):
    """(edges, records) of flagCrossStrandReadGraphEdges1 on read graph g when it flags exactly `flagged_edges`:
    crossesStrands set on them and cleared on every other edge, isInReadGraph cleared on their alignments. Where two edge
    pairs of a strand jump region tie on markerCount, only the reference's unstable sort decides which edges it flags
    (oracle/readgraph_flags_bindings.py), so the chain after that stage is rebuilt from the reference's own choice."""
    edges = np.array(g["edges"], np.uint32, copy=True).reshape(-1, 4)
    rec = np.array(g["records"], np.uint32, copy=True).reshape(-1, 16)
    edges[:, 3] &= ~F.CROSS
    e = np.asarray(flagged_edges, np.int64)
    edges[e, 3] |= F.CROSS
    rec[edges[e, 2].astype(np.int64) | ((edges[e, 3] & 0x3FFFFFFF).astype(np.int64) << 32), 15] &= ~np.uint32(1)
    return edges, rec


def ref_chimeric(g, d):
    r = F.ref_chimeric(g, d, threads=4)
    assert r["status"] == 0
    return dict(flags=r["flags"], records=r["records"], chimeric=r["chimeric"])


def ref_vertices(toc, kmer, edges, ctoc, cdata, flags, params):
    r = MB.ref_create_marker_graph_vertices(toc, kmer, edges, ctoc, cdata, flags, threads=4, **params)
    assert r["status"] == 0
    st, rc = MB.ref_find_rc_vertices(toc, r["table"], r["vtoc"], r["vdata"])
    assert st == 0
    return vertices_outputs(r["table"], r["vtoc"], r["vdata"], rc, r["histogram"], **{k: r[k] for k in VERTEX_COUNTS})


def ref_edges(toc, table, vtoc, vdata, rcv):
    s = EB.ref_create_marker_graph_edges(toc, table, vtoc, vdata, threads=1)
    assert s["status"] == 0
    msg, rc = EB.ref_find_rc_edges(toc, rcv, s, threads=1)
    assert msg is None
    return edges_outputs(s, rc)


def reference(name, stage, fn, *args):
    """The reference's digest of a stage: computed by fn(*args) under SHB_RECORD_REFERENCE=1, else as recorded."""
    return recorded("pipeline", f"{name}/{stage}", lambda *a: digest(fn(*a)), *args)


def recorded_digest(name, stage):
    """The reference's digest of a stage as recorded (never calls the reference)."""
    return stored("pipeline", f"{name}/{stage}")
