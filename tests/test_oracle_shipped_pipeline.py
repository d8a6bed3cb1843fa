"""The oracle chain from bases to marker graph edges at the shipped configurations (tests/golden/pipeline_inputs.py),
each stage compared with the reference's compiled code given the same upstream outputs. The reference's outputs are
stored as SHA-256 digests (raw where small) in tests/golden/reference_pipeline.npz (tests/golden/pipeline_reference.py), and
tests/test_gpu_shipped_pipeline.py checks the device's chain against the same digests.

Stages with reference code: flagPalindromicReads, LowHash0, createReadGraph / createReadGraph2, flagCrossStrandReadGraphEdges1,
flagChimericReads, createMarkerGraphVertices, findMarkerGraphReverseComplementVertices, createMarkerGraphEdges,
findMarkerGraphReverseComplementEdges; for computeAlignments the reference's AlignmentInfo and compressAlignment check every
stored record and its compressed bytes (the DP itself is the oracle's: SeqAn is absent). Markers at k 8 and 15 are
oracle-only."""
import numpy as np
import pytest

from oracle import bindings as B
from oracle import markergraph_bindings as MB
from oracle import markergraph_edges_bindings as EB
from oracle import palindromic_bindings as PB
from oracle import readgraph_flags_bindings as F

import support  # noqa: F401  (puts tests/golden on sys.path)
import pipeline_inputs as P
import pipeline_reference as PR
from pipeline_reference import reference, same

NAMES = list(P.CONFIGS)


# ---- the chain ---------------------------------------------------------------------------------------------------------
def markers(name):
    """(inputs, toc, data7, kmer ids) of the oracle's MarkerFinder on the configuration's reads."""
    cfg = P.CONFIGS[name]
    d = P.inputs(name)
    is_marker, _ = P.marker_set(cfg["k"], cfg["probability"])
    toc, data = B.oracle_find_markers(d["word_offsets"], d["words"], d["base_counts"], is_marker, cfg["k"])
    return d, toc, data, P.kmer_ids(data)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_chain_equals_reference(name):
    cfg = P.CONFIGS[name]
    rg = cfg["readgraph"]
    d, toc, data, kmer = markers(name)
    R = len(d["base_counts"])
    assert (np.diff(toc.astype(np.int64))[2 * d["short"]] == 0).all()

    pal = PB.oracle_flag_palindromic(toc, kmer, **cfg["palindromic"])
    exact = pal["survives"] == 1            # the other reads carry the prefilter's bounds
    same(PR.palindromic_outputs(pal["flags"], pal["aligned"], pal["nearDiagonal"], exact),
         reference(name, "palindromic", PR.ref_palindromic, toc, kmer, cfg["palindromic"], exact), "flagPalindromicReads")
    flags = pal["flags"].copy()
    assert flags[d["palindromic"]].all(), "the injected palindromic reads are flagged"

    cand, stats, _ = B.oracle_lowhash0(toc, data, flags, B.LowHashParams(**cfg["minhash"]))
    same(PR.lowhash_outputs(cand, stats), reference(name, "lowhash", PR.ref_lowhash, toc, data, flags, cfg["minhash"]), "LowHash0")

    rec, ctoc, cdata, _ = B.oracle_compute_alignments(toc, kmer, cand, B.make_align_options(**cfg["align"]), threads=8)
    same(PR.alignment_outputs(rec[:, 3:15], ctoc, cdata), reference(name, "alignments", PR.ref_alignments, toc, rec, ctoc, cdata),
         "alignments")

    aligned = rec
    if rg["creationMethod"] == 0:
        crit = {}
        rec, keep, edges, gtoc, gdata = B.oracle_create_read_graph(aligned, R, rg["maxAlignmentCount"])
    else:
        crit, rec, keep, edges, gtoc, gdata = B.oracle_create_read_graph2(aligned, R, rg["maxAlignmentCount"], rg["percentiles"])
    same(dict(PR.readgraph_outputs(rec, keep, edges, gtoc, gdata), **crit), reference(name, "readgraph", PR.ref_readgraph, aligned, R, rg),
         "read graph")

    g = dict(edges=edges, toc=gtoc, data=gdata, records=rec, flags=flags)
    if rg["strandSeparationMethod"] == 1:
        dist = rg["crossStrandMaxDistance"]
        c = F.py_cross_strand(g, dist)
        r = reference(name, "cross", PR.ref_cross, g, dist)
        if not F.region_ties(g, dist):
            same({k: c[k] for k in ("edges", "records", "reported", "regions", "flagged")}, r, "flagCrossStrandReadGraphEdges1")
        # The chain goes on from the reference's choice of edges (the restatement's, where no region ties).
        edges, rec = PR.cross_outputs(g, r["flaggedEdges"])
        same(dict(edges=edges, records=rec, flagged=len(r["flaggedEdges"])), r, "flagCrossStrandReadGraphEdges1 (flagged edges)")
        g = dict(g, edges=edges, records=rec)
    ch = F.py_chimeric(g, rg["maxChimericReadDistance"])
    same({k: ch[k] for k in ("flags", "records", "chimeric")}, reference(name, "chimeric", PR.ref_chimeric, g, rg["maxChimericReadDistance"]),
         "flagChimericReads")
    assert ch["chimeric"] > 0 and (ch["flags"][d["chimeric"]] & 2).any(), "an injected chimeric read is flagged"

    v = MB.oracle_create_marker_graph_vertices(toc, kmer, g["edges"], ctoc, cdata, ch["flags"], **cfg["markergraph"])
    assert v["status"] == 0
    st, rcv = MB.oracle_find_rc_vertices(toc, v["table"], v["vtoc"], v["vdata"])
    assert st == 0
    same(PR.vertices_outputs(v["table"], v["vtoc"], v["vdata"], rcv, v["histogram"], **{k: v[k] for k in PR.VERTEX_COUNTS}),
         reference(name, "vertices", PR.ref_vertices, toc, kmer, g["edges"], ctoc, cdata, ch["flags"], cfg["markergraph"]), "vertices")

    e = EB.oracle_create_marker_graph_edges(toc, v["table"], v["vtoc"], v["vdata"])
    assert e["status"] == 0
    msg, rce = EB.oracle_find_rc_edges(toc, rcv, e)
    assert msg is None
    same(PR.edges_outputs(e, rce), reference(name, "edges", PR.ref_edges, toc, v["table"], v["vtoc"], v["vdata"], rcv), "edges")

