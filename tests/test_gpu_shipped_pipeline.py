"""The device pipeline from bases to marker graph edges at the shipped configurations (tests/golden/pipeline_inputs.py), in
the reference's order (srcMain/main.cpp:650-938), on one context per configuration. Each stage runs on the device's own
upstream outputs and is compared bit for bit with the oracle given the same inputs, and with the reference's outputs
recorded by tests/test_oracle_shipped_pipeline.py for the oracle's chain (the same chain when every stage agrees).

Each configuration also asserts that it is not vacuous: the injected palindromic and chimeric reads are flagged, there are
hundreds of candidates and alignments, the peak finder succeeds where minCoverage is 0, there are thousands of vertices and
edges, and at k = 8 some marker set holds two markers of one read and a read aligned exactly against its reverse complement
has a k-mer at exactly maxMarkerFrequency. The Align4 grid path (more than 512 existing cells) is not reached by these inputs:
the count of such candidates is printed, and tests/test_gpu_align.py reaches the path through SHB_ALIGN4_SMEM_CELLS."""
import os
import time

import numpy as np
import pytest

from oracle import bindings as B
from oracle import markergraph_bindings as MB
from oracle import markergraph_edges_bindings as EB
from oracle import palindromic_bindings as PB
from oracle import readgraph_flags_bindings as F

import support  # noqa: F401  (puts tests/golden on sys.path)
import pipeline_inputs as P
import pipeline_reference as T

pytestmark = pytest.mark.gpu
NAMES = list(P.CONFIGS)


def align4_grid_candidates(toc, kmer, cand, a):
    """Candidates whose Align4 grid has more existing cells than fit in shared memory (kAlign4SmemCells = 512): the
    createAlignmentMatrix / createCells count (src/Align4.cpp:195-267, 380-436) in numpy."""
    n = 0
    for r0, r1, same in np.asarray(cand, np.int64):
        o0, o1 = 2 * r0, 2 * r1 + (0 if same else 1)
        x_k, y_k = kmer[toc[o0]:toc[o0 + 1]], kmer[toc[o1]:toc[o1 + 1]]
        nx = len(x_k)
        order = np.argsort(y_k, kind="stable")
        lo, hi = np.searchsorted(y_k[order], x_k, "left"), np.searchsorted(y_k[order], x_k, "right")
        reps = hi - lo
        x = np.repeat(np.arange(nx), reps)
        y = order[np.repeat(lo, reps) + np.arange(reps.sum()) - np.repeat(np.cumsum(reps) - reps, reps)]
        X, Y = x + y, nx + y - x - 1
        nIX = (nx + len(y_k) - 2) // a["align4DeltaX"] + 1
        _, counts = np.unique((Y // a["align4DeltaY"]) * nIX + X // a["align4DeltaX"], return_counts=True)
        n += int((counts >= max(1, a["align4MinEntryCountPerCell"])).sum() > 512)
    return n


def frequency_at_limit(toc, kmer, reads, limit):
    """Reads among `reads` with a k-mer that occurs exactly `limit` times in the read (the maxMarkerFrequency edge)."""
    hits = 0
    for r in reads:
        _, counts = np.unique(kmer[toc[2 * r]:toc[2 * r + 1]], return_counts=True)
        hits += int((counts == limit).any())
    return hits


@pytest.mark.parametrize("name", NAMES)
def test_device_chain(name):
    from shasta_b200 import capi
    cfg = P.CONFIGS[name]
    rg, mg, a = cfg["readgraph"], cfg["markergraph"], cfg["align"]
    d = P.inputs(name)
    is_marker, bitmap = P.marker_set(cfg["k"], cfg["probability"])
    R = len(d["base_counts"])
    ref = {stage: T.recorded_digest(name, stage) for stage in T.STAGES if stage != "cross" or rg["strandSeparationMethod"] == 1}
    ms, counts = {}, {}
    c = capi.Context(0)
    try:
        # findMarkers: the markers stay on the device; the host copy goes to the oracle.
        t = time.perf_counter()
        toc, data, _ = c.find_markers(cfg["k"], d["word_offsets"], d["words"], d["base_counts"], np.zeros(R, np.uint8),
                                      is_marker_bitmap=bitmap)
        ms["markers"] = 1e3 * (time.perf_counter() - t)
        otoc, odata = B.oracle_find_markers(d["word_offsets"], d["words"], d["base_counts"], is_marker, cfg["k"])
        assert np.array_equal(toc, otoc) and np.array_equal(data, odata), "markers"
        kmer = P.kmer_ids(data)
        counts["markers"] = int(toc[-1])

        # flagPalindromicReads, on the markers the context holds; the flags stay in the context for LowHash0.
        flags = np.zeros(R, np.uint8)
        t = time.perf_counter()
        aligned, near, pres = capi.flag_palindromic_reads(c, capi.make_palindromic_params(**cfg["palindromic"]), read_flags=flags)
        ms["palindromic"] = 1e3 * (time.perf_counter() - t)
        o = PB.oracle_flag_palindromic(toc, kmer, **cfg["palindromic"])
        assert np.array_equal(flags, o["flags"]) and np.array_equal(aligned, o["aligned"]) and np.array_equal(near, o["nearDiagonal"])
        assert pres.palindromicReadCount == int(o["flags"].sum()) and pres.exactReadCount == int(o["survives"].sum())
        exact = o["survives"] == 1
        T.same(T.palindromic_outputs(flags, aligned, near, exact), ref["palindromic"], "flagPalindromicReads")
        assert flags[d["palindromic"]].all(), "the injected palindromic reads are flagged"
        counts["palindromic"] = int(flags.sum())

        # LowHash0 on the flags the previous step left in the context.
        t = time.perf_counter()
        cand, stats, _, _ = c.lowhash0(capi.make_lowhash_params(**cfg["minhash"]))
        ms["lowhash"] = 1e3 * (time.perf_counter() - t)
        oc, ostats, _ = B.oracle_lowhash0(toc, data, flags, B.LowHashParams(**cfg["minhash"]))
        assert np.array_equal(cand, oc) and np.array_equal(stats, ostats), "LowHash0"
        T.same(T.lowhash_outputs(cand, stats), ref["lowhash"], "LowHash0")
        counts["candidates"] = len(cand)

        t = time.perf_counter()
        rec, ctoc, cdata, _ = capi.compute_alignments(c, cand, capi.make_align_options(**a))
        ms["alignments"] = 1e3 * (time.perf_counter() - t)
        orec, octoc, ocdata, _ = B.oracle_compute_alignments(toc, kmer, cand, B.make_align_options(**a), threads=os.cpu_count())
        assert np.array_equal(rec, orec) and np.array_equal(ctoc, octoc) and np.array_equal(cdata, ocdata), "computeAlignments"
        T.same(T.alignment_outputs(rec[:, 3:15], ctoc, cdata), ref["alignments"], "computeAlignments")
        counts["alignments"] = len(rec)
        assert len(cand) > 300 and len(rec) > 300

        rec = np.array(rec, np.uint32)
        if rg["creationMethod"] == 0:
            crit = ocrit = {}
            o = B.oracle_create_read_graph(rec, R, rg["maxAlignmentCount"])
            t = time.perf_counter()
            keep, edges, gtoc, gdata = capi.create_read_graph(c, rec, R, rg["maxAlignmentCount"])
        else:
            ocrit, *o = B.oracle_create_read_graph2(rec, R, rg["maxAlignmentCount"], rg["percentiles"])
            t = time.perf_counter()
            crit, keep, edges, gtoc, gdata = capi.create_read_graph2(c, rec, R, rg["maxAlignmentCount"], *rg["percentiles"])
        ms["readgraph"] = 1e3 * (time.perf_counter() - t)
        assert crit == ocrit
        edges, gtoc, gdata = np.array(edges), np.array(gtoc), np.array(gdata)
        for got, want, what in zip((rec, keep, edges, gtoc, gdata), o, ("records", "keep", "edges", "toc", "data")):
            assert np.array_equal(got, want), f"read graph {what}"
        T.same(dict(T.readgraph_outputs(rec, keep, edges, gtoc, gdata), **crit), ref["readgraph"], "read graph")
        counts["readGraphEdges"] = len(edges)

        # Strand separation method 1 only: method 2 goes on without flagCrossStrandReadGraphEdges1.
        g = dict(edges=edges.copy(), toc=gtoc, data=gdata, records=rec.copy(), flags=flags.copy())
        if rg["strandSeparationMethod"] == 1:
            dist = rg["crossStrandMaxDistance"]
            t = time.perf_counter()
            res = capi.flag_cross_strand_read_graph_edges1(c, dist, edges, gtoc, gdata, rec)
            ms["cross"] = 1e3 * (time.perf_counter() - t)
            got = dict(edges=edges, records=rec, reported=res["nearStrandJumpReportedCount"], regions=res["regionCount"],
                       flagged=res["crossStrandEdgeCount"])
            if not F.region_ties(g, dist):
                p = F.py_cross_strand(g, dist)
                T.same(got, T.digest(p), "cross-strand (restatement)")
            T.same(got, ref["cross"], "cross-strand")
            counts["crossStrand"] = res["crossStrandEdgeCount"]
            g = dict(g, edges=edges.copy(), records=rec.copy())
        t = time.perf_counter()
        res = capi.flag_chimeric_reads(c, rg["maxChimericReadDistance"], edges, gtoc, gdata, flags, rec)
        ms["chimeric"] = 1e3 * (time.perf_counter() - t)
        p = F.py_chimeric(g, rg["maxChimericReadDistance"])
        got = dict(flags=flags, records=rec, chimeric=res["chimericReadCount"])
        assert np.array_equal(flags, p["flags"]) and np.array_equal(rec, p["records"]) and res["chimericReadCount"] == p["chimeric"]
        T.same(got, ref["chimeric"], "flagChimericReads")
        counts["chimeric"] = res["chimericReadCount"]
        assert (flags[d["chimeric"]] & 2).any(), "an injected chimeric read is flagged"

        t = time.perf_counter()
        table, vtoc, vdata, hist, vres = capi.create_marker_graph_vertices(c, capi.make_marker_graph_params(**mg), edges, ctoc,
                                                                          cdata, flags)
        rcv = capi.find_marker_graph_reverse_complement_vertices(c, table, vtoc, vdata)
        ms["vertices"] = 1e3 * (time.perf_counter() - t)
        ov = MB.oracle_create_marker_graph_vertices(toc, kmer, edges, ctoc, cdata, flags, **mg)
        assert ov["status"] == 0
        t64, vtoc64 = capi.uint40_to_uint64(table), capi.uint40_to_uint64(vtoc)
        assert np.array_equal(t64, ov["table"]) and np.array_equal(vtoc64, ov["vtoc"]) and np.array_equal(vdata, ov["vdata"])
        assert np.array_equal(hist, ov["histogram"])
        for key in T.VERTEX_COUNTS + ("edgePairsUsed", "edgePairsSkipped", "alignedMarkerPairs"):
            assert getattr(vres, key) == ov[key], key
        assert vres.peakFinderObservedAreaFraction == ov["observedAreaFraction"]
        st, orcv = MB.oracle_find_rc_vertices(toc, ov["table"], ov["vtoc"], ov["vdata"])
        assert st == 0 and np.array_equal(rcv, orcv)
        T.same(T.vertices_outputs(t64, vtoc64, vdata, rcv, hist, **{k: getattr(vres, k) for k in T.VERTEX_COUNTS}), ref["vertices"],
               "vertices")
        if mg["minCoverage"] == 0:
            assert not vres.peakFinderFailed
        counts["vertices"] = vres.vertexCount
        counts["badDisjointSets"] = vres.badDisjointSetCount

        t = time.perf_counter()
        out, eres = capi.create_marker_graph_edges(c, table, vtoc, vdata)
        rce, _ = capi.find_marker_graph_reverse_complement_edges(c, rcv, out["edges"], out["intervalsToc"], out["intervalsData"],
                                                                 out["bySourceToc"], out["bySourceData"])
        ms["edges"] = 1e3 * (time.perf_counter() - t)
        oe = EB.oracle_create_marker_graph_edges(toc, ov["table"], ov["vtoc"], ov["vdata"])
        s = dict(out, bySourceData=EB.rows_from_uint40(out["bySourceData"]), byTargetData=EB.rows_from_uint40(out["byTargetData"]))
        for k in ("edges", "intervalsToc", "intervalsData", "bySourceToc", "bySourceData", "byTargetToc", "byTargetData"):
            assert np.array_equal(np.asarray(s[k]).reshape(-1), np.asarray(oe[k]).reshape(-1)), k
        assert eres.saturatedEdgeCount == oe["saturated"] and eres.markerIntervalCount == len(oe["intervalsData"])
        msg, orce = EB.oracle_find_rc_edges(toc, orcv, oe)
        assert msg is None and np.array_equal(rce, orce)
        T.same(T.edges_outputs(s, rce), ref["edges"], "edges")
        counts["edges"] = eres.edgeCount
        assert vres.vertexCount > 1000 and eres.edgeCount > 1000
    finally:
        c.close()
    counts["align4GridPathCandidates"] = align4_grid_candidates(toc, kmer, cand, a) if a["alignMethod"] == 4 else 0
    counts["exactReadsAtMaxMarkerFrequency"] = frequency_at_limit(toc, kmer, np.nonzero(exact)[0],
                                                                  cfg["palindromic"]["maxMarkerFrequency"])
    print(f"\n{name}: " + ", ".join(f"{k} {v}" for k, v in counts.items()) + "; device ms " +
          ", ".join(f"{k} {v:.0f}" for k, v in ms.items()))
    if cfg["k"] == 8:
        assert counts["badDisjointSets"] > 0, "a marker set holds two markers of one read"
        assert counts["exactReadsAtMaxMarkerFrequency"] > 0, "a k-mer at exactly maxMarkerFrequency in an exactly aligned read"
