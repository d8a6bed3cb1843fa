"""createMarkerGraphVertices and findMarkerGraphReverseComplementVertices: the C restatement (oracle/markergraph_oracle.c)
against the reference's own DisjointSets, decompress and PeakFinder driven in the member's control flow
(oracle/ref_glue/ref_markergraph.cpp), in canonical form (vertices by first marker). PeakFinder alone: the library's
restatement (shb_peak_finder_cutoff) and the oracle's against the reference on a few hundred histograms. The reference's
outputs are stored in tests/golden/reference_markergraph.npz."""
import numpy as np
import pytest

from oracle import markergraph_bindings as MB
import support  # noqa: F401  (tests/golden on sys.path)

from markergraph_inputs import PARAMS, START_INDEX, cases, histograms
from reference_outputs import recorded, shrink

CASES = cases()
HISTOGRAMS = histograms()


def _ref_peaks():
    out = {}
    for name, y in HISTOGRAMS.items():
        for fraction in (0.08, 0.3):
            out[f"{name}/{fraction}"] = np.array(MB.ref_peak_finder_cutoff(y, fraction, START_INDEX.get(name, 2)), np.float64)
    return out


def test_peak_finder():
    ref = recorded("markergraph", "peaks", _ref_peaks)
    from shasta_b200 import capi
    seen = set()
    for name, y in HISTOGRAMS.items():
        for fraction in (0.08, 0.3):
            threw, cutoff, observed = ref[f"{name}/{fraction}"].tolist()
            expected = (int(threw), int(cutoff) if not threw else None, observed)
            start = START_INDEX.get(name, 2)
            o = MB.oracle_peak_finder_cutoff(y, fraction, start)
            g = capi.peak_finder_cutoff(y, fraction, start)
            for got in (o, g):
                assert (got[0], got[1] if not got[0] else None, got[2]) == expected, (name, fraction)
            seen.add(int(threw))
    assert seen == {0, 1}
    assert ref["single/0.08"][0] == 1 and ref["one_peak/0.08"][0] == 1
    # The empty histogram (no markers) is undefined in the reference; here it is a throw with observed area 0.
    assert MB.oracle_peak_finder_cutoff(np.zeros(0, np.uint64)) == (1, 0, 0.0)
    assert capi.peak_finder_cutoff(np.zeros(0, np.uint64)) == (1, 0, 0.0)


def pack(table, vtoc, vdata):
    """Canonical vertices in a form that compresses: table as marker id minus first marker (2^40-1 kept), vertex sizes,
    and the differences of consecutive vertex markers. Arrays of the long-read case are stored as their SHA-256."""
    table = np.asarray(table, np.uint64)
    inv = np.uint64((1 << 40) - 1)
    delta = np.where(table == inv, inv, np.arange(len(table), dtype=np.uint64) - table)
    out = dict(table=delta, sizes=np.diff(np.asarray(vtoc, np.uint64)), steps=np.diff(np.asarray(vdata, np.uint64), prepend=np.uint64(0)))
    return {k: shrink(np.asarray(v, np.uint64), 50_000) for k, v in out.items()}


def _ref_case(name, pname):
    d = CASES[name]
    r = MB.ref_create_marker_graph_vertices(d["toc"], d["kmer"], d["edges"], d["ctoc"], d["cdata"], d["flags"], threads=4,
                                            **PARAMS[pname])
    assert r["status"] == 0
    table, vtoc, vdata, _ = MB.canonical(r["table"], r["vtoc"], r["vdata"])
    st, rc = MB.ref_find_rc_vertices(d["toc"], r["table"], r["vtoc"], r["vdata"])
    assert st == 0
    rank = MB.canonical(r["table"], r["vtoc"], r["vdata"])[3]
    crc = np.zeros(len(rc), np.int64)
    crc[rank] = rank[rc.astype(np.int64)]
    keys = ("histogram", "minCoverageUsed", "peakFinderFailed", "disjointSetCount", "keptDisjointSetCount",
            "badDisjointSetCount", "vertexCount", "observedAreaFraction")
    return dict(rc=shrink(np.asarray(crc, np.uint64), 50_000), **pack(table, vtoc, vdata), **{k: r[k] for k in keys})


@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference(name, pname):
    ref = recorded("markergraph", f"{name}/{pname}", _ref_case, name, pname)
    d = CASES[name]
    o = MB.oracle_create_marker_graph_vertices(d["toc"], d["kmer"], d["edges"], d["ctoc"], d["cdata"], d["flags"], **PARAMS[pname])
    assert o["status"] == 0
    # The oracle numbers vertices by first marker already: its canonical form is itself.
    table, vtoc, vdata, rank = MB.canonical(o["table"], o["vtoc"], o["vdata"])
    assert np.array_equal(rank, np.arange(len(rank)))
    for key, got in list(pack(table, vtoc, vdata).items()) + [("histogram", o["histogram"])]:
        assert np.array_equal(got, np.asarray(ref[key]).reshape(-1)), key
    for key in ("minCoverageUsed", "peakFinderFailed", "disjointSetCount", "keptDisjointSetCount", "badDisjointSetCount",
                "vertexCount", "observedAreaFraction"):
        assert o[key] == ref[key], key
    st, rc = MB.oracle_find_rc_vertices(d["toc"], o["table"], o["vtoc"], o["vdata"])
    assert st == 0 and np.array_equal(shrink(np.asarray(rc, np.uint64), 50_000), np.asarray(ref["rc"]).reshape(-1))
    assert o["edgePairsUsed"] + o["edgePairsSkipped"] == len(d["edges"]) // 2


def test_cases_reach_every_branch():
    """The inputs exercise what the comparison above is meant to cover."""
    tags = set()
    for d in CASES.values():
        for a in range(len(d["ctoc"]) - 1):
            p, e = int(d["ctoc"][a]), int(d["ctoc"][a + 1])
            while p < e:
                t = int(d["cdata"][p])
                n = 1 if t & 1 == 0 else {1: 2, 3: 4, 5: 8, 7: 16}[t & 7]
                tags.add(n)
                p += n
    assert tags == {1, 2, 4, 8, 16}
    flags = np.concatenate([d["edges"][:, 3] >> 30 for d in CASES.values()])
    assert {1, 2, 3} <= set(flags.tolist())
    assert any((d["flags"] & 2).any() for d in CASES.values())
    o = MB.oracle_create_marker_graph_vertices(**{k: CASES["deep"][k] for k in ("toc", "kmer", "edges", "ctoc", "cdata", "flags")},
                                               **PARAMS["cov2"])
    assert o["badDisjointSetCount"] > 0 and o["keptDisjointSetCount"] > o["badDisjointSetCount"]
    sizes = [recorded("markergraph", f"{name}/strand1", _ref_case, name, "strand1")["histogram"] for name in CASES]
    assert any(len(h) > 1 and h[1] > 0 for h in sizes)          # singletons meet minCoveragePerStrand 1 (kept) and 2 (bad)


@pytest.mark.parametrize("status,mutate", [
    (1, lambda d: d.update(edges=d["edges"][:-1])),
    (2, lambda d: d["edges"].__setitem__((1, 0), d["edges"][1, 0] ^ 2)),
    (3, lambda d: d["edges"].__setitem__((slice(0, 2), slice(0, 2)), d["edges"][0:2, [1, 0]])),
    (4, lambda d: d["edges"].__setitem__((0, 2), len(d["ctoc"]) + 5)),
    (5, lambda d: d["kmer"].__setitem__(int(d["toc"][d["edges"][0, 0]]) + int(MB_first_ordinal(d)), 1 << 21)),
])
def test_oracle_assertions(status, mutate):
    d = {k: np.array(v) for k, v in CASES["genome_in_order"].items()}
    mutate(d)
    o = MB.oracle_create_marker_graph_vertices(d["toc"], d["kmer"], d["edges"], d["ctoc"], d["cdata"], d["flags"], **PARAMS["cov2"])
    assert o["status"] == status


def MB_first_ordinal(d):
    from oracle import bindings as B
    a = int(d["edges"][0, 2])
    return B.oracle_decompress(d["cdata"][int(d["ctoc"][a]):int(d["ctoc"][a + 1])])[0, 0]
