"""GPU (run with -m gpu): shb_create_read_graph, shb_create_read_graph2 (ReadGraph.creationMethod 0 and 2),
shb_compute_alignment_table and shb_compute_candidate_table against the reference's own code, on the input families of
tests/test_oracle_readgraph.py, at scale, and on the alignments the device itself computed.

Where oracle/_ref is present with the read graph glue (oracle/ref_glue/ref_readgraph.cpp) the device is compared with it
directly; elsewhere with the outputs recorded from it in tests/golden/reference_readgraph.npz. Always also with the oracle, which the
CPU tests pin to the same outputs."""
import numpy as np
import pytest

from oracle import bindings as B
from shasta_b200 import synth

from test_oracle_readgraph import (DEFAULT_PERCENTILES, assert_same, outcome, read_graph2_families, read_graph_families,
                                   scale_family, summary, table_summary, unordered2_cases, unordered_cases)
from reference_outputs import recorded

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from shasta_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


def _reference(key, fn, *args):
    return fn(*args) if B.have_ref_readgraph() else recorded("readgraph", key, fn, *args)


def device_outcome(ctx, rec, reads, k, percentiles=None):
    """summary() of the device's read graph, or "refused" (SHB_ERR_INVALID, records left as they were)."""
    from shasta_b200 import capi
    work = np.ascontiguousarray(rec, np.uint32).copy()
    try:
        if percentiles is None:
            crit = None
            keep, edges, toc, data = capi.create_read_graph(ctx, work, reads, k)
        else:
            crit, keep, edges, toc, data = capi.create_read_graph2(ctx, work, reads, k, *percentiles)
    except capi.ShastaB200Error as e:
        assert e.status == 1 and "not in increasing order" in str(e), str(e)
        assert np.array_equal(work, rec)
        return "refused"
    assert np.array_equal(work[:, :15], rec[:, :15]) and np.array_equal(work[:, 15] >> 1, rec[:, 15] >> 1)
    return summary(work, keep, edges, toc, data, criteria=crit)


def test_read_graph_families(ctx):
    for name, rec, reads, ks in read_graph_families():
        for k in ks:
            got = device_outcome(ctx, rec, reads, k)
            assert_same(_reference(f"rg0_{name}_{k}", outcome, B.ref_create_read_graph, rec, reads, k), got, (name, k))
            assert_same(outcome(B.oracle_create_read_graph, rec, reads, k), got, (name, k))


def test_read_graph2_families(ctx):
    for name, rec, reads, ks, pc in read_graph2_families():
        for k in ks:
            got = device_outcome(ctx, rec, reads, k, pc)
            assert_same(_reference(f"rg2_{name}_{k}", outcome, B.ref_create_read_graph2, rec, reads, k, pc), got, (name, k))
            assert_same(outcome(B.oracle_create_read_graph2, rec, reads, k, pc), got, (name, k))


def test_unordered_kept_edge_is_refused(ctx):
    """A kept alignment with readIds[0] > readIds[1], or of a read with itself, is refused with SHB_ERR_INVALID; the same
    input with that alignment out-selected is accepted and equals the reference. The context keeps working after a refusal."""
    for name, rec, reads, k, refused in unordered_cases():
        got = device_outcome(ctx, rec, reads, k)
        assert (got == "refused") == refused, name
        assert_same(_reference(f"unordered_{name}", outcome, B.ref_create_read_graph, rec, reads, k), got, name)
    for name, rec, reads, k, refused in unordered2_cases():
        got = device_outcome(ctx, rec, reads, k, (0.0,) * 5)
        assert (got == "refused") == refused, name
        assert_same(_reference(f"unordered2_{name}", outcome, B.ref_create_read_graph2, rec, reads, k, (0.0,) * 5), got, name)


def test_tables(ctx):
    from shasta_b200 import capi
    for name, rec, reads, _ in read_graph_families() + [c[:3] + (None,) for c in unordered_cases()[::2]]:
        got = table_summary(*capi.compute_alignment_table(ctx, rec, reads))
        want = _reference(f"alignment_table_{name}", lambda: table_summary(*B.ref_compute_alignment_table(rec, reads)))
        assert_same(want, got, name)
        cand = np.ascontiguousarray(rec[:, :3])
        got = table_summary(*capi.compute_candidate_table(ctx, cand, reads))
        want = _reference(f"candidate_table_{name}", lambda: table_summary(*B.ref_compute_candidate_table(cand, reads)))
        assert_same(want, got, name)


def test_scale(ctx):
    """3 M alignments over 100 k reads: the selection sort (6 M items) and the connectivity sort run over many tiles."""
    rec, reads, ks = scale_family()
    for k in ks:
        got = device_outcome(ctx, rec, reads, k)
        assert_same(_reference(f"rg0_scale_{k}", outcome, B.ref_create_read_graph, rec, reads, k), got, k)


def test_device_pipeline(ctx):
    """LowHash0 -> computeAlignments -> the tables and both read graphs, on the device's own AlignmentData, against the
    reference glue (or, without oracle/_ref, the oracle)."""
    from shasta_b200 import capi
    R = 400
    d = synth.generate(synth.SynthParams(reads=R, k=10, genome_markers=40000, n50_bases=12000, min_bases=6000, seed=9))
    kw = dict(m=4, hashFraction=0.01, minHashIterationCount=10, minBucketSize=2, maxBucketSize=30, minFrequency=2)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    cand, _, _, _ = ctx.lowhash0(capi.make_lowhash_params(**kw))
    akw = dict(alignMethod=3, k=10, maxSkip=30, maxDrift=30, maxTrim=30, minAlignedMarkerCount=50, minAlignedFraction=0.3,
               downsamplingFactor=0.1, bandExtend=10, maxBand=1000)
    rec, _, _, _ = capi.compute_alignments(ctx, cand, capi.make_align_options(**akw))
    rec = np.ascontiguousarray(rec, np.uint32)
    assert len(rec) > 500
    ref = B.have_ref_readgraph()
    for k in (1, 6, 20):
        want = outcome(B.ref_create_read_graph if ref else B.oracle_create_read_graph, rec, R, k)
        assert_same(want, device_outcome(ctx, rec, R, k), k)
        want = outcome(B.ref_create_read_graph2 if ref else B.oracle_create_read_graph2, rec, R, k, DEFAULT_PERCENTILES)
        assert_same(want, device_outcome(ctx, rec, R, k, DEFAULT_PERCENTILES), k)
    want = (B.ref_compute_alignment_table if ref else B.oracle_compute_alignment_table)(rec, R)
    assert_same(table_summary(*want), table_summary(*capi.compute_alignment_table(ctx, rec, R)), "alignment table")
    c = np.ascontiguousarray(np.asarray(cand, np.uint32).reshape(-1, 3))
    want = (B.ref_compute_candidate_table if ref else B.oracle_compute_candidate_table)(c, R)
    assert_same(table_summary(*want), table_summary(*capi.compute_candidate_table(ctx, c, R)), "candidate table")
