"""GPU parity (run with -m gpu): shb_create_read_graph against the oracle, on random AlignmentData and on the alignments the
CUDA path itself produced for a synthetic read set."""
import numpy as np
import pytest

from oracle import bindings as B
from support import ctx, device_alignments  # noqa: F401

from readgraph_inputs import quality_records, records

pytestmark = pytest.mark.gpu


def _check(ctx, rec, reads, k):
    from shasta_b200 import capi
    orec, okeep, oedges, otoc, odata = B.oracle_create_read_graph(rec, reads, k)
    work = rec.copy()
    keep, edges, toc, data = capi.create_read_graph(ctx, work, reads, k)
    assert np.array_equal(keep, okeep)
    assert np.array_equal(edges, oedges)
    assert np.array_equal(toc, otoc) and np.array_equal(data, odata)
    assert np.array_equal(work, orec)


def test_random_alignment_data(ctx):
    rng = np.random.default_rng(11)
    for n, reads, k in [(0, 5, 3), (1, 4, 6), (60, 12, 3), (5000, 300, 6), (5000, 300, 1), (200, 10, 0), (150, 8, 1000),
                        (200000, 9000, 6)]:
        _check(ctx, records(rng, n, reads), reads, k)


def test_on_computed_alignments(ctx):
    _, _, rec, _, _ = device_alignments(ctx)
    assert len(rec) > 500
    for k in (1, 6, 20):
        _check(ctx, rec, 400, k)


def test_creation_method_2(ctx):
    """createReadGraph2: thresholds from the histograms (host, alignment order) + the device selection over the alignments that pass."""
    from shasta_b200 import capi
    rng = np.random.default_rng(21)
    pc = (0.015, 0.12, 0.12, 0.12, 0.015)
    for n, reads, k in [(0, 4, 6), (400, 30, 6), (3000, 120, 6), (3000, 120, 2), (150000, 6000, 6)]:
        rec = quality_records(rng, n, reads)
        ocrit, orec, okeep, oedges, otoc, odata = B.oracle_create_read_graph2(rec, reads, k, pc)
        work = rec.copy()
        crit, keep, edges, toc, data = capi.create_read_graph2(ctx, work, reads, k, *pc)
        assert crit == ocrit
        assert np.array_equal(keep, okeep) and np.array_equal(edges, oedges)
        assert np.array_equal(toc, otoc) and np.array_equal(data, odata) and np.array_equal(work, orec)
