"""flagCrossStrandReadGraphEdges1 and flagChimericReads: the restatement in oracle/readgraph_flags_bindings.py against the
reference's own ReadGraph code (oracle/_ref/libshasta_ref_readgraph_flags.so) on read graphs built directly. Where that
build is absent the comparisons use its outputs recorded in tests/golden/reference_readgraph_flags.npz."""
import numpy as np
import pytest

from oracle import readgraph_flags_bindings as F

import support  # noqa: F401  (puts tests/golden on sys.path)
from readgraph_flags_inputs import DISTANCES, bad_graphs, expected, families, hub

FAM = families()
need_ref = pytest.mark.skipif(not F.have_ref(), reason="the reference build oracle/_ref/libshasta_ref_readgraph_flags.so is absent")


def _same(a, b, keys):
    assert a["status"] == b["status"]
    if a["status"] == 0:
        for k in keys:
            assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


@pytest.mark.parametrize("name", sorted(FAM))
@pytest.mark.parametrize("d", DISTANCES)
def test_cross_strand_restatement_equals_reference(name, d):
    g = FAM[name]
    ref = expected("cross", name, g, d)
    py = F.py_cross_strand(g, d)
    if ref["status"] == 0 and F.region_ties(g, d):
        # Only the reference's unstable sort decides the order of tied pairs; the sets of near reads and regions still agree.
        assert (py["reported"], py["regions"]) == (ref["reported"], ref["regions"])
        return
    _same(py, ref, ["edges", "records", "reported", "regions", "flagged"])


@pytest.mark.parametrize("name", sorted(FAM))
@pytest.mark.parametrize("d", DISTANCES)
def test_chimeric_restatement_equals_reference(name, d):
    g = FAM[name]
    _same(F.py_chimeric(g, d), expected("chimeric", name, g, d), ["flags", "records", "chimeric"])


def test_ties_are_decided_by_the_unstable_sort():
    """On the tie family the reference's std::sort flags other edges than a stable sort would: the tie cases are the ones
    that tell the device's ordering apart."""
    g = FAM["ties"]
    assert F.region_ties(g, 6)
    assert not np.array_equal(expected("cross", "ties", g, 6)["edges"], F.py_cross_strand(g, 6)["edges"])


@pytest.mark.parametrize("what", sorted(bad_graphs()))
def test_region_assertions(what):
    assert expected("cross", what, bad_graphs()[what], 6)["status"] == 1
    assert F.py_cross_strand(bad_graphs()[what], 6)["status"] == 1


HUB_CASES = [("hub300", 7, 300, "cross", 2), ("hub300", 7, 300, "cross", 6), ("hub300", 7, 300, "cross", 254),
             ("hub300", 7, 300, "chimeric", 2), ("hub300", 7, 300, "chimeric", 6), ("hub300", 7, 300, "chimeric", 254),
             ("hub3000", 8, 3000, "chimeric", 3), ("hub3000", 8, 3000, "cross", 6)]


@pytest.mark.parametrize("key,seed,R,kind,d", HUB_CASES)
def test_hubs(key, seed, R, kind, d):
    """The hubs whose balls overflow the device's shared-memory table (the GPU tests use these outputs)."""
    g = hub(R, seed)
    ref = expected(kind, key, g, d)
    assert ref["status"] == 0
    if R <= 300:
        py = F.py_cross_strand(g, d) if kind == "cross" else F.py_chimeric(g, d)
        keys = ["flags", "records", "chimeric"] if kind == "chimeric" else (["regions", "reported"] if F.region_ties(g, d) else
                                                                              ["edges", "records", "regions", "flagged"])
        _same(py, ref, keys)


@need_ref
def test_reference_threads_do_not_change_the_result():
    g = FAM["several_regions"]
    for d in (2, 6):
        _same(F.ref_cross_strand(g, d, threads=4), F.ref_cross_strand(g, d), ["edges", "records", "flagged"])
        _same(F.ref_chimeric(g, d, threads=4), F.ref_chimeric(g, d), ["flags", "records", "chimeric"])


@need_ref
def test_recordings_are_the_reference_outputs():
    """The recorded outputs equal what the reference build computes now (for every recorded family input)."""
    from reference_outputs import RECORD, recorded
    if RECORD:
        pytest.skip("the recordings are being rewritten")
    for name, g in FAM.items():
        for d in DISTANCES:
            for kind, fn in (("cross", F.ref_cross_strand), ("chimeric", F.ref_chimeric)):
                rec = recorded("readgraph_flags", f"{kind}/{name}/{d}", None)
                live = fn(g, d)
                assert rec["status"] == live["status"]
                for k, v in live.items():
                    assert np.array_equal(np.asarray(rec[k]), np.asarray(v)), (kind, name, d, k)


def test_families_cover_what_they_claim():
    assert F.py_cross_strand(FAM["one_region"], 6)["regions"] == 1
    assert F.py_cross_strand(FAM["several_regions"], 6)["regions"] == 3
    assert F.py_cross_strand(FAM["one_region"], 6)["flagged"] > 0
    assert F.region_ties(FAM["ties"], 6)
    assert F.py_chimeric(FAM["chimeric"], 2)["flags"][20] & 2
    assert not (F.py_chimeric(FAM["near_chimeric"], 2)["flags"] & 2).any()
    assert (FAM["flagged_on_input"]["edges"][:, 3] & F.CROSS).any()


def test_refusals():
    g = FAM["one_region"]
    assert F.py_chimeric(g, 255)["status"] == 1 and F.py_cross_strand(g, -1)["status"] == 1
    assert expected("chimeric", "one_region", g, 255)["status"] == 1
