"""flagPalindromicReads: the C restatement (oracle/palindromic_oracle.c) against the unmodified reference build
(shasta::align of src/AlignmentGraph.cpp and the thresholds of src/AssemblerAlign.cpp:741-766), read for read and path
for path. The reference's outputs are stored in tests/golden/reference_palindromic.npz."""
import numpy as np
import pytest

from oracle import palindromic_bindings as B

import support  # noqa: F401  (puts tests/golden on sys.path)
from palindromic_inputs import cases, killer_case
from reference_outputs import recorded

CASES = cases()


def _ref(toc, ids, params):
    R = (len(toc) - 1) // 2
    out = B.ref_flag_palindromic(toc, ids, **params)
    for r in range(R):
        out[f"path{r}"] = B.ref_flag_palindromic(toc, ids, path_read=r, **params)["path"]
    return out


def _check(name, toc, ids, params):
    R = (len(toc) - 1) // 2
    ref = recorded("palindromic", name, _ref, toc, ids, params)
    o = B.oracle_flag_palindromic(toc, ids, exact_all=True, **params)
    for key in ("flags", "aligned", "nearDiagonal"):
        assert np.array_equal(o[key], ref[key]), key
    for r in range(R):
        p = B.oracle_flag_palindromic(toc, ids, path_read=r, **params)["path"]
        assert np.array_equal(p, np.asarray(ref[f"path{r}"]).reshape(-1, 2)), f"read {r}"
    # Every read the reference flags survives the prefilter, and the prefilter's bounds hold.
    assert np.all(o["survives"][ref["flags"] == 1] == 1)
    assert np.all(o["vBound"] >= ref["aligned"]) and np.all(o["vNearBound"] >= ref["nearDiagonal"])
    # Without exact_all the rejected reads carry their bounds and the flags are unchanged.
    q = B.oracle_flag_palindromic(toc, ids, **params)
    assert np.array_equal(q["flags"], ref["flags"])
    return o, ref


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference(name):
    toc, ids, params = CASES[name]
    o, ref = _check(name, toc, ids, params)
    if name == "noisy_palindromes":
        assert ref["flags"].sum() >= 3 and (ref["flags"] == 0).sum() >= 3
    if name == "streaks":
        # The input reaches both sides of maxMarkerFrequency in both strands.
        mmf = params["maxMarkerFrequency"]
        lengths = set()
        for row in range(len(toc) - 1):
            _, counts = np.unique(ids[toc[row]:toc[row + 1]], return_counts=True)
            lengths.update(counts.tolist())
        assert mmf in lengths and mmf + 1 in lengths
    if name == "zero_thresholds":
        assert np.all(ref["flags"] == 1)
    if name == "tiny":
        assert ref["flags"][0] == 1                 # zero markers: 0/0 is NaN, neither test rejects the read
        assert o["vBound"][3] == 5 and o["survives"][3] == 1    # V/n == alignedFractionThreshold exactly


def test_heapsort_fallback():
    keys = B.oracle_sort_killer_keys(3000)
    k, o, fallbacks = B.oracle_std_sort_markers(keys, np.arange(len(keys)))
    assert fallbacks > 0 and np.all(np.diff(k.astype(np.int64)) >= 0)
    toc, ids, params = killer_case(keys)
    o, ref = _check("killer", toc, ids, params)
    assert o["counters"]["heapsortFallbacks"] > 0


def test_counters():
    toc, ids, params = CASES["noisy_palindromes"]
    o = B.oracle_flag_palindromic(toc, ids, exact_all=True, **params)
    c = o["counters"]
    assert c["exactReads"] == (len(toc) - 1) // 2
    assert c["vertices"] > 0 and c["edges"] >= 2 * c["vertices"] and c["heapPushes"] > 0
