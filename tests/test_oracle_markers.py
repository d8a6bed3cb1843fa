"""CPU test: the marker-finding oracle (oracle/markers_oracle.c) against the golden output of the UNMODIFIED reference
MarkerFinder on TinyTest (tests/golden/tinytest_markers.npz; inputs tests/golden/tinytest_reads.npz), and against the
reference's ReadLoader + MarkerFinder run on synthetic FASTA files (recorded in tests/golden/reference_markers.npz)."""
import hashlib
import os

import numpy as np

from oracle import bindings as B
from support import reference_markers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (reads, seed, k) of the synthetic FASTA files: this test's, then the GPU test's (tests/test_gpu_markers.py)
SYNTHETIC_CASES = [(40, 3, 8), (40, 3, 10), (60, 6, 6), (60, 10, 10), (60, 14, 14)]


def _golden():
    r = np.load(os.path.join(ROOT, "tests", "golden", "tinytest_reads.npz"))
    m = np.load(os.path.join(ROOT, "tests", "golden", "tinytest_markers.npz"))
    is_marker = np.unpackbits(r["is_marker_bitmap"].view(np.uint8), bitorder="little")
    return r, m, is_marker


def test_marker_oracle_reproduces_reference_tinytest():
    r, m, is_marker = _golden()
    assert int(r["k"]) == 10 and len(is_marker) == 4 ** 10
    toc, data = B.oracle_find_markers(r["word_offsets"], r["words"], r["base_counts"], is_marker, 10)
    assert toc[-1] == 124036                    # SURVEY.md F5
    assert np.array_equal(toc, m["toc"]) and np.array_equal(data, m["data"])


def test_marker_oracle_against_live_reference(tmp_path):
    for reads, seed, k in SYNTHETIC_CASES:
        g = reference_markers(tmp_path, reads, seed, k)
        is_marker = np.zeros(4 ** k, np.uint8)
        is_marker[g["marker_kmers"]] = 1
        toc, data = B.oracle_find_markers(g["word_offsets"], g["words"], g["base_counts"], is_marker, k)
        assert toc[-1] > 1000
        assert np.array_equal(toc, g["toc"]) and hashlib.sha256(data.tobytes()).hexdigest() == g["data_sha256"]
