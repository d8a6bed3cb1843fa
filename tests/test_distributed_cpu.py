"""CPU test of the read-range split that a read-sharded run gives its ranks (shasta_b200/distributed.py)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_balanced_read_ranges():
    from shasta_b200 import distributed as D
    b = D.balanced_read_ranges([1] * 10, 4)
    assert b[0] == 0 and b[-1] == 10 and all(b[i] <= b[i + 1] for i in range(4))
    b = D.balanced_read_ranges([100, 1, 1, 1, 100], 2)
    w = [100, 1, 1, 1, 100]
    assert b[0] == 0 and b[2] == 5 and abs(sum(w[:b[1]]) - sum(w[b[1]:])) <= 100
