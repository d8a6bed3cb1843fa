"""CPU tests: the host side of the digests every bench line carries (include/shasta_b200.h: shb_digest_records /
shb_digest_compressed) against an independent numpy statement of the same formula; the oracle's tie-break policy switch
and tie-exposure flags (include/shb_dp_policy.h, oracle/align_oracle.c); the candidate-table oracle against a direct
restatement of src/AssemblerAlignmentCandidates.cpp:379-448."""
import numpy as np

from oracle import bindings as B
from support import candidate_set

M64 = (1 << 64) - 1
FNV_OFFSET, FNV_PRIME = 0xcbf29ce484222325, 0x100000001b3


def _fnv_words(words):
    h = FNV_OFFSET
    for w in words:
        h = ((h ^ int(w)) * FNV_PRIME) & M64
    return h ^ (h >> 32)


def test_record_digest_matches_formula_and_is_order_independent():
    from shasta_b200 import capi
    rng = np.random.default_rng(1)
    rec = rng.integers(0, 2**32, (500, 16), dtype=np.uint64).astype(np.uint32)
    want = sum(_fnv_words(r) for r in rec) & M64
    assert capi.digest_records(rec, 16) == want
    assert capi.digest_records(rec[rng.permutation(len(rec))], 16) == want
    # additive over any partition (multi-GPU: the ranks' digests sum to the single-GPU digest)
    assert (capi.digest_records(rec[:123], 16) + capi.digest_records(rec[123:], 16)) & M64 == want
    cand = np.stack([rng.integers(0, 1000, 300), rng.integers(1000, 2000, 300), rng.integers(0, 2, 300)], 1).astype(np.uint32)
    assert capi.digest_candidates(cand) == sum(_fnv_words(r) for r in cand) & M64
    assert capi.digest_records(rec[:0], 16) == 0


def test_compressed_digest_matches_formula():
    from shasta_b200 import capi
    rng = np.random.default_rng(2)
    n = 200
    rec = rng.integers(0, 2**31, (n, 16), dtype=np.int64).astype(np.uint32)
    rec[:, 2] = rng.integers(0, 2, n)
    lens = rng.integers(1, 40, n)
    toc = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    data = rng.integers(0, 256, int(toc[-1])).astype(np.uint8)
    want = 0
    for i in range(n):
        want += _fnv_words(list(rec[i, :3]) + list(data[int(toc[i]):int(toc[i + 1])]))
    assert capi.digest_compressed(rec, toc, data) == want & M64


def _random_pair(rng, n=400, alphabet=6):
    a = rng.integers(0, alphabet, n).astype(np.uint32)
    b = a.copy()
    drop = rng.random(n) < 0.15
    b = b[~drop]
    b[rng.random(len(b)) < 0.1] = alphabet + 1
    return a, b


def test_every_policy_gives_an_optimal_path_of_the_same_score():
    # The policies only choose among co-optimal paths: same score, and each path re-scores to that score.
    rng = np.random.default_rng(5)
    default = B.default_dp_policy()
    try:
        for trial in range(20):
            a, b = _random_pair(rng)
            scores, paths = [], []
            for policy in range(8):
                B.set_dp_policy(policy)
                s, path = B.overlap_align(a, b, 6, -1, -1)
                scores.append(s)
                paths.append(path)
                # re-score the path: diagonal steps + gaps between consecutive steps. Gap moves before the first or after the
                # last diagonal step (to reach the border of the matrix) are not visible in the list of diagonal steps: the
                # re-scored total can exceed the DP score by their number, never fall below it.
                total = 0
                for k in range(len(path)):
                    x, y = int(path[k, 0]), int(path[k, 1])
                    total += 6 if a[x] == b[y] else -1
                    if k:
                        px, py = int(path[k - 1, 0]), int(path[k - 1, 1])
                        assert x > px and y > py
                        total -= (x - px - 1) + (y - py - 1)
                assert s <= total <= s + 8
            assert len(set(scores)) == 1
            # a small alphabet makes ties common: the policies must actually differ somewhere
            if trial == 0:
                first = paths
        assert any(not np.array_equal(first[0], p) for p in first[1:])
    finally:
        B.set_dp_policy(default)


def test_tie_flags_bound_the_policy_exposure():
    # A candidate whose tie flags are clear has a unique optimum: every policy must return the same alignment.
    d, cand = candidate_set(150, 10, 11, genome_markers=12000, n50=12000, min_bases=6000)
    cand = cand[:400]
    oo = B.make_align_options(alignMethod=3, k=10, minAlignedMarkerCount=30, minAlignedFraction=0.2)
    default = B.default_dp_policy()
    try:
        base = B.oracle_compute_alignments(d["toc"], d["kmer"], cand, oo, threads=4)
        ties = base[3]
        exposed = (ties & 6) != 0
        assert 0 < exposed.sum() < len(cand)        # some pairs are tie free, some are not
        kept = {tuple(r[:3]): (r.tobytes(), base[2][int(base[1][i]):int(base[1][i + 1])].tobytes()) for i, r in enumerate(base[0])}
        differing = set()
        for policy in range(8):
            if policy == default:
                continue
            B.set_dp_policy(policy)
            rec, ctoc, cdata, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], cand, oo, threads=4)
            other = {tuple(r[:3]): (r.tobytes(), cdata[int(ctoc[i]):int(ctoc[i + 1])].tobytes()) for i, r in enumerate(rec)}
            for key in set(kept) | set(other):
                if kept.get(key) != other.get(key):
                    differing.add(key)
        index = {tuple(int(x) for x in c): i for i, c in enumerate(cand)}
        for key in differing:
            assert exposed[index[key]], "a pair without tie flags changed under another tie-break policy"
    finally:
        B.set_dp_policy(default)


def test_candidate_table_oracle_against_direct_restatement():
    rng = np.random.default_rng(3)
    R = 40
    a = rng.integers(0, R, 300)
    b = rng.integers(0, R, 300)
    ok = a < b
    cand = np.unique(np.stack([a[ok], b[ok], rng.integers(0, 2, ok.sum())], 1), axis=0).astype(np.uint32)
    toc, table = B.oracle_compute_candidate_table(cand, R)
    rows = [[] for _ in range(2 * R)]
    for i, (r0, r1, same) in enumerate(cand.tolist()):
        o0, o1 = 2 * r0, 2 * r1 + (0 if same else 1)
        rows[o0].append((o1, i)); rows[o1].append((o0, i))
        rows[o0 ^ 1].append((o1 ^ 1, i)); rows[o1 ^ 1].append((o0 ^ 1, i))
    want = []
    for o in range(2 * R):
        assert toc[o] == len(want)
        want += [i for _, i in sorted(rows[o])]
    assert toc[-1] == len(want) == 4 * len(cand)
    assert table.tolist() == want
