"""Marker rows for the palindromic-read tests (tests/test_oracle_palindromic.py, tests/test_gpu_palindromic.py).

Each case is (toc uint64[2R+1], kmerIds uint32[], params dict of flagPalindromicReads); read r is rows 2r (strand 0)
and 2r+1 (strand 1). All rows come from fixed seeds."""
import numpy as np

K = 14


def reverse_complement(ids, k=K):
    ids = np.asarray(ids, np.uint64)
    out = np.zeros_like(ids)
    x = ids.copy()
    for _ in range(k):
        out = (out << np.uint64(2)) | (np.uint64(3) - (x & np.uint64(3)))
        x >>= np.uint64(2)
    return out.astype(np.uint32)


def rows_to_case(reads, **params):
    """reads: list of (strand0, strand1) id arrays."""
    toc = [0]
    ids = []
    for s0, s1 in reads:
        for s in (s0, s1):
            ids.append(np.asarray(s, np.uint32))
            toc.append(toc[-1] + len(s))
    return np.array(toc, np.uint64), (np.concatenate(ids) if ids else np.zeros(0, np.uint32)), params


def oriented(s0):
    """A read and its reverse complement, as the marker finder stores them."""
    return s0, reverse_complement(np.asarray(s0)[::-1])


def palindrome(rng, n, noise=0.02, k=K):
    """n markers whose second half is the reverse complement of the first, with a fraction noise of ids replaced."""
    s = rng.integers(0, 1 << (2 * k), n).astype(np.uint32)
    h = n // 2
    s[n - h:] = reverse_complement(s[:h][::-1], k)
    hit = rng.random(n) < noise
    s[hit] = rng.integers(0, 1 << (2 * k), int(hit.sum()))
    return s


def cases():
    rng = np.random.default_rng(2024)
    out = {}
    out["random"] = rows_to_case([oriented(rng.integers(0, 1 << (2 * K), int(rng.integers(20, 1500)))) for _ in range(40)])
    noisy = [oriented(palindrome(rng, n)) for n in (2, 7, 15, 16, 17, 33, 300, 2500, 4000)]
    noisy += [oriented(rng.integers(0, 1 << (2 * K), n)) for n in (16, 17, 900)]
    out["noisy_palindromes"] = rows_to_case(noisy)
    # Few distinct k-mers: streaks of every length, among them exactly maxMarkerFrequency and maxMarkerFrequency + 1,
    # with many equal keys for both unstable sorts to order.
    streaky = []
    for i in range(30):
        n = int(rng.integers(40, 400))
        alphabet = int(rng.integers(8, 40))
        s0 = rng.integers(0, alphabet, n).astype(np.uint32)
        if i % 2:
            s0[n // 2:] = s0[:n - n // 2][::-1]      # palindromic in marker space (ids equal their own complement here)
        streaky.append((s0, s0[::-1].copy()))
    out["streaks"] = rows_to_case(streaky, maxMarkerFrequency=4, maxSkip=30, maxDrift=30, deltaThreshold=20)
    # maxDrift < maxSkip enables the drift test; maxDrift >= maxSkip disables it.
    drift_reads = [oriented(palindrome(rng, int(rng.integers(50, 2000)), noise=0.1)) for _ in range(12)]
    out["drift_below_skip"] = rows_to_case(drift_reads, maxSkip=100, maxDrift=7)
    out["drift_above_skip"] = rows_to_case(drift_reads, maxSkip=50, maxDrift=200)
    out["zero_thresholds"] = rows_to_case(drift_reads[:6] + noisy[:4], alignedFractionThreshold=0.0,
                                          nearDiagonalFractionThreshold=0.0)
    # A zero-marker read, one-marker reads (matching and not), and a read whose V/n is exactly the threshold.
    ten = rng.integers(0, 1 << (2 * K), 10).astype(np.uint32)
    half = np.concatenate([ten[:5], rng.integers(1 << 27, 1 << 28, 5).astype(np.uint32)])
    out["tiny"] = rows_to_case([(ten[:0], ten[:0]), (ten[:1], ten[:1]), (ten[:1], ten[1:2]), (ten, half[::-1].copy())],
                               alignedFractionThreshold=0.5, nearDiagonalFractionThreshold=0.0)
    return out


def killer_case(killer_keys):
    """A read whose strand-0 row drives introsort to its depth limit (keys from oracle_sort_killer_keys)."""
    s0 = np.asarray(killer_keys, np.uint32)
    return rows_to_case([(s0, s0[::-1].copy()), oriented(palindrome(np.random.default_rng(7), 600))])
