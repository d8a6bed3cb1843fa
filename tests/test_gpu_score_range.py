"""The alignment DP at the edges of its score range.

The DP kernels run in int32 and stand for "minus infinity" with sentinels: kNegInf = -2^29 for cells outside the matrix,
the gap score kGapBarrier = -2^28 on the two barrier offsets beside a wavefront band, -2^30 for "no end cell yet", and the
scan kernel adds e * gap to every cell of a column. computeAlignments therefore refuses scores with
M * (2L + 16384) >= 2^28 (M = max |score|, L = the longest read the call aligns, in markers; derivation in
csrc/align.cu).

Host part (no GPU):
- exact_dp states the banded overlap DP of the oracle (default tie-break policy) in int64 numpy, with have-flags and no
  sentinels. On every DP problem the GPU part runs, the oracle's score and path equal it: the oracle does not overflow.
- kernel_model restates the recurrence as the kernels compute it: the wavefront kernels' physical offsets with the two
  barriers, unmasked cells above and below the matrix, the lanes' skewed start and the wrap-around shuffles of the first
  and last lane; the scan kernel's A - e * gap prefix maximum in wrapping int32; the -2^30 end-cell start; the traceback
  on the 2-bit codes. At the largest scores the bound admits it equals exact_dp on every problem and no value leaves
  int32; at twice those scores, on a long exact run one offset outside a stage-2 band, a barrier value leaks into the band
  and the model stores a different alignment: by the model, the refusal is needed, and the bound is within a small factor
  of the edge. Only this model tests how close a barrier comes to a real score; the GPU never runs scores beyond the bound.
- The shipped configurations sit far inside the bound, and every case reaches the path it is built for.

GPU part (-m gpu): device/oracle parity, bit for bit, at the largest scores the bound admits, under methods 1 and 3 and
through the single-pair entry point, on four families: (a) reads against identical copies (scores up to +L*M); (b) a shared
seed followed by unrelated tails, so that the stage-2 band holds no boundary end cell and every end cell is reached through
a long mismatch run; (c) a long exact run of k-mers the downsampling drops, one offset outside the stage-2 band on either
side; (d) the widest bands (method 1 at 16 381 offsets, stage 2 at maxBand 16 317). One score step beyond the bound, each
family is refused with SHB_ERR_INVALID before any kernel runs, and the same context then aligns correctly. Out-of-range
scores never reach the kernels on the GPU.
For reads of a few thousand markers the 16384 term of the bound sets M, so the real scores there stay far from the barrier
(copies: L = 3000, M = 11 992, scores up to 36 M against -2^28); what these cases test at full range is the scan kernel's
e * gap transform and the int32 range of the recurrence. Only the widest family brings 2 * L * M near 2^27."""
import functools
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import bindings as B  # noqa: E402
from support import (CONFIGS, FORWARD_MAX_MARKERS, FORWARD_MAX_ROWS, K, MAX_BAND_WIDTH, PERMISSIVE, assemble,  # noqa: E402,F401
                     compare_alignments, ctx, downsampled, downsampling_hash, downsampling_threshold, expected_single_pair,
                     padded_width, single_pair_options, wide_band_class)

SCORE_LIMIT = 1 << 28
NEG_INF, GAP_BARRIER, END_NONE = -(1 << 29), -(1 << 28), -(1 << 30)     # kNegInf, kGapBarrier, kNegInf * 2
INT32 = (-(1 << 31), (1 << 31) - 1)
DROP_FACTOR = 0.5           # tails and runs use k-mers this downsampling (and every smaller factor) drops


def in_bound(m, longest):
    return m * (2 * longest + MAX_BAND_WIDTH) < SCORE_LIMIT


def largest_score(longest):
    """The largest M the bound admits for reads of up to `longest` markers."""
    return (SCORE_LIMIT - 1) // (2 * longest + MAX_BAND_WIDTH)


def score_opts(m):
    return dict(matchScore=m, mismatchScore=-m, gapScore=-m)


# ---- exact DP ----------------------------------------------------------------------------------------------------------
VERT, HORZ, DIAG = 1, 2, 0


def exact_dp(a, b, match, mismatch, gap, band=None):
    """The oracle's banded overlap DP (orc_overlap_align) under the default policy, in int64: diagonal wins ties with a
    gap move, vertical wins ties with horizontal, the end cell is the first strict maximum in column-major order over the
    last row and the last column. Returns (score, (i, j), path int64[n, 2] of the diagonal steps), or None."""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    nx, ny = len(a), len(b)
    lo, hi = band if band is not None else (-ny, nx)
    if lo > hi or hi < -ny or lo > nx:
        return None
    lo, hi = max(lo, -ny), min(hi, nx)
    none = np.int64(-(1 << 62))
    codes, ranges = [], []
    prev, prev_lo, prev_hi = np.array([none]), 0, -1
    best = None
    for i in range(nx + 1):
        jlo, jhi = max(0, i - hi), min(ny, i - lo)
        j = np.arange(jlo, jhi + 1)
        if i == 0 or jlo > jhi:
            H = np.zeros(len(j), np.int64)
            code = np.zeros(len(j), np.int8)
        else:
            inner = j >= 1
            jj = np.maximum(j, 1)
            d = np.where(inner, prev[np.clip(jj - 1 - prev_lo, 0, len(prev) - 1)] + np.where(a[i - 1] == b[jj - 1], match, mismatch), 0)
            have_h = (j >= prev_lo) & (j <= prev_hi)
            h = np.where(have_h, prev[np.clip(j - prev_lo, 0, max(len(prev) - 1, 0))] + gap, none)
            A = np.where(inner, np.maximum(d, h), 0)
            H = gap * j + np.maximum.accumulate(A - gap * j)       # H(j) = max(A(j), H(j-1) + gap); j = 0 comes first
            v = np.concatenate([[none], H[:-1] + gap])
            g = np.maximum(v, h)
            code = np.where(d >= g, DIAG, np.where(v >= h, VERT, HORZ)).astype(np.int8)
        codes.append(code)
        ranges.append(jlo)
        if len(j):
            cells = [(len(j) - 1)] if (i < nx and jhi == ny) else (range(len(j)) if i == nx else [])
            for k in cells:
                if best is None or H[k] > best[0]:
                    best = (int(H[k]), i, int(j[k]))
        prev, prev_lo, prev_hi = (H if len(H) else np.array([none])), jlo, jhi
    if best is None:
        return None
    score, i, j = best
    path = []
    while i > 0 and j > 0:
        c = codes[i][j - ranges[i]]
        if c == DIAG:
            path.append((i - 1, j - 1))
            i, j = i - 1, j - 1
        elif c == VERT:
            j -= 1
        else:
            i -= 1
    return score, (best[1], best[2]), np.array(path[::-1], np.int64).reshape(-1, 2)


# ---- the kernels' arithmetic -------------------------------------------------------------------------------------------
def band_shape(lo, hi):
    """(lanes, c, padded width) of a band (dpBandShape); c = 0 is the scan kernel."""
    need = hi - lo + 3
    if need <= 128:
        return 8, max(2, -(-need // 16)), padded_width(hi - lo + 1)
    return 32, next((c for c in (3, 4, 6, 8, 12, 16) if need <= 64 * c), 0), padded_width(hi - lo + 1)


def _row_kmers(b, j):
    """b[j - 1] for rows j, 0xffffffff outside 1 .. ny (the kernels' sentinel)."""
    idx = j - 1
    ok = (idx >= 0) & (idx < len(b))
    return np.where(ok, b[np.clip(idx, 0, max(len(b) - 1, 0))], 0xffffffff)


class _Range:
    def __init__(self):
        self.lo, self.hi = 0, 0

    def see(self, *xs):
        for x in xs:
            if len(x):
                self.lo, self.hi = min(self.lo, int(x.min())), max(self.hi, int(x.max()))

    def wrapped(self):
        return self.lo < INT32[0] or self.hi > INT32[1]


def _wavefront(a, b, match, mismatch, gap, lo, hi):
    """bandedOverlapDpSystolic in exact int64, with the range of every value it forms (the kernel wraps at int32)."""
    nx, ny = len(a), len(b)
    G, C, _ = band_shape(lo, hi)
    W, n = hi - lo + 1, 2 * G * C
    p = np.arange(n)
    e = p - 1
    inband = (e >= 0) & (e < W)
    first = np.where(inband, np.maximum(0, hi - e), 1 << 40)         # column of the cell's boundary cell
    g = np.where((e == -1) | (e == W), GAP_BARRIER, gap).astype(np.int64)
    S = np.cumsum(g)
    lane = p // (2 * C)
    i_first, i_last = max(0, lo), min(nx, ny + hi)
    H = np.full(n, NEG_INF, np.int64)
    rng = _Range()
    codes, best = {}, None
    big = np.int64(1 << 50)
    for i in range(i_first - (G - 1), i_last + 1):
        p0 = 2 * C * max(0, i_first - i)                              # lanes start G - 1 .. 0 columns early, lane G-1 first
        ai = int(a[i - 1]) if 1 <= i <= nx else 0xfffffffe
        bw = _row_kmers(b, e + i - hi)
        d1 = H + mismatch
        diag = np.where(bw == ai, d1 + (match - mismatch), d1)
        horz = np.concatenate([H[1:], [0]])                           # (i-1, p+1); the last offset's is set below
        vin = H[2 * C - 1] if p0 == 0 else H[p0 - 1]                  # lane 0 reads its own previous B; or a lane not started
        s = slice(p0, n - 1)
        x = np.maximum(diag[s], horz[s] + g[s])
        x[0] = max(x[0], vin + g[p0])
        reset = (first[s] == i)
        seg = np.cumsum(reset).astype(np.int64)
        y = np.where(reset, -S[s], x - S[s]) + seg * big
        h = np.maximum.accumulate(y) - seg * big + S[s]
        Hn = H.copy()
        Hn[s] = h
        top = Hn[2 * C * (G - 1)]                                     # lane G-1 reads its own A of this column
        horz[n - 1] = top
        Hn[n - 1] = max(diag[n - 1], max(Hn[n - 2], top) + g[n - 1])
        vert = np.concatenate([[vin], Hn[p0:n - 1]])
        gap_in = np.maximum(vert, horz[p0:]) + g[p0:]
        rng.see(d1[p0:], diag[p0:], gap_in, Hn[p0:])
        code = np.zeros(n, np.int8)
        code[p0:] = (gap_in > diag[p0:]).astype(np.int8) | ((horz[p0:] > vert).astype(np.int8) << 1)
        if i >= 1:
            codes[i] = code
        if 0 <= i <= nx:
            j = e + i - hi
            cand = inband & (i >= first) & (j <= ny) & ((j == ny) | (i == nx)) & (p >= p0)
            for k in np.flatnonzero(cand):                             # column-major: j ascending
                if (best is None and Hn[k] >= END_NONE) or (best is not None and Hn[k] > best[0]):
                    best = (int(Hn[k]), i, int(j[k]))
        H = Hn
    return best, codes, (lambda i, j: j - i + hi + 1), n, rng


def _scan(a, b, match, mismatch, gap, lo, hi):
    """bandedOverlapDp (the scan kernel) in wrapping int32, as the kernel computes it."""
    nx, ny = len(a), len(b)
    W = hi - lo + 1
    _, _, wpad = band_shape(lo, hi)
    i32 = np.int32
    e = np.arange(wpad, dtype=i32)
    eg = e * i32(gap)
    h_prev = np.full(wpad + 1, NEG_INF, i32)
    rng = _Range()
    codes, best = {}, None
    with np.errstate(over="ignore"):
        for i in range(nx + 1):
            j = e.astype(np.int64) + i - hi
            valid = (e < W) & (j >= 0) & (j <= ny)
            boundary = (j == 0) | (i == 0)
            ai = int(a[i - 1]) if i > 0 else 0
            d = h_prev[:wpad] + np.where(_row_kmers(b, j) == ai, i32(match), i32(mismatch)).astype(i32)
            horz = h_prev[1:] + i32(gap)
            A = np.where(valid, np.where(boundary, i32(0), np.maximum(d, horz)), i32(NEG_INF)).astype(i32)
            P = np.maximum(np.maximum.accumulate(A - eg), i32(END_NONE))
            H = (P + eg).astype(i32)
            H = np.where(valid, np.where(boundary, i32(0), H), i32(NEG_INF)).astype(i32)
            vert = np.concatenate([[i32(NEG_INF)], H[:-1]]).astype(i32) + i32(gap)
            wide = np.int64
            d64 = h_prev[:wpad].astype(wide) + np.where(_row_kmers(b, j) == ai, match, mismatch)
            rng.see(A[valid].astype(wide) - eg[valid].astype(wide), d64[valid], P.astype(wide) + eg.astype(wide))
            code = np.where(valid & ~boundary, (np.maximum(horz, vert) > d).astype(np.int8) | ((horz > vert).astype(np.int8) << 1), 0)
            codes[i] = code.astype(np.int8)
            if i == nx:
                for k in np.flatnonzero(valid):
                    if (best is None and H[k] > END_NONE) or (best is not None and H[k] > best[0]):
                        best = (int(H[k]), i, int(j[k]))
            else:
                k = ny - i + hi
                if 0 <= k < W and (best is None and H[k] > END_NONE or best is not None and H[k] > best[0]):
                    best = (int(H[k]), i, ny)
            h_prev[:wpad] = H
    return best, codes, (lambda i, j: j - i + hi), wpad, rng


def kernel_model(a, b, match, mismatch, gap, band=None):
    """The DP as the device computes it. Returns dict(result=(score, (i, j), path) or None, kernel, wrapped, escaped):
    wrapped = a value left int32 (the wavefront model is exact in int64, the kernel would wrap); escaped = the traceback
    left the trace (a leaked barrier value steered it out of the band)."""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    nx, ny = len(a), len(b)
    lo, hi = band if band is not None else (-ny, nx)
    lo, hi = max(lo, -ny), min(hi, nx)
    _, c, _ = band_shape(lo, hi)
    best, codes, offset, width, rng = (_wavefront if c else _scan)(a, b, match, mismatch, gap, lo, hi)
    out = dict(kernel="wavefront" if c else "scan", wrapped=rng.wrapped(), escaped=False, result=None)
    if best is None:
        return out
    i, j = best[1], best[2]
    path = []
    while i > 0 and j > 0:
        q = offset(i, j)
        if i not in codes or not 0 <= q < width:
            out["escaped"] = True
            break
        code = codes[i][q]
        if not code & 1:
            path.append((i - 1, j - 1))
            i, j = i - 1, j - 1
        elif code & 2:
            i -= 1
        else:
            j -= 1
    out["result"] = (best[0], (best[1], best[2]), np.array(path[::-1], np.int64).reshape(-1, 2))
    return out


def same_result(x, y):
    if x is None or y is None:
        return x is None and y is None
    return x[0] == y[0] and x[1] == y[1] and np.array_equal(x[2], y[2])


# ---- the families ------------------------------------------------------------------------------------------------------
class Pool:
    """Distinct random k-mer ids, optionally only ones the downsampling at DROP_FACTOR drops."""

    def __init__(self, seed):
        self.ids = np.random.default_rng(seed).permutation(1 << (2 * K)).astype(np.uint32)
        self.used = np.zeros(len(self.ids), bool)

    def take(self, n, dropped=False):
        ok = ~self.used
        if dropped:
            ok &= downsampling_hash(self.ids, K) >= downsampling_threshold(DROP_FACTOR)
        pick = np.flatnonzero(ok)[:n]
        assert len(pick) == n
        self.used[pick] = True
        return self.ids[pick]


M3 = dict(PERMISSIVE, alignMethod=3, downsamplingFactor=0.1, bandExtend=10, maxBand=1000)
M3_TRACED = dict(M3, downsamplingFactor=DROP_FACTOR, bandExtend=200)
M1 = dict(PERMISSIVE, alignMethod=1)
WIDE_EXTEND, WIDE_MAX_BAND = 8158, 16317


@functools.lru_cache(None)
def family(name):
    """(rows, candidates, option sets) of a family; every candidate is (2i, 2i+1, same strand)."""
    pool = Pool({"copies": 1, "tails": 2, "outside": 3, "widest": 4}[name])
    pairs, opts = [], [M1, M3]
    if name == "copies":            # (a) values up to +L*M; method 1 on the 8-lane, whole-warp and scan classes
        for n in (40, 300, 3000):
            x = pool.take(n)
            pairs.append((x, x.copy()))
        opts = [M1, M3, M3_TRACED]
    elif name == "tails":           # (b) seed, then long unrelated tails that stage 1 does not see
        for seed, tail in ((30, 300), (200, 2800)):
            s = pool.take(seed)
            pairs.append((np.concatenate([s, pool.take(tail, True)]), np.concatenate([s, pool.take(tail + 7, True)])))
    elif name == "outside":         # (c) an exact run on the diagonal just below (lo - 1) or above (hi + 1) the band
        ext = M3["bandExtend"]
        for seed, run in ((120, 400), (200, 2800)):
            s, r, z = pool.take(seed), pool.take(run, True), pool.take(ext + 1, True)
            pairs.append((np.concatenate([s, r]), np.concatenate([s, z, r])))
            s, r, z = pool.take(seed), pool.take(run, True), pool.take(ext + 1, True)
            pairs.append((np.concatenate([s, z, r]), np.concatenate([s, r])))
        opts = [M3]
    elif name == "widest":          # (d) method 1 at 16 381 offsets, stage 2 at 16 317
        x = pool.take(8190)
        pairs.append((x, x.copy()))
        opts = [M1, dict(M3, bandExtend=WIDE_EXTEND, maxBand=WIDE_MAX_BAND)]
    rows = [r for pair in pairs for r in pair]
    cand = np.array([(2 * k, 2 * k + 1, 1) for k in range(len(pairs))], np.uint32)
    return rows, cand, opts


FAMILIES = ("copies", "tails", "outside", "widest")


def longest(name):
    return max(len(r) for r in family(name)[0])


def family_scores(name):
    return score_opts(largest_score(longest(name)))


def dp_problems(a, b, opts, sc):
    """The DP problems the device runs for one candidate: [(kind, a, b, band or None)], kind in 'method1', 'forward',
    'traced', 'stage2'. Method 3's stage-2 band comes from the exact stage-1 path (src/AssemblerAlign3.cpp:193-239)."""
    if opts["alignMethod"] == 1:
        return [("method1", a, b, None)]
    (da, oa), (db, ob) = downsampled(a, opts["downsamplingFactor"]), downsampled(b, opts["downsamplingFactor"])
    if not len(da) or not len(db):
        return []
    traced = len(db) > FORWARD_MAX_ROWS or max(len(a), len(b)) > FORWARD_MAX_MARKERS
    out = [("traced" if traced else "forward", da, db, None)]
    r = exact_dp(da, db, *sc)
    eq = da[r[2][:, 0]] == db[r[2][:, 1]] if len(r[2]) else np.zeros(0, bool)
    if eq.any():
        off = oa[r[2][eq, 0]] - ob[r[2][eq, 1]]
        lo, hi = int(off.min()) - opts["bandExtend"], int(off.max()) + opts["bandExtend"]
        if hi - lo <= opts["maxBand"]:
            out.append(("stage2", a, b, (lo, hi)))
    return out


@functools.lru_cache(None)
def problems(name):
    rows, cand, opts = family(name)
    sc = tuple(family_scores(name).values())
    out = []
    for o in opts:
        for r0, r1, _ in cand:
            # both orders: computeAlignments runs (r0, r1), the single-pair test also (r1, r0); a read against its own
            # copy gives the same problem either way
            orders = [(r0, r1)] + ([] if np.array_equal(rows[r0], rows[r1]) else [(r1, r0)])
            for x, y in orders:
                for kind, a, b, band in dp_problems(rows[x], rows[y], o, sc):
                    out.append((o["alignMethod"], kind, a, b, band, exact_dp(a, b, *sc, band=band)))
    return sc, out


# ---- host tests --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FAMILIES)
def test_exact_dp_matches_oracle(name):
    # The oracle uses int32 with have-flags: at these scores it must not overflow (undefined behaviour) anywhere.
    sc, probs = problems(name)
    assert len(probs) >= 2
    for method, kind, a, b, band, want in probs:
        score, path = B.overlap_align(a, b, *sc, band=band)
        assert want is not None and score == want[0], (name, method, kind, band)
        assert np.array_equal(path.astype(np.int64), want[2]), (name, method, kind, band)


@pytest.mark.parametrize("name", FAMILIES)
def test_kernel_model_is_exact_at_the_bound(name):
    sc, probs = problems(name)
    assert in_bound(sc[0], longest(name)) and not in_bound(sc[0] + 1, longest(name))
    for method, kind, a, b, band, want in probs:
        if kind == "forward":           # the forward kernel has no sentinels: values within +-L*M, exact by range alone
            continue
        got = kernel_model(a, b, *sc, band=band)
        assert not got["wrapped"] and not got["escaped"], (name, method, kind, band)
        assert same_result(got["result"], want), (name, method, kind, band, got["kernel"])


def leak_case(run):
    """A seed of 200 k-mers, then an exact run of `run` k-mers on the diagonal one offset outside a band of +-10, on the
    barrier side of each edge: the barrier gains match after match while every in-band cell loses."""
    pool = Pool(5)
    s, r, z = pool.take(200), pool.take(run, True), pool.take(11, True)
    below = (np.concatenate([s, r]), np.concatenate([s, z, r]))
    s, r, z = pool.take(200), pool.take(run, True), pool.take(11, True)
    above = (np.concatenate([s, z, r]), np.concatenate([s, r]))
    return [below, above]


def test_kernel_model_diverges_beyond_the_bound():
    # At the largest scores the bound admits, the model is exact on reads of 16 211 markers; at twice those scores (the
    # refusal's side), the barrier's value on the exact run overtakes the in-band cells, and the model of the kernels takes
    # a barrier move and stores a different alignment. This is the model's prediction; it is not run on the device.
    diverged = []
    for a, b in leak_case(16000):
        L = max(len(a), len(b))
        m = largest_score(L)
        for factor, expect_exact in ((1, True), (2, False)):
            sc = (factor * m, -factor * m, -factor * m)
            assert in_bound(sc[0], L) == expect_exact
            want = exact_dp(a, b, *sc, band=(-10, 10))
            got = kernel_model(a, b, *sc, band=(-10, 10))
            assert not got["wrapped"]                       # the divergence is the barrier's, not a wrap-around
            assert want is not None and len(want[2]) > 100
            if expect_exact:
                assert same_result(got["result"], want) and not got["escaped"]
            else:
                diverged.append(got["escaped"] or not same_result(got["result"], want))
    assert any(diverged), "the model did not diverge beyond the bound"


def test_scan_kernel_wraps_far_beyond_the_bound():
    # Failure mode of the scan kernel: with |e * gap| plus a cell value reaching 2^31 its prefix maximum compares wrapped
    # values. A read against its copy in a 2 049-offset band (the scan kernel) at M = 2^20, 200 times the bound's M.
    x = Pool(6).take(1024)
    sc = (1 << 20, -(1 << 20), -(1 << 20))
    assert not in_bound(sc[0], len(x)) and band_shape(-1024, 1024)[1] == 0
    got = kernel_model(x, x, *sc, band=(-1024, 1024))
    assert got["wrapped"] and not same_result(got["result"], exact_dp(x, x, *sc, band=(-1024, 1024)))


def test_shipped_configurations_sit_far_inside_the_bound():
    sets = [dict(B.ALIGN_DEFAULTS, **cfg["align"]) for cfg in CONFIGS.values()] + [dict(bench.ALIGN_DEFAULT)]
    for o in sets:
        m = 6 if o["alignMethod"] == 4 else max(abs(o["matchScore"]), abs(o["mismatchScore"]), abs(o["gapScore"]))
        assert m == 6
        assert 5 * m * (2 * 4_000_000 + MAX_BAND_WIDTH) < SCORE_LIMIT        # reads of 4 M markers, 5x margin
        assert in_bound(m, (1 << 24) - 1)                                        # every read the reference can store
    assert largest_score(4_000_000) >= 30


def test_cases_reach_their_paths():
    kinds, classes = set(), set()
    for name in FAMILIES:
        sc, probs = problems(name)
        m, L = sc[0], longest(name)
        widths = []
        for method, kind, a, b, band, want in probs:
            kinds.add((method, kind))
            lo, hi = band if band else (-len(b), len(a))
            lo, hi = max(lo, -len(b)), min(hi, len(a))
            widths.append(hi - lo + 1)
            if kind != "forward":
                lanes, c, _ = band_shape(lo, hi)
                classes.add((kind, "scan" if c == 0 else lanes))
        stage2 = [p for p in probs if p[1] == "stage2"]
        if name == "copies":            # a read against its copy ends at (nx, ny) with +L*M
            assert max(p[5][0] for p in probs) == L * m
        if name == "tails":             # no boundary end cell in the band; the best end is far below zero
            assert len(stage2) == 4
            for _, _, a, b, (lo, hi), want in stage2:
                assert lo > -len(b) and hi < len(a) and want[0] < -(len(a) // 2) * m
        if name == "outside":           # the exact run is one offset outside the band, below it and above it
            sides = []
            for _, _, a, b, (lo, hi), _ in stage2:
                off = np.unique(exact_dp(a, b, *sc)[2] @ np.array([1, -1]))
                sides.append((lo - 1 in off, hi + 1 in off))
            assert len(stage2) == 8 and (True, False) in sides and (False, True) in sides
        if name == "widest":
            assert sorted(widths)[-2:] == [WIDE_MAX_BAND, 16381]
            assert wide_band_class(16381) == wide_band_class(WIDE_MAX_BAND) == 16384
    assert {(1, "method1"), (3, "forward"), (3, "traced"), (3, "stage2")} <= kinds
    assert {("method1", 8), ("method1", 32), ("method1", "scan"), ("stage2", 8), ("stage2", 32), ("stage2", "scan"),
            ("traced", "scan")} <= classes


# ---- GPU tests ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", FAMILIES)
def test_device_matches_oracle_at_the_bound(ctx, name):
    rows, cand, opts = family(name)
    d = assemble(rows, K)
    for o in opts:
        compare_alignments(ctx, d, cand, **o, **family_scores(name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", FAMILIES)
def test_single_pair_at_the_bound(ctx, name):
    from shasta_b200 import capi
    rows, cand, opts = family(name)
    d = assemble(rows, K)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    stored = 0
    for o in opts:
        o = dict(o, **family_scores(name))
        go = capi.make_align_options(**o)
        for r0, r1, _ in cand:
            for o0, o1 in ((2 * int(r0), 2 * int(r1)), (2 * int(r1), 2 * int(r0))):
                ords, info = capi.align_oriented_reads(ctx, o0, o1, go)
                exp = expected_single_pair(rows[o0 // 2], rows[o1 // 2], o)
                if exp is None:
                    assert len(ords) == 0 and not info.any(), (o0, o1)
                    continue
                stored += 1
                assert np.array_equal(info, exp[0][3:16]), (o0, o1)
                assert np.array_equal(ords, exp[1]), (o0, o1)
    assert stored >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("name", FAMILIES)
def test_refused_beyond_the_bound(ctx, name):
    from shasta_b200 import capi
    rows, cand, opts = family(name)
    d = assemble(rows, K)
    ctx.set_markers(d["toc"], d["data"], d["flags"])
    m = largest_score(longest(name)) + 1
    for o in opts:
        for sc in (score_opts(m), dict(matchScore=1, mismatchScore=-1, gapScore=-m), dict(matchScore=-m, mismatchScore=0, gapScore=0)):
            go = capi.make_align_options(**o, **sc)
            with pytest.raises(capi.ShastaB200Error, match="scores too large") as err:
                capi.compute_alignments(ctx, cand, go)
            assert err.value.status == 1                                    # SHB_ERR_INVALID
            with pytest.raises(capi.ShastaB200Error, match="scores too large"):
                capi.align_oriented_reads(ctx, 2 * int(cand[-1, 0]), 2 * int(cand[-1, 1]), go)   # the longest pair
    # Only the reads a call aligns count: a pair of shorter reads is within the bound at these scores.
    if len(cand) > 1:
        short = max(len(rows[int(cand[0, 0])]), len(rows[int(cand[0, 1])]))
        assert in_bound(m, short)
        compare_alignments(ctx, d, cand[:1], **opts[0], **score_opts(m))
    # Align4 scores 6/-1/-1 whatever the options say: never refused for them, and bit-exact with the oracle's Align4,
    # which hard-codes those scores too.
    compare_alignments(ctx, d, cand, **dict(single_pair_options(4), **score_opts(m)))
    # The same context then aligns in range, bit-exact.
    compare_alignments(ctx, d, cand, **opts[-1], **family_scores(name))
