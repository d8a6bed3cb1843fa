"""The alignment kernels under all eight DP tie-break policies (include/shb_dp_policy.h), against the oracle.

The policy is a compile-time choice of the kernels: build() makes shasta_b200/lib/dp_policy/libshasta_b200_policy<N>.so for
the seven non-default policies N (bit 0 SHB_DP_DIAG_WINS_TIES, bit 1 SHB_DP_VERT_BEFORE_HORZ, bit 2 SHB_DP_END_FIRST_MAX);
policy 7, the default, is the production library. capi loads one library per process, so each policy runs in a
subprocess (this file run as a script) that writes its outputs, and the test compares them bit for bit with the
oracle's under B.set_dp_policy(N): records, compressed toc and bytes, and the device digests.

Most cases run on reads cut from a genome of eight k-mer ids, where ties are everywhere. They cover every kernel whose
output depends on the policy: method 3 stage 2 on the 8-lane group classes, the whole-warp classes and the scan kernel;
method 3 stage 1 on the forward kernel (groups of 8, 16 and 32 lanes) and on the traced path; method 1 up to the scan
kernel; method 4; the single-pair entry point with methods 1, 3 and 4; eight score sets, from the shipped 6/-1/-1 to 0/0/0,
2/5/-1 (a mismatch above a match), 6/0/0 and 1/-1000/-1; the k = 10 synthetic reads; and
pairs built so that the best end score is 0 and is reached both in the last row and at the boundary cell (nx, 0), where
the last-maximum end-cell rule must pick (nx, 0) and store nothing.

The host checks (no GPU) make sure each case reaches its path, that each policy bit on its own changes the oracle's stored
output somewhere in the cases (so a variant that ignores a bit or has it backwards fails), and that the end-cell pairs
are what they are built to be, against a plain numpy statement of the DP."""
import functools
import os
import subprocess
import sys
from typing import Callable, NamedTuple

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _path in (HERE, ROOT):                      # run as the per-policy subprocess
    if _path not in sys.path:
        sys.path.insert(0, _path)

from oracle import bindings as B  # noqa: E402
from support import (PERMISSIVE, K, Genome, assemble, candidate_set, downsampled, downsampling_hash,  # noqa: E402
                     downsampling_threshold, expected_single_pair, oracle_options, row, single_pair_options)

DEFAULT_POLICY = 7
POLICY_DIR = os.path.join(ROOT, "shasta_b200", "lib", "dp_policy")
# The shipped 6/-1/-1 and variants, then unusual but legal sets: every path ties (0/0/0), a mismatch scoring above a match
# (2/5/-1: stage-1 paths of diagonal steps with no matching k-mer, whose band wraps around and is skipped), free gaps and
# mismatches (6/0/0), and a mismatch far costlier than a gap (1/-1000/-1).
SCORES = {"6_1_1": (6, -1, -1), "6_1_3": (6, -1, -3), "6_1_0": (6, -1, 0), "3_2_1": (3, -2, -1),
          "0_0_0": (0, 0, 0), "2_5_1": (2, 5, -1), "6_0_0": (6, 0, 0), "1_1000_1": (1, -1000, -1)}
FORWARD_GROUPS = ((128, 8), (256, 16), (512, 32))      # dpForwardClassAt: rows held by groups of 8, 16, 32 lanes
SCAN_MIN_WIDTH = 1023                                   # bands of more offsets run on the scan kernel (dpClassAt)


def policy_library(policy):
    if policy == DEFAULT_POLICY:
        return os.path.join(ROOT, "shasta_b200", "lib", "libshasta_b200.so")
    return os.path.join(POLICY_DIR, f"libshasta_b200_policy{policy}.so")


def scores(name):
    m, x, g = SCORES[name]
    return dict(matchScore=m, mismatchScore=x, gapScore=g)


# ---- datasets --------------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def k10_set():
    """The k = 10 synthetic reads with their LowHash candidates."""
    return candidate_set(150, K, 11, genome_markers=12000, n50=12000, min_bases=6000)


def few_kmer_values(count, factor, seed, kept=True):
    """`count` k-mer ids that the downsampling at `factor` keeps (kept) or drops."""
    ids = np.random.default_rng(seed).integers(0, 1 << (2 * K), 256).astype(np.uint32)
    keep = downsampling_hash(ids, K) < downsampling_threshold(factor)
    return ids[keep == kept][:count]


TIE_FACTOR = 0.5
TIE_LENGTHS = (20, 35, 60, 110, 200, 260, 400, 520, 700, 900, 1100, 1300, 1600, 2000)
TIE_STARTS = (40, 50, 0, 30, 100, 150, 250, 300, 400, 500, 600, 800, 900, 1000)


@functools.lru_cache(None)
def tie_set():
    """Reads of 20 to 2 000 markers cut from a genome of eight k-mer ids (inserted markers are random), four of which the
    downsampling at TIE_FACTOR keeps: ties everywhere, in both stages of method 3. Every pair on the same strand, and a
    few on opposite strands."""
    genome = Genome(6000, seed=5, drop=0.04, ins=0.02)
    values = np.concatenate([few_kmer_values(4, TIE_FACTOR, 3), few_kmer_values(4, TIE_FACTOR, 3, kept=False)])
    genome.kmer = genome.rng.choice(values, len(genome.kmer)).astype(np.uint32)
    rows = [genome.read(s, L)[0] for s, L in zip(TIE_STARTS, TIE_LENGTHS)]
    n = len(rows)
    cand = [(i, j, 1) for i in range(n) for j in range(i + 1, n)] + [(i, i + 1, 0) for i in range(0, n - 1, 3)]
    return assemble(rows, K), np.array(cand, np.uint32)


END_CELL_M = (1, 5, 20, 40, 75)        # ny = 7m: forward groups of 8, 8, 16, 32 lanes; 525 > 512 rows: the traced path


def end_cell_rows(m, rng):
    """a = m shared k-mers + 8m found nowhere else, b = the same m + 6m found nowhere else (6/-1/-1): the best end score is
    0, reached in row ny (from (m, m), 6m steps of -1) and at the boundary cell (nx, 0); column nx is negative above row 0."""
    ids = rng.choice(1 << (2 * K), 15 * m, replace=False).astype(np.uint32)
    return np.concatenate([ids[:m], ids[m:9 * m]]), np.concatenate([ids[:m], ids[9 * m:]])


@functools.lru_cache(None)
def end_cell_set():
    rng = np.random.default_rng(37)
    rows = []
    for m in END_CELL_M:
        rows += end_cell_rows(m, rng)
    return assemble(rows, K), np.array([(2 * i, 2 * i + 1, 1) for i in range(len(END_CELL_M))], np.uint32)


TIE_PAIRS = ((2, 5), (4, 9), (6, 8), (8, 9), (3, 4), (0, 2))


@functools.lru_cache(None)
def tie_pair_set():
    """Single-pair calls on the tie-rich reads: both orders on both strands, and reads against their reverse complement."""
    d, _ = tie_set()
    pairs = []
    for i, j in TIE_PAIRS:
        pairs += [(2 * i, 2 * j), (2 * j, 2 * i), (2 * i + 1, 2 * j + 1), (2 * j + 1, 2 * i + 1)]
    pairs += [(6, 7), (15, 14)]
    return d, np.array(pairs, np.int64)


# ---- cases -----------------------------------------------------------------------------------------------------------
class Case(NamedTuple):
    name: str
    data: Callable              # () -> (markers, candidates), or (markers, oriented read pairs) when oriented
    opts: dict
    oriented: bool = False


M3_TIES = dict(PERMISSIVE, alignMethod=3, downsamplingFactor=TIE_FACTOR, maxBand=2000)
TIE_EXTENDS = (2, 10, 30, 100, 600)     # stage-2 bands on the 8-lane groups, the whole-warp classes and the scan kernel
END_CELL_OPTS = dict(PERMISSIVE, alignMethod=3, downsamplingFactor=1.0, bandExtend=2, maxBand=1000)


def k10_candidates():
    d, cand = k10_set()
    return d, cand[:300]


def cases():
    # Method 3 on the tie-rich reads: stage 1 on every forward class and on the traced path, stage 2 on every band class.
    out = [Case(f"m3_ties_e{e}", tie_set, dict(M3_TIES, bandExtend=e)) for e in TIE_EXTENDS]
    for s in SCORES:
        out.append(Case(f"m1_ties_s{s}", tie_set, dict(PERMISSIVE, alignMethod=1, **scores(s))))
        if s != "6_1_1":
            out.append(Case(f"m3_ties_s{s}", tie_set, dict(M3_TIES, bandExtend=10, **scores(s))))
    out.append(Case("m4_ties", tie_set, single_pair_options(4)))
    for s in ("6_1_1", "6_1_3"):
        out.append(Case(f"m3_k10_s{s}", k10_candidates, dict(PERMISSIVE, alignMethod=3, minAlignedMarkerCount=30,
                                                           minAlignedFraction=0.2, **scores(s))))
    out.append(Case("m4_k10", k10_candidates, single_pair_options(4)))
    out.append(Case("m3_end_cell", end_cell_set, END_CELL_OPTS))
    for method in (1, 3, 4):
        opts = dict(single_pair_options(method), **(dict(downsamplingFactor=TIE_FACTOR) if method == 3 else {}))
        out.append(Case(f"oriented_m{method}", tie_pair_set, opts, oriented=True))
    return out


# ---- the device side (one subprocess per policy) ---------------------------------------------------------------------
def run_device(lib_path, out_dir):
    """Every case on the library at lib_path; the outputs go to out_dir/<case>.npz."""
    from shasta_b200 import capi
    assert capi._lib is None, "the library is already loaded"
    capi.LIB_PATH = lib_path
    ctx = capi.Context(0)
    for case in cases():
        d, work = case.data()
        ctx.set_markers(d["toc"], d["data"], d["flags"])
        go = capi.make_align_options(**case.opts)
        path = os.path.join(out_dir, case.name + ".npz")
        if case.oriented:
            ords, infos = [], []
            for o0, o1 in work:
                o, info = capi.align_oriented_reads(ctx, int(o0), int(o1), go)
                ords.append(np.asarray(o, np.uint32).reshape(-1, 2))
                infos.append(info)
            np.savez(path, ords=np.concatenate(ords), counts=np.array([len(o) for o in ords]), infos=np.stack(infos))
        else:
            rec, ctoc, cdata, res = capi.compute_alignments(ctx, work, go)
            np.savez(path, rec=rec, ctoc=ctoc, cdata=cdata, too_wide=res.tooWideCount,
                     digests=np.array([res.alignmentDataDigest, res.compressedDigest], np.uint64))
    ctx.close()


# ---- the oracle side -------------------------------------------------------------------------------------------------
def _oracle_case(case):
    d, work = case.data()
    if case.oriented:
        expected = []
        for o0, o1 in work:
            exp = expected_single_pair(row(d, o0), row(d, o1), case.opts)
            expected.append(None if exp is None else (exp[0][3:16].copy(), exp[1]))
        return expected
    return B.oracle_compute_alignments(d["toc"], d["kmer"], work, oracle_options(case.opts), threads=8)[:3]


@functools.lru_cache(None)
def oracle_outputs(policy):
    """{case name: the oracle's outputs} under `policy`."""
    old = B.set_dp_policy(policy)
    try:
        return {case.name: _oracle_case(case) for case in cases()}
    finally:
        B.set_dp_policy(old)


def _stored(rec, ctoc, cdata):
    """{(readId0, readId1, isSameStrand): (record bytes, compressed bytes)} of compute_alignments' outputs."""
    return {tuple(int(x) for x in r[:3]): (r.tobytes(), cdata[int(ctoc[i]):int(ctoc[i + 1])].tobytes()) for i, r in enumerate(rec)}


def compare_case(case, got, want):
    """Differences of the device outputs `got` (the case's npz) from the oracle's `want`, as text; empty when bit-exact."""
    from shasta_b200 import capi
    if case.oriented:
        ords = np.split(got["ords"], np.cumsum(got["counts"])[:-1])
        bad = []
        for k, exp in enumerate(want):
            o, info = ords[k], got["infos"][k]
            ok = (len(o) == 0 and not info.any()) if exp is None else (np.array_equal(info, exp[0]) and np.array_equal(o, exp[1]))
            if not ok:
                bad.append(k)
        return [f"pairs {bad} of {len(want)} differ"] if bad else []
    orec, otoc, odata = want
    errors = []
    if not (got["rec"].shape == orec.shape and np.array_equal(got["rec"], orec)):
        g, w = _stored(got["rec"], got["ctoc"], got["cdata"]), _stored(orec, otoc, odata)
        diff = sorted(key for key in set(g) | set(w) if g.get(key, (None,))[0] != w.get(key, (None,))[0])
        errors.append(f"{len(got['rec'])} records, the oracle {len(orec)}; differing candidates {diff[:6]}")
    if not np.array_equal(got["ctoc"], otoc) or not np.array_equal(got["cdata"], odata):
        errors.append("compressed alignments differ")
    if int(got["too_wide"]) != 0:
        errors.append(f"tooWideCount {int(got['too_wide'])}")
    if int(got["digests"][0]) != capi.digest_records(orec, 16) or int(got["digests"][1]) != capi.digest_compressed(orec, otoc, odata):
        errors.append("digests differ from the oracle's outputs")
    return errors


@pytest.mark.gpu
@pytest.mark.parametrize("policy", range(8))
def test_policy_matches_oracle(policy, tmp_path):
    lib_path = policy_library(policy)
    if not os.path.exists(lib_path):
        pytest.fail(f"{lib_path} is missing: build() makes it (make -C shasta_b200/csrc policies)")
    # the worker starts like this interpreter: without the user's site-packages when this one runs without them
    flags = [f for f, on in (("-I", sys.flags.isolated), ("-E", sys.flags.ignore_environment), ("-s", sys.flags.no_user_site)) if on]
    cmd = [sys.executable, *flags, os.path.abspath(__file__), lib_path, str(tmp_path)]
    proc = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert proc.returncode == 0, f"policy {policy} worker failed:\n{proc.stdout[-3000:]}\n{proc.stderr[-3000:]}"
    want = oracle_outputs(policy)
    failures = {}
    for case in cases():
        errors = compare_case(case, np.load(tmp_path / (case.name + ".npz")), want[case.name])
        if errors:
            failures[case.name] = errors
    assert not failures, f"policy {policy}: " + "; ".join(f"{name}: {', '.join(e)}" for name, e in failures.items())


# ---- host checks -----------------------------------------------------------------------------------------------------
def candidate_rows(d, c):
    r0, r1, same = (int(x) for x in c)
    return row(d, 2 * r0), row(d, 2 * r1 + (0 if same else 1))


def band_class(W):
    """('group', C) / ('warp', C) / ('scan', 0) of a band of W offsets (dpClassAt / dpBandShape)."""
    need = W + 2
    if need <= 128:
        return ("group", max(2, -(-need // 16)))
    for c in (3, 4, 6, 8, 12, 16):
        if need <= 64 * c:
            return ("warp", c)
    return ("scan", 0)


def forward_lanes(ny):
    """Lanes per job of the forward kernel for ny downsampled rows; None: the traced path."""
    return next((g for rows, g in FORWARD_GROUPS if ny <= rows), None)


def stage1_band(a, b, opts):
    """Method 3's stage 1 under the oracle's current policy: the stage-2 band (lo, hi), or None."""
    (da, oa), (db, ob) = downsampled(a, opts["downsamplingFactor"]), downsampled(b, opts["downsamplingFactor"])
    if not len(da) or not len(db):
        return None
    sc = [opts.get(k, B.ALIGN_DEFAULTS[k]) for k in ("matchScore", "mismatchScore", "gapScore")]
    _, path = B.overlap_align(da, db, *sc)
    eq = da[path[:, 0]] == db[path[:, 1]] if len(path) else np.zeros(0, bool)
    if not eq.any():
        return None
    off = oa[path[eq, 0]] - ob[path[eq, 1]]
    lo, hi = int(off.min()) - opts["bandExtend"], int(off.max()) + opts["bandExtend"]
    return (lo, hi) if hi - lo <= opts["maxBand"] else None


def policy_sensitive(case):
    """Candidates (readId0, readId1, isSameStrand) whose stored output is not the same under all eight policies."""
    stored = [_stored(*oracle_outputs(p)[case.name]) for p in range(8)]
    return {key for key in set().union(*stored) if len({s.get(key) for s in stored}) > 1}


def test_cases_reach_their_paths():
    # Each path is reached by candidates whose output depends on the policy: the kernels' tie-break code is exercised.
    by_name = {c.name: c for c in cases()}
    d, cand = tie_set()
    keys = [tuple(int(x) for x in c) for c in cand]
    rows = [candidate_rows(d, c) for c in cand]
    # stage 2: every 8-lane group class, every whole-warp class, the scan kernel
    reached = set()
    for e in TIE_EXTENDS:
        case = by_name[f"m3_ties_e{e}"]
        sensitive = policy_sensitive(case)
        for key, (a, b) in zip(keys, rows):
            band = stage1_band(a, b, case.opts)
            if band is not None and key in sensitive:
                reached.add(band_class(min(band[1], len(a)) - max(band[0], -len(b)) + 1))
    want = {("group", c) for c in range(2, 9)} | {("warp", c) for c in (3, 4, 6, 8, 12, 16)} | {("scan", 0)}
    assert want <= reached, sorted(want - reached)
    # stage 1: the forward kernel on groups of 8, 16 and 32 lanes (rows = downsampled markers of the second read) and the
    # traced path, each with candidates whose stage-2 band depends on the policy
    opts = by_name["m3_ties_e10"].opts
    default = B.default_dp_policy()
    try:
        bands = []
        for p in range(8):
            B.set_dp_policy(p)
            bands.append([stage1_band(a, b, opts) for a, b in rows])
    finally:
        B.set_dp_policy(default)
    lanes = [forward_lanes(len(downsampled(b, TIE_FACTOR)[0])) for _, b in rows]
    for g in (8, 16, 32, None):
        assert any(lanes[k] == g and len({bands[p][k] for p in range(8)}) > 1 for k in range(len(rows))), g
    # method 1: one unbanded DP on the full rows, from the 8-lane groups to the scan kernel
    sensitive = set().union(*(policy_sensitive(by_name[f"m1_ties_s{s}"]) for s in SCORES))
    assert {band_class(len(a) + len(b) + 1)[0] for key, (a, b) in zip(keys, rows) if key in sensitive} == {"group", "warp", "scan"}
    # method 4 and the single-pair calls store alignments, and some depend on the policy
    assert policy_sensitive(by_name["m4_ties"])
    for m in (1, 3, 4):
        out = [oracle_outputs(p)[f"oriented_m{m}"] for p in range(8)]
        assert sum(e is not None for e in out[DEFAULT_POLICY]) >= 8
        assert any(any((x is None) != (y is None) or (x is not None and not np.array_equal(x[1], y[1])) for x, y in zip(o, out[0]))
                   for o in out[1:]), m
    # tie-rich: eight k-mer ids make up all but the inserted markers, and the downsampling keeps four of them
    strand0 = np.concatenate([row(d, 2 * r) for r in range(len(d["flags"]))])
    values, counts = np.unique(strand0, return_counts=True)
    top = values[np.argsort(counts)[-8:]]
    assert np.isin(strand0, top).mean() > 0.95 and len(downsampled(top, TIE_FACTOR)[0]) == 4
    # the end-cell pairs: ny = 7m rows of stage 1 (every k-mer kept), on each forward group size and on the traced path
    d, cand = end_cell_set()
    for m, c in zip(END_CELL_M, cand):
        a, b = candidate_rows(d, c)
        assert len(downsampled(a, 1.0)[0]) == len(a) == 9 * m and len(downsampled(b, 1.0)[0]) == len(b) == 7 * m
    assert [forward_lanes(7 * m) for m in END_CELL_M] == [8, 8, 16, 32, None]


def test_each_policy_bit_changes_the_stored_output():
    # For every policy and every bit, the policy with that bit flipped stores something else on some candidate.
    stored = {}
    for policy in range(8):
        out = oracle_outputs(policy)
        stored[policy] = {c.name: _stored(*out[c.name]) for c in cases() if not c.oriented}
    for policy in range(8):
        for bit in range(3):
            other = policy ^ (1 << bit)
            if other < policy:
                continue
            assert any(stored[policy][name] != stored[other][name] for name in stored[policy]), (policy, other)


INT32_MAX, INT32_MIN = (1 << 31) - 1, -(1 << 31)


def wrap32(x):
    return (x - INT32_MIN) % (1 << 32) + INT32_MIN


def stage1_outcome(a, b, opts, sc):
    """What method 3's stage 1 leaves for stage 2 under the oracle's current policy: 'none' (no diagonal step), 'no_match'
    (diagonal steps, none on equal k-mers) or 'band'."""
    (da, _), (db, _) = downsampled(a, opts["downsamplingFactor"]), downsampled(b, opts["downsamplingFactor"])
    _, path = B.overlap_align(da, db, *sc)
    if not len(path):
        return "none"
    return "band" if (da[path[:, 0]] == db[path[:, 1]]).any() else "no_match"


def test_stage1_without_a_matching_step_is_reached():
    # 2/5/-1 prefers mismatches: stage-1 paths with diagonal steps and no matching k-mer (kPairNoMatchingStep on the forward
    # kernel, INT32_MAX / INT32_MIN offsets on the traced path). setStage2Band widens them by bandExtend in 32-bit
    # wrap-around arithmetic: the band's width wraps to 2 * bandExtend <= maxBand, but bandMin > bandMax, so the candidate
    # is skipped (the reference's SeqAn throw); the oracle stores nothing for it.
    case = {c.name: c for c in cases()}["m3_ties_s2_5_1"]
    opts, sc = case.opts, SCORES["2_5_1"]
    band_min, band_max = wrap32(INT32_MAX - opts["bandExtend"]), wrap32(INT32_MIN + opts["bandExtend"])
    assert wrap32(band_max - band_min) <= opts["maxBand"] and band_min > band_max
    d, cand = tie_set()
    reached = set()
    for c in cand:
        a, b = candidate_rows(d, c)
        if stage1_outcome(a, b, opts, sc) == "no_match":
            reached.add(forward_lanes(len(downsampled(b, opts["downsamplingFactor"])[0])) is not None)
            status, ords, _ = B.oracle_align_pair(a, b, oracle_options(opts))
            assert status == 1 and len(ords) == 0
    assert reached == {True, False}         # on the forward kernel and on the traced path
    # ... and the candidates are not stored: none of them appears in the oracle's output of the case.
    stored = _stored(*oracle_outputs(DEFAULT_POLICY)[case.name])
    keys = {tuple(int(x) for x in c) for c in cand
            if stage1_outcome(*candidate_rows(d, c), opts, sc) == "no_match"}
    assert keys and not keys & set(stored)


def dp_scores(a, b, match, mismatch, gap):
    """H[i, j] (int64) of the overlap DP of a (columns i) against b (rows j): free end gaps (row 0 and column 0 score 0),
    linear gaps. Column i: H = max(A, H(i, j-1) + gap) with A = max(diagonal, horizontal), as a running maximum."""
    nx, ny = len(a), len(b)
    H = np.zeros((nx + 1, ny + 1), np.int64)
    down = np.arange(ny + 1, dtype=np.int64) * gap
    for i in range(1, nx + 1):
        A = np.zeros(ny + 1, np.int64)
        A[1:] = np.maximum(H[i - 1, :-1] + np.where(b == a[i - 1], match, mismatch), H[i - 1, 1:] + gap)
        H[i] = np.maximum.accumulate(A - down) + down
    return H


def end_cells(H):
    """The end-cell candidates (i, j) in column-major order: row ny of every column, then every row of column nx."""
    nx, ny = H.shape[0] - 1, H.shape[1] - 1
    return [(i, ny) for i in range(nx)] + [(nx, j) for j in range(ny + 1)]


def test_end_cell_case_is_real():
    d, cand = end_cell_set()
    default = B.default_dp_policy()
    try:
        for m, c in zip(END_CELL_M, cand):
            a, b = candidate_rows(d, c)
            nx, ny = len(a), len(b)
            H = dp_scores(a, b, 6, -1, -1)
            cells = end_cells(H)
            best = max(H[c] for c in cells)
            last = [c for c in cells if H[c] == best][-1]
            assert best == 0 and last == (nx, 0), (m, best, last)
            assert (H[nx, 1:] < 0).all()
            row_zero = [i for i in range(1, nx) if H[i, ny] == 0]
            assert row_zero and max(row_zero) == 7 * m, (m, row_zero[-3:])
            # the path into (7m, 7m) holds the m matches at the start: a kernel that ends there would find a band
            assert H[m, m] == 6 * m
            for policy in range(8):
                B.set_dp_policy(policy)
                score, path = B.overlap_align(a, b, 6, -1, -1)
                assert score == 0 and len(path) == 0, (m, policy, score, len(path))
                rec, _, _, _ = B.oracle_compute_alignments(d["toc"], d["kmer"], c[None], oracle_options(END_CELL_OPTS))
                assert len(rec) == 0, (m, policy)
    finally:
        B.set_dp_policy(default)


def test_numpy_dp_scores_match_the_oracle():
    d, cand = tie_set()
    for c in cand[:12]:
        a, b = candidate_rows(d, c)
        for s in SCORES.values():
            H = dp_scores(a, b, *s)
            assert max(H[c] for c in end_cells(H)) == B.overlap_align(a, b, *s)[0]


if __name__ == "__main__":
    run_device(sys.argv[1], sys.argv[2])
