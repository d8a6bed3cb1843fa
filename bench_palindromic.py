"""Measures shb_flag_palindromic_reads (Assembler::flagPalindromicReads on the GPU) and prints one JSON line.

  1. the default bench.py workload (nanopore-may2022-500k, device-generated): nearly every read is decided by the prefilter;
  2. a ~20 k-read sample of it in which every 50th read is made palindromic in marker space, next to the reference build
     (oracle/_ref, one process per core) with a check that flags and counts are identical;
  3. one UL-length palindromic read (>= 7 000 markers per strand), the longest single phase-B job.

    python bench_palindromic.py [--reads 500000] [--sample 20000] [--repeats 3]

The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.dont_write_bytecode = True          # the tree may be read-only

PARAMS = dict(maxSkip=100, maxDrift=100, maxMarkerFrequency=10, alignedFractionThreshold=0.1,
              nearDiagonalFractionThreshold=0.1, deltaThreshold=100)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _ref_chunk(args):
    toc, ids = args
    from oracle import palindromic_bindings as B
    r = B.ref_flag_palindromic(toc, ids, **PARAMS)
    return r["flags"], r["aligned"], r["nearDiagonal"]


def ref_all_cores(toc, ids, reads_per_chunk=200):
    R = (len(toc) - 1) // 2
    jobs = []
    for b in range(0, R, reads_per_chunk):
        e = min(R, b + reads_per_chunk)
        t = toc[2 * b:2 * e + 1]
        jobs.append(((t - t[0]).astype(np.uint64), ids[int(t[0]):int(t[-1])]))
    t0 = time.perf_counter()
    with ProcessPoolExecutor(os.cpu_count()) as ex:
        parts = list(ex.map(_ref_chunk, jobs))
    sec = time.perf_counter() - t0
    return [np.concatenate([p[i] for p in parts]) for i in range(3)], sec


def make_palindromic(toc, kmer, k, every=50):
    from palindromic_inputs import reverse_complement
    kmer = kmer.copy()
    R = (len(toc) - 1) // 2
    for r in range(0, R, every):
        b, m, e = int(toc[2 * r]), int(toc[2 * r + 1]), int(toc[2 * r + 2])
        s0 = kmer[b:m].copy()
        h = len(s0) // 2
        s0[len(s0) - h:] = reverse_complement(s0[:h][::-1], k)
        kmer[b:m] = s0
        kmer[m:e] = reverse_complement(s0[::-1], k)
    return kmer


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=500_000)
    ap.add_argument("--sample", type=int, default=20_000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    os.environ.setdefault("TMPDIR", tempfile.gettempdir())
    import bench
    from shasta_b200 import capi, synth
    from palindromic_inputs import oriented, palindrome, rows_to_case
    out = {"card": card(), "params": PARAMS}
    params = capi.make_palindromic_params(**PARAMS)
    wl = bench.WORKLOADS["nanopore-may2022-500k"]
    ctx = capi.Context(0)

    # 1. the default workload
    p = bench.synth_params(wl, reads=args.reads, seed=1)
    dm = capi.synth_generate_device(ctx, p, want_data7=False)
    ctx.set_markers_device(dm.toc, dm.kmer_ptr, dm.flags, keepalive=dm)
    capi.flag_palindromic_reads(ctx, params, want_counts=False)           # warm-up
    runs = []
    for _ in range(args.repeats):
        _, _, res = capi.flag_palindromic_reads(ctx, params, want_counts=False)
        runs.append(res.asdict())
    out["workload"] = dict(reads=args.reads, markers=int(dm.marker_count), ms=[r["totalMs"] for r in runs], last=runs[-1])
    dm.free(("kmer_ptr",))

    # 2. the sample with injected palindromes, against the reference build on all cores
    ps = bench.synth_params(wl, reads=args.sample, seed=3)
    d = synth.generate(ps)
    kmer = make_palindromic(d["toc"], d["kmer"], ps.k)
    ctx.set_markers(d["toc"], synth.pack_markers(kmer, d["pos"]), d["flags"])
    flags = np.zeros(len(d["flags"]), np.uint8)
    aligned, near, res = capi.flag_palindromic_reads(ctx, params, read_flags=flags)
    sample = dict(reads=args.sample, gpu=res.asdict())
    from oracle import palindromic_bindings as B
    if B.have_ref():
        (rf, ra, rn), sec = ref_all_cores(d["toc"], kmer)
        o = B.oracle_flag_palindromic(d["toc"], kmer, **PARAMS)
        exact = o["survives"] == 1
        sample.update(ref_seconds_all_cores=sec, cpu_count=os.cpu_count(),
                      identical=bool(np.array_equal(flags & 1, rf) and np.array_equal(aligned[exact], ra[exact])
                                     and np.array_equal(near[exact], rn[exact])))
    out["sample"] = sample

    # 3. one UL-length palindromic read: reported, its own time not separated from the call's
    toc, ids, _ = rows_to_case([oriented(palindrome(np.random.default_rng(5), 8000, noise=0.03))])
    ctx.set_markers(toc, synth.pack_markers(ids, np.concatenate([np.arange(8000, dtype=np.uint32)] * 2)), np.zeros(1, np.uint8))
    _, _, res = capi.flag_palindromic_reads(ctx, params)
    out["ul_read"] = dict(markers_per_strand=8000, result=res.asdict())
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
