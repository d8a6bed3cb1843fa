"""Measures shb_flag_cross_strand_read_graph_edges1 (maxDistance 6) and shb_flag_chimeric_reads (maxDistance 2), the
reference's defaults, and prints one JSON line.

  1. the default bench.py workload (nanopore-may2022-500k, device-generated): LowHash0, computeAlignments and createReadGraph2
     (Nanopore-May2022 percentiles, maxAlignmentCount 6) on the GPU build its read graph; both calls are then timed over
     repeats after a warm-up. Reported: wall and device times, the host part of the cross-strand call, the histogram of
     the ball sizes the searches reached (the work done), the reads that took the overflow path, the peak device bytes;
  2. a ~20 k-read sample of the same workload, next to the reference's own ReadGraph code in the members' control flow
     (oracle/_ref, all cores, batches of 10 000 reads), with a check that the results are identical;
  3. the overflow path: a 20 k-read graph with one hub read aligned to every other read, where every read's search
     reaches the whole graph and is run again with its table in device memory.

    python bench_readgraph_flags.py [--reads 500000] [--sample 20000] [--repeats 3] [--hub-reads 20000]

The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True          # the tree may be read-only

from bench_markergraph import READ_GRAPH2, card  # noqa: E402

CROSS_DISTANCE, CHIMERIC_DISTANCE = 6, 2


def read_graph(ctx, wl, R):
    from shasta_b200 import capi
    cand, _, _, _ = ctx.lowhash0(capi.make_lowhash_params(**wl["minhash"]), want_stats=False)
    rec, _, _, _ = capi.compute_alignments(ctx, cand, capi.make_align_options(**wl["align"]))
    rec = np.array(rec, np.uint32)
    _, _, edges, toc, data = capi.create_read_graph2(ctx, rec, R, *READ_GRAPH2)
    return np.array(edges), np.array(toc), np.array(data), rec


def run_both(ctx, edges, toc, data, rec, flags):
    from shasta_b200 import capi
    e, r = edges.copy(), rec.copy()
    t0 = time.perf_counter()
    cross = capi.flag_cross_strand_read_graph_edges1(ctx, CROSS_DISTANCE, e, toc, data, r)
    t1 = time.perf_counter()
    f = flags.copy()
    chim = capi.flag_chimeric_reads(ctx, CHIMERIC_DISTANCE, e, toc, data, f, r)
    t2 = time.perf_counter()
    return e, r, f, dict(cross, wallMs=(t1 - t0) * 1e3), dict(chim, wallMs=(t2 - t1) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=500_000)
    ap.add_argument("--sample", type=int, default=20_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--hub-reads", type=int, default=20_000)
    args = ap.parse_args()
    os.environ.setdefault("TMPDIR", tempfile.gettempdir())
    import bench
    from shasta_b200 import capi, synth
    wl = bench.WORKLOADS["nanopore-may2022-500k"]
    out = {"card": card(), "crossStrandMaxDistance": CROSS_DISTANCE, "maxChimericReadDistance": CHIMERIC_DISTANCE}

    p = bench.synth_params(wl, reads=args.reads, seed=1)
    gen = capi.Context(0)
    dm = capi.synth_generate_device(gen, p, want_data7=False)
    gen.set_markers_device(dm.toc, dm.kmer_ptr, dm.flags, keepalive=dm)
    edges, toc, data, rec = read_graph(gen, wl, p.reads)
    flags = np.array(dm.flags, np.uint8)
    gen.close()
    dm.free(("kmer_ptr",))
    ctx = capi.Context(0)
    for _ in range(2):
        run_both(ctx, edges, toc, data, rec, flags)
    runs = [run_both(ctx, edges, toc, data, rec, flags)[3:] for _ in range(args.repeats)]
    cross, chim = runs[-1]
    out["workload"] = dict(reads=args.reads, edges=len(edges), alignments=len(rec),
                           cross_ms=[c["wallMs"] for c, _ in runs], cross_device_ms=[c["deviceMs"] for c, _ in runs],
                           cross_host_ms=[c["hostMs"] for c, _ in runs],
                           chimeric_ms=[c["wallMs"] for _, c in runs], chimeric_device_ms=[c["deviceMs"] for _, c in runs],
                           cross=cross, chimeric=chim)
    ctx.close()

    ps = bench.synth_params(wl, reads=args.sample, seed=3)
    d = synth.generate(ps)
    c = capi.Context(0)
    c.set_markers(d["toc"], d["data"], d["flags"])
    edges, toc, data, rec = read_graph(c, wl, args.sample)
    flags = np.array(d["flags"], np.uint8)
    e, r, f, cr, ch = run_both(c, edges, toc, data, rec, flags)
    sample = dict(reads=args.sample, edges=len(edges), cross=cr, chimeric=ch)
    from oracle import readgraph_flags_bindings as F
    if F.have_ref():
        g = dict(edges=edges, toc=toc, data=data, records=rec, flags=flags)
        t0 = time.perf_counter()
        rc = F.ref_cross_strand(g, CROSS_DISTANCE, threads=os.cpu_count())
        t1 = time.perf_counter()
        rh = F.ref_chimeric(dict(g, edges=rc["edges"], records=rc["records"]), CHIMERIC_DISTANCE, threads=os.cpu_count())
        t2 = time.perf_counter()
        identical = (rc["status"] == 0 and rh["status"] == 0 and np.array_equal(e, rc["edges"]) and np.array_equal(f, rh["flags"])
                     and np.array_equal(r, rh["records"]))
        sample.update(ref_cross_seconds_all_cores=t1 - t0, ref_chimeric_seconds_all_cores=t2 - t1, cpu_count=os.cpu_count(),
                      identical=bool(identical))
    c.close()
    out["sample"] = sample

    # 3. the overflow path: a hub read aligned to every other read of a small graph, so every read's ball holds the whole
    # graph and outgrows the shared-memory table (tests/golden/readgraph_flags_inputs.hub)
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from readgraph_flags_inputs import hub
    g = hub(args.hub_reads, 8)
    c = capi.Context(0)
    run_both(c, g["edges"], g["toc"], g["data"], g["records"], g["flags"])
    _, _, _, cr, ch = run_both(c, g["edges"], g["toc"], g["data"], g["records"], g["flags"])
    c.close()
    out["hub"] = dict(reads=args.hub_reads, edges=len(g["edges"]), cross=cr, chimeric=ch)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
