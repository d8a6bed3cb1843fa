"""Times the device -> host copy of the LowHash0 and computeAlignments results on the bench.py workload.

One process, the calls a one-shot caller and a caller that keeps its previous results make: the first lowhash0 and
compute_alignments call of the process (fresh host blocks), a second call of each while the first call's results are still
held (fresh blocks again), and a third after both were freed (recycled, page-locked blocks). Prints one JSON line: per call
the host wall time, the library's outputCopyMs (computeAlignments: the time from the end of the last batch to the last byte
on the host) and hostWallMs, and the bytes copied. Writes nothing to disk.

    python bench_result_copy.py [--workload nanopore-may2022-500k]
"""
import argparse
import gc
import json
import os
import time

import bench


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="nanopore-may2022-500k", choices=list(bench.WORKLOADS))
    args = ap.parse_args()
    wl = bench.WORKLOADS[args.workload]
    import torch
    from shasta_b200 import capi

    torch.cuda.set_device(0)
    # the host placement bench.py uses for its timed legs
    _, cpus = bench.gpu_numa_cpus(torch, 0)
    if cpus and len(cpus & os.sched_getaffinity(0)) >= 8:
        os.sched_setaffinity(0, cpus & os.sched_getaffinity(0))
    p = bench.synth_params(wl, seed=1)
    ctx = capi.Context(0)
    dm = capi.synth_generate_device(ctx, p, want_data7=False)
    ctx.set_markers_device(dm.toc, dm.kmer_ptr, dm.flags, keepalive=dm, read_count_total=p.reads, total_marker_count=dm.marker_count)
    lparams = capi.make_lowhash_params(**wl["minhash"])
    aopts = capi.make_align_options(**wl["align"])
    out = {"workload": args.workload, "gpu": torch.cuda.get_device_name(0), "lowhash0": {}, "compute_alignments": {}}

    def lowhash(name):
        t0 = time.perf_counter()
        cand, _, _, res = ctx.lowhash0(lparams, want_stats=True)
        wall = 1e3 * (time.perf_counter() - t0)
        out["lowhash0"][name] = {"host_wall_ms": round(wall, 1), "total_ms": round(res.totalMs, 1), "bytes": int(cand.nbytes),
                                 "candidate_digest": int(res.candidateDigest)}
        return cand

    def align(name, cand):
        t0 = time.perf_counter()
        rec, ctoc, cdata, res = capi.compute_alignments(ctx, cand, aopts)
        wall = 1e3 * (time.perf_counter() - t0)
        out["compute_alignments"][name] = {
            "host_wall_ms": round(wall, 1), "output_copy_ms": round(res.outputCopyMs, 1), "lib_host_wall_ms": round(res.hostWallMs, 1),
            "dp_ms": round(res.dpMs, 1), "bytes": int(rec.nbytes + ctoc.nbytes + cdata.nbytes), "alignments": int(len(rec)),
            "digests": [int(res.alignmentDataDigest), int(res.compressedDigest)]}
        return rec, ctoc, cdata

    first = lowhash("first")
    held = lowhash("held")
    cand = held
    del first
    gc.collect()
    lowhash("recycled")
    a1 = align("first", cand)
    a2 = align("held", cand)
    del a1, a2
    gc.collect()
    align("recycled", cand)
    print(json.dumps(out), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
