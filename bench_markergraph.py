"""Measures shb_create_marker_graph_vertices (Assembler::createMarkerGraphVertices on the GPU) and prints one JSON line.

  1. the default bench.py workload (nanopore-may2022-500k, device-generated): LowHash0, computeAlignments and createReadGraph2
     (Nanopore-May2022 percentiles, maxAlignmentCount 6) on the GPU build its read graph; the call is then timed with the
     May2022 marker graph values (minCoverage 0, maxCoverage 100, the rest at their defaults) over repeats after a warm-up;
  2. a ~20 k-read sample of the same workload, next to the reference's own DisjointSets / decompress / PeakFinder in the
     member's control flow (oracle/_ref, all cores), with a check that the two agree in canonical form.

    python bench_markergraph.py [--reads 500000] [--sample 20000] [--repeats 3]

The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True          # the tree may be read-only

MARKER_GRAPH = dict(minCoverage=0, maxCoverage=100, minCoveragePerStrand=0, allowDuplicateMarkers=False,
                    peakFinderMinAreaFraction=0.08, peakFinderAreaStartIndex=2)
READ_GRAPH2 = (6, 0.015, 0.12, 0.12, 0.12, 0.015)      # maxAlignmentCount and the five percentiles of Nanopore-May2022.conf


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def read_graph(ctx, wl, R):
    """LowHash0 -> computeAlignments -> createReadGraph2 on the markers ctx holds. Returns (edges, ctoc, cdata, seconds)."""
    from shasta_b200 import capi
    t0 = time.perf_counter()
    cand, _, _, _ = ctx.lowhash0(capi.make_lowhash_params(**wl["minhash"]), want_stats=False)
    rec, ctoc, cdata, _ = capi.compute_alignments(ctx, cand, capi.make_align_options(**wl["align"]))
    rec = np.array(rec, np.uint32)
    _, _, edges, _, _ = capi.create_read_graph2(ctx, rec, R, *READ_GRAPH2)
    return np.array(edges), np.array(ctoc), np.array(cdata), time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=500_000)
    ap.add_argument("--sample", type=int, default=20_000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    os.environ.setdefault("TMPDIR", tempfile.gettempdir())
    import bench
    from shasta_b200 import capi, synth
    wl = bench.WORKLOADS["nanopore-may2022-500k"]
    params = capi.make_marker_graph_params(**MARKER_GRAPH)
    out = {"card": card(), "params": MARKER_GRAPH}

    # 1. the default workload. The read graph is built in a context of its own, which is then closed: the timed context
    # holds only the markers (the same device k-mer ids) and what the call allocates.
    p = bench.synth_params(wl, reads=args.reads, seed=1)
    gen = capi.Context(0)
    dm = capi.synth_generate_device(gen, p, want_data7=False)
    gen.set_markers_device(dm.toc, dm.kmer_ptr, dm.flags, keepalive=dm)
    edges, ctoc, cdata, rg_s = read_graph(gen, wl, p.reads)
    gen.close()
    ctx = capi.Context(0)
    ctx.set_markers_device(dm.toc, dm.kmer_ptr, dm.flags, keepalive=dm)
    flags = np.array(dm.flags, np.uint8)
    # Warm-up: two calls. The second is the first to reuse the library's large host result blocks, which page-locks them
    # once (csrc/hostpool.cuh); from the third call on the outputs go to page-locked memory directly.
    # The outputs of a call are dropped before the next one, so that it can reuse their blocks, as a steady caller would.
    for _ in range(2):
        capi.create_marker_graph_vertices(ctx, params, edges, ctoc, cdata, flags)
    runs = []
    for _ in range(args.repeats):
        table = vtoc = vdata = hist = None
        t0 = time.perf_counter()
        table, vtoc, vdata, hist, res = capi.create_marker_graph_vertices(ctx, params, edges, ctoc, cdata, flags)
        wall = time.perf_counter() - t0
        runs.append(dict(res.asdict(), wallMs=wall * 1e3))
    digest = [int(np.frombuffer(a.tobytes(), np.uint64, len(a.tobytes()) // 8).sum(dtype=np.uint64)) for a in (vdata, hist)]
    last = runs[-1]
    out["workload"] = dict(reads=args.reads, markers=int(dm.marker_count), edges=len(edges), read_graph_seconds=rg_s,
                           ms=[r["totalMs"] for r in runs], device_ms=[r["deviceMs"] for r in runs],
                           aligned_pairs_per_s=last["alignedMarkerPairs"] / (last["totalMs"] / 1e3),
                           vertices=last["vertexCount"], min_coverage_used=last["minCoverageUsed"],
                           peak_device_bytes_of_call=last["peakDeviceBytes"], marker_kmer_bytes=4 * int(dm.marker_count),
                           output_digest=digest, last=last)
    del table, vtoc, vdata, hist
    ctx.close()
    dm.free(("kmer_ptr",))

    # 2. the sample, against the reference's components on all cores
    ps = bench.synth_params(wl, reads=args.sample, seed=3)
    d = synth.generate(ps)
    c = capi.Context(0)
    c.set_markers(d["toc"], d["data"], d["flags"])
    edges, ctoc, cdata, _ = read_graph(c, wl, args.sample)
    flags = np.array(d["flags"], np.uint8)
    table, vtoc, vdata, hist, res = capi.create_marker_graph_vertices(c, params, edges, ctoc, cdata, flags)
    sample = dict(reads=args.sample, markers=int(d["toc"][-1]), edges=len(edges), gpu=res.asdict())
    from oracle import markergraph_bindings as MB
    if MB.have_ref():
        t0 = time.perf_counter()
        r = MB.ref_create_marker_graph_vertices(d["toc"], d["kmer"], edges, ctoc, cdata, flags, threads=os.cpu_count(), **MARKER_GRAPH)
        sec = time.perf_counter() - t0
        ref_form = MB.canonical(r["table"], r["vtoc"], r["vdata"])[:3]
        gpu_form = MB.canonical(capi.uint40_to_uint64(table), capi.uint40_to_uint64(vtoc), vdata)[:3]
        identical = (all(np.array_equal(a, b) for a, b in zip(gpu_form, ref_form)) and np.array_equal(hist, r["histogram"])
                     and res.minCoverageUsed == r["minCoverageUsed"] and res.badDisjointSetCount == r["badDisjointSetCount"])
        sample.update(ref_seconds_all_cores=sec, cpu_count=os.cpu_count(), identical=bool(identical))
    c.close()
    out["sample"] = sample
    print(json.dumps(out))


if __name__ == "__main__":
    main()
