"""Measures shb_create_marker_graph_edges and shb_find_marker_graph_reverse_complement_edges (Assembler::createMarkerGraphEdges
and findMarkerGraphReverseComplementEdges on the GPU) and prints one JSON line.

  1. the default bench.py workload (nanopore-may2022-500k, device-generated): LowHash0, computeAlignments, createReadGraph2
     (Nanopore-May2022 values) and createMarkerGraphVertices (minCoverage 0, maxCoverage 100) with its reverse complement
     vertices on the GPU give the vertices; both calls are then timed over repeats after a warm-up;
  2. a ~20 k-read sample of the same workload, next to the reference's own MarkerGraph code in the members' control flow
     (oracle/_ref, all cores), with a check that the two agree in canonical form.

    python bench_markergraph_edges.py [--reads 500000] [--sample 20000] [--repeats 3]

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

from bench_markergraph import MARKER_GRAPH, card, read_graph  # noqa: E402


def vertices(ctx, edges, ctoc, cdata, flags):
    from shasta_b200 import capi
    table, vtoc, vdata, _, res = capi.create_marker_graph_vertices(ctx, capi.make_marker_graph_params(**MARKER_GRAPH), edges, ctoc,
                                                                   cdata, flags)
    rc = capi.find_marker_graph_reverse_complement_vertices(ctx, table, vtoc, vdata)
    return table, vtoc, vdata, rc


def digest(a):
    b = np.ascontiguousarray(a).tobytes()
    b += b"\0" * (-len(b) % 8)
    return int(np.frombuffer(b, np.uint64).sum(dtype=np.uint64))


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
    out = {"card": card()}

    # 1. the default workload: the read graph in a context of its own, then the vertices and the timed calls in a context that
    # holds only the markers.
    p = bench.synth_params(wl, reads=args.reads, seed=1)
    gen = capi.Context(0)
    dm = capi.synth_generate_device(gen, p, want_data7=False)
    gen.set_markers_device(dm.toc, dm.kmer_ptr, dm.flags, keepalive=dm)
    edges, ctoc, cdata, _ = read_graph(gen, wl, p.reads)
    gen.close()
    ctx = capi.Context(0)
    ctx.set_markers_device(dm.toc, dm.kmer_ptr, dm.flags, keepalive=dm)
    table, vtoc, vdata, rcv = vertices(ctx, edges, ctoc, cdata, np.array(dm.flags, np.uint8))
    del edges, ctoc, cdata
    for _ in range(2):                                  # warm-up (the second call reuses the host result blocks)
        o, _ = capi.create_marker_graph_edges(ctx, table, vtoc, vdata)
        capi.find_marker_graph_reverse_complement_edges(ctx, rcv, o["edges"], o["intervalsToc"], o["intervalsData"], o["bySourceToc"],
                                                        o["bySourceData"])
        del o
    runs, rc_runs = [], []
    for _ in range(args.repeats):
        o = None
        o, res = capi.create_marker_graph_edges(ctx, table, vtoc, vdata)
        rc, rres = capi.find_marker_graph_reverse_complement_edges(ctx, rcv, o["edges"], o["intervalsToc"], o["intervalsData"],
                                                                   o["bySourceToc"], o["bySourceData"])
        runs.append(res.asdict())
        rc_runs.append(rres.asdict())
    last = runs[-1]
    out["workload"] = dict(reads=args.reads, markers=int(dm.marker_count), vertices=len(rcv), vertex_markers=len(vdata),
                           edges=last["edgeCount"], intervals=last["markerIntervalCount"], saturated=last["saturatedEdgeCount"],
                           create_ms=[r["totalMs"] for r in runs], create_device_ms=[r["deviceMs"] for r in runs],
                           create_peak_device_bytes=last["peakDeviceBytes"], rc_ms=[r["totalMs"] for r in rc_runs],
                           rc_device_ms=[r["deviceMs"] for r in rc_runs], rc_peak_device_bytes=rc_runs[-1]["peakDeviceBytes"],
                           output_digest=[digest(o[k]) for k in sorted(o)] + [digest(rc)])
    del o, rc
    ctx.close()
    dm.free(("kmer_ptr",))

    # 2. the sample, against the reference's MarkerGraph code on all cores
    ps = bench.synth_params(wl, reads=args.sample, seed=3)
    d = synth.generate(ps)
    c = capi.Context(0)
    c.set_markers(d["toc"], d["data"], d["flags"])
    edges, ctoc, cdata, _ = read_graph(c, wl, args.sample)
    table, vtoc, vdata, rcv = vertices(c, edges, ctoc, cdata, np.array(d["flags"], np.uint8))
    o, res = capi.create_marker_graph_edges(c, table, vtoc, vdata)
    rc, rres = capi.find_marker_graph_reverse_complement_edges(c, rcv, o["edges"], o["intervalsToc"], o["intervalsData"], o["bySourceToc"],
                                                               o["bySourceData"])
    sample = dict(reads=args.sample, vertices=len(rcv), gpu=res.asdict(), gpu_rc=rres.asdict())
    from oracle import markergraph_edges_bindings as EB
    if EB.have_ref():
        t64, v64 = capi.uint40_to_uint64(table), capi.uint40_to_uint64(vtoc)
        t0 = time.perf_counter()
        r = EB.ref_create_marker_graph_edges(d["toc"], t64, v64, vdata, threads=os.cpu_count())
        msg, rrc = EB.ref_find_rc_edges(d["toc"], rcv, r, threads=os.cpu_count())
        sec = time.perf_counter() - t0
        g = dict(o)
        g["bySourceData"] = EB.rows_from_uint40(o["bySourceData"])
        g["byTargetData"] = EB.rows_from_uint40(o["byTargetData"])
        a, b = EB.canonical(g, rc), EB.canonical(r, rrc)
        identical = msg is None and all(np.array_equal(np.asarray(x).reshape(-1), np.asarray(y).reshape(-1)) for x, y in zip(a, b))
        sample.update(ref_seconds_all_cores=sec, cpu_count=os.cpu_count(), identical=bool(identical))
    c.close()
    out["sample"] = sample
    print(json.dumps(out))


if __name__ == "__main__":
    main()
