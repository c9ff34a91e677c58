#!/usr/bin/env python3
"""Throughput of `abyss-bloom graph` on one GPU.

Workload `m1_k64_H4`: a -b1G -H4 rolling-hash filter (`abyss-bloom build -t rolling-hash`) of 1 M x 150 bp reads of a 5 Mbp genome
(abyss_b200.synth seed 7, 0.5 % errors) at k = 64; roots from -f of the first 2 000 reads; default depth (k).  Reports, as one JSON
line:
  kernel[]              k_graph_neighbors alone, on one 65 536-vertex frontier made of read k-mers (not a level of a search), in
                        two configurations: the graph only (H = 4: one probe per lane), and the graph with two -A filters of
                        H = 4 (lanes 0 and 1 then make five probes, the
                        others one).  Per configuration:
    kernel_ms           CUDA events around each launch (abb_filter_set_profiling; abb_insert_stats::ms_graph), over --launches calls
    call_ms             the whole abb_graph_neighbors call, copies in and out included: CUDA events on the library's stream
    vertices_per_s      frontier vertices per second of kernel_ms
    alg_bytes_per_vertex  (8 H + sum of the attribute filters' H) x 32 B: one 32-byte sector per probe
    hbm_frac            alg bytes / kernel_ms over 3.35 TB/s (H100 SXM HBM3 data sheet)
  cli_graph_s           wall time of the whole command, text output to a file included
  gpu, power_limit      the card and its power limit, queried in the same run
Everything it writes goes to a temporary directory.

    python scripts/bench_bloom_graph.py [--launches 50]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from abyss_b200 import capi  # noqa: E402
from abyss_b200.synth import ReadSet, write_fastq_fast  # noqa: E402

K, H, PIECE = 64, 4, 1 << 16
EXE = os.path.join(ROOT, "abyss_b200", "lib", "abyss-bloom")


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    return [x.strip() for x in out.split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_bloom_graph measures the GPU: no CUDA device"
    name, power = card()
    rs = ReadSet(7, 5_000_000, 1_000_000, 150, 0.005)
    res = {"workload": "m1_k64_H4: 1 M x 150 bp, k=64, -b1G -H4, -f 2000 reads, depth k", "gpu": name, "power_limit": power}
    with tempfile.TemporaryDirectory() as d:
        reads, roots, bloom = os.path.join(d, "r.fq"), os.path.join(d, "roots.fa"), os.path.join(d, "g.bloom")
        write_fastq_fast(rs, reads, 0, rs.n)
        rs.write_fastq(roots, 0, 2000, fasta=True)
        subprocess.run([EXE, "build", f"-k{K}", "-t", "rolling-hash", "-b1G", f"-H{H}", bloom, reads], check=True, capture_output=True)
        t0 = time.perf_counter()
        with open(os.path.join(d, "g.dot"), "wb") as out:
            subprocess.run([EXE, "graph", f"-k{K}", "-f", roots, bloom], check=True, stdout=out)
        res["cli_graph_s"] = round(time.perf_counter() - t0, 3)
        res["dot_lines"] = sum(1 for _ in open(os.path.join(d, "g.dot"), "rb"))
        raw = open(bloom, "rb").read()
        body = raw[raw.index(b"[HeaderEnd]\n") + len(b"[HeaderEnd]\n"):]
    # the kernel alone: one piece of read k-mers (a frontier of that size), many launches
    import numpy as np
    f = capi.Filter.bits(len(body) * 8, H, K)
    f.upload(np.frombuffer(body, dtype=np.uint8))
    attr_bytes = 64 << 20
    attrs = [capi.Filter.bits(attr_bytes * 8, H, K) for _ in range(2)]
    for i, x in enumerate(attrs):
        x.upload(np.frombuffer(body[i * attr_bytes:(i + 1) * attr_bytes], dtype=np.uint8))
    asc = rs.ascii(0, PIECE)
    buf = b"".join(bytes(asc[i, 10:10 + K]) for i in range(PIECE))
    lib = capi.load()
    out = (capi.NbrInfo * PIECE)()
    st = torch.cuda.ExternalStream(lib.abb_filter_stream(f.handle))
    res["kernel"] = []
    for name_cfg, use in (("graph H=4", []), ("graph H=4 + two -A H=4", attrs)):
        handles = (capi._vp * max(1, len(use)))(*[x.handle for x in use])
        for _ in range(3):  # warm-up
            capi.check(lib.abb_graph_neighbors(f.handle, buf, PIECE, handles, len(use), out))
        capi.check(lib.abb_filter_set_profiling(f.handle, 1))
        capi.check(lib.abb_filter_insert_stats(f.handle, None, 1))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(a.launches):
            capi.check(lib.abb_graph_neighbors(f.handle, buf, PIECE, handles, len(use), out))
        e1.record(st)
        e1.synchronize()
        stats = capi.InsertStats()
        capi.check(lib.abb_filter_insert_stats(f.handle, C.byref(stats), 1))
        capi.check(lib.abb_filter_set_profiling(f.handle, 0))
        assert stats.graph_launches == a.launches, stats.graph_launches
        ms = stats.ms_graph / a.launches
        alg = (8 * H + H * len(use)) * 32
        res["kernel"].append({"config": name_cfg, "kernel_ms": round(ms, 4), "call_ms": round(e0.elapsed_time(e1) / a.launches, 4),
                              "vertices": PIECE, "vertices_per_s": round(PIECE / (ms / 1e3)), "alg_bytes_per_vertex": alg,
                              "hbm_frac": round(PIECE * alg / (ms / 1e3) / 3.35e12, 4)})
    for x in attrs + [f]:
        x.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
