#!/usr/bin/env python3
"""Throughput of the Konnector filter family (abyss-bloom build -t konnector / kmers) on one GPU.

Workload `m1_k64`: 1 M x 150 bp reads of a 5 Mbp genome (abyss_b200.synth seed 7, 0.5 % errors), k = 64, -b1G -l2.
Reports, as one JSON line:
  build_kmers_per_s   abb_insert_reads on the whole batch (reads already in host memory), best of --steps
  query_kmers_per_s   abb_contains_reads (the kmers command's query) on the same reads against the built filter
  trim_reads_per_s, trim_ms   abb_trim_reads on the same reads against the built filter (minBranchLen from its population):
                      host wall time of the call (copies included, it ends in a synchronise) and CUDA events on the library's
                      stream around it
  cli_build_s / cli_kmers_s / cli_trim_s   wall time of `abyss-bloom build`, `kmers --raw` and `trim` on the FASTQ (parse + GPU + file I/O)
  ref_build_s / ref_kmers_s / ref_trim_s   the same commands of the reference (oracle/_ref/abyss-bloom-ref, -j8 for build) when built
  gpu, power_limit    the card and its power limit, queried in the same run
Everything it writes goes to a temporary directory.

    python scripts/bench_konnector.py [--steps 3] [--no-ref]
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from abyss_b200 import capi  # noqa: E402
from abyss_b200.synth import ReadSet  # noqa: E402

K, BYTES, LEVELS = 64, 1 << 30, 2


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:
        return None, None


def timed(cmd, **kw):
    t0 = time.perf_counter()
    subprocess.run(cmd, check=True, **kw)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true")
    a = ap.parse_args()
    rs = ReadSet(7, 5_000_000, 1_000_000, 150, 0.005)
    bases, offs = capi.fixed_length_reads(rs.ascii(0, rs.n))
    n_kmers = rs.n * (rs.L - K + 1)
    lib = capi.load()
    res = {"workload": "m1_k64: 1 M x 150 bp, k=64, -b1G -l2", "kmer_windows": n_kmers}
    bits = BYTES * 8 // LEVELS
    best_ins, best_q, best_t, best_t_ev = float("inf"), float("inf"), float("inf"), float("inf")
    import torch
    for _ in range(a.steps):
        f = capi.Filter.konnector(bits, K, LEVELS)
        t0 = time.perf_counter()
        f.insert_reads((bases, offs))
        best_ins = min(best_ins, time.perf_counter() - t0)
        q = capi.Filter.konnector(bits, K, 1)
        q.read_bits(f.download(), bits)
        f.close()
        flag = np.zeros(n_kmers, np.uint8)
        valid = np.zeros(n_kmers, np.uint8)
        n = C.c_uint64(0)
        t0 = time.perf_counter()
        capi.check(lib.abb_contains_reads(q.handle, capi._ptr(bases), capi._ptr(offs), rs.n, capi._ptr(flag), capi._ptr(valid), n_kmers,
                                          C.byref(n)))
        best_q = min(best_q, time.perf_counter() - t0)
        mbl = math.ceil(math.log(0.0001) / math.log(q.level_popcount() / bits))
        stream = torch.cuda.ExternalStream(q.stream())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t0 = time.perf_counter()
        q.trim_reads((bases, offs), mbl)
        best_t = min(best_t, time.perf_counter() - t0)
        e1.record(stream)
        e1.synchronize()
        best_t_ev = min(best_t_ev, e0.elapsed_time(e1))
        q.close()
    res["build_kmers_per_s"] = n_kmers / best_ins
    res["query_kmers_per_s"] = n_kmers / best_q
    res["trim_min_branch_len"] = mbl
    res["trim_reads_per_s"] = rs.n / best_t
    res["trim_ms"] = best_t_ev
    exe = os.path.join(ROOT, "abyss_b200", "lib", "abyss-bloom")
    ref = os.path.join(ROOT, "oracle", "_ref", "abyss-bloom-ref")
    with tempfile.TemporaryDirectory() as d:
        fq = os.path.join(d, "r.fq")
        rs.write_fastq(fq)
        dn = subprocess.DEVNULL
        res["cli_build_s"] = timed([exe, "build", f"-k{K}", "-b1G", f"-l{LEVELS}", os.path.join(d, "g.bloom"), fq], stderr=dn)
        res["cli_kmers_s"] = timed([exe, "kmers", f"-k{K}", "--raw", os.path.join(d, "g.bloom"), fq], stdout=dn)
        res["cli_trim_s"] = timed([exe, "trim", f"-k{K}", os.path.join(d, "g.bloom"), fq], stdout=dn)
        if os.path.exists(ref) and not a.no_ref:
            res["ref_build_s"] = timed([ref, "build", f"-k{K}", "-b1G", f"-l{LEVELS}", "-j8", os.path.join(d, "r.bloom"), fq], stderr=dn)
            res["ref_kmers_s"] = timed([ref, "kmers", f"-k{K}", "--raw", os.path.join(d, "r.bloom"), fq], stdout=dn)
            res["ref_trim_s"] = timed([ref, "trim", f"-k{K}", os.path.join(d, "r.bloom"), fq], stdout=dn)
        else:
            res["ref"] = "oracle/_ref/abyss-bloom-ref not built: no CPU figures"
    res["gpu"], res["power_limit"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
