#!/usr/bin/env python3
"""Pass 1 and pass 2 at k = 192 (Kmer<6>, the 256-entry K1 ring) and k = 256 (Kmer<8>, the 512-entry ring) on one GPU, in one run.

Workload: --reads x 300 bp of a --genome bp genome (abyss_b200.synth seed 12, 0.1 % errors: k-mers of 256 bases need a low
error rate to be solid), --kc=3 -H4, a filter of --bloom bytes.  For each k: one warm-up of pass 1 and pass 2, then --runs
timed runs of each, alternating the two k.  pass 1 = Filter.insert_reads (K1 + ordered insert), pass 2 = the whole of
abb_assembler_process_reads; both are host clocks around work that ends in a device synchronise.  Reports one JSON line with
the median, min and max of each, the contig count and FASTA md5 of each k, and the card and its power limit, queried in the
same run.  Nothing is written outside a temporary directory.

    python scripts/bench_kwidth.py [--reads 4000000] [--genome 30000000] [--runs 3]
"""
import argparse
import hashlib
import json
import statistics
import subprocess
import sys
import time
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from abyss_b200 import capi  # noqa: E402
from abyss_b200.synth import ReadSet  # noqa: E402

KC, H, L = 3, 4, 300
KS = (192, 256)


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    return [x.strip() for x in out.split(",")]


def one_run(k, counters, reads):
    f = capi.Filter.counting(counters, H, k, KC)
    t0 = time.perf_counter()
    f.insert_reads(reads)
    pass1 = (time.perf_counter() - t0) * 1e3
    a = capi.Assembler(f)
    h = hashlib.md5()
    n = 0
    t0 = time.perf_counter()
    for _, seq, cov in a.process_reads(reads):
        h.update(f">{n} {len(seq)} {cov}\n{seq}\n".encode())
        n += 1
    pass2 = (time.perf_counter() - t0) * 1e3
    a.close()
    f.close()
    return pass1, pass2, n, h.hexdigest()


def stats(v):
    return {"median": round(statistics.median(v), 1), "min": round(min(v), 1), "max": round(max(v), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=4_000_000)
    ap.add_argument("--genome", type=int, default=30_000_000)
    ap.add_argument("--bloom", default="4G", help="filter size in bytes, with k/M/G (abyss-bloom-dbg -b)")
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_kwidth measures the GPU: no CUDA device"
    name, power = card()
    capi.set_max_kmer(256)  # MAX_KMER is 192 until raised
    mult = {"k": 1 << 10, "M": 1 << 20, "G": 1 << 30}
    counters = int(float(a.bloom[:-1]) * mult[a.bloom[-1]] / 1.125 + 0.5)
    counters += (64 - counters % 64) % 64
    rs = ReadSet(12, a.genome, a.reads, L, 0.001)
    reads = capi.fixed_length_reads(rs.ascii(0, rs.n))
    res = {k: {"pass1": [], "pass2": [], "md5": set(), "contigs": set()} for k in KS}
    for k in KS:  # warm-up
        one_run(k, counters, reads)
    for _ in range(a.runs):
        for k in KS:
            p1, p2, n, m = one_run(k, counters, reads)
            r = res[k]
            r["pass1"].append(p1)
            r["pass2"].append(p2)
            r["md5"].add(m)
            r["contigs"].add(n)
    out = {"workload": f"{a.reads} x {L} bp of a {a.genome} bp genome (seed 12, 0.1 % errors), --kc={KC} -H{H} -b{a.bloom}",
           "gpu": name, "power_limit": power}
    for k in KS:
        r = res[k]
        assert len(r["md5"]) == 1, f"k={k}: runs gave different FASTA"
        out[f"k{k}"] = {"pass1_ms": stats(r["pass1"]), "pass2_ms": stats(r["pass2"]), "contigs": r["contigs"].pop(),
                        "fasta_md5": r["md5"].pop()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
