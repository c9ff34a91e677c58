#!/usr/bin/env python3
"""Pass 2 of a spaced-seed assembly on one GPU, with tiles and vertex by vertex (ABB_NO_TILES=1).

Workload: --reads x 150 bp of a --genome bp genome (abyss_b200.synth seed 12, 0.5 % errors), -k80 with kmerPair(80, 32) (the
seed shape of config 4, `abyss-bloom-dbg -k80 -K32`), --kc=3 -H4, a filter of --bloom bytes.  Pass 1 runs once; pass 2 then
runs on that filter with a fresh assembler per run, tiles and no tiles alternating, after one warm-up run of each.  Reports,
as one JSON line:
  tiles / no_tiles      per run: ms_tiles (marker enumeration and tile production), ms_extend (K4 walks), ms_replay (K5),
                        ms_total (the whole of abb_assembler_process_reads, host clock around work that ends in a device
                        synchronise), and their median, min and max over the runs
  markers, tiles        tile-store counters of the tiled run
  fasta_md5             of each side's FASTA; they must be equal (the script fails otherwise)
  gpu, power_limit      the card and its power limit, queried in the same run
Nothing is written outside a temporary directory.

    python scripts/bench_spaced_seed.py [--reads 8000000] [--genome 30000000] [--runs 3]
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from abyss_b200 import capi  # noqa: E402
from abyss_b200.synth import ReadSet  # noqa: E402

K, KC, H = 80, 3, 4


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    return [x.strip() for x in out.split(",")]


def assemble(f, reads, tiles):
    """one pass 2 on filter f: (stats fields, fasta md5, wall ms)"""
    if tiles:
        os.environ.pop("ABB_NO_TILES", None)
    else:
        os.environ["ABB_NO_TILES"] = "1"  # read when the assembler is created
    a = capi.Assembler(f)
    h = hashlib.md5()
    t0 = time.perf_counter()
    n = 0
    for _, seq, cov in a.process_reads(reads):
        h.update(f">{n} {len(seq)} {cov}\n{seq}\n".encode())
        n += 1
    wall = (time.perf_counter() - t0) * 1e3
    st = a.stats()
    a.close()
    os.environ.pop("ABB_NO_TILES", None)
    row = {x: round(getattr(st, x), 1) for x in ("ms_tiles", "ms_extend", "ms_replay", "ms_total")}
    row.update(markers=st.markers, tiles=st.tiles, contigs=n, wall_ms=round(wall, 1))
    return row, h.hexdigest()


def summary(rows):
    out = {"runs": rows}
    for x in ("ms_tiles", "ms_extend", "ms_replay", "ms_total"):
        v = [r[x] for r in rows]
        out[x] = {"median": round(statistics.median(v), 1), "min": min(v), "max": max(v)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=8_000_000)
    ap.add_argument("--genome", type=int, default=30_000_000)
    ap.add_argument("--bloom", default="4G", help="filter size in bytes, with k/M/G (abyss-bloom-dbg -b)")
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_spaced_seed measures the GPU: no CUDA device"
    name, power = card()
    mask = capi.kmer_pair_seed(K, 32)
    mult = {"k": 1 << 10, "M": 1 << 20, "G": 1 << 30}
    counters = int(float(a.bloom[:-1]) * mult[a.bloom[-1]] / 1.125 + 0.5)
    counters += (64 - counters % 64) % 64
    rs = ReadSet(12, a.genome, a.reads, 150, 0.005)
    reads = capi.fixed_length_reads(rs.ascii(0, rs.n))
    f = capi.Filter.counting(counters, H, K, KC, mask=mask)
    t0 = time.perf_counter()
    f.insert_reads(reads)
    pass1 = (time.perf_counter() - t0) * 1e3
    assemble(f, reads, True)  # warm-up of both paths
    assemble(f, reads, False)
    rows = {True: [], False: []}
    md5s = {True: set(), False: set()}
    for _ in range(a.runs):
        for tiles in (True, False):
            row, m = assemble(f, reads, tiles)
            rows[tiles].append(row)
            md5s[tiles].add(m)
    f.close()
    assert len(md5s[True] | md5s[False]) == 1, md5s
    res = {"workload": f"{a.reads} x 150 bp of a {a.genome} bp genome (seed 12, 0.5 % errors), -k{K} -K32 --kc={KC} -H{H} -b{a.bloom}",
           "mask": mask, "gpu": name, "power_limit": power, "pass1_ms": round(pass1, 1), "fasta_md5": md5s[True].pop(),
           "tiles": summary(rows[True]), "no_tiles": summary(rows[False])}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
