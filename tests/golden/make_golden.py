#!/usr/bin/env python
"""Regenerate the committed golden fixtures from the UNMODIFIED reference compiled in
oracle/_ref (see oracle/Makefile; make -C oracle ref REF=<reference source tree>).

    make -C oracle ref && python tests/golden/make_golden.py

Fixtures (all small, committed):
  seqs_edge.txt            hand-written edge-case reads (N runs, lower case, short, non-ACGT letters)
  hashes_k{K}.npz          RollingHashIterator output (pos, H hashes) for seqs_edge + seeded reads
  hashes_mask.npz          same with a spaced seed
  count_*.npz              CountingBloomFilter<uint8_t> arrays after inserting seeded reads (tiny m => collisions)
  bits_*.npz / casc_*.npz  BloomFilter / HashAgnosticCascadingBloom arrays
  e2e_*.fa                 abyss-bloom-dbg -j1 FASTA for seeded synthetic read sets (reads regenerated
                           by abyss_b200.synth from the seeds recorded in e2e_cases.json)
"""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from abyss_b200.synth import ReadSet  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
ARITH = os.path.join(REF, "ref_arith")
DBG = os.path.join(REF, "abyss-bloom-dbg-ref")
BLOOM = os.path.join(REF, "abyss-bloom-ref")

EDGE = [
    "ACGTACACTGGACTGAGTCT",                      # vendor/nthash/unittest/UnitTests.cpp:45 vector
    "GCAATGT", "AAANAAA", "ACGT", "A", "",
    "acgtacgtNNacgtacgtacgtacgtacgtacgtacgtacgtacgtacg",
    "ACGTNACGTACGTACGTACGTRACGTACGTACGTACGTACGTACGTACGTUACGTACGATCGATCGATCGATCGACTAGCTAGCTAGCTAGCATCGATCG",
    "NNNNNNNNNNNNNNNNNNNNNNNNNNNNNNNNNNNNNNNN",
    "TTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTT",
    "ACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTACGTN",
    "GATTACAGATTACAGATTACAGATTACAGATTACAGATTACAGATTACAGATTACAGATTACAGATTACAGATTACAGATTACAnGATTACAGATTACA",
]


def si_bytes(s):
    mult = {"k": 1 << 10, "M": 1 << 20, "G": 1 << 30}
    return int(s[:-1]) * mult[s[-1]] if s[-1] in mult else int(s)


def counters_for_budget(b):
    x = si_bytes(b) / 1.125
    r = int(x + 0.5)
    return r if r % 64 == 0 else r + 64 - r % 64


def run(cmd, stdin=None):
    r = subprocess.run(cmd, input=stdin, capture_output=True, check=True)
    return r.stdout


def seeded_reads(seed, genome, n, L, err=0.01):
    rs = ReadSet(seed, genome, n, L, err)
    return [a.tobytes().decode() for a in rs.ascii(0, n)]


def hashes_fixture(name, seqs, k, H, mask=None):
    inp = ("\n".join(seqs) + "\n").encode()
    cmd = [ARITH, "hashes", str(k), str(H)] + ([mask] if mask else [])
    out = run(cmd, inp).decode().split("\n")
    rows = [list(map(int, l.split())) for l in out if l]
    arr = np.array(rows, dtype=np.uint64).reshape(-1, 2 + H)
    np.savez_compressed(os.path.join(HERE, name), seq=arr[:, 0].astype(np.uint32), pos=arr[:, 1].astype(np.uint32),
                        h=arr[:, 2:], k=k, H=H, mask=mask or "")
    print(name, arr.shape)


def filter_fixture(name, kind, seqs, k, H, m, L=None):
    # empty lines would be read as empty sequences by ref_arith's getline loop, same as ours
    inp = ("\n".join(seqs) + "\n").encode()
    cmd = [ARITH, kind, str(k), str(H), str(m)] + ([str(L)] if L else [])
    raw = np.frombuffer(run(cmd, inp), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, name), data=raw, k=k, H=H, m=m, L=L or 0)
    print(name, raw.shape, int(raw.sum()))


def main():
    with open(os.path.join(HERE, "seqs_edge.txt"), "w") as f:
        f.write("\n".join(EDGE) + "\n")
    reads60 = seeded_reads(11, 3000, 1500, 60)
    reads150 = seeded_reads(12, 20000, 600, 150)
    for k in (5, 20, 32, 64):
        hashes_fixture(f"hashes_k{k}.npz", EDGE + reads150[:40], k, 4)
    hashes_fixture("hashes_mask.npz", EDGE + reads150[:40], 11, 3, "10100011101")
    hashes_fixture("hashes_mask33.npz", EDGE + reads150[:40], 33, 4, "101000111010000000000010111000101")
    # tiny filters => many shared counters => order dependence is exercised
    filter_fixture("count_m4096.npz", "count", EDGE + reads60, 20, 4, 4096)
    filter_fixture("count_m65536_H3.npz", "count", reads150, 32, 3, 65536)
    filter_fixture("count_sat.npz", "count", [EDGE[9]] * 40 + reads60[:200], 20, 2, 1024)   # saturates at 255
    filter_fixture("bits_m8192.npz", "bits", EDGE + reads60, 20, 4, 8192)
    filter_fixture("casc_m8192_L3.npz", "casc", EDGE + reads60 + reads60[:700], 20, 4, 8192, 3)

    # end-to-end FASTA goldens (-j1 is deterministic)
    cases = [
        dict(name="e2e_g20k_k32", seed=21, genome=20000, cov=30, L=150, err=0.005, k=32, kc=2, b="1M", H=4),
        dict(name="e2e_g30k_k64", seed=22, genome=30000, cov=40, L=150, err=0.005, k=64, kc=3, b="2M", H=4),
        dict(name="e2e_g10k_k25_small", seed=23, genome=10000, cov=25, L=100, err=0.01, k=25, kc=2, b="64k", H=3),
    ]
    tmp = "/tmp/abyss_golden"
    os.makedirs(tmp, exist_ok=True)
    for c in cases:
        rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
        fq = os.path.join(tmp, c["name"] + ".fq")
        rs.write_fastq(fq)
        out = os.path.join(HERE, c["name"] + ".fa")
        log = os.path.join(HERE, c["name"] + ".readlog.tsv")
        cmd = f"ulimit -s 65536; {DBG} -k{c['k']} --kc={c['kc']} -b{c['b']} -H{c['H']} -j1 --read-log={log} {fq} > {out}"
        subprocess.run(["bash", "-c", cmd], check=True)
        c["n_reads"] = rs.n
        c["n_contigs"] = sum(1 for l in open(out) if l.startswith(">"))
        # counting filter from `abyss-bloom build -t counting` with the counter count that
        # abyss-bloom-dbg derives from -b (bloom-dbg.cc:359-367): sha256 of the raw array
        counters = counters_for_budget(c["b"])
        bf = os.path.join(tmp, c["name"] + ".bloom")
        subprocess.run([BLOOM, "build", "-k", str(c["k"]), "-t", "counting", f"-b{counters}", f"-H{c['H']}", "-j1", bf, fq],
                       check=True, capture_output=True)
        blob = open(bf, "rb").read()
        tag = b"[HeaderEnd]\n"
        raw = blob[blob.index(tag) + len(tag):]
        assert len(raw) == counters, (len(raw), counters)
        c["counters"] = counters
        c["bloom_header"] = blob[:blob.index(tag) + len(tag)].decode()
        c["counters_sha256"] = hashlib.sha256(raw).hexdigest()
        c["counters_nonzero"] = int(np.count_nonzero(np.frombuffer(raw, dtype=np.uint8)))
        # `abyss-bloom build -t rolling-hash -l 2`: whole file (header + last level) sha256
        rh = os.path.join(tmp, c["name"] + ".rh.bloom")
        subprocess.run([BLOOM, "build", "-k", str(c["k"]), "-t", "rolling-hash", "-l", "2", f"-H{c['H']}", f"-b{counters // 4}", "-j1", rh, fq],
                       check=True, capture_output=True)
        c["rolling_hash_l2_b"] = counters // 4
        c["rolling_hash_l2_file_sha256"] = hashlib.sha256(open(rh, "rb").read()).hexdigest()
        c["counting_file_sha256"] = hashlib.sha256(blob).hexdigest()
        print(c["name"], c["n_reads"], c["n_contigs"], counters, c["counters_nonzero"])
    json.dump(cases, open(os.path.join(HERE, "e2e_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
