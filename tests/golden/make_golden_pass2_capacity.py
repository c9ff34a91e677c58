#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: goldens for pass 2 when its bounded tile scratch fills up, from the UNMODIFIED reference compiled in
oracle/_ref (`make -C oracle ref`; -j1 is deterministic).  Writes pass2_capacity.json: per case the md5 of the reference's
FASTA and --read-log, the sha256 of the counters of `abyss-bloom build -t counting`, unitig count, total bases and the
longest unitig, and the overflow precondition computed here from those counters:

  mset_fresh   marker-set entries the library sizes for a fresh assembler (ensure_tile_store in abb_assemble.cu)
  mset_reset   the same after the small first assembly of `first` (a reused handle keeps that store)
  solid_markers  distinct canonical hashes of valid, solid k-mer windows of the reads that are markers (low 8 bits clear)

  g12m_k64         12 Mbp genome (seed 11) at 20x, 1.6 M x 150 bp, -k64 --kc=3 -b1G -H4.  solid_markers > mset_reset, so a
                   handle first sized by 400 reads of a 10 kbp genome overflows its marker set; a fresh one does not.
  overload_k25_H1  13 333 reads of a 20 kbp genome at 100x followed by 200 000 reads of a 250 Mbp genome (0.12x) in a
                   256 KiB filter with one hash, kc chosen so that about half the counters are >= kc: the marker set
                   of a fresh handle overflows.

Run in the build container only:  python tests/golden/make_golden_pass2_capacity.py [case ...]"""
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from abyss_b200.synth import ReadSet  # noqa: E402
import oracle_py  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
DBG = os.path.join(REF, "abyss-bloom-dbg-ref")
BLOOM = os.path.join(REF, "abyss-bloom-ref")
TMP = "/tmp/abyss_golden_pass2_capacity"
MARKER_MASK = 255  # kMarkerMask, abb_walk.cuh

CASES = [
    dict(name="g12m_k64", parts=[dict(prefix="r", seed=11, genome=12_000_000, n_reads=1_600_000)], L=150, err=0.005, k=64, kc=3,
         b="1G", H=4, first=dict(prefix="s", seed=12, genome=10_000, n_reads=400)),
    dict(name="overload_k25_H1", parts=[dict(prefix="f", seed=13, genome=20_000, n_reads=13_333),
                                        dict(prefix="b", seed=14, genome=250_000_000, n_reads=200_000)], L=150, err=0.005, k=25,
         kc=None, b="256k", H=1, first=None),
]


def counters_for_budget(b):  # bloom-dbg.cc:359-367
    mult = {"k": 1 << 10, "M": 1 << 20, "G": 1 << 30}
    x = int(b[:-1]) * mult[b[-1]] / 1.125
    r = int(x + 0.5)
    return r if r % 64 == 0 else r + 64 - r % 64


def read_chunks(parts, L, err, chunk=1 << 16):
    """(ids, (n, L) ASCII array) of the reads of `parts` in file order; tests/test_gpu_pass2_capacity.py builds the same"""
    for p in parts:
        rs = ReadSet(p["seed"], p["genome"], p["n_reads"], L, err)
        for lo in range(0, rs.n, chunk):
            hi = min(rs.n, lo + chunk)
            yield [f"{p['prefix']}{i}" for i in range(lo, hi)], rs.ascii(lo, hi)


def write_reads(c, path, parts=None):
    with open(path, "wb") as f:
        for ids, a in read_chunks(parts or c["parts"], c["L"], c["err"]):
            q = b"I" * c["L"]
            f.write(b"".join(b"@" + i.encode() + b"\n" + a[j].tobytes() + b"\n+\n" + q + b"\n" for j, i in enumerate(ids)))


def md5_file(path):
    h = hashlib.md5()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 22), b""):
            h.update(blk)
    return h.hexdigest()


def mset_size(counters, kc, H):
    """the marker-set entries ensure_tile_store allocates for a filter with these counters"""
    solid = int((counters >= kc).sum()) // max(1, H) + 1024
    markers = solid // (MARKER_MASK + 1) * 2 + 4096
    m = 1
    while m < markers * 4:
        m <<= 1
    return m


def solid_markers(orc, c, counters, kc):
    """distinct canonical hashes of valid windows that are markers and whose H counters are all >= kc"""
    m = np.uint64(counters.size)
    found = []
    for _, a in read_chunks(c["parts"], c["L"], c["err"]):
        hs = [orc.hash_seq(a[j].tobytes(), c["k"], c["H"])[0] for j in range(a.shape[0])]
        h = np.concatenate(hs)
        h = h[(h[:, 0] & np.uint64(MARKER_MASK)) == 0]
        ok = np.ones(len(h), dtype=bool)
        for i in range(c["H"]):
            ok &= counters[(h[:, i] % m).astype(np.int64)] >= kc
        found.append(np.unique(h[ok, 0]))
    return int(np.unique(np.concatenate(found)).size)


def oracle_counters(orc, parts, c, n):
    counters = np.zeros(n, dtype=np.uint8)
    for _, a in read_chunks(parts, c["L"], c["err"]):
        orc.cbf_load(counters, [a[j].tobytes() for j in range(a.shape[0])], c["k"], c["H"])
    return counters


def main():
    os.makedirs(TMP, exist_ok=True)
    orc = oracle_py.load()
    path = os.path.join(HERE, "pass2_capacity.json")
    done = {c["name"]: c for c in json.load(open(path))} if os.path.exists(path) else {}
    want = set(sys.argv[1:])
    for c in CASES:
        if want and c["name"] not in want:
            continue
        c = dict(c)
        fq, fa, log, bf = (os.path.join(TMP, c["name"] + x) for x in (".fq", ".fa", ".readlog.tsv", ".bloom"))
        write_reads(c, fq)
        n = counters_for_budget(c["b"])
        counters = None
        if c["kc"] is None:  # about half the counters at or above kc
            counters = oracle_counters(orc, c["parts"], c, n)
            c["kc"] = int(np.median(counters))
        t0 = time.time()
        cmd = f"ulimit -s 65536; {DBG} -k{c['k']} --kc={c['kc']} -b{c['b']} -H{c['H']} -j1 --read-log={log} {fq} > {fa}"
        subprocess.run(["bash", "-c", cmd], check=True, capture_output=True)
        c["ref_seconds_j1"] = round(time.time() - t0, 1)
        subprocess.run([BLOOM, "build", "-k", str(c["k"]), "-t", "counting", f"-b{n}", f"-H{c['H']}", "-j1", bf, fq],
                       check=True, capture_output=True)
        blob = open(bf, "rb").read()
        tag = b"[HeaderEnd]\n"
        raw = np.frombuffer(blob[blob.index(tag) + len(tag):], dtype=np.uint8)
        assert raw.size == n
        if counters is not None:
            assert (raw == counters).all(), "oracle counters differ from abyss-bloom build"
        os.remove(bf)
        seqs = [l.strip() for l in open(fa) if not l.startswith(">")]
        c.update(counters=n, counters_sha256=hashlib.sha256(raw.tobytes()).hexdigest(), fasta_md5=md5_file(fa),
                 readlog_md5=md5_file(log), n_contigs=len(seqs), bases=sum(map(len, seqs)), longest=max(map(len, seqs)))
        c["solid_fraction"] = round(float((raw >= c["kc"]).mean()), 4)
        c["mset_fresh"] = mset_size(raw, c["kc"], c["H"])
        c["solid_markers"] = solid_markers(orc, c, raw, c["kc"])
        # the set overflows where the test needs it to, and only there
        if c["first"]:
            c["mset_reset"] = mset_size(oracle_counters(orc, [c["first"]], c, n), c["kc"], c["H"])
            assert c["solid_markers"] > c["mset_reset"], c
            assert c["solid_markers"] < c["mset_fresh"] // 2, c
        else:
            assert c["solid_markers"] > c["mset_fresh"], c
        done[c["name"]] = c
        print(c, flush=True)
        json.dump([done[k] for k in sorted(done)], open(path, "w"), indent=1)


if __name__ == "__main__":
    main()
