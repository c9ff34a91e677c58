#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: regenerates tests/golden/spaced_tiles_cases.json, the pass-2 goldens of spaced-seed runs (-K,
--qr-seed) large enough for the tile store to do real work, from the UNMODIFIED reference binaries built by oracle/Makefile
(oracle/_ref, -j1 is deterministic).  Every read is made here from seeds, so the tests rebuild the same files and no read
file is committed.

With a spaced seed, tiles are named by the canonical hash of the full k-mer (tile_key, abyss_b200/csrc/abb_walk.cuh), not by
the vertex identity, which ignores the don't-care positions.  The cases:

  sp_cfg1_k64_K24        config 1's reads (200 kbp genome seed 1, 53 333 x 150 bp, 0.5 % errors) at -k64 -K24
  sp_cfg1_k80_K32        the same reads at -k80 -K32: kmerPair(80, 32), the seed shape of config 4
  sp_m1_k80_K32          1 M x 150 bp of a 5 Mbp genome (30x, 0.5 % errors) at -k80 -K32 -b1G --kc=3: more new markers in one
                         batch than the marker list of a tile store sized for a small assembly holds
  sp_lr_k64_qr31         the long reads of lr_repeats (make_golden_longreads.py) at -k64 --qr-seed=31: unitigs of 2^15 k-mers
                         and more, built from tiles under a mask
  sp_adversary_k64_K24   a don't-care adversary: a k-mer X occurs at one locus and X', which differs from X at one don't-care
                         position only, at another, with unrelated sequence around each.  X and X' are one vertex to the
                         reference (equal identity) and a marker under identity keying (identity & 255 == 0), but they
                         continue differently: a tile named by the identity would splice one locus's continuation into
                         the other's unitig.

For each case the script records md5 of the FASTA and the read log, sha256 of the -T trace (the length cell of redundant rows
blanked, as make_golden_trace.py does), the mask, the unitig count, bases and longest unitig, and the counts its
preconditions are asserted on.  It prints the reference's wall time per case: 35, 44, 204, 14 and 3 s in the order above on one
core, about 5 minutes with the read generation.

    python tests/golden/make_golden_spaced_tiles.py

Run where the reference binaries are built (oracle/_ref: make -C oracle ref REF=...)."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from abyss_b200.synth import ReadSet, revcomp  # noqa: E402
from make_golden_kwidth import blank_trace, counters_for_budget, write_fastq  # noqa: E402
from make_golden_longreads import long_reads  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
DBG = os.path.join(REF, "abyss-bloom-dbg-ref")
BIG = 1 << 15  # kBigContig (abb_assemble.cu)
MARKER_MASK = 255  # kMarkerMask (abb_walk.cuh)


# ---- ntHash of a k-mer (nthash.hpp), for the adversary's identity ---------------------------------------------------------

_SEED = {"A": 0x3c8bfbb395c60474, "C": 0x3193c18562a02b4c, "G": 0x20323ed082572324, "T": 0x295549f54be24456}


def _srol_n(x, n):
    """ntHash's split rotation: the top 31 bits and the low 33 bits rotate separately"""
    n31, n33 = n % 31, n % 33
    hi, lo = x >> 33, x & ((1 << 33) - 1)
    hi = ((hi << n31) | (hi >> (31 - n31))) & ((1 << 31) - 1) if n31 else hi
    lo = ((lo << n33) | (lo >> (33 - n33))) & ((1 << 33) - 1) if n33 else lo
    return (hi << 33) | lo


def identity(kmer, mask):
    """the reference's vertex identity under a spaced seed (RollingBloomDBG.h:92-158): the masked forward hash of the
    orientation of the FULL k-mer that is not greater than its reverse complement (what Vtx::id holds)"""
    cs = min(kmer, revcomp(kmer))
    k, h = len(kmer), 0
    for i in range(k):
        if mask[i] == "1":
            h ^= _srol_n(_SEED[cs[i]], k - 1 - i)
    return h


# ---- read sets -----------------------------------------------------------------------------------------------------------

def _rand(rng, n):
    return "".join(np.array(list("ACGT"))[rng.integers(0, 4, n)])


def adversary_genome(spec):
    """a random genome with X at spec['at'][0] and X' at spec['at'][1].  X starts and ends with 'A', so X and X' are both
    the canonical orientation; X' has the other base at don't-care position spec['p']; the seed is searched so that the
    shared identity is a marker (make_golden_spaced_tiles.py finds it, the case records it)"""
    rng = np.random.default_rng(spec["seed"])
    k, p = spec["k"], spec["p"]
    g = list(_rand(rng, spec["genome"]))
    x = "A" + _rand(rng, k - 2) + "A"
    alt = "ACGT"[("ACGT".index(x[p]) + 1 + int(rng.integers(0, 3))) % 4]
    x2 = x[:p] + alt + x[p + 1:]
    a, b = spec["at"]
    g[a:a + k] = x
    g[b:b + k] = x2
    return "".join(g), x, x2


def raw_reads(spec):
    """[(id, sequence)] of a case's read set, in file order"""
    kind = spec["kind"]
    if kind == "readset":
        rs = ReadSet(spec["seed"], spec["genome"], spec["n_reads"], spec["L"], spec["err"])
        return [(rs.read_id(i), a.tobytes().decode()) for i, a in enumerate(rs.ascii(0, rs.n))]
    if kind == "repeats":
        return long_reads(spec)
    if kind == "adversary":
        g = adversary_genome(spec)[0]
        rng = np.random.default_rng(spec["seed"] + 1)
        n, L = int(len(g) * spec["cov"] / spec["L"]), spec["L"]
        out = []
        for i in range(n):
            q = int(rng.integers(0, len(g) - L + 1))
            s = g[q:q + L]
            out.append((f"a{i}", revcomp(s) if rng.random() < 0.5 else s))
        return out
    raise ValueError(kind)


def find_adversary_seed(k, mask, p, first=1):
    """the first seed from `first` whose X has a marker identity"""
    seed = first
    while True:
        spec = dict(kind="adversary", seed=seed, k=k, p=p, genome=20000, at=[6000, 14000], cov=30, L=150)
        _, x, x2 = adversary_genome(spec)
        if identity(x, mask) & MARKER_MASK == 0:
            assert identity(x2, mask) == identity(x, mask)
            return spec
        seed += 1


def kmer_pair(k, K):
    return "1" * K + "0" * (k - 2 * K) + "1" * K


def qr_seed_pair(k, length):
    qr = ["1"] * length
    for i in range(length):
        if any(j * j % length == i for j in range(1, length)):
            qr[i] = "0"
    m = ["0"] * k
    for i, c in enumerate(qr):
        m[i] = m[k - 1 - i] = c
    return "".join(m)


# ---- cases ---------------------------------------------------------------------------------------------------------------

CFG1 = dict(kind="readset", seed=1, genome=200000, n_reads=53333, L=150, err=0.005)
M1 = dict(kind="readset", seed=2, genome=5000000, n_reads=1000000, L=150, err=0.005)


def cases():
    out = []

    def case(name, k, opt, mask, reads, kc=2, b="64M"):
        out.append(dict(name=name, k=k, kc=kc, H=4, b=b, counters=counters_for_budget(b), opt=opt, mask=mask, reads=reads))
    case("sp_cfg1_k64_K24", 64, "-K24", kmer_pair(64, 24), CFG1)
    case("sp_cfg1_k80_K32", 80, "-K32", kmer_pair(80, 32), CFG1)
    case("sp_m1_k80_K32", 80, "-K32", kmer_pair(80, 32), M1, kc=3, b="1G")
    case("sp_lr_k64_qr31", 64, "--qr-seed=31", qr_seed_pair(64, 31), dict(kind="repeats", seed=31), b="16M")
    m = kmer_pair(64, 24)
    case("sp_adversary_k64_K24", 64, "-K24", m, find_adversary_seed(64, m, 31), b="16M")
    return out


# ---- the reference and the preconditions ---------------------------------------------------------------------------------

def md5(data):
    return hashlib.md5(data).hexdigest()


def sha256(data):
    return hashlib.sha256(data).hexdigest()


def preconditions(c, fasta, log):
    k = c["k"]
    seqs = [l for l in fasta.splitlines() if not l.startswith(">")]
    codes = [l.split("\t")[1] for l in log.splitlines()[1:]]
    p = dict(unitig_kmers=sorted(len(s) - k + 1 for s in seqs)[-3:], generating_reads=codes.count("GENERATED_CONTIGS"))
    if c["name"].startswith(("sp_cfg1", "sp_m1")):
        # unitigs of thousands of k-mers: walks pass many markers
        assert p["unitig_kmers"][-1] > 10000 and p["generating_reads"] > 10, p
    elif c["name"].startswith("sp_lr"):
        p["big_unitigs"] = sum(len(s) - k + 1 >= BIG for s in seqs)
        assert p["big_unitigs"] >= 3, p
    elif c["name"].startswith("sp_adversary"):
        _, x, x2 = adversary_genome(c["reads"])
        assert x != x2 and c["mask"][c["reads"]["p"]] == "0"
        assert identity(x, c["mask"]) == identity(x2, c["mask"]) and identity(x, c["mask"]) & MARKER_MASK == 0
        # both loci are in the output, each with its own continuation: X and X' each lie inside an emitted unitig
        p["x_in"] = sum(x in s or revcomp(x) in s for s in seqs)
        p["x2_in"] = sum(x2 in s or revcomp(x2) in s for s in seqs)
        assert p["x_in"] >= 1 and p["x2_in"] >= 1, p
    return p


def run_case(c, d):
    fq = os.path.join(d, c["name"] + ".fq")
    write_fastq(raw_reads(c["reads"]), fq)
    log, tr = (os.path.join(d, c["name"] + x) for x in (".log", ".trace"))
    t0 = time.time()
    r = subprocess.run(["bash", "-c", "ulimit -s 65536; exec " + " ".join([DBG, "-j1", f"-k{c['k']}", c["opt"], f"--kc={c['kc']}",
                        f"-b{c['b']}", f"-H{c['H']}", "-v", f"--read-log={log}", "-T", tr, fq])], capture_output=True)
    secs = time.time() - t0
    if r.returncode:
        raise SystemExit(r.stderr.decode())
    used = [l.split()[3] for l in r.stderr.decode().splitlines() if l.startswith("Using spaced seed")]
    assert used == [c["mask"]], (used, c["mask"])
    fasta, logtext, trace = r.stdout.decode(), open(log).read(), open(tr).read()
    seqs = [l for l in fasta.splitlines() if not l.startswith(">")]
    out = dict(c, fasta_md5=md5(r.stdout), readlog_md5=md5(logtext.encode()), trace_sha256=sha256(blank_trace(trace).encode()),
               n_contigs=len(seqs), bases=sum(map(len, seqs)), longest=max(map(len, seqs), default=0),
               reads_md5=md5(open(fq, "rb").read()), pre=preconditions(c, fasta, logtext))
    return out, secs


def main():
    out = []
    with tempfile.TemporaryDirectory() as d:
        for c in cases():
            res, secs = run_case(c, d)
            out.append(res)
            print(f"{c['name']}: {res['n_contigs']} unitigs, reference {secs:.1f} s, {res['pre']}", flush=True)
    json.dump(out, open(os.path.join(HERE, "spaced_tiles_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
