#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: regenerates tests/golden/longread_cases.json, the pass-2 goldens of long reads (5 to 80 kbp), from the
UNMODIFIED reference binaries built by oracle/Makefile (oracle/_ref, -j1 is deterministic).  Every read is made here from
seeds, so the tests rebuild the same files and no read file is committed.

A long read seeds an extension at every k-mer that no earlier unitig of the same read covers (processRead, bloom-dbg.h:783-882),
so it yields many unitigs: unique stretches, repeat copies and the length-k branch k-mers between them.  The cases reach the
kernel paths that short reads never do: unitigs of 2^15 k-mers and more (the whole-grid replay of K5), reads of more than
1 024 k-mers (the strided read-level loops of K2, K3 and K5), overflow of the K4 record buffer, and long ballot loops in the
coverage marking of the walks.

  lr_repeats_k{32,64,160}        255 kbp of unique segments joined by copies of a 300 bp and a 2 kbp repeat; 60 error-free
                                 reads of 5, 20 and 80 kbp on both strands and reads at both genome ends
  lr_boundary_k{64,128}_{N}      a linear random genome of N + k - 1 bp, N = 32 767 and 32 768, tiled by 6 kbp reads on both
                                 strands: one unitig of exactly N k-mers, on both sides of the replay's 2^15 threshold
  lr_dense_k64                   600 x (800 bp unique + one 200 bp repeat), 512 reads of 20 kbp: every read is a candidate
                                 and each generating read yields well over 100 unitigs
  lr_mixed_k64                   the long reads of lr_repeats_k64 among 150 bp reads of the same genome (30x, 0.5 % errors);
                                 three long reads carry one substitution past base 2 000 and must come out NOT_SOLID

For each case the script records md5 of the FASTA and the read log, sha256 of the -T trace (the length cell of redundant rows
blanked, as make_golden_trace.py does), sha256 of the counters of `abyss-bloom build -t counting`, the unitig count, bases and
longest unitig, and the counts its preconditions are asserted on.  It asserts those preconditions, so a change of seed cannot
quietly drop the paths a case is there to reach.  It prints the reference's wall time per case.

    python tests/golden/make_golden_longreads.py

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
from abyss_b200.synth import revcomp  # noqa: E402
from make_golden_kwidth import blank_trace, counters_for_budget, write_fastq  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
DBG = os.path.join(REF, "abyss-bloom-dbg-ref")
BLOOM = os.path.join(REF, "abyss-bloom-ref")
BIG = 1 << 15  # kBigContig (abb_assemble.cu): unitigs of this many k-mers and more are replayed by the whole grid


# ---- genomes and reads ---------------------------------------------------------------------------------------------------

def _rand(rng, n):
    return "".join(np.array(list("ACGT"))[rng.integers(0, 4, n)])


def repeat_genome(seed):
    """unique segments of 600 bp to 52 kbp, six of them long enough for a unitig of 2^15 k-mers at k = 160, joined
    alternately by copies of a 300 bp and a 2 kbp repeat"""
    rng = np.random.default_rng(seed)
    reps = [_rand(rng, 300), _rand(rng, 2000)]
    uniq = [600, 52000, 900, 34000, 1500, 41000, 700, 36000, 2500, 47000, 800, 33500, 1200]
    parts = []
    for i, n in enumerate(uniq):
        parts.append(_rand(rng, n))
        if i + 1 < len(uniq):
            parts.append(reps[i % 2])
    return "".join(parts)


def dense_genome(seed, units=600):
    """units x (800 bp unique + the same 200 bp repeat)"""
    rng = np.random.default_rng(seed)
    rep = _rand(rng, 200)
    return "".join(_rand(rng, 800) + rep for _ in range(units))


def _strand(rng, s):
    return revcomp(s) if rng.random() < 0.5 else s


def long_reads(spec):
    """lr_repeats: 60 error-free reads of 5, 20 and 80 kbp at random places on either strand, then a 20 kbp read at each
    genome end on both strands"""
    g = repeat_genome(spec["seed"])
    rng = np.random.default_rng(spec["seed"] + 1)
    out = []
    for i in range(60):
        L = (5000, 20000, 80000)[i % 3]
        p = int(rng.integers(0, len(g) - L + 1))
        out.append((f"r{i}", _strand(rng, g[p:p + L])))
    for j, s in enumerate((g[:20000], g[-20000:])):
        out += [(f"e{2 * j}", s), (f"e{2 * j + 1}", revcomp(s))]
    return out


MUTATED = (7, 22, 40)  # long reads of lr_mixed with one substitution past base 2 000


def raw_reads(spec):
    """[(id, sequence)] of a case's read set, in file order"""
    kind = spec["kind"]
    if kind == "repeats":
        return long_reads(spec)
    if kind == "boundary":  # reads of 6 kbp every 2 kbp, the last one flush with the genome end, each on both strands
        rng = np.random.default_rng(spec["seed"])
        g = _rand(rng, spec["kmers"] + spec["k"] - 1)
        starts = list(range(0, len(g) - 6000, 2000)) + [len(g) - 6000]
        out = []
        for i, p in enumerate(starts):
            out += [(f"b{2 * i}", g[p:p + 6000]), (f"b{2 * i + 1}", revcomp(g[p:p + 6000]))]
        return out
    if kind == "dense":
        g = dense_genome(spec["seed"])
        rng = np.random.default_rng(spec["seed"] + 1)
        out = []
        for i in range(spec["n"]):
            p = int(rng.integers(0, len(g) - 20000 + 1))
            out.append((f"d{i}", _strand(rng, g[p:p + 20000])))
        return out
    if kind == "mixed":
        longs = long_reads(spec)
        rng = np.random.default_rng(spec["seed"] + 2)
        for i in MUTATED:
            name, s = longs[i]
            p = int(rng.integers(2000, len(s) - 2000))
            longs[i] = (name, s[:p] + "ACGT"[("ACGT".index(s[p]) + 1) % 4] + s[p + 1:])
        g = repeat_genome(spec["seed"])
        n, L = int(len(g) * spec["cov"] / 150), 150
        pos = rng.integers(0, len(g) - L + 1, n)
        flip = rng.random(n) < 0.5
        err = rng.random((n, L)) < spec["err"]
        shift = rng.integers(1, 4, (n, L))
        codes = np.frombuffer(g.encode(), dtype=np.uint8)
        lut = np.zeros(256, dtype=np.uint8)
        lut[np.frombuffer(b"ACGT", dtype=np.uint8)] = np.arange(4)
        gc = lut[codes]
        acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
        shorts = []
        for i in range(n):
            c = gc[pos[i]:pos[i] + L]
            c = np.where(err[i], (c + shift[i]) % 4, c)
            s = acgt[c].tobytes().decode()
            shorts.append((f"s{i}", revcomp(s) if flip[i] else s))
        # one long read after every n / len(longs) short reads
        step = n // len(longs)
        out = []
        for j, lr in enumerate(longs):
            out += shorts[j * step:(j + 1) * step] + [lr]
        return out + shorts[len(longs) * step:]
    raise ValueError(kind)


def write_fasta(records, path, width=60):
    with open(path, "w") as f:
        for i, s in records:
            f.write(f">{i}\n" + "".join(s[j:j + width] + "\n" for j in range(0, len(s), width)))


# ---- cases ---------------------------------------------------------------------------------------------------------------

def cases():
    out = []

    def case(name, k, reads, kc=2, b="16M"):
        out.append(dict(name=name, k=k, kc=kc, H=4, b=b, counters=counters_for_budget(b), reads=reads))
    for k in (32, 64, 160):
        case(f"lr_repeats_k{k}", k, dict(kind="repeats", seed=31))
    for k in (64, 128):
        for n in (BIG - 1, BIG):
            case(f"lr_boundary_k{k}_{n}", k, dict(kind="boundary", seed=40 + k, k=k, kmers=n))
    case("lr_dense_k64", 64, dict(kind="dense", seed=51, n=512), b="64M")
    case("lr_mixed_k64", 64, dict(kind="mixed", seed=31, cov=30, err=0.005), kc=3)
    return out


# ---- the reference and the preconditions ---------------------------------------------------------------------------------

def md5(data):
    return hashlib.md5(data).hexdigest()


def sha256(data):
    return hashlib.sha256(data).hexdigest()


def trace_rows(text, k):
    """the -T rows as (read_id, redundant, k-mers): printed rows from their length, redundant rows from the untrimmed path
    (left + right extension + 1), less the at most two vertices trimming removes"""
    out = []
    for line in text.splitlines()[1:]:
        r = line.split("\t")
        red = r[2] == "1"
        if red:
            n = sum(int(x) for x in (r[5], r[7]) if x != "NA") + 1 - 2
        else:
            n = int(r[1]) - k + 1
        out.append((r[3], red, n))
    return out


def preconditions(c, fasta, log, trace):
    k, rows = c["k"], trace_rows(trace, c["k"])
    codes = dict(l.split("\t") for l in log.splitlines()[1:])
    big = [n >= BIG for _, _, n in rows]
    p = dict(rows=len(rows), printed_big=sum(b and not red for b, (_, red, _) in zip(big, rows)),
             redundant_big=sum(b and red for b, (_, red, _) in zip(big, rows)))
    firsts = {}
    for i, (rid, _, _) in enumerate(rows):
        firsts.setdefault(rid, i)
    p["big_first_with_more"] = sum(big[i] and i + 1 < len(rows) and rows[i + 1][0] == rid for rid, i in firsts.items())
    p["big_then_same_read"] = sum(big[i] and rows[i + 1][0] == rows[i][0] for i in range(len(rows) - 1))
    p["big_adjacent"] = sum(big[i] and big[i + 1] for i in range(len(rows) - 1))
    # rows shorter than k + 4 bases; a redundant row's untrimmed path is an upper bound of its length
    p["short_printed"] = sum(not red and n + k - 1 < k + 4 for _, red, n in rows)
    p["short_redundant"] = sum(red and n + 2 + k - 1 < k + 4 for _, red, n in rows)
    p["candidates"] = sum(v in ("GENERATED_CONTIGS", "ALL_KMERS_VISITED") for v in codes.values())
    gen = [rid for rid, v in codes.items() if v == "GENERATED_CONTIGS"]
    p["generating_reads"] = len(gen)
    p["rows_per_generating_read"] = round(len(rows) / max(1, len(gen)), 1)
    seqs = [l for l in fasta.splitlines() if not l.startswith(">")]
    p["unitig_kmers"] = sorted(len(s) - k + 1 for s in seqs)[-3:]
    name = c["name"]
    if name.startswith("lr_repeats"):
        assert p["printed_big"] >= 3 and p["redundant_big"] >= 2, p
        assert p["big_first_with_more"] >= 1 and p["big_then_same_read"] >= 1 and p["big_adjacent"] >= 1, p
        assert p["short_printed"] >= 1 and p["short_redundant"] >= 1, p
    elif name.startswith("lr_boundary"):
        assert len(seqs) == 1 and len(seqs[0]) - k + 1 == c["reads"]["kmers"], p
    elif name == "lr_dense_k64":
        assert p["candidates"] >= 500 and p["rows_per_generating_read"] >= 100, p
    elif name == "lr_mixed_k64":
        p["mutated_not_solid"] = sum(codes[f"r{i}"] == "NOT_SOLID" for i in MUTATED)
        assert p["mutated_not_solid"] == len(MUTATED), p
        assert p["candidates"] >= 1000, p
    return p


def run_case(c, d):
    fq = os.path.join(d, c["name"] + ".fq")
    write_fastq(raw_reads(c["reads"]), fq)
    fa, log, tr, bf = (os.path.join(d, c["name"] + x) for x in (".fa", ".log", ".trace", ".bloom"))
    t0 = time.time()
    r = subprocess.run(["bash", "-c", "ulimit -s 65536; exec " + " ".join([DBG, "-j1", f"-k{c['k']}", f"--kc={c['kc']}", f"-b{c['b']}",
                        f"-H{c['H']}", f"--read-log={log}", "-T", tr, fq])], capture_output=True)
    secs = time.time() - t0
    if r.returncode:
        raise SystemExit(r.stderr.decode())
    subprocess.run([BLOOM, "build", "-k", str(c["k"]), "-t", "counting", f"-b{c['counters']}", f"-H{c['H']}", "-j1", bf, fq],
                   check=True, capture_output=True)
    blob = open(bf, "rb").read()
    raw = blob[blob.index(b"[HeaderEnd]\n") + 12:]
    assert len(raw) == c["counters"]
    fasta, logtext, trace = r.stdout.decode(), open(log).read(), open(tr).read()
    seqs = [l for l in fasta.splitlines() if not l.startswith(">")]
    out = dict(c, fasta_md5=md5(r.stdout), readlog_md5=md5(logtext.encode()), trace_sha256=sha256(blank_trace(trace).encode()),
               counters_sha256=sha256(raw), n_contigs=len(seqs), bases=sum(map(len, seqs)), longest=max(map(len, seqs), default=0),
               reads_md5=md5(open(fq, "rb").read()), pre=preconditions(c, fasta, logtext, trace))
    return out, secs


def main():
    out = []
    with tempfile.TemporaryDirectory() as d:
        for c in cases():
            res, secs = run_case(c, d)
            out.append(res)
            print(f"{c['name']}: {res['n_contigs']} unitigs, reference {secs:.1f} s, {res['pre']}", flush=True)
    json.dump(out, open(os.path.join(HERE, "longread_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
