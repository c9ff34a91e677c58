#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: regenerates tests/golden/kwidth_cases.json and kwidth_graph_*.dot.gz, the goldens of every k-mer width
the pass-2 kernels are compiled for (Kmer<KW>, KW = ceil(2k / 64): 1, 2, 3, 4 and 6 words up to k = 192), from the UNMODIFIED
reference binaries built by oracle/Makefile (oracle/_ref, -j1 is deterministic).  Every input is made here from seeds, so the
tests rebuild the same files and no read file is committed.

  assembler   abyss-bloom-dbg-ref -j1 --read-log -T       md5 of the FASTA and read log, sha256 of the trace (the length cell
                                                          of redundant rows blanked, as make_golden_trace.py does)
              abyss-bloom-ref build -t counting -j1       sha256 of the counters (not for spaced seeds)
              k = 31 .. 192 around every word boundary; H = 1 and 9; N / lower-case / short reads; mixed read lengths;
              circular, hairpin and tandem genomes; -K and --qr-seed spaced seeds
  dbg_graph   abyss-bloom-dbg-ref -g                      size, line count and sha256 of the GraphViz dump
  covtrack    abyss-bloom-dbg-ref -C -R                   size, line count and sha256 of the WIG track
  graph       abyss-bloom-ref graph                       the dump, kept whole as kwidth_graph_<case>.dot.gz
  trim        abyss-bloom-ref trim                        md5 of the trimmed reads, stderr and the exit status

    python tests/golden/make_golden_kwidth.py

Run where the reference binaries are built (oracle/_ref: make -C oracle ref REF=...)."""
import gzip
import hashlib
import json
import os
import random
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from abyss_b200.synth import ReadSet, edge_mutate, revcomp  # noqa: E402
from make_golden_bloom_graph import filt as graph_filt, genome_text  # noqa: E402
from make_golden_covtrack import ref_fasta  # noqa: E402
from make_golden_konnector import write_reads as write_konnector_reads  # noqa: E402
from make_golden_trim import filt as trim_filt  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
DBG = os.path.join(REF, "abyss-bloom-dbg-ref")
BLOOM = os.path.join(REF, "abyss-bloom-ref")
KS = [31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 140, 159, 160, 161, 191, 192]
WIDE_KS = [97, 128, 129, 160, 192]  # the graph and trim cases


def counters_for_budget(b):  # bloom-dbg.cc:359-367
    mult = {"k": 1 << 10, "M": 1 << 20, "G": 1 << 30}
    r = int(float(b[:-1]) * mult[b[-1]] / 1.125 + 0.5)
    return r if r % 64 == 0 else r + 64 - r % 64


# ---- read sets -----------------------------------------------------------------------------------------------------------

def _sampled(rng, genome, n, L, circular, prefix):
    """n reads of length L from random positions of genome (wrapping around when circular), either strand"""
    g = genome + genome[:L] if circular else genome
    out = []
    for i in range(n):
        p = rng.randrange(len(genome) if circular else len(genome) - L + 1)
        s = g[p:p + L]
        out.append((f"{prefix}{i}", revcomp(s) if rng.random() < 0.5 else s))
    return out


def raw_reads(spec):
    """[(id, sequence)] of a read set as the FASTQ file holds it (before the reader trims lower-case ends)"""
    kind, seed = spec["kind"], spec["seed"]
    if kind in ("plain", "edge"):
        rs = ReadSet.from_coverage(seed, spec["genome"], spec["cov"], spec["L"], spec["err"])
        seqs = [a.tobytes().decode() for a in rs.ascii(0, rs.n)]
        if kind == "edge":  # N, lower-case ends, reads cut to 40 bases
            seqs = edge_mutate(seqs, every_n=13, every_lc=17, every_short=29)
        return [(rs.read_id(i), s) for i, s in enumerate(seqs)]
    if kind == "mixed":  # 150, 250 and 400 bp reads of one genome, interleaved
        sets = [ReadSet.from_coverage(seed, spec["genome"], spec["cov"] / 3, L, spec["err"]) for L in (150, 250, 400)]
        seqs = [[a.tobytes().decode() for a in rs.ascii(0, rs.n)] for rs in sets]
        n = min(len(s) for s in seqs)
        return [(f"m{3 * i + j}", seqs[j][i]) for i in range(n) for j in range(3)]
    rng = random.Random(seed)
    rand = lambda n: "".join(rng.choice("ACGT") for _ in range(n))  # noqa: E731
    n = int(spec["genome"] * spec["cov"] / spec["L"])
    if kind == "circ":  # a plasmid: the walk comes back to its seed (ER_CYCLE)
        return _sampled(rng, rand(spec["genome"]), n, spec["L"], True, "c")
    if kind == "hairpin":  # a sequence followed by its own reverse complement: the path folds back onto its vertices
        arm = rand(spec["genome"] // 2 - 10)
        return _sampled(rng, arm + rand(20) + revcomp(arm), n, spec["L"], False, "h")
    if kind == "tandem":  # units shorter and longer than k repeated in tandem between unique flanks
        u1, u2 = rand(70), rand(230)
        g = rand(1500) + u1 * 8 + rand(1500) + u2 * 5 + rand(1500)
        return _sampled(rng, g, int(len(g) * spec["cov"] / spec["L"]), spec["L"], False, "t")
    raise ValueError(kind)


def reader_view(records):
    """the reads as the reference's reader hands them to the assembler: lower-case ends removed (trimMasked,
    FastaReader.cpp:236-250), the rest folded to upper case"""
    out = []
    for i, s in records:
        a, b = 0, len(s)
        while a < b and s[a].islower():
            a += 1
        while b > a and s[b - 1].islower():
            b -= 1
        out.append((i, s[a:b].upper()))
    return out


def write_fastq(records, path):
    with open(path, "w") as f:
        for i, s in records:
            f.write(f"@{i}\n{s}\n+\n{'I' * len(s)}\n")


# ---- cases ---------------------------------------------------------------------------------------------------------------

def _plain(seed):
    return dict(kind="plain", seed=seed, genome=15000, cov=30, L=250, err=0.005)


def assembler_cases():
    out = []

    def case(name, k, reads, H=4, opt=""):
        out.append(dict(name=name, k=k, kc=2, H=H, b="1M", counters=counters_for_budget("1M"), opt=opt, reads=reads))
    for k in KS:
        case(f"asm_k{k}", k, _plain(500 + k))
    for k in (128, 192):
        for H in (1, 9):
            case(f"asm_k{k}_H{H}", k, _plain(500 + k), H=H)
    for k in (33, 129, 192):
        case(f"asm_edge_k{k}", k, dict(_plain(600 + k), kind="edge"))
    case("asm_mixed_k160", 160, dict(_plain(760), kind="mixed"))
    for k in (128, 129, 160):
        for kind in ("circ", "hairpin", "tandem"):
            case(f"asm_{kind}_k{k}", k, dict(kind=kind, seed=800 + k, genome=6000, cov=30, L=250))
    # spaced seeds; k = 140 and 160 are in the six-word instance with a whole word to drop in kmer_revcomp
    for k, opt in ((128, "-K40"), (140, "--qr-seed=23"), (160, "-K50"), (160, "--qr-seed=31"), (192, "--qr-seed=47"), (192, "-K90")):
        case(f"asm_seed_k{k}_{opt.strip('-').replace('=', '').replace('-', '')}", k, _plain(900 + k), opt=opt)
    return out


def dbg_graph_cases():
    return [dict(name=f"dbg_graph_k{k}", k=k, kc=2, H=3, b="256k", reads=dict(kind="plain", seed=700 + k, genome=4000, cov=20, L=250, err=0.01))
            for k in (97, 128, 192)]


def covtrack_cases():
    return [dict(name=f"covtrack_k{k}", k=k, kc=2, H=4, b="1M", reads=_plain(500 + k)) for k in (97, 128, 192)]


# abyss-bloom graph: reads of the 6 kb genome of make_golden_bloom_graph.py (seed 11) long enough for k = 192
GRAPH_FILTERS = {}
for _k in WIDE_KS:
    for _H in (1, 4):
        GRAPH_FILTERS[f"L{_k}_H{_H}.bloom"] = graph_filt(f"L{_k}_H{_H}.bloom", _k, "256K", _H, ["L.fq"])
    GRAPH_FILTERS[f"Lsub{_k}.bloom"] = graph_filt(f"Lsub{_k}.bloom", _k, "256K", 1, ["Lsub.fq"])


def graph_cases():
    g = genome_text(11, 6000)
    out = []
    for k in WIDE_KS:
        for H in (1, 4):
            gf, af = f"L{k}_H{H}.bloom", f"Lsub{k}.bloom"
            roots = ["-R", g[4000:4000 + k], "-R", revcomp(g[1500:1500 + k])]
            rec = lambda f: ",".join(map(str, GRAPH_FILTERS[f]["recipe"]))  # noqa: E731
            out.append(dict(name=f"graph_k{k}_H{H}", args=["graph", f"-k{k}", "-d30", "-A", f"sub:{af}"] + roots + [gf],
                            harness=[str(k), "30", rec(gf)] + roots + ["-A", "sub:" + rec(af)]))
    return out


def write_graph_inputs(d):
    rs = ReadSet.from_coverage(11, 6000, 12, 300, 0.003)
    recs = [(f"l{i}", a.tobytes().decode()) for i, a in enumerate(rs.ascii(0, rs.n))]
    write_fastq(recs, os.path.join(d, "L.fq"))
    write_fastq(recs[:len(recs) // 3], os.path.join(d, "Lsub.fq"))


# abyss-bloom trim: A.fq of make_golden_konnector.py (250 bp; N, lower-case ends, 40 bp reads) and reads of another genome
TRIM_FILTERS = [trim_filt(f"a{k}.bloom", k, "64K", ["A.fq"]) for k in WIDE_KS]


def write_trim_inputs(d):
    write_konnector_reads(d)
    rs = ReadSet.from_coverage(14, 20000, 8, 300, 0.01)
    write_fastq(list(zip((rs.read_id(i) for i in range(rs.n)), edge_mutate([a.tobytes().decode() for a in rs.ascii(0, rs.n)]))),
                os.path.join(d, "O.fq"))


def trim_cases():
    out = []
    for k in WIDE_KS:
        out.append(dict(name=f"trim_self_k{k}", args=["trim", "-vv", f"-k{k}", f"a{k}.bloom", "A.fq"], harness=[k, f"a{k}.bloom", "A.fq"]))
        out.append(dict(name=f"trim_other_k{k}", args=["trim", f"-k{k}", f"a{k}.bloom", "O.fq"], harness=[k, f"a{k}.bloom", "O.fq"]))
    return out


# ---- the reference -------------------------------------------------------------------------------------------------------

def md5(data):
    return hashlib.md5(data).hexdigest()


def sha256(data):
    return hashlib.sha256(data).hexdigest()


def blank_trace(text):
    """the reference leaves `length` uninitialised in redundant rows (make_golden_trace.py): blank it"""
    rows = [l.rstrip("\n").split("\t") for l in text.splitlines(True)]
    for r in rows[1:]:
        if r[2] == "1":
            r[1] = "-"
    return "".join("\t".join(r) + "\n" for r in rows)


def _dbg(args, d):
    r = subprocess.run(["bash", "-c", "ulimit -s 65536; exec " + " ".join([DBG, "-j1", *args])], cwd=d, capture_output=True)
    if r.returncode:
        raise SystemExit(r.stderr.decode())
    return r


def run_assembler(c, d):
    fq = os.path.join(d, c["name"] + ".fq")
    write_fastq(raw_reads(c["reads"]), fq)
    fa, log, tr = (os.path.join(d, c["name"] + x) for x in (".fa", ".log", ".trace"))
    r = _dbg([f"-k{c['k']}", c["opt"], f"--kc={c['kc']}", f"-b{c['b']}", f"-H{c['H']}", "-v", f"--read-log={log}", "-T", tr, fq], d)
    open(fa, "wb").write(r.stdout)
    out = dict(c)
    for line in r.stderr.decode().splitlines():
        if line.startswith("Using spaced seed"):
            out["mask"] = line.split()[3]
    if c["opt"]:
        assert "mask" in out, r.stderr.decode()
    else:
        bf = os.path.join(d, c["name"] + ".bloom")
        subprocess.run([BLOOM, "build", "-k", str(c["k"]), "-t", "counting", f"-b{c['counters']}", f"-H{c['H']}", "-j1", bf, fq],
                       check=True, capture_output=True)
        blob = open(bf, "rb").read()
        raw = blob[blob.index(b"[HeaderEnd]\n") + 12:]
        assert len(raw) == c["counters"]
        out["counters_sha256"] = sha256(raw)
    out.update(n_contigs=r.stdout.count(b">"), fasta_md5=md5(r.stdout), readlog_md5=md5(open(log, "rb").read()),
               trace_sha256=sha256(blank_trace(open(tr).read()).encode()))
    return out


def main():
    out = {"assembler": [], "dbg_graph": [], "covtrack": [], "graph": [], "trim": []}
    with tempfile.TemporaryDirectory() as d:
        for c in assembler_cases():
            out["assembler"].append(run_assembler(c, d))
            print(c["name"], out["assembler"][-1]["n_contigs"], out["assembler"][-1].get("mask", ""), flush=True)
        for c in dbg_graph_cases():
            fq, dot = os.path.join(d, c["name"] + ".fq"), os.path.join(d, c["name"] + ".dot")
            write_fastq(raw_reads(c["reads"]), fq)
            _dbg([f"-k{c['k']}", f"--kc={c['kc']}", f"-b{c['b']}", f"-H{c['H']}", "-g", dot, "-o", "/dev/null", fq], d)
            data = open(dot, "rb").read()
            out["dbg_graph"].append(dict(c, bytes=len(data), lines=data.count(b"\n"), sha256=sha256(data)))
            print(c["name"], len(data), flush=True)
        for c in covtrack_cases():
            fq, ref, wig = (os.path.join(d, c["name"] + x) for x in (".fq", ".ref.fa", ".wig"))
            write_fastq(raw_reads(c["reads"]), fq)
            s = c["reads"]
            ref_fasta(ReadSet.from_coverage(s["seed"], s["genome"], s["cov"], s["L"], s["err"]), ref)
            _dbg([f"-k{c['k']}", f"--kc={c['kc']}", f"-b{c['b']}", f"-H{c['H']}", "-C", wig, "-R", ref, "-o", "/dev/null", fq], d)
            data = open(wig, "rb").read()
            out["covtrack"].append(dict(c, bytes=len(data), lines=data.count(b"\n"), sha256=sha256(data)))
            print(c["name"], len(data), flush=True)
        write_graph_inputs(d)
        for f in GRAPH_FILTERS.values():
            subprocess.run([BLOOM, *f["args"]], cwd=d, check=True, capture_output=True)
        for c in graph_cases():
            r = subprocess.run([BLOOM, *c["args"]], cwd=d, capture_output=True)
            assert r.returncode == 0 and r.stdout, r.stderr.decode()
            with gzip.GzipFile(os.path.join(HERE, f"kwidth_{c['name']}.dot.gz"), "wb", mtime=0) as z:
                z.write(r.stdout)
            out["graph"].append(dict(c, rc=r.returncode, bytes=len(r.stdout), lines=r.stdout.count(b"\n"), sha256=sha256(r.stdout),
                                     stderr=r.stderr.decode()))
            print(c["name"], len(r.stdout), flush=True)
        write_trim_inputs(d)
        for f in TRIM_FILTERS:
            subprocess.run([BLOOM, *f["args"]], cwd=d, check=True, capture_output=True)
        for c in trim_cases():
            r = subprocess.run([BLOOM, *c["args"]], cwd=d, capture_output=True)
            out["trim"].append(dict(c, rc=r.returncode, stdout_md5=md5(r.stdout), stdout_bytes=len(r.stdout), stderr=r.stderr.decode()))
            print(c["name"], r.returncode, len(r.stdout), flush=True)
    json.dump(out, open(os.path.join(HERE, "kwidth_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
