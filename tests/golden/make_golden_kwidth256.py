#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: regenerates tests/golden/kwidth256_cases.json and kwidth256_graph_*.dot.gz, the goldens of k = 193..256
(Kmer<8> in pass 2, the 512-entry K1 ring above k = 224, eight-word Konnector k-mers), from the UNMODIFIED reference built
with MAX_KMER = 256 (configure --enable-maxk=256; oracle/maxk256.mk builds it into oracle/_ref/maxk256).  The cases, the read
sets and the way each program is run are those of make_golden_kwidth.py; reads are 300 bp where k > 250 so that every k has
windows.

Before it writes anything it checks that the MAX_KMER = 256 build is the same program as the MAX_KMER = 192 one on a k <= 192
case: both must give the bytes of kwidth_cases.json's asm_k192.

    python tests/golden/make_golden_kwidth256.py

Run where the reference binaries are built (oracle/_ref and oracle/_ref/maxk256: make -C oracle ref REF=...
and make -C oracle -f maxk256.mk REF=...)."""
import gzip
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden_kwidth as kw  # noqa: E402
import overlap_cases as oc  # noqa: E402
from make_golden_bloom_graph import filt as graph_filt, genome_text  # noqa: E402
from make_golden_trim import filt as trim_filt  # noqa: E402

from abyss_b200.synth import ReadSet, revcomp  # noqa: E402

REF256 = os.path.join(ROOT, "oracle", "_ref", "maxk256")
DBG256 = os.path.join(REF256, "abyss-bloom-dbg-ref")
BLOOM256 = os.path.join(REF256, "abyss-bloom-ref")
ADJ256 = os.path.join(REF256, "AdjList-ref")
ASM_KS = [193, 200, 224, 225, 255, 256]
WIDE_KS = [193, 256]  # the graph, trim and Konnector cases


def _plain(seed, k):
    """k-mers this long are solid only at a higher coverage and a lower error rate than make_golden_kwidth's reads have"""
    return dict(kind="plain", seed=seed, genome=15000, cov=60, L=250 if k <= 240 else 300, err=0.001)


def assembler_cases():
    out = []

    def case(name, k, reads, H=4, opt=""):
        out.append(dict(name=name, k=k, kc=2, H=H, b="1M", counters=kw.counters_for_budget("1M"), opt=opt, reads=reads))
    for k in ASM_KS:
        case(f"asm_k{k}", k, _plain(500 + k, k))
    for H in (1, 9):
        case(f"asm_k256_H{H}", 256, _plain(756, 256), H=H)
    for k in (193, 256):
        case(f"asm_edge_k{k}", k, dict(_plain(600 + k, k), kind="edge"))
    case("asm_mixed_k225", 225, dict(_plain(825, 225), kind="mixed"))  # 150 bp reads have no window, 250 and 400 bp do
    for kind in ("circ", "hairpin", "tandem"):
        case(f"asm_{kind}_k256", 256, dict(kind=kind, seed=1056, genome=6000, cov=60, L=300))
    for k, opt in ((224, "-K100"), (224, "--qr-seed=61"), (256, "-K120"), (256, "--qr-seed=59")):
        case(f"asm_seed_k{k}_{opt.strip('-').replace('=', '').replace('-', '')}", k, _plain(900 + k, k), opt=opt)
    return out


def dbg_graph_cases():
    return [dict(name=f"dbg_graph_k{k}", k=k, kc=2, H=3, b="256k", reads=dict(kind="plain", seed=700 + k, genome=4000, cov=40, L=300, err=0.002))
            for k in (224, 256)]


def covtrack_cases():
    return [dict(name=f"covtrack_k{k}", k=k, kc=2, H=4, b="1M", reads=_plain(500 + k, k)) for k in (224, 256)]


# abyss-bloom graph: the 300 bp reads of make_golden_kwidth.write_graph_inputs
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


# Konnector filters and trim, over make_golden_kwidth.write_trim_inputs: O.fq (300 bp; N, lower-case ends, 40 bp reads) and
# A.fq (250 bp, the same edits).  Each k builds a filter of O.fq whole and in two -w windows, the union of the windows, the
# k-mers of A.fq in the filter, and trims O.fq (the filter's own reads) and A.fq (another genome's).
def konnector_cases():
    out = []
    for k in WIDE_KS:
        f = trim_filt(f"o{k}.bloom", k, "64K", ["O.fq"])
        out.append(dict(name=f"kon_build_k{k}", args=f["args"], file=f["file"], harness=f["harness"]))
        for w in (1, 2):
            f = trim_filt(f"o{k}w{w}.bloom", k, "64K", ["O.fq"], levels=2, window=(w, 2))
            out.append(dict(name=f"kon_window_{w}of2_k{k}", args=f["args"], file=f["file"], harness=f["harness"]))
        out.append(dict(name=f"kon_union_k{k}", args=["union", f"-k{k}", f"u{k}.bloom", f"o{k}w1.bloom", f"o{k}w2.bloom"],
                        file=f"u{k}.bloom", harness=["union", k, f"u{k}.bloom", f"o{k}w1.bloom", f"o{k}w2.bloom"]))
        for fmt in ("--fasta", "--raw"):
            out.append(dict(name=f"kon_kmers{fmt[1:]}_k{k}", args=["kmers", f"-k{k}", fmt, f"o{k}.bloom", "A.fq"]))
    return out


def trim_cases():
    out = []
    for k in WIDE_KS:
        out.append(dict(name=f"trim_self_k{k}", args=["trim", "-vv", f"-k{k}", f"o{k}.bloom", "O.fq"], harness=[k, f"o{k}.bloom", "O.fq"]))
        out.append(dict(name=f"trim_other_k{k}", args=["trim", f"-k{k}", f"o{k}.bloom", "A.fq"], harness=[k, f"o{k}.bloom", "A.fq"]))
    return out


def adjlist_cases():
    """AdjList at k = 256 in every output format: contigs of 257..400 bp overlapping by k-1 = 255 bases or by -m 200..254"""
    return [dict(name=f"adj_k256_{oc.FORMATS[n][2:]}", seed=40 + n, genome=60000, k=256, m=200, n_fmt=n) for n in range(len(oc.FORMATS))]


def adjlist_input(c):
    return oc.tiled_case(c["seed"], c["genome"], c["k"], c["m"], c["n_fmt"])


def _run_case(c, d, binary):
    r = subprocess.run([binary, *c["args"]], cwd=d, capture_output=True)
    rec = dict(rc=r.returncode, stdout_md5=kw.md5(r.stdout), stdout_bytes=len(r.stdout), stderr=r.stderr.decode())
    if "file" in c:
        rec["sha256"] = kw.sha256(open(os.path.join(d, c["file"]), "rb").read())
    return r, rec


def same_program_check(d):
    """the MAX_KMER = 256 build gives the MAX_KMER = 192 build's bytes, and the committed golden's, on asm_k192"""
    c = {x["name"]: x for x in kw.assembler_cases()}["asm_k192"]
    got = {}
    for label, dbg, bloom in (("192", kw.DBG, kw.BLOOM), ("256", DBG256, BLOOM256)):
        kw.DBG, kw.BLOOM = dbg, bloom
        sub = os.path.join(d, "same" + label)
        os.makedirs(sub)
        got[label] = kw.run_assembler(c, sub)
    committed = {x["name"]: x for x in json.load(open(os.path.join(HERE, "kwidth_cases.json")))["assembler"]}["asm_k192"]
    keys = ("n_contigs", "fasta_md5", "readlog_md5", "trace_sha256", "counters_sha256")
    assert all(got["192"][x] == got["256"][x] == committed[x] for x in keys), (got, committed)
    return {x: committed[x] for x in keys}


def main():
    out = {}
    with tempfile.TemporaryDirectory() as d:
        out["same_program_k192"] = same_program_check(d)
        print("MAX_KMER = 192 and 256 give the same bytes at k = 192", flush=True)
        kw.DBG, kw.BLOOM = DBG256, BLOOM256
        out["assembler"] = []
        for c in assembler_cases():
            out["assembler"].append(kw.run_assembler(c, d))
            print(c["name"], out["assembler"][-1]["n_contigs"], out["assembler"][-1].get("mask", ""), flush=True)
        out["dbg_graph"], out["covtrack"] = [], []
        for c in dbg_graph_cases():
            fq, dot = os.path.join(d, c["name"] + ".fq"), os.path.join(d, c["name"] + ".dot")
            kw.write_fastq(kw.raw_reads(c["reads"]), fq)
            kw._dbg([f"-k{c['k']}", f"--kc={c['kc']}", f"-b{c['b']}", f"-H{c['H']}", "-g", dot, "-o", "/dev/null", fq], d)
            data = open(dot, "rb").read()
            out["dbg_graph"].append(dict(c, bytes=len(data), lines=data.count(b"\n"), sha256=kw.sha256(data)))
            print(c["name"], len(data), flush=True)
        for c in covtrack_cases():
            fq, ref, wig = (os.path.join(d, c["name"] + x) for x in (".fq", ".ref.fa", ".wig"))
            kw.write_fastq(kw.raw_reads(c["reads"]), fq)
            s = c["reads"]
            kw.ref_fasta(ReadSet.from_coverage(s["seed"], s["genome"], s["cov"], s["L"], s["err"]), ref)
            kw._dbg([f"-k{c['k']}", f"--kc={c['kc']}", f"-b{c['b']}", f"-H{c['H']}", "-C", wig, "-R", ref, "-o", "/dev/null", fq], d)
            data = open(wig, "rb").read()
            out["covtrack"].append(dict(c, bytes=len(data), lines=data.count(b"\n"), sha256=kw.sha256(data)))
            print(c["name"], len(data), flush=True)
        kw.write_graph_inputs(d)
        for f in GRAPH_FILTERS.values():
            subprocess.run([BLOOM256, *f["args"]], cwd=d, check=True, capture_output=True)
        out["graph"] = []
        for c in graph_cases():
            r, rec = _run_case(c, d, BLOOM256)
            assert r.returncode == 0 and r.stdout.count(b"->") > 10, r.stderr.decode()
            with gzip.GzipFile(os.path.join(HERE, f"kwidth256_{c['name']}.dot.gz"), "wb", mtime=0) as z:
                z.write(r.stdout)
            out["graph"].append(dict(c, rc=r.returncode, bytes=len(r.stdout), lines=r.stdout.count(b"\n"), sha256=kw.sha256(r.stdout),
                                     stderr=r.stderr.decode()))
            print(c["name"], len(r.stdout), flush=True)
        kw.write_trim_inputs(d)
        out["konnector"], out["trim"] = [], []
        for c in konnector_cases():  # in order: later cases read the files earlier ones wrote
            r, rec = _run_case(c, d, BLOOM256)
            assert r.returncode == 0, r.stderr.decode()
            out["konnector"].append(dict(c, **rec))
            print(c["name"], rec["stdout_bytes"], flush=True)
        for c in trim_cases():
            r, rec = _run_case(c, d, BLOOM256)
            assert r.returncode == 0, r.stderr.decode()
            out["trim"].append(dict(c, **rec))
            print(c["name"], r.returncode, len(r.stdout), flush=True)
        out["adjlist"] = []
        for c in adjlist_cases():
            t = adjlist_input(c)
            fa = os.path.join(d, c["name"] + ".fa")
            oc.write_fasta(t, fa)
            r = subprocess.run([ADJ256] + oc.command_args(t, fa), capture_output=True, check=True)
            data = oc.normalise(r.stdout, ADJ256).replace(fa.encode(), b"IN.fa")
            out["adjlist"].append(dict(c, contigs=len(t["records"]), bytes=len(data), sha256=kw.sha256(data)))
            print(c["name"], len(t["records"]), len(data), flush=True)
    for c in out["assembler"]:
        assert c["n_contigs"] > 0, c["name"]
    json.dump(out, open(os.path.join(HERE, "kwidth256_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
