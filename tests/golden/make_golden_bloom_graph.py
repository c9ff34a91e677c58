"""Goldens of `abyss-bloom graph` (Bloom/bloom.cc:984-1153): the unmodified reference binary (oracle/_ref/abyss-bloom-ref) builds
every filter of FILTERS with `build -t rolling-hash` and runs every case of cases() in one directory, on the inputs write_inputs()
makes from seeded abyss_b200.synth read sets.  bloom_graph_cases.json keeps, per case, the size, line count and sha256 of stdout,
stderr and the exit status; the dumps of up to 64 KiB are kept whole as bloom_graph_<case>.dot.gz.  A case with "harness" is one
the CPU harness tests/host_bloom_graph runs: its filters are given by how they were built, so the harness can rebuild them with
the C oracle.  A case with "ref" is one where this project does not follow the reference (DESIGN.md, section 3, K7b): the reference's
outcome is kept there and the case's own fields say what `abyss-bloom graph` does instead.

    python tests/golden/make_golden_bloom_graph.py
"""
import gzip
import hashlib
import json
import os
import random
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)
from abyss_b200.synth import ReadSet  # noqa: E402

COMP = str.maketrans("ACGTacgt", "TGCAtgca")


def rc(s):
    return s.translate(COMP)[::-1]


def rand_seq(rng, n):
    return "".join(rng.choice("ACGT") for _ in range(n))


def genome_text(seed, n):
    return "".join("ACGT"[c] for c in ReadSet(seed, n, 1, 50).genome)


def write_inputs(d, large=False):
    """the read sets, root and attribute FASTA files of every case"""
    ReadSet.from_coverage(11, 6000, 10, 100, 0.003).write_fastq(os.path.join(d, "g.fq"))    # a 6 kb genome, some errors
    ReadSet.from_coverage(12, 2000, 8, 100, 0.0).write_fastq(os.path.join(d, "c.fq"))       # a 2 kb genome, no errors
    g = genome_text(11, 6000)
    rng = random.Random(5)
    with open(os.path.join(d, "roots.fa"), "w") as f:       # about 5 900 distinct roots: the root set rehashes many times
        f.write(f">r0\n{g[:3000]}\n>r1 reverse strand\n{rc(g[2500:6000])}\n>r2\nNNNN{g[100:200]}N{g[300:400]}\n")
    with open(os.path.join(d, "few.fa"), "w") as f:         # a handful of roots, one of them twice on opposite strands
        f.write(f">a\n{g[1000:1040]}\n>b\n{rc(g[1000:1040])}\n>c\n{rand_seq(rng, 60)}\n")
    with open(os.path.join(d, "attr1.fa"), "w") as f:       # k-mers of the genome
        f.write(f">x\n{g[1000:1100]}\n>y\n{g[4000:4500]}\n")
    with open(os.path.join(d, "attr2.fa"), "w") as f:       # disjoint from the genome
        f.write(f">z\n{rand_seq(rng, 300)}\n")
    with open(os.path.join(d, "sub.fq"), "w") as f:         # a third of the reads: the -A filters
        lines = open(os.path.join(d, "g.fq")).read().split("\n")
        f.write("\n".join(lines[:len(lines) // 12 * 4]) + "\n")
    # special shapes: a homopolymer run, and at k = 24 reverse-complement palindromes (a vertex whose in-edge is itself)
    with open(os.path.join(d, "s.fa"), "w") as f:
        f.write(f">h\n{rand_seq(rng, 50)}{'A' * 60}{rand_seq(rng, 50)}\n")
        for i in range(6):
            half = rand_seq(rng, 12)
            f.write(f">p{i}\n{rand_seq(rng, 40)}{half}{rc(half)}{rand_seq(rng, 40)}\n")
            f.write(f">q{i}\n{half[1:]}{rc(half)}{rand_seq(rng, 30)}\n")
        f.write(f">t\n{g[:400]}\n")
    if large:
        ReadSet.from_coverage(13, 200000, 75, 150, 0.005).write_fastq(os.path.join(d, "big.fq"))  # 100 000 reads
        big = genome_text(13, 200000)
        with open(os.path.join(d, "bigroots.fa"), "w") as f:
            for i in range(40):
                f.write(f">b{i}\n{big[i * 5000:i * 5000 + 150]}\n")


def filt(name, k, b, H, reads, levels=1):
    """a filter: the command line of `abyss-bloom build -t rolling-hash` and its recipe for the harness (H, levels, bits per level,
    read files)"""
    size = {"16K": 16384, "64K": 65536, "256K": 262144, "2M": 2 << 20, "16M": 16 << 20}[b]
    bits = size * 8 // levels
    bits += -bits % 64
    args = ["build", f"-k{k}", "-t", "rolling-hash", f"-b{b}", f"-H{H}"] + ([f"-l{levels}"] if levels > 1 else []) + [name] + reads
    return {"file": name, "args": args, "recipe": [H, levels, bits, "+".join(reads)]}


FILTERS = [filt(f"g{k}_H{H}.bloom", k, "256K", H, ["g.fq"]) for k, H in ((21, 2), (32, 1), (33, 4), (64, 2), (96, 4), (25, 2))] + [
    filt("g25_l2.bloom", 25, "256K", 2, ["g.fq", "g.fq"], levels=2),
    filt("c25.bloom", 25, "64K", 2, ["c.fq"]),
    filt("s24.bloom", 24, "64K", 2, ["s.fa"]),
    filt("s25.bloom", 25, "64K", 3, ["s.fa"]),
    filt("sub25_H1.bloom", 25, "256K", 1, ["sub.fq"]),    # an -A filter with fewer hashes than the graph
    filt("sub25_big.bloom", 25, "2M", 2, ["sub.fq"]),     # an -A filter of another size
    filt("sub25_H3.bloom", 25, "256K", 3, ["sub.fq"]),    # more hashes than the graph
    # more than 4 hashes: a lane of the kernel probes several of its neighbour's hashes, and an attribute filter's hashes on top
    filt("g25_H6.bloom", 25, "256K", 6, ["g.fq"]),
    filt("g25_H20.bloom", 25, "2M", 20, ["g.fq"]),
    filt("sub25_H5.bloom", 25, "256K", 5, ["sub.fq"]),
    filt("sub25_H20.bloom", 25, "2M", 20, ["sub.fq"]),
]
OTHER_FILTERS = [["build", "-k25", "-t", "counting", "-b64K", "count25.bloom", "c.fq"], ["build", "-k25", "-b64K", "kon25.bloom", "c.fq"]]
LARGE_FILTERS = [filt("big64.bloom", 64, "16M", 4, ["big.fq"])]
RECIPES = {f["file"]: f["recipe"] for f in FILTERS + LARGE_FILTERS}


def cases(g):
    """g: the 6 kb genome's text.  Each case: name, the command line after `graph`, and whether the harness runs it."""
    out = []

    def case(name, args, harness=True, **extra):
        out.append({"name": name, "args": ["graph"] + args, "harness": harness, **extra})

    r = g[1000:1025]
    case("one_root", ["-k25", f"-R{r}", "g25_H2.bloom"])
    case("root_and_rc", ["-k25", "-R", r, "-R", rc(r), "-R", rand_seq(random.Random(3), 25), "g25_H2.bloom"])
    case("lower_case_root", ["-k25", "-R", g[2000:2025].lower(), "g25_H2.bloom"])
    case("fasta_roots", ["-v", "-k25", "-d2", "-f", "roots.fa", "g25_H2.bloom"])
    case("fasta_few_and_R", ["-k25", "-d", "3", "-f", "few.fa", "-R", g[5000:5025], "g25_H2.bloom"])
    for d in (0, 1, 2):
        case(f"depth{d}", ["-k25", f"-d{d}", "-R", g[3000:3025], "-R", g[3010:3035], "g25_H2.bloom"])
    case("depth_exhausts_component", ["-k25", "-d", "100000", "-R", genome_text(12, 2000)[700:725], "c25.bloom"])
    case("homopolymer", ["-k25", "-d", "4", "-R", "A" * 25, "s25.bloom"])
    case("palindromes_k24", ["-k24", "-f", "s.fa", "s24.bloom"])
    for k, H in ((21, 2), (32, 1), (33, 4), (64, 2), (96, 4)):
        case(f"k{k}_H{H}", ["-k", str(k), "-R", g[4000:4000 + k], "-R", rc(g[1500:1500 + k]), f"g{k}_H{H}.bloom"])
    case("levels2", ["-k25", "-d5", "-R", r, "g25_l2.bloom"])
    case("fasta_attrs", ["-v", "-k25", "-d30", "-a", "color=red:attr1.fa", "--node-attr=shape=box:attr2.fa", "--fasta-attr", "mark:attr1.fa",
                         "-R", g[1020:1045], "g25_H2.bloom"])
    case("bloom_attrs", ["-v", "-k25", "-d30", "-A", "color=blue:sub25_H1.bloom", "--bloom-attr=style=bold:sub25_big.bloom",
                         "-a", "x:attr1.fa", "-R", g[990:1015], "-R", g[3990:4015], "g25_H2.bloom"])
    case("k25_H6", ["-k25", "-d8", "-R", g[4000:4025], "-R", rc(g[1500:1525]), "g25_H6.bloom"])
    case("H6_attrs", ["-k25", "-d20", "-A", "five:sub25_H5.bloom", "-A", "one:sub25_H1.bloom", "-R", g[990:1015], "g25_H6.bloom"])
    case("H20_attrs", ["-k25", "-d20", "-A", "twenty:sub25_H20.bloom", "-A", "five:sub25_H5.bloom", "-R", g[2990:3015], "g25_H20.bloom"])
    case("fasta_attr_progress", ["-v", "-k25", "-d3", "-a", "reads:g.fq", "-R", g[1020:1045], "g25_H2.bloom"])  # > 10 000 k-mers
    case("depth_wraps", ["-k25", "-d", "4294967297", "-R", g[3000:3025], "g25_H2.bloom"])  # kept as an unsigned: depth 1
    # errors
    case("no_roots", ["-k25", "g25_H2.bloom"], False)
    case("missing_arguments", ["-k25", "-R", r], False)
    case("two_files", ["-k25", "-R", r, "g25_H2.bloom", "g21_H2.bloom"], False)
    case("missing_k", ["-R", r, "g25_H2.bloom"], False)
    case("invalid_depth", ["-k25", "-d", "x3", "-R", r, "g25_H2.bloom"], False)
    case("invalid_attr", ["-k25", "-a", "noseparator", "-R", r, "g25_H2.bloom"], False)
    case("k_after_command_option", ["-k25", "-R", r, "-k25", "g25_H2.bloom"], False)
    case("counting_file", ["-k25", "-R", r, "count25.bloom"], False)
    case("konnector_file", ["-k25", "-R", r, "kon25.bloom"], False)
    case("no_root_in_filter", ["-k25", "-R", "ACGT" * 6 + "A", "c25.bloom"])
    # where the reference asserts or reads uninitialised memory: refused
    case("root_not_k", ["-k25", "-R", r[:20], "g25_H2.bloom"], False,
         expect={"rc": 1, "stderr": f"abyss-bloom: root `{r[:20]}' is not a 25-mer\n"})
    case("k_not_the_files", ["-k24", "-R", r[:24], "g25_H2.bloom"], False,
         expect={"rc": 1, "stderr": "abyss-bloom: `g25_H2.bloom' holds 25-mers, not the 24-mers of -k\n"})
    case("attr_more_hashes", ["-k25", "-A", "c:sub25_H3.bloom", "-R", r, "g25_H2.bloom"], False,
         expect={"rc": 1, "stderr": "abyss-bloom: `sub25_H3.bloom' uses 3 hash functions, more than the 2 of the graph's filter\n"})
    case("root_with_N", ["-k25", "-R", r[:12] + "N" + r[13:], "g25_H2.bloom"], False,
         expect={"rc": 1, "stderr": f"abyss-bloom: root `{r[:12] + 'N' + r[13:]}' has a character other than A, C, G, T\n"})
    return out


def large_case():
    return {"name": "large", "args": ["graph", "-k64", "-f", "bigroots.fa", "big64.bloom"], "harness": True}


def run(exe, d, args):
    return subprocess.run([exe, *args], cwd=d, capture_output=True)


def record(c, r):
    o = {"rc": r.returncode, "bytes": len(r.stdout), "lines": r.stdout.count(b"\n"), "sha256": hashlib.sha256(r.stdout).hexdigest(),
         "stderr": r.stderr.decode()}
    exp = c.pop("expect", None)
    if exp is None:
        return {**c, **o}
    # the reference's outcome, kept for the record; what this program does instead
    ref = {"rc": o["rc"], "bytes": o["bytes"], "sha256": o["sha256"], "stderr": re.sub(r"\S*/(Bloom/)", r"\1", o["stderr"])}
    return {**c, "ref": ref, "rc": exp["rc"], "bytes": 0, "lines": 0,
            "sha256": hashlib.sha256(b"").hexdigest(), "stderr": exp["stderr"]}


def main():
    exe = os.path.join(ROOT, "oracle", "_ref", "abyss-bloom-ref")
    large = "--large" in sys.argv
    out = []
    with tempfile.TemporaryDirectory() as d:
        write_inputs(d, large)
        for f in FILTERS + (LARGE_FILTERS if large else []):
            r = run(exe, d, f["args"])
            assert r.returncode == 0, r.stderr.decode()
        for a in OTHER_FILTERS:
            r = run(exe, d, a)
            assert r.returncode == 0, r.stderr.decode()
        for c in cases(genome_text(11, 6000)) + ([large_case()] if large else []):
            r = run(exe, d, c["args"])
            rec = record(c, r)
            out.append(rec)
            if c["name"] != "large" and "ref" not in rec and 0 < len(r.stdout) <= 65536:
                with gzip.GzipFile(os.path.join(GOLD, f"bloom_graph_{c['name']}.dot.gz"), "wb", mtime=0) as z:
                    z.write(r.stdout)
            print(c["name"], r.returncode, len(r.stdout), r.stdout.count(b"\n"), r.stderr.decode().replace("\n", " | ")[-200:])
    path = os.path.join(GOLD, "bloom_graph_cases.json")
    if not large and os.path.exists(path):  # keep the large case of an earlier --large run
        out += [c for c in json.load(open(path)) if c["name"] == "large"]
    json.dump(out, open(path, "w"), indent=1)
    print(len(out), "cases")


if __name__ == "__main__":
    main()
