"""Goldens of `abyss-bloom trim` (Bloom/bloom.cc:1233-1382): the unmodified reference binary (oracle/_ref/abyss-bloom-ref)
builds every filter of FILTERS and runs every case of cases() in one directory, on the read sets write_inputs() makes.
trim_cases.json keeps, per case, the md5 of stdout (the trimmed reads), stderr and the exit status; the cases with a
"harness" entry are the ones the CPU harness tests/host_trim can run (it prints no messages).  The hand-made cases also keep,
per surviving read, the (left, right) trim lengths that the reference's output shows (lengths_of).

    python tests/golden/make_golden_trim.py
"""
import gzip
import hashlib
import json
import os
import random
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_konnector import write_reads  # noqa: E402  (A.fq: 800 x 250 bp, B.fq: 1066 x 150 bp; N, lower-case ends, 40 bp reads)

COMP = str.maketrans("ACGTacgtN", "TGCAtgcaN")


def rc(s):
    return s.translate(COMP)[::-1]


def rand_seq(rng, n):
    return "".join(rng.choice("ACGT") for _ in range(n))


def fastq_records(path):
    lines = open(path).read().split("\n")
    return [(lines[i][1:], lines[i + 1], lines[i + 3]) for i in range(0, len(lines) - 3, 4)]


def hand_graph(rng, k):
    """sequences whose k-mers make a small graph with known shapes, and reads that end on them.  Returns (graph, reads)."""
    S = rand_seq(rng, 600)                       # backbone
    graph, reads = [S], []
    for at, n in ((100, 1), (160, 2), (220, 3), (280, 6), (340, 12), (400, 30)):
        # a branch that leaves the backbone after S[at + k - 2] and dead-ends after n k-mers: a tip of n vertices
        b = "ACGT"[("ACGT".index(S[at + k - 1]) + 1) % 4]
        tip = S[at:at + k - 1] + b + rand_seq(rng, n - 1)
        graph.append(tip)
        reads.append(tip + "")                    # a read that is the tip: its right end is the dead end
        reads.append(rc(tip))                     # the same on the other strand: the left end
        reads.append(S[at - 40:at + k - 1] + b + rand_seq(rng, n - 1 + 8))  # runs past the tip into k-mers that are not there
        reads.append(S[at - 30:at + k + 30])     # spans the fork along the backbone
        reads.append(S[at + 1:at + k + 40])      # the first k-mer is the vertex right after the fork
    # in-branches: a sequence that joins the backbone
    for at, n in ((460, 2), (500, 9)):
        b = "ACGT"[("ACGT".index(S[at - 1]) + 2) % 4]
        tip = rand_seq(rng, n - 1) + b + S[at:at + k - 1]
        graph.append(tip)
        reads += [tip, rc(tip), tip + S[at + k - 1:at + k + 30]]
    # X: two paths that share exactly one k-mer (what a Bloom false positive makes)
    mid = rand_seq(rng, k)
    p1, p2 = rand_seq(rng, 3), rand_seq(rng, 3)
    while p1[-1] == p2[-1]:
        p2 = rand_seq(rng, 3)
    q1, q2 = rand_seq(rng, 3), rand_seq(rng, 3)
    while q1[0] == q2[0]:
        q2 = rand_seq(rng, 3)
    graph += [p1 + mid + q1, p2 + mid + q2]
    reads += [p1 + mid + q1, p2 + mid + q2, rc(p1 + mid + q2), mid + q1, p2 + mid]
    # longer arms: the same X with arms past fpTrim
    mid2 = rand_seq(rng, k)
    a1, a2, c1, c2 = rand_seq(rng, 9), rand_seq(rng, 9), rand_seq(rng, 9), rand_seq(rng, 9)
    a2 = a2[:-1] + "ACGT"[("ACGT".index(a1[-1]) + 1) % 4]
    c2 = "ACGT"[("ACGT".index(c1[0]) + 1) % 4] + c2[1:]
    graph += [a1 + mid2 + c1, a2 + mid2 + c2]
    reads += [a1 + mid2 + c1, rc(a2 + mid2 + c2), a1 + mid2 + c2]
    # the strand matters: a read that holds a k-mer and later its reverse complement (a hairpin); with even k a k-mer that is
    # its own reverse complement
    stem = rand_seq(rng, k + 10)
    hp = stem + rand_seq(rng, 4) + rc(stem)
    graph.append(hp)
    reads += [hp, hp[5:], hp[:len(stem) + 20]]
    if k % 2 == 0:
        half = rand_seq(rng, k // 2)
        pal = rand_seq(rng, 30) + half + rc(half) + rand_seq(rng, 30)
        graph.append(pal)
        reads += [pal, pal[30:], rc(pal)[:30 + k]]
    # plain reads of the backbone: no tip at all; and reads with an N, reads of length k and k - 1, reads of nothing in the graph
    reads += [S[10:160], rc(S[300:450]), S[50:50 + k], S[60:60 + k - 1], S[200:230] + "N" + S[231:300], "N" * (k + 5), rand_seq(rng, 120),
              rand_seq(rng, k), S[0:k - 1] + rand_seq(rng, 60), S[150:210].lower() + S[210:300] + S[300:320].lower()]
    return graph, reads


def strand_graph(rng, k, n=40, filler=24000):
    """Graphs that only a strand-specific vertex identity gets right (k odd).  Each is a sequence G = u + c + tail that nothing
    precedes, and a stub X = u[1:] + b that forks off its first vertex u, with u[2:] + b an even-length reverse-complement
    palindrome: then the stub's second vertex is rc(X) and its third rc(u), which has no successor, so the stub is
    X -> rc(X) -> rc(u), a dead end of three vertices.  trueBranch must find it false at trim >= 3; if it took rc(X) for the
    already visited X ("branches with cycles are true branches") u would be a fork and the read G would not be trimmed.
    `filler` bases of random sequence bring the filter to the occupancy where minBranchLen is 3.  Returns (graph, reads)."""
    graph, reads = [rand_seq(rng, filler)], []
    for _ in range(n):
        h = rand_seq(rng, (k - 1) // 2)
        q = h + rc(h)                              # u[2:] + b
        u = rand_seq(rng, 2) + q[:-1]
        c = "ACGT"[("ACGT".index(q[-1]) + 1 + rng.randrange(3)) % 4]
        g = u + c + rand_seq(rng, 60)
        graph += [g, u[1:] + q[-1]]
        reads += [g, rc(g)]
    return graph, reads


def write_inputs(d):
    write_reads(d)
    b = fastq_records(os.path.join(d, "B.fq"))
    with open(os.path.join(d, "few.fq"), "w") as f:        # 20 reads: a nearly empty filter
        for i, s, q in b[:20]:
            f.write(f"@{i}\n{s}\n+\n{q}\n")
    with open(os.path.join(d, "short.fa"), "w") as f:      # no k-mer at all: an empty filter
        f.write(">s\nACGTACGTAC\n")
    # FASTA, every other record on several lines.  The reference cuts the (empty) quality string of a FASTA record with
    # substr(startPos) and aborts on the first record whose left trim is not 0, so only records that trim echoes (shorter
    # than the k = 64 they are used with) can be compared.
    with open(os.path.join(d, "C.fa"), "w") as f:
        for n, (i, s, q) in enumerate(r for r in b if len(r[1]) < 64):
            body = s if n % 2 else "\n".join(s[j:j + 15] for j in range(0, len(s), 15))
            f.write(f">{i} len={len(s)}\n{body}\n")
    with open(os.path.join(d, "D.fq"), "w") as f:          # Casava 1.8 comments; every seventh read fails the chastity filter
        for n, (i, s, q) in enumerate(b[300:600]):
            q = "".join(chr(33 + (5 if j < 7 or j >= len(s) - 9 else 40)) for j in range(len(s)))  # low-quality ends for -q
            f.write(f"@{i.replace('/', '_')} {1 + n % 2}:{'Y' if n % 7 == 0 else 'N'}:0:ACGT\n{s}\n+\n{q}\n")
    with open(os.path.join(d, "Dq.fq"), "w") as f:         # D.fq as the reader's -q 10 leaves it: 7 and 9 bases of quality 5 cut
        for i, s, q in fastq_records(os.path.join(d, "D.fq")):
            f.write(f"@{i}\n{s[7:-9]}\n+\n{q[7:-9]}\n")
    with gzip.open(os.path.join(d, "B.fq.gz"), "wb") as f:
        f.write(open(os.path.join(d, "B.fq"), "rb").read())
    for k in (24, 25, 33, "s25"):
        graph, reads = strand_graph(random.Random(77), 25) if k == "s25" else hand_graph(random.Random(1000 + k), k)
        with open(os.path.join(d, f"G{k}.fa"), "w") as f:
            for n, s in enumerate(graph):
                f.write(f">g{n}\n{s}\n")
        qrng = random.Random(5)
        with open(os.path.join(d, f"H{k}.fq"), "w") as f:   # random qualities: where a trimmed record came from shows in them
            for n, s in enumerate(reads):
                f.write(f"@h{n}\n{s}\n+\n{''.join(chr(qrng.randrange(35, 75)) for _ in s)}\n")


def filt(name, k, b, reads, levels=1, window=None):
    """a filter: the command line of `abyss-bloom build` and the argument list of tests/host_konnector's build"""
    bits = {"16K": 16384, "64K": 65536, "4M": 4 << 20, "8M": 8 << 20}[b] * 8 // levels
    args = ["build", f"-k{k}", f"-b{b}"] + ([f"-l{levels}"] if levels > 1 else [])
    start, end = 0, bits - 1
    if window:
        w, n = window
        args += ["-w", f"{w}/{n}"]
        per = bits // n
        start, end = (w - 1) * per, (w * per - 1 if w < n else bits - 1)
    return {"file": name, "args": args + [name] + reads, "harness": ["build", k, bits, levels, 0, start, end, name] + reads}


FILTERS = (
    [filt(f"a{k}.bloom", k, "64K", ["A.fq"]) for k in (25, 32, 33, 64, 96)] +
    [filt("b25.bloom", 25, "64K", ["B.fq"]),                 # minBranchLen 4
     filt("empty25.bloom", 25, "64K", ["short.fa"]),         # 0
     filt("few25.bloom", 25, "8M", ["few.fq"]),              # 1
     filt("b25_4M.bloom", 25, "4M", ["B.fq"]),               # 2
     filt("b25_16K.bloom", 25, "16K", ["B.fq"]),             # >= 8
     filt("b64_l2.bloom", 64, "64K", ["B.fq", "B.fq"], levels=2),  # a cascading build: its file is the last level
     filt("b25_w2.bloom", 25, "64K", ["B.fq"], window=(2, 4)),
     filt("g24.bloom", 24, "64K", ["G24.fa"]), filt("g25.bloom", 25, "64K", ["G25.fa"]), filt("g33.bloom", 33, "64K", ["G33.fa"]),
     filt("g25_4M.bloom", 25, "4M", ["G25.fa"]), filt("s25.bloom", 25, "64K", ["Gs25.fa"])])


def cases():
    out = []

    def case(name, args, harness=None):
        out.append({"name": name, "args": ["trim"] + args, **({"harness": harness} if harness else {})})
    for k in (25, 32, 33, 64, 96):
        case(f"self_k{k}", ["-vv", f"-k{k}", f"a{k}.bloom", "A.fq"], [k, f"a{k}.bloom", "A.fq"])
        case(f"other_k{k}", [f"-k{k}", f"a{k}.bloom", "B.fq"], [k, f"a{k}.bloom", "B.fq"])   # the k - 2 quirk: reads of another genome
    for name, f in (("mbl0", "empty25"), ("mbl1", "few25"), ("mbl2", "b25_4M"), ("mbl4", "b25"), ("mbl8", "b25_16K")):
        case(name, ["-vv", "-k25", f"{f}.bloom", "B.fq"], [25, f"{f}.bloom", "B.fq"])
    case("cascade_last_level", ["-vv", "-k64", "b64_l2.bloom", "B.fq"], [64, "b64_l2.bloom", "B.fq"])
    case("window_file", ["-vv", "-k25", "b25_w2.bloom", "B.fq"], [25, "b25_w2.bloom", "B.fq"])
    for k, f in ((24, "g24"), (25, "g25"), (33, "g33"), (25, "g25_4M")):
        case(f"hand_{f}", ["-vv", f"-k{k}", f"{f}.bloom", f"H{k}.fq"], [k, f"{f}.bloom", f"H{k}.fq"])
    case("hand_strand", ["-vv", "-k25", "s25.bloom", "Hs25.fq"], [25, "s25.bloom", "Hs25.fq"])
    case("fasta_multiline", ["-k64", "a64.bloom", "C.fa"], [64, "a64.bloom", "C.fa"])
    case("casava", ["-k25", "b25.bloom", "D.fq"], [25, "b25.bloom", "D.fq"])
    # (the reference's trim parses only the options every command shares: it takes -q, --no-chastity and --no-trim-masked for
    # file names, so there is nothing to compare for them)
    # the reader's -q through trim: what the reference prints for the file cut beforehand
    case("trim_quality", ["-k25", "b25.bloom", "Dq.fq"], [25, "-q", "10", "b25.bloom", "D.fq"])
    case("two_files_gz", ["-v", "-k64", "a64.bloom", "B.fq.gz", "C.fa"], [64, "a64.bloom", "B.fq.gz", "C.fa"])
    case("verbose", ["-v", "-k25", "b25.bloom", "A.fq", "B.fq"])
    case("missing_arguments", ["-k25", "b25.bloom"])
    case("missing_k", ["b25.bloom", "B.fq"])
    case("wrong_k", ["-k31", "b25.bloom", "B.fq"])
    return out


def lengths_of(d, reads_file, stdout):
    """{id: [left, right]} for the records of reads_file that the output holds, from where the trimmed quality string lies in
    the record's own (the H files carry random qualities).  Records the reader changes (lower-case ends, which it cuts) and
    the rare ambiguous position are left out."""
    lines = stdout.decode().split("\n")
    got = {lines[i][1:]: lines[i + 3] for i in range(0, len(lines) - 3, 4)}
    out = {}
    for i, s, q in fastq_records(os.path.join(d, reads_file)):
        t = got.get(i)
        if t is None or s != s.upper() or q.count(t) != 1:
            continue
        out[i] = [q.find(t), len(q) - q.find(t) - len(t)]
    return out


def run(exe, d, args):
    r = subprocess.run([exe, *args], cwd=d, capture_output=True)
    return r


def main():
    exe = os.path.join(ROOT, "oracle", "_ref", "abyss-bloom-ref")
    out = []
    with tempfile.TemporaryDirectory() as d:
        write_inputs(d)
        for f in FILTERS:
            r = run(exe, d, f["args"])
            assert r.returncode == 0, r.stderr.decode()
        for c in cases():
            r = run(exe, d, c["args"])
            out.append({**c, "rc": r.returncode, "stdout_md5": hashlib.md5(r.stdout).hexdigest(), "stdout_bytes": len(r.stdout),
                        "stderr": r.stderr.decode()})
            if c["name"].startswith("hand_"):
                out[-1]["lengths"] = lengths_of(d, c["args"][-1], r.stdout)
            print(c["name"], r.returncode, len(r.stdout), r.stderr.decode().replace("\n", " | ")[-160:])
    json.dump(out, open(os.path.join(ROOT, "tests", "golden", "trim_cases.json"), "w"), indent=1)
    print(len(out), "cases")


if __name__ == "__main__":
    main()
