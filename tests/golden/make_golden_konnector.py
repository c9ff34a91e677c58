"""Goldens of `abyss-bloom` on Konnector filters (-t konnector, union, intersect, info, compare, kmers): the unmodified
reference binary (oracle/_ref/abyss-bloom-ref) runs every case of CASES, in order, in one directory, on two seeded read sets
with N and lower-case ends (write_reads); later cases read the files earlier ones wrote.  konnector_cases.json keeps, per
case, the sha256 of the file written, the md5 of stdout, stderr and the exit status.

    python tests/golden/make_golden_konnector.py
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from abyss_b200.synth import ReadSet, edge_mutate  # noqa: E402

HASH_KS = [1, 3, 4, 5, 16, 17, 31, 32, 33, 63, 64, 65, 96, 128, 129, 191, 192]  # every CityHash length branch
SEEDS = [0, 1, 4294967301]


def write_reads(d):
    """A.fq: 800 x 250 bp of a 20 kbp genome; B.fq: 1066 x 150 bp of another; both with N, lower-case ends and 40 bp reads"""
    for name, (seed, L) in {"A.fq": (11, 250), "B.fq": (12, 150)}.items():
        rs = ReadSet.from_coverage(seed, 20000, 8, L, 0.01)
        seqs = edge_mutate([rs.ascii(i, i + 1)[0].tobytes().decode() for i in range(rs.n)])
        with open(os.path.join(d, name), "w") as f:
            for i, s in enumerate(seqs):
                f.write(f"@{rs.read_id(i)}\n{s}\n+\n{'I' * len(s)}\n")


def cases():
    out = []
    for k in HASH_KS:
        for h in SEEDS:
            out.append({"name": f"hash_k{k}_h{h}", "args": ["build", f"-k{k}", "-b64K", f"-h{h}", "out.bloom", "A.fq"], "file": "out.bloom",
                        "harness": ["build", k, 524288, 1, h, 0, 524287, "out.bloom", "A.fq"]})
    for k in (25, 32, 64, 96):
        for l in (1, 2, 3):
            bits = 524288 // l
            out.append({"name": f"build_k{k}_l{l}", "args": ["build", f"-k{k}", "-b64K", f"-l{l}", f"k{k}l{l}.bloom", "A.fq", "B.fq"],
                        "file": f"k{k}l{l}.bloom", "harness": ["build", k, bits, l, 0, 0, bits - 1, f"k{k}l{l}.bloom", "A.fq", "B.fq"]})
    out.append({"name": "build_k64_l2_seed", "args": ["build", "-k64", "-b64K", "-l2", "-h18446744073709551557", "seed.bloom", "A.fq"],
                "file": "seed.bloom", "harness": ["build", 64, 262144, 2, 18446744073709551557, 0, 262143, "seed.bloom", "A.fq"]})
    for w in (1, 2, 3):
        per = 174762 // 3
        start, end = (w - 1) * per, (w * per - 1 if w < 3 else 174761)
        out.append({"name": f"window_{w}of3", "args": ["build", "-k25", "-b64K", "-l3", "-w", f"{w}/3", f"w{w}.bloom", "A.fq"],
                    "file": f"w{w}.bloom", "harness": ["build", 25, 174762, 3, 0, start, end, f"w{w}.bloom", "A.fq"]})
    out.append({"name": "full_l3", "args": ["build", "-k25", "-b64K", "-l3", "full.bloom", "A.fq"], "file": "full.bloom",
                "harness": ["build", 25, 174762, 3, 0, 0, 174761, "full.bloom", "A.fq"]})
    out.append({"name": "union_windows", "args": ["union", "-k25", "u.bloom", "w1.bloom", "w2.bloom", "w3.bloom"], "file": "u.bloom",
                "harness": ["union", 25, "u.bloom", "w1.bloom", "w2.bloom", "w3.bloom"]})
    out.append({"name": "a_k25", "args": ["build", "-k25", "-b64K", "a.bloom", "A.fq"], "file": "a.bloom",
                "harness": ["build", 25, 524288, 1, 0, 0, 524287, "a.bloom", "A.fq"]})
    out.append({"name": "b_k25", "args": ["build", "-k25", "-b64K", "b.bloom", "B.fq"], "file": "b.bloom",
                "harness": ["build", 25, 524288, 1, 0, 0, 524287, "b.bloom", "B.fq"]})
    out.append({"name": "union_ab", "args": ["union", "-k25", "ab_or.bloom", "a.bloom", "b.bloom"], "file": "ab_or.bloom",
                "harness": ["union", 25, "ab_or.bloom", "a.bloom", "b.bloom"]})
    out.append({"name": "intersect_ab", "args": ["intersect", "-k25", "ab_and.bloom", "a.bloom", "b.bloom"], "file": "ab_and.bloom",
                "harness": ["intersect", 25, "ab_and.bloom", "a.bloom", "b.bloom"]})
    out.append({"name": "level1_src", "args": ["build", "-k25", "-b32K", "lvl.bloom", "B.fq"], "file": "lvl.bloom"})
    out.append({"name": "init_level", "args": ["build", "-k25", "-b64K", "-l2", "-L", "1=lvl.bloom", "init.bloom", "A.fq"], "file": "init.bloom"})
    out.append({"name": "level2_seed_src", "args": ["build", "-k25", "-b32K", "-h7", "lvl7.bloom", "B.fq"], "file": "lvl7.bloom"})
    out.append({"name": "init_last_level_seed", "args": ["build", "-k25", "-b64K", "-l2", "-L", "2=lvl7.bloom", "init7.bloom", "A.fq"],
                "file": "init7.bloom"})
    out.append({"name": "build_verbose", "args": ["build", "-v", "-k25", "-b64K", "-l2", "vb.bloom", "A.fq", "B.fq"], "file": "vb.bloom"})
    out.append({"name": "info_a", "args": ["info", "-k25", "a.bloom"]})
    out.append({"name": "info_options_last", "args": ["info", "a.bloom", "-k", "25"]})
    out.append({"name": "bad_seed", "args": ["build", "-k25", "-b64K", "-hx", "bad.bloom", "A.fq"]})
    out.append({"name": "bad_window", "args": ["build", "-k25", "-b64K", "-w", "1/3abc", "bad.bloom", "A.fq"]})
    out.append({"name": "info_window", "args": ["info", "-k25", "w2.bloom"]})
    for m in ("jaccard", "forbes", "czekanowski"):
        out.append({"name": f"compare_{m}", "args": ["compare", "-k25", "-m", m, "a.bloom", "b.bloom"]})
    for fmt in ("--fasta", "--bed", "--raw"):
        for inv in ([], ["-r"]):
            out.append({"name": f"kmers{fmt[1:]}{'_r' if inv else ''}", "args": ["kmers", "-k25", *inv, fmt, "a.bloom", "B.fq"]})
    out.append({"name": "kmers_verbose", "args": ["kmers", "-v", "-k25", "--raw", "a.bloom", "B.fq"]})
    return out


def run(exe, d, c):
    r = subprocess.run([exe, *c["args"]], cwd=d, capture_output=True)
    rec = {"rc": r.returncode, "stdout_md5": hashlib.md5(r.stdout).hexdigest(), "stderr": r.stderr.decode()}
    if "file" in c:
        rec["sha256"] = hashlib.sha256(open(os.path.join(d, c["file"]), "rb").read()).hexdigest()
    return rec


def main():
    exe = os.path.join(ROOT, "oracle", "_ref", "abyss-bloom-ref")
    out = []
    with tempfile.TemporaryDirectory() as d:
        write_reads(d)
        for c in cases():
            out.append({**c, **run(exe, d, c)})
    json.dump(out, open(os.path.join(ROOT, "tests", "golden", "konnector_cases.json"), "w"), indent=1)
    print(len(out), "cases")


if __name__ == "__main__":
    main()
