#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: regenerates tests/golden/hashnum_cases.json, pass 1 and pass 2 at hash counts other than the e2e
cases' 3 and 4, from the UNMODIFIED reference binaries built by oracle/Makefile (oracle/_ref, -j1 is deterministic):

  abyss-bloom-dbg-ref -H<H> -j1 --read-log      md5 of the unitig FASTA and of the read log
  abyss-bloom-ref build -t counting -H<H> -j1   sha256 of the counters (the file without its header)

on the e2e_g20k_k32 and e2e_g10k_k25_small read sets (tests/golden/e2e_cases.json) at H = 1, 2, 5, 8 and 9, plus the
whole file of `abyss-bloom-ref build -t rolling-hash -l 2 -b 1000` on the smaller set: each level rounds up to 504
bytes, which is not a multiple of 16.

Run in the build container only (needs the reference binaries in oracle/_ref: make -C oracle ref REF=...)."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from abyss_b200.synth import ReadSet  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
DBG = os.path.join(REF, "abyss-bloom-dbg-ref")
BLOOM = os.path.join(REF, "abyss-bloom-ref")
READ_SETS = ["e2e_g20k_k32", "e2e_g10k_k25_small"]
HASH_NUMS = [1, 2, 5, 8, 9]


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def main():
    e2e = {c["name"]: c for c in json.load(open(os.path.join(HERE, "e2e_cases.json")))}
    tmp = tempfile.mkdtemp(prefix="abyss_golden_hashnum_")
    cases = []
    for name in READ_SETS:
        c = e2e[name]
        rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
        fq = os.path.join(tmp, name + ".fq")
        rs.write_fastq(fq)
        for H in HASH_NUMS:
            out, log, bf = (os.path.join(tmp, f"{name}_H{H}.{x}") for x in ("fa", "readlog.tsv", "bloom"))
            cmd = f"ulimit -s 65536; {DBG} -k{c['k']} --kc={c['kc']} -b{c['b']} -H{H} -j1 --read-log={log} {fq} > {out}"
            subprocess.run(["bash", "-c", cmd], check=True, capture_output=True)
            subprocess.run([BLOOM, "build", "-k", str(c["k"]), "-t", "counting", f"-b{c['counters']}", f"-H{H}", "-j1", bf, fq],
                           check=True, capture_output=True)
            blob = open(bf, "rb").read()
            tag = b"[HeaderEnd]\n"
            raw = blob[blob.index(tag) + len(tag):]
            assert len(raw) == c["counters"], (len(raw), c["counters"])
            n_contigs = sum(1 for l in open(out) if l.startswith(">"))
            cases.append(dict(name=f"{name}_H{H}", reads=name, H=H, n_contigs=n_contigs, fasta_md5=md5(out), readlog_md5=md5(log),
                              counters_sha256=hashlib.sha256(raw).hexdigest()))
            print(cases[-1]["name"], n_contigs)
    name = "e2e_g10k_k25_small"
    c = e2e[name]
    rh = os.path.join(tmp, name + ".rh1000.bloom")
    subprocess.run([BLOOM, "build", "-k", str(c["k"]), "-t", "rolling-hash", "-l", "2", f"-H{c['H']}", "-b1000", "-j1", rh,
                    os.path.join(tmp, name + ".fq")], check=True, capture_output=True)
    rolling = dict(name=name + "_rh_l2_b1000", reads=name, H=c["H"], levels=2, b=1000, file_bytes=os.path.getsize(rh),
                   file_sha256=hashlib.sha256(open(rh, "rb").read()).hexdigest())
    print(rolling["name"], rolling["file_bytes"])
    json.dump({"dbg": cases, "rolling_hash": rolling}, open(os.path.join(HERE, "hashnum_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
