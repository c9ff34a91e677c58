#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: regenerates the pass-2 goldens that are not part of make_golden.py from the UNMODIFIED reference
binary built by oracle/Makefile (oracle/_ref/abyss-bloom-dbg-ref, -j1 is deterministic):

  cyc_<case>.fa       circular / hairpin / tandem-repeat read sets (the committed cyc_*.fa.gz ARE the fixture inputs)
  mask_<case>.fa      spaced seeds: -K (kmerPair), --qr-seed (qrSeedPair) and the reads above; the mask is recorded
                      in mask_cases.json so that the tests do not depend on the option parser
  mask_<case>.readlog.tsv for the cases marked readlog

Run in the build container only (needs the reference binaries in oracle/_ref: make -C oracle ref REF=...)."""
import gzip
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from abyss_b200.synth import ReadSet  # noqa: E402

DBG = os.path.join(ROOT, "oracle", "_ref", "abyss-bloom-dbg-ref")
TMP = "/tmp/abyss_golden"


def reads_of(case, e2e):
    """path of a FASTQ/FASTA file with the reads of the case"""
    os.makedirs(TMP, exist_ok=True)
    if case["reads"].endswith(".gz"):
        out = os.path.join(TMP, case["reads"][:-3])
        with gzip.open(os.path.join(HERE, case["reads"]), "rb") as f, open(out, "wb") as g:
            g.write(f.read())
        return out
    c = e2e[case["reads"]]
    rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
    out = os.path.join(TMP, c["name"] + ".fq")
    rs.write_fastq(out)
    return out


def run_ref(opts, reads, out, log=None):
    cmd = f"ulimit -s 65536; {DBG} {opts} -j1 -v {'--read-log=' + log if log else ''} {reads} > {out}"
    r = subprocess.run(["bash", "-c", cmd], capture_output=True, text=True)
    if r.returncode:
        raise SystemExit(r.stderr)
    info = {}
    for line in r.stderr.splitlines():
        if line.startswith("Using spaced seed"):
            info["mask"] = line.split()[3]
        if "#counters" in line:
            info["counters"] = int(line.split("=")[1])
    return info


def main():
    e2e = {c["name"]: c for c in json.load(open(os.path.join(HERE, "e2e_cases.json")))}
    cyc = json.load(open(os.path.join(HERE, "cyc_cases.json")))
    for c in cyc:
        out = os.path.join(HERE, c["name"] + ".fa")
        run_ref(f"-k{c['k']} --kc={c['kc']} -b{c['b']} -H{c['H']} -t{c['trim']}", reads_of(c, e2e), out)
        c["n_contigs"] = sum(1 for l in open(out) if l[0] == ">")
        print(c["name"], c["n_contigs"])
    json.dump(cyc, open(os.path.join(HERE, "cyc_cases.json"), "w"), indent=1)

    mask_cases = [
        dict(name="mask_g20k_K20", reads="e2e_g20k_k32", k=50, kc=2, b="1M", H=4, opt="-K20"),
        dict(name="mask_g20k_qr11", reads="e2e_g20k_k32", k=32, kc=2, b="1M", H=4, opt="--qr-seed=11"),
        dict(name="mask_g10k_K5", reads="e2e_g10k_k25_small", k=25, kc=2, b="1M", H=4, opt="-K5", readlog=True),
        dict(name="mask_g10k_K2", reads="e2e_g10k_k25_small", k=25, kc=2, b="1M", H=4, opt="-K2"),
        dict(name="mask_g30k_K12", reads="e2e_g30k_k64", k=80, kc=2, b="2M", H=4, opt="-K12"),
        dict(name="mask_tandem_qr15", reads="cyc_tandem.fa.gz", k=50, kc=2, b="400000", H=4, opt="--qr-seed=15"),
        dict(name="mask_hairpin_K10", reads="cyc_hairpin.fa.gz", k=25, kc=2, b="400000", H=4, opt="-K10"),
        dict(name="mask_circ_K3", reads="cyc_circ.fa.gz", k=25, kc=2, b="400000", H=3, opt="-K3"),
        dict(name="mask_circ_qr17", reads="cyc_circ.fa.gz", k=40, kc=2, b="400000", H=4, opt="--qr-seed=17"),
    ]
    for c in mask_cases:
        out = os.path.join(HERE, c["name"] + ".fa")
        log = os.path.join(HERE, c["name"] + ".readlog.tsv") if c.get("readlog") else None
        info = run_ref(f"-k{c['k']} {c['opt']} --kc={c['kc']} -b{c['b']} -H{c['H']}", reads_of(c, e2e), out, log)
        c.update(info)
        body = "".join(l for l in open(out) if l[0] != ">")
        c["n_contigs"] = sum(1 for l in open(out) if l[0] == ">")
        c["n_N"] = body.count("N")
        print(c["name"], c["mask"], c["counters"], c["n_contigs"], c["n_N"])
    json.dump(mask_cases, open(os.path.join(HERE, "mask_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
