#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: the scale golden of `abyss-bloom build -t konnector`, from the UNMODIFIED reference in oracle/_ref.
1 M x 150 bp of a 5 Mbp genome (seed 7, the reads of make_golden_scale.py's m1_k64), -k64 -b1G -l2: the sha256 of the
512 MiB file goes to konnector_scale.json.  The Konnector insert does not depend on order, so the reference's -j8 file is
its -j1 file.

Run in the build container only:  python tests/golden/make_golden_konnector_scale.py"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from abyss_b200.synth import ReadSet  # noqa: E402

CASES = [dict(name="m1_k64_b1G_l2", seed=7, genome=5000000, n_reads=1000000, L=150, err=0.005, args=["-k64", "-b1G", "-l2"])]


def sha256_file(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 22), b""):
            h.update(blk)
    return h.hexdigest()


def main():
    out = []
    with tempfile.TemporaryDirectory() as d:
        for c in CASES:
            fq = os.path.join(d, "r.fq")
            ReadSet(c["seed"], c["genome"], c["n_reads"], c["L"], c["err"]).write_fastq(fq)
            t0 = time.time()
            r = subprocess.run([os.path.join(ROOT, "oracle", "_ref", "abyss-bloom-ref"), "build", *c["args"], "-j8",
                                os.path.join(d, "o.bloom"), fq], capture_output=True, text=True, check=True)
            out.append({**c, "sha256": sha256_file(os.path.join(d, "o.bloom")), "stderr": r.stderr})
            print(c["name"], f"{time.time() - t0:.1f} s")
    json.dump(out, open(os.path.join(HERE, "konnector_scale.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
