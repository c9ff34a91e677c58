#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: the scale golden of `abyss-bloom trim`, from the UNMODIFIED reference in oracle/_ref.  The reads and
the filter of konnector_scale.json (1 M x 150 bp of a 5 Mbp genome, seed 7; build -k64 -b1G -l2, whose file is the last
level); `trim -vv -k64` on those reads: the md5 of the trimmed FASTQ, its size, stderr (minBranchLen and the "Processed N
reads" lines) go to trim_scale.json, with the reference's wall time as context (one thread; not a baseline).

    python tests/golden/make_golden_trim_scale.py"""
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


def main():
    exe = os.path.join(ROOT, "oracle", "_ref", "abyss-bloom-ref")
    out = []
    for c in json.load(open(os.path.join(HERE, "konnector_scale.json"))):
        with tempfile.TemporaryDirectory() as d:
            ReadSet(c["seed"], c["genome"], c["n_reads"], c["L"], c["err"]).write_fastq(os.path.join(d, "r.fq"))
            subprocess.run([exe, "build", *c["args"], "-j8", "o.bloom", "r.fq"], cwd=d, capture_output=True, check=True)
            k = [a for a in c["args"] if a.startswith("-k")][0]
            t0 = time.time()
            with open(os.path.join(d, "t.fq"), "wb") as f:
                r = subprocess.run([exe, "trim", "-vv", k, "o.bloom", "r.fq"], cwd=d, stdout=f, stderr=subprocess.PIPE, check=True)
            wall = time.time() - t0
            h = hashlib.md5()
            with open(os.path.join(d, "t.fq"), "rb") as f:
                for blk in iter(lambda: f.read(1 << 22), b""):
                    h.update(blk)
            keys = ("name", "seed", "genome", "n_reads", "L", "err", "args")
            out.append({**{x: c[x] for x in keys}, "trim_args": ["-vv", k], "stdout_md5": h.hexdigest(),
                        "stdout_bytes": os.path.getsize(os.path.join(d, "t.fq")), "stderr": r.stderr.decode(),
                        "reference_wall_s": round(wall, 1)})
            print(c["name"], f"{wall:.1f} s")
    json.dump(out, open(os.path.join(HERE, "trim_scale.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
