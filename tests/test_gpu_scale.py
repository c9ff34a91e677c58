"""GPU parity at the sizes SURVEY.md 8(d) names, through the C++ command-line programs (the drop-in boundary):
config 1 (53 333 x 150 bp, -b64M) at k = 32, 40, 48, 64, 96, the same reads with N / lower-case ends / short reads,
and 1 M reads at -k64 --kc=3 -b1G, each in the default batch and split into batches (--batch-reads).  Goldens: md5 of the reference's -j1 FASTA and --read-log, sha256 of the
counters of `abyss-bloom build -t counting -j1` (tests/golden/make_golden_scale.py, scale_cases.json)."""
import hashlib
import json
import os
import subprocess

import pytest

from abyss_b200.synth import ReadSet, edge_mutate

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "abyss_b200", "lib")
CASES = json.load(open(os.path.join(ROOT, "tests", "golden", "scale_cases.json")))


def md5_file(path):
    h = hashlib.md5()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 22), b""):
            h.update(blk)
    return h.hexdigest()


def write_reads(c, path):
    rs = ReadSet(c["seed"], c["genome"], c["n_reads"], c["L"], c["err"])
    if not c["edge"]:
        rs.write_fastq(path)
        return
    seqs = edge_mutate([a.tobytes().decode() for a in rs.ascii(0, rs.n)])
    with open(path, "w") as f:
        for i, s in enumerate(seqs):
            f.write(f"@{rs.read_id(i)}\n{s}\n+\n{'I' * len(s)}\n")


def _batches(c):
    # the default batch (4 M reads: one batch here) and a split one: a prime for config 1, so that batch boundaries fall at every
    # offset of the read order; 131 072 for the 1 M-read case.  The reference's output does not depend on the batch size.
    yield pytest.param(c, None, id=c["name"])
    split = 131072 if c["name"] == "m1_k64" else 7919 if c["name"].startswith("cfg1_") else None
    if split:
        yield pytest.param(c, split, id=f"{c['name']}-batch{split}")


@pytest.mark.parametrize("case,batch", [p for c in CASES for p in _batches(c)])
def test_scale_case_identical_to_reference(abb, tmp_path, case, batch):
    c = case
    fq = str(tmp_path / "reads.fq")
    write_reads(c, fq)
    fa, log, bf = str(tmp_path / "out.fa"), str(tmp_path / "read.log"), str(tmp_path / "c.bloom")
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"-k{c['k']}", f"--kc={c['kc']}", f"-b{c['b']}", f"-H{c['H']}",
                        f"--read-log={log}", "-o", fa, fq] + ([f"--batch-reads={batch}"] if batch else []), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    seqs = [l.strip() for l in open(fa) if not l.startswith(">")]
    assert (len(seqs), sum(map(len, seqs))) == (c["n_contigs"], c["bases"])
    assert md5_file(fa) == c["fasta_md5"]
    assert md5_file(log) == c["readlog_md5"]
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), "build", "-k", str(c["k"]), "-t", "counting", f"-b{c['counters']}",
                        f"-H{c['H']}", bf, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    blob = open(bf, "rb").read()
    tag = b"[HeaderEnd]\n"
    raw = blob[blob.index(tag) + len(tag):]
    assert len(raw) == c["counters"]
    assert hashlib.sha256(raw).hexdigest() == c["counters_sha256"]
