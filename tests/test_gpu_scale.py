"""GPU parity at the sizes SURVEY.md 8(d) names, through the C++ command-line programs (the drop-in boundary):
config 1 (53 333 x 150 bp, -b64M) at k = 32, 40, 48, 64, 96, the same reads with N / lower-case ends / short reads,
and 1 M reads at -k64 --kc=3 -b1G, each in the default batch and split into batches (--batch-reads).  Goldens: md5 of the reference's -j1 FASTA and --read-log, sha256 of the
counters of `abyss-bloom build -t counting -j1` (tests/golden/make_golden_scale.py, scale_cases.json)."""
import json
import os

import pytest

import parity
from abyss_b200.synth import ReadSet, edge_mutate

pytestmark = pytest.mark.gpu
CASES = json.load(open(os.path.join(parity.GOLD, "scale_cases.json")))


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
    fasta, log, _ = parity.bloom_dbg_cli(c, fq, tmp_path, *([f"--batch-reads={batch}"] if batch else []))
    parity.check_unitigs(c, fasta, log)
    assert sum(map(len, fasta.split(b"\n")[1::2])) == c["bases"]
    parity.check_counting_build(c, fq, tmp_path)
