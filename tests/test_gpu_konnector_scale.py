"""GPU: `abyss-bloom build -t konnector` at scale -- 1 M x 150 bp, -k64 -b1G -l2 (two 512 MiB levels, positions past 2^32
bits) -- writes the sha256 and the statistics of the unmodified reference's file (tests/golden/make_golden_konnector_scale.py),
in one batch and in four."""
import hashlib
import json
import os
import subprocess

import pytest

from abyss_b200.synth import ReadSet

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "abyss_b200", "lib", "abyss-bloom")
CASES = json.load(open(os.path.join(ROOT, "tests", "golden", "konnector_scale.json")))


def sha256_file(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 22), b""):
            h.update(blk)
    return h.hexdigest()


@pytest.fixture(scope="module")
def reads(tmp_path_factory):
    d = tmp_path_factory.mktemp("konscale")
    out = {}
    for c in CASES:
        fq = str(d / (c["name"] + ".fq"))
        ReadSet(c["seed"], c["genome"], c["n_reads"], c["L"], c["err"]).write_fastq(fq)
        out[c["name"]] = fq
    return d, out


@pytest.mark.parametrize("batch", [None, 250000])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_konnector_scale(abb, reads, case, batch):
    d, fqs = reads
    out = str(d / "o.bloom")
    extra = [f"--batch-reads={batch}"] if batch else []
    r = subprocess.run([EXE, "build", *case["args"], *extra, out, fqs[case["name"]]], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stderr == case["stderr"]
    assert sha256_file(out) == case["sha256"]
    os.remove(out)
