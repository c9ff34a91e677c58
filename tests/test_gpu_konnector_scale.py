"""GPU: `abyss-bloom build -t konnector` at scale -- 1 M x 150 bp, -k64 -b1G -l2 (two 512 MiB levels, positions past 2^32
bits) -- writes the sha256 and the statistics of the unmodified reference's file (tests/golden/make_golden_konnector_scale.py),
in one batch and in four."""
import hashlib
import json
import os

import pytest

import parity
from abyss_b200.synth import ReadSet

pytestmark = pytest.mark.gpu
CASES = json.load(open(os.path.join(parity.GOLD, "konnector_scale.json")))


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
    r = parity.run(os.path.join(parity.BIN, "abyss-bloom"), "build", *case["args"], *extra, out, fqs[case["name"]])
    assert r.stderr.decode() == case["stderr"]
    with open(out, "rb") as f:
        assert hashlib.file_digest(f, "sha256").hexdigest() == case["sha256"]
    os.remove(out)
