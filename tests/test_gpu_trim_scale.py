"""GPU: `abyss-bloom trim` at scale -- 1 M x 150 bp against the last level of a -k64 -b1G -l2 filter that `abyss-bloom build`
writes here (minBranchLen 2), two million tasks so that every warp of k_kon_trim works through hundreds of them -- prints the
md5 of the unmodified reference's trimmed FASTQ and its stderr, with the "Processed N reads" line that a dropped read
skips (tests/golden/make_golden_trim_scale.py), in one batch and in four."""
import hashlib
import json
import os
import subprocess

import pytest

from abyss_b200.synth import ReadSet

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "abyss_b200", "lib", "abyss-bloom")
CASES = json.load(open(os.path.join(ROOT, "tests", "golden", "trim_scale.json")))


@pytest.fixture(scope="module")
def work(tmp_path_factory, abb):
    out = {}
    for c in CASES:
        d = str(tmp_path_factory.mktemp("trimscale"))
        ReadSet(c["seed"], c["genome"], c["n_reads"], c["L"], c["err"]).write_fastq(os.path.join(d, "r.fq"))
        r = subprocess.run([EXE, "build", *c["args"], "o.bloom", "r.fq"], cwd=d, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out[c["name"]] = d
    return out


@pytest.mark.parametrize("batch", [None, 250000])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_trim_scale(work, case, batch):
    extra = [f"--batch-reads={batch}"] if batch else []
    p = subprocess.Popen([EXE, "trim", *case["trim_args"], *extra, "o.bloom", "r.fq"], cwd=work[case["name"]], stdout=subprocess.PIPE,
                         stderr=subprocess.PIPE)
    h, n = hashlib.md5(), 0
    for blk in iter(lambda: p.stdout.read(1 << 22), b""):
        h.update(blk)
        n += len(blk)
    err = p.stderr.read().decode()
    assert p.wait() == 0, err
    assert "min length threshold for true branches (k-mers): 2\n" in err
    assert err == case["stderr"]
    assert (n, h.hexdigest()) == (case["stdout_bytes"], case["stdout_md5"])
