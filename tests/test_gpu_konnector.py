"""GPU: `abyss-bloom` on Konnector filters (build -t konnector with levels, seeds, -L and -w windows, union, intersect, info,
compare, kmers) over libabyssb200 writes the files, stdout, stderr and exit status of the unmodified reference
(tests/golden/make_golden_konnector.py)."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
EXE = os.path.join(ROOT, "abyss_b200", "lib", "abyss-bloom")
sys.path.insert(0, GOLD)
from make_golden_konnector import write_reads  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "konnector_cases.json")))


def _run(d, args):
    r = subprocess.run([EXE, *args], cwd=d, capture_output=True)
    return r


@pytest.fixture(scope="module")
def results(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("kon"))
    write_reads(d)
    out = {}
    for c in CASES:  # in file order: later cases read the files earlier ones wrote
        r = _run(d, c["args"])
        rec = {"rc": r.returncode, "stdout_md5": hashlib.md5(r.stdout).hexdigest(), "stderr": r.stderr.decode()}
        if "file" in c and os.path.exists(os.path.join(d, c["file"])):
            rec["sha256"] = hashlib.sha256(open(os.path.join(d, c["file"]), "rb").read()).hexdigest()
        out[c["name"]] = rec
    return d, out


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_konnector_cli(results, case):
    got = results[1][case["name"]]
    assert got["rc"] == case["rc"], got["stderr"]
    assert got["stderr"] == case["stderr"]
    assert got["stdout_md5"] == case["stdout_md5"]
    if "sha256" in case:
        assert got["sha256"] == case["sha256"]


@pytest.mark.parametrize("name", ["build_k64_l3", "window_2of3", "init_level"])
def test_batch_size_does_not_change_the_file(results, name):
    # the level walk is order free: any split of the reads into batches gives the same bytes
    d, _ = results
    c = {x["name"]: x for x in CASES}[name]
    args = list(c["args"])
    args[args.index(c["file"])] = "small_batches.bloom"
    r = _run(d, ["build", "--batch-reads=1000", *args[1:]])
    assert r.returncode == 0, r.stderr.decode()
    assert hashlib.sha256(open(os.path.join(d, "small_batches.bloom"), "rb").read()).hexdigest() == c["sha256"]


def test_compare_counts_every_bit_once(abb):
    # a size that is no multiple of 32 KiB and a partial last byte: the four counts add up to the bit count
    bits = 100_003
    rng = np.random.default_rng(5)
    a = abb.Filter.konnector(bits, 25)
    b = abb.Filter.konnector(bits, 25)
    ra = rng.integers(0, 256, (bits + 7) // 8, dtype=np.uint8)
    rb = rng.integers(0, 256, (bits + 7) // 8, dtype=np.uint8)
    a.read_bits(ra, bits)
    b.read_bits(rb, bits)
    n = a.compare(b)
    assert sum(n) == bits
    ua, ub = np.unpackbits(ra)[:bits].astype(bool), np.unpackbits(rb)[:bits].astype(bool)
    assert n[:3] == (int((ua & ub).sum()), int((ua & ~ub).sum()), int((~ua & ub).sum()))
    assert a.level_popcount() == int(ua.sum()) == a.popCount()


def test_ntHash_entry_points_refuse_konnector(abb):
    f = abb.Filter.konnector(1 << 16, 25)
    with pytest.raises(abb.AbbError) as e:
        f.insert(np.zeros(4, dtype=np.uint64))
    assert e.value.code == abb.ABB_ESTATE


def test_too_large_filter_suggests_windows(tmp_path):
    fq = tmp_path / "r.fq"
    fq.write_text("@r/1\nACGTACGTACGTACGTACGTACGTACGT\n+\nIIIIIIIIIIIIIIIIIIIIIIIIIIII\n")
    r = subprocess.run([EXE, "build", "-k25", "-b200000G", str(tmp_path / "o.bloom"), str(fq)], capture_output=True, text=True)
    assert r.returncode != 0
    assert "-w M/N" in r.stderr
