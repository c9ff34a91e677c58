"""GPU: `abyss-bloom trim` over libabyssb200 prints the stdout, stderr and exit status of the unmodified reference on every case
of tests/golden/trim_cases.json (tests/golden/make_golden_trim.py), whatever the batch size; Filter.trim_reads gives, read by
read, the lengths the CPU harness tests/host_trim computes with the same code; other filter kinds are refused."""
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
from make_golden_trim import FILTERS, fastq_records, write_inputs  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "trim_cases.json")))


def _run(d, args):
    return subprocess.run([EXE, *args], cwd=d, capture_output=True)


@pytest.fixture(scope="module")
def work(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("trim"))
    write_inputs(d)
    for f in FILTERS:
        r = _run(d, f["args"])
        assert r.returncode == 0, r.stderr.decode()
    return d


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_trim_cli(work, case):
    r = _run(work, case["args"])
    assert r.returncode == case["rc"], r.stderr.decode()
    assert r.stderr.decode() == case["stderr"]
    assert hashlib.md5(r.stdout).hexdigest() == case["stdout_md5"]


@pytest.mark.parametrize("name", ["self_k64", "mbl8", "hand_g25", "hand_strand", "two_files_gz"])
def test_batch_size_does_not_change_the_output(work, name):
    c = {x["name"]: x for x in CASES}[name]
    r = _run(work, ["trim", "--batch-reads=1000" if not name.startswith("hand_") else "--batch-reads=7", *c["args"][1:]])
    assert r.returncode == 0, r.stderr.decode()
    assert hashlib.md5(r.stdout).hexdigest() == c["stdout_md5"]


@pytest.mark.parametrize("k,filt,reads,mbl", [(25, "b25_16K.bloom", "B.fq", 8), (96, "a96.bloom", "A.fq", 5), (24, "g24.bloom", "H24.fq", 2)])
def test_trim_reads_equals_the_host_harness(work, abb, tmp_path, k, filt, reads, mbl):
    exe = str(tmp_path / "host_trim")
    subprocess.run(["g++", "-std=c++17", "-O2", "-pthread", "-o", exe, os.path.join(ROOT, "tests", "host_trim", "host_trim.cpp")],
                   check=True, capture_output=True)
    r = subprocess.run([exe, str(k), "--no-trim-masked", "--lengths", str(tmp_path / "len.txt"), filt, reads], cwd=work, capture_output=True)
    assert r.returncode == 0 and f"minBranchLen {mbl} " in r.stderr.decode(), r.stderr.decode()
    want = [l.split() for l in open(tmp_path / "len.txt").read().splitlines()]
    seqs = [s.upper() for _, s, _ in fastq_records(os.path.join(work, reads))]  # the reader folds case; masked ends kept (--no-trim-masked)
    assert len(seqs) == len(want)
    raw = open(os.path.join(work, filt), "rb").read()
    header = raw.split(b"\n", 4)
    full = int(header[2].split(b"\t")[0])
    f = abb.Filter.konnector(full, k, seed=int(header[3]))
    f.read_bits(np.frombuffer(header[4], dtype=np.uint8), full)
    left, right = f.trim_reads(seqs, mbl)
    f.close()
    for i, (s, w) in enumerate(zip(seqs, want)):
        assert (int(left[i]), int(right[i])) == (int(w[0]), int(w[1])), (i, s)


def test_reader_options_through_trim(work):
    # -q cuts the low-quality ends before the scan: the reference's output for the file cut beforehand (case trim_quality)
    c = {x["name"]: x for x in CASES}["trim_quality"]
    r = _run(work, ["trim", "-k25", "-q", "10", "b25.bloom", "D.fq"])
    assert r.returncode == 0, r.stderr.decode()
    assert hashlib.md5(r.stdout).hexdigest() == c["stdout_md5"]


def test_other_filter_kinds_are_refused(abb):
    for f in (abb.Filter.cascading(1 << 16, 2, 2, 25), abb.Filter.bits(1 << 16, 2, 25)):
        with pytest.raises(abb.AbbError) as e:
            f.trim_reads(["ACGT" * 20], 2)
        assert e.value.code == abb.ABB_ESTATE
        f.close()
