"""GPU: `abyss-bloom trim` over libabyssb200 prints the stdout, stderr and exit status of the unmodified reference on every case
of tests/golden/trim_cases.json (tests/golden/make_golden_trim.py), whatever the batch size; Filter.trim_reads gives, read by
read, the lengths the CPU harness tests/host_trim computes with the same code; other filter kinds are refused."""
import json
import os

import numpy as np
import pytest

import parity
from make_golden_trim import FILTERS, fastq_records, write_inputs

pytestmark = pytest.mark.gpu
CASES = json.load(open(os.path.join(parity.GOLD, "trim_cases.json")))
host_trim = parity.harness("host_trim", "tests/host_trim/host_trim.cpp")


@pytest.fixture(scope="module")
def work(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("trim"))
    write_inputs(d)
    parity.build_filters(FILTERS, d)
    return d


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_trim_cli(work, case):
    parity.check_trim_cli(case, work)


@pytest.mark.parametrize("name", ["self_k64", "mbl8", "hand_g25", "hand_strand", "two_files_gz"])
def test_batch_size_does_not_change_the_output(work, name):
    c = {x["name"]: x for x in CASES}[name]
    r = parity.abyss_bloom("trim", "--batch-reads=1000" if not name.startswith("hand_") else "--batch-reads=7", *c["args"][1:], cwd=work)
    assert r.returncode == 0, r.stderr.decode()
    assert parity.md5(r.stdout) == c["stdout_md5"]


@pytest.mark.parametrize("k,filt,reads,mbl", [(25, "b25_16K.bloom", "B.fq", 8), (96, "a96.bloom", "A.fq", 5), (24, "g24.bloom", "H24.fq", 2)])
def test_trim_reads_equals_the_host_harness(work, abb, host_trim, tmp_path, k, filt, reads, mbl):
    r = parity.run(host_trim, k, "--no-trim-masked", "--lengths", tmp_path / "len.txt", filt, reads, cwd=work)
    assert f"minBranchLen {mbl} " in r.stderr.decode(), r.stderr.decode()
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
    r = parity.abyss_bloom("trim", "-k25", "-q", "10", "b25.bloom", "D.fq", cwd=work)
    assert r.returncode == 0, r.stderr.decode()
    assert parity.md5(r.stdout) == c["stdout_md5"]


def test_other_filter_kinds_are_refused(abb):
    for f in (abb.Filter.cascading(1 << 16, 2, 2, 25), abb.Filter.bits(1 << 16, 2, 25)):
        with pytest.raises(abb.AbbError) as e:
            f.trim_reads(["ACGT" * 20], 2)
        assert e.value.code == abb.ABB_ESTATE
        f.close()
