"""CPU: the pass-2 templates (abb_walk.cuh through tests/host_walk) on long reads of 5 to 80 kbp against the unmodified reference
(tests/golden/longread_cases.json, tests/golden/make_golden_longreads.py), vertex by vertex and with tiles spliced in.  This
covers walk_read, extend_seed and the tile splicing over many unitigs per read and unitigs of 2^15 k-mers and more; the
whole-grid replay of K5 and the device coverage marking run only on the GPU (tests/test_gpu_longreads.py)."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, GOLD)
from make_golden_longreads import raw_reads, write_fastq  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "longread_cases.json")))


def md5(data):
    return hashlib.md5(data).hexdigest()


@pytest.fixture(scope="module")
def host_walk(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("hw") / "host_walk")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wno-unknown-pragmas", "-o", exe, os.path.join(ROOT, "tests", "host_walk", "host_walk.cpp"),
                    os.path.join(ROOT, "oracle", "abyss_oracle.c")], check=True, capture_output=True)
    return exe


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_reads_are_rebuilt(tmp_path, case):
    """the generator's seeds still give the reads the goldens were made from"""
    fq = str(tmp_path / "reads.fq")
    write_fastq(raw_reads(case["reads"]), fq)
    assert md5(open(fq, "rb").read()) == case["reads_md5"]


WALKS = [(c, t) for c in CASES for t in (False, True)]


@pytest.mark.parametrize("case,tiles", WALKS, ids=[c["name"] + ("-tiles" if t else "-vertex") for c, t in WALKS])
def test_assembler(host_walk, tmp_path, case, tiles):
    fq, log = str(tmp_path / "reads.fq"), str(tmp_path / "read.log")
    write_fastq(raw_reads(case["reads"]), fq)
    env = {k: v for k, v in os.environ.items() if not k.startswith("HOST_WALK_")}
    if tiles:
        env["HOST_WALK_TILES"] = "1"
    r = subprocess.run([host_walk, str(case["k"]), str(case["kc"]), str(case["H"]), str(case["counters"]), str(case["k"]), fq, log],
                       capture_output=True, env=env)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout.count(b">") == case["n_contigs"]
    assert md5(r.stdout) == case["fasta_md5"]
    assert md5(open(log, "rb").read()) == case["readlog_md5"]
