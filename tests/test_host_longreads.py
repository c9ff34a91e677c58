"""CPU: the pass-2 templates (abb_walk.cuh through tests/host_walk) on long reads of 5 to 80 kbp against the unmodified reference
(tests/golden/longread_cases.json, tests/golden/make_golden_longreads.py), vertex by vertex and with tiles spliced in.  This
covers walk_read, extend_seed and the tile splicing over many unitigs per read and unitigs of 2^15 k-mers and more; the
whole-grid replay of K5 and the device coverage marking run only on the GPU (tests/test_gpu_longreads.py)."""
import json
import os

import pytest

import parity
from make_golden_longreads import raw_reads, write_fastq

CASES = json.load(open(os.path.join(parity.GOLD, "longread_cases.json")))
host_walk = parity.harness("host_walk", "tests/host_walk/host_walk.cpp", parity.ORACLE)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_reads_are_rebuilt(tmp_path, case):
    """the generator's seeds still give the reads the goldens were made from"""
    fq = str(tmp_path / "reads.fq")
    write_fastq(raw_reads(case["reads"]), fq)
    assert parity.md5(open(fq, "rb").read()) == case["reads_md5"]


WALKS = [(c, t) for c in CASES for t in (False, True)]


@pytest.mark.parametrize("case,tiles", WALKS, ids=[c["name"] + ("-tiles" if t else "-vertex") for c, t in WALKS])
def test_assembler(host_walk, tmp_path, case, tiles):
    fq, log = str(tmp_path / "reads.fq"), str(tmp_path / "read.log")
    write_fastq(raw_reads(case["reads"]), fq)
    parity.check_unitigs(case, *parity.run_host_walk(host_walk, case, fq, log, tiles)[:2])
