"""CPU: the pass-2 templates (abb_walk.cuh through tests/host_walk), `abyss-bloom graph` (tests/host_bloom_graph) and `abyss-bloom
trim` (tests/host_trim) at every k-mer width the kernels are compiled for, up to k = 192, against the unmodified reference
(tests/golden/kwidth_cases.json, tests/golden/make_golden_kwidth.py).  The harnesses instantiate the same Kmer<KW> templates
the CUDA kernels do, so a template that is wrong only for four or six words fails here without a GPU."""
import gzip
import hashlib
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, GOLD)
from make_golden_kwidth import TRIM_FILTERS, raw_reads, reader_view, write_fastq, write_graph_inputs, write_trim_inputs  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "kwidth_cases.json")))
ASM = CASES["assembler"]


def kw(k):
    return {1: 1, 2: 2, 3: 3, 4: 4}.get((2 * k + 63) // 64, 6)


def md5(data):
    return hashlib.md5(data).hexdigest()


def test_every_width_is_covered():
    """each instance of the pass-2 kernels, and the word boundaries of the issue, have cases"""
    widths = {kw(c["k"]) for c in ASM}
    assert widths == {1, 2, 3, 4, 6}
    ks = {c["k"] for c in ASM}
    assert {33, 65, 97, 129, 160, 192} <= ks
    for section in ("graph", "trim"):
        assert {97, 129, 160, 192} <= {int(re.search(r"_k(\d+)", c["name"]).group(1)) for c in CASES[section]}
    assert {c["k"] for c in ASM if c["opt"]} >= {128, 140, 160, 192}
    assert {c["H"] for c in ASM} >= {1, 4, 9}


@pytest.fixture(scope="module")
def host_walk(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("hw") / "host_walk")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wno-unknown-pragmas", "-o", exe, os.path.join(ROOT, "tests", "host_walk", "host_walk.cpp"),
                    os.path.join(ROOT, "oracle", "abyss_oracle.c")], check=True, capture_output=True)
    return exe


# the assembler builds no tiles for a spaced seed (abb_assemble.cu: tiles_on), so those cases run vertex by vertex only
WALKS = [(c, t) for c in ASM for t in (False, True) if not (t and c["opt"])]


@pytest.mark.parametrize("case,tiles", WALKS, ids=[c["name"] + ("-tiles" if t else "-vertex") for c, t in WALKS])
def test_assembler(host_walk, tmp_path, case, tiles):
    fq, log = str(tmp_path / "reads.fq"), str(tmp_path / "read.log")
    write_fastq(reader_view(raw_reads(case["reads"])), fq)
    env = dict(os.environ, HOST_WALK_MASK=case.get("mask", ""))
    env.pop("HOST_WALK_TILES", None)
    if tiles:
        env["HOST_WALK_TILES"] = "1"
    r = subprocess.run([host_walk, str(case["k"]), str(case["kc"]), str(case["H"]), str(case["counters"]), str(case["k"]), fq, log],
                       capture_output=True, env=env)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout.count(b">") == case["n_contigs"]
    assert md5(r.stdout) == case["fasta_md5"]
    assert md5(open(log, "rb").read()) == case["readlog_md5"]


@pytest.fixture(scope="module")
def graph_work(tmp_path_factory):
    d = tmp_path_factory.mktemp("kwg")
    exe = str(d / "host_bloom_graph")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wno-unknown-pragmas", "-pthread", "-o", exe,
                    os.path.join(ROOT, "tests", "host_bloom_graph", "host_bloom_graph.cpp"), os.path.join(ROOT, "oracle", "abyss_oracle.c")],
                   check=True, capture_output=True)
    write_graph_inputs(str(d))  # the harness rebuilds each filter from the recipe in the case's command line
    return str(d), exe


@pytest.mark.parametrize("case", CASES["graph"], ids=[c["name"] for c in CASES["graph"]])
def test_bloom_graph(graph_work, case):
    d, exe = graph_work
    r = subprocess.run([exe, *case["harness"]], cwd=d, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert (len(r.stdout), r.stdout.count(b"\n")) == (case["bytes"], case["lines"])
    assert r.stdout == gzip.open(os.path.join(GOLD, f"kwidth_{case['name']}.dot.gz"), "rb").read()
    assert hashlib.sha256(r.stdout).hexdigest() == case["sha256"]


@pytest.fixture(scope="module")
def trim_work(tmp_path_factory):
    d = tmp_path_factory.mktemp("kwt")
    exes = {}
    for name in ("host_konnector", "host_trim"):
        exes[name] = str(d / name)
        subprocess.run(["g++", "-std=c++17", "-O2", "-pthread", "-o", exes[name], os.path.join(ROOT, "tests", name, name + ".cpp")],
                       check=True, capture_output=True)
    write_trim_inputs(str(d))
    for f in TRIM_FILTERS:
        r = subprocess.run([exes["host_konnector"], *map(str, f["harness"])], cwd=str(d), capture_output=True)
        assert r.returncode == 0, r.stderr.decode()
    return str(d), exes["host_trim"]


@pytest.mark.parametrize("case", CASES["trim"], ids=[c["name"] for c in CASES["trim"]])
def test_trim(trim_work, case):
    d, exe = trim_work
    r = subprocess.run([exe, *map(str, case["harness"])], cwd=d, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert md5(r.stdout) == case["stdout_md5"]
    m = re.search(r"min length threshold for true branches \(k-mers\): (\d+)", case["stderr"])
    if m:
        assert f"minBranchLen {m.group(1)} " in r.stderr.decode()
