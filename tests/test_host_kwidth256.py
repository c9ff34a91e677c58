"""CPU: k = 193..256 against the unmodified reference built with MAX_KMER = 256 (tests/golden/kwidth256_cases.json,
tests/golden/make_golden_kwidth256.py): the pass-2 templates at eight words (tests/host_walk/host_walk_kw8), `abyss-bloom graph`
(tests/host_bloom_graph), Konnector filters and `trim` over the eight-word Konnector k-mer (tests/host_konnector/
host_konnector_kw8, tests/host_trim/host_trim_kw8), and AdjList's overlap joins at k = 256 (tests/host_overlap).  The harnesses
instantiate the templates the kernels do, so a template that is wrong only at eight words fails here without a GPU."""
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
from make_golden_kwidth import raw_reads, reader_view, write_fastq, write_graph_inputs, write_trim_inputs  # noqa: E402
from make_golden_kwidth256 import adjlist_input  # noqa: E402
import overlap_cases as oc  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "kwidth256_cases.json")))
ASM = CASES["assembler"]


def md5(data):
    return hashlib.md5(data).hexdigest()


def _compile(out, *srcs):
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wno-unknown-pragmas", "-pthread", "-o", out, *srcs], check=True, capture_output=True)
    return out


def test_every_boundary_is_covered():
    """the eight-word instance, both K1 rings and both Konnector widths have cases"""
    ks = {c["k"] for c in ASM}
    assert {193, 224, 225, 256} <= ks
    assert {c["k"] for c in ASM if c["opt"]} >= {224, 256}
    assert {c["H"] for c in ASM if c["k"] == 256} >= {1, 4, 9}
    assert all(c["n_contigs"] > 0 for c in ASM)
    for section in ("graph", "trim", "konnector"):
        assert {193, 256} <= {int(re.search(r"_k(\d+)", c["name"]).group(1)) for c in CASES[section]}


@pytest.fixture(scope="module")
def host_walk(tmp_path_factory):
    d = tmp_path_factory.mktemp("hw8")
    return _compile(str(d / "host_walk_kw8"), os.path.join(ROOT, "tests", "host_walk", "host_walk_kw8.cpp"),
                    os.path.join(ROOT, "oracle", "abyss_oracle.c"))


# host_walk builds tiles without a mask only; spaced-seed cases run vertex by vertex here (the GPU test runs them with tiles)
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
    d = tmp_path_factory.mktemp("kwg256")
    exe = _compile(str(d / "host_bloom_graph"), os.path.join(ROOT, "tests", "host_bloom_graph", "host_bloom_graph.cpp"),
                   os.path.join(ROOT, "oracle", "abyss_oracle.c"))
    write_graph_inputs(str(d))
    return str(d), exe


@pytest.mark.parametrize("case", CASES["graph"], ids=[c["name"] for c in CASES["graph"]])
def test_bloom_graph(graph_work, case):
    d, exe = graph_work
    r = subprocess.run([exe, *case["harness"]], cwd=d, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == gzip.open(os.path.join(GOLD, f"kwidth256_{case['name']}.dot.gz"), "rb").read()
    assert hashlib.sha256(r.stdout).hexdigest() == case["sha256"]


@pytest.fixture(scope="module")
def konnector_work(tmp_path_factory):
    """the Konnector filters of the cases built by the harness, in file order (the union reads the windows)"""
    d = tmp_path_factory.mktemp("kwk256")
    exes = {name: _compile(str(d / name), os.path.join(ROOT, "tests", name.replace("_kw8", ""), name + ".cpp"))
            for name in ("host_konnector_kw8", "host_trim_kw8")}
    write_trim_inputs(str(d))
    files = {}
    for c in CASES["konnector"]:
        if "harness" in c:
            r = subprocess.run([exes["host_konnector_kw8"], *map(str, c["harness"])], cwd=str(d), capture_output=True)
            assert r.returncode == 0, r.stderr.decode()
            files[c["name"]] = hashlib.sha256(open(os.path.join(d, c["file"]), "rb").read()).hexdigest()
    return str(d), exes["host_trim_kw8"], files


@pytest.mark.parametrize("case", [c for c in CASES["konnector"] if "harness" in c],
                         ids=[c["name"] for c in CASES["konnector"] if "harness" in c])
def test_konnector_filter(konnector_work, case):
    assert konnector_work[2][case["name"]] == case["sha256"]


@pytest.mark.parametrize("case", CASES["trim"], ids=[c["name"] for c in CASES["trim"]])
def test_trim(konnector_work, case):
    d, exe, _ = konnector_work
    r = subprocess.run([exe, *map(str, case["harness"])], cwd=d, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert md5(r.stdout) == case["stdout_md5"]
    m = re.search(r"min length threshold for true branches \(k-mers\): (\d+)", case["stderr"])
    if m:
        assert f"minBranchLen {m.group(1)} " in r.stderr.decode()


@pytest.fixture(scope="module")
def overlap_harness(tmp_path_factory):
    return _compile(str(tmp_path_factory.mktemp("ho256") / "AdjList"), os.path.join(ROOT, "tests", "host_overlap", "host_overlap.cpp"))


@pytest.mark.parametrize("case", CASES["adjlist"], ids=[c["name"] for c in CASES["adjlist"]])
def test_adjlist(overlap_harness, tmp_path, case):
    t = adjlist_input(case)
    fa = str(tmp_path / "in.fa")
    oc.write_fasta(t, fa)
    r = subprocess.run([overlap_harness] + oc.command_args(t, fa), capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    got = oc.normalise(r.stdout, overlap_harness).replace(fa.encode(), b"IN.fa")
    assert (len(got), hashlib.sha256(got).hexdigest()) == (case["bytes"], case["sha256"])
