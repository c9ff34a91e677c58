"""CPU: k = 193..256 against the unmodified reference built with MAX_KMER = 256 (tests/golden/kwidth256_cases.json,
tests/golden/make_golden_kwidth256.py): the pass-2 templates at eight words (tests/host_walk/host_walk_kw8), `abyss-bloom graph`
(tests/host_bloom_graph), Konnector filters and `trim` over the eight-word Konnector k-mer (tests/host_konnector/
host_konnector_kw8, tests/host_trim/host_trim_kw8), and AdjList's overlap joins at k = 256 (tests/host_overlap).  The harnesses
instantiate the templates the kernels do, so a template that is wrong only at eight words fails here without a GPU."""
import json
import os
import re
import subprocess

import pytest

import overlap_cases as oc
import parity
from make_golden_kwidth import write_graph_inputs, write_trim_inputs
from make_golden_kwidth256 import adjlist_input

CASES = json.load(open(os.path.join(parity.GOLD, "kwidth256_cases.json")))
ASM = CASES["assembler"]
host_walk = parity.harness("host_walk_kw8", "tests/host_walk/host_walk_kw8.cpp", parity.ORACLE)
host_bloom_graph = parity.harness("host_bloom_graph", "tests/host_bloom_graph/host_bloom_graph.cpp", parity.ORACLE)
host_konnector = parity.harness("host_konnector_kw8", "tests/host_konnector/host_konnector_kw8.cpp")
host_trim = parity.harness("host_trim_kw8", "tests/host_trim/host_trim_kw8.cpp")
overlap_harness = parity.harness("AdjList", "tests/host_overlap/host_overlap.cpp")


def test_every_boundary_is_covered():
    """the eight-word instance, both K1 rings and both Konnector widths have cases"""
    ks = {c["k"] for c in ASM}
    assert {193, 224, 225, 256} <= ks
    assert {c["k"] for c in ASM if c["opt"]} >= {224, 256}
    assert {c["H"] for c in ASM if c["k"] == 256} >= {1, 4, 9}
    assert all(c["n_contigs"] > 0 for c in ASM)
    for section in ("graph", "trim", "konnector"):
        assert {193, 256} <= {int(re.search(r"_k(\d+)", c["name"]).group(1)) for c in CASES[section]}


# host_walk builds tiles without a mask only; spaced-seed cases run vertex by vertex here (the GPU test runs them with tiles)
WALKS = [(c, t) for c in ASM for t in (False, True) if not (t and c["opt"])]


@pytest.mark.parametrize("case,tiles", WALKS, ids=[c["name"] + ("-tiles" if t else "-vertex") for c, t in WALKS])
def test_assembler(host_walk, tmp_path, case, tiles):
    parity.check_host_assembler(host_walk, case, tmp_path, tiles)


@pytest.fixture(scope="module")
def graph_work(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("kwg256"))
    write_graph_inputs(d)
    return d


@pytest.mark.parametrize("case", CASES["graph"], ids=[c["name"] for c in CASES["graph"]])
def test_bloom_graph(host_bloom_graph, graph_work, case):
    parity.check_host_bloom_graph(host_bloom_graph, case, graph_work, os.path.join(parity.GOLD, f"kwidth256_{case['name']}.dot.gz"))


@pytest.fixture(scope="module")
def konnector_work(tmp_path_factory, host_konnector):
    """the Konnector filters of the cases built by the harness, in file order (the union reads the windows)"""
    d = str(tmp_path_factory.mktemp("kwk256"))
    write_trim_inputs(d)
    files = {}
    for c in CASES["konnector"]:
        if "harness" in c:
            parity.run(host_konnector, *c["harness"], cwd=d)
            files[c["name"]] = parity.sha256(open(os.path.join(d, c["file"]), "rb").read())
    return d, files


@pytest.mark.parametrize("case", [c for c in CASES["konnector"] if "harness" in c],
                         ids=[c["name"] for c in CASES["konnector"] if "harness" in c])
def test_konnector_filter(konnector_work, case):
    assert konnector_work[1][case["name"]] == case["sha256"]


@pytest.mark.parametrize("case", CASES["trim"], ids=[c["name"] for c in CASES["trim"]])
def test_trim(host_trim, konnector_work, case):
    parity.check_host_trim(host_trim, case, konnector_work[0])


@pytest.mark.parametrize("case", CASES["adjlist"], ids=[c["name"] for c in CASES["adjlist"]])
def test_adjlist(overlap_harness, tmp_path, case):
    t = adjlist_input(case)
    fa = str(tmp_path / "in.fa")
    oc.write_fasta(t, fa)
    r = subprocess.run([overlap_harness] + oc.command_args(t, fa), capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    got = oc.normalise(r.stdout, overlap_harness).replace(fa.encode(), b"IN.fa")
    assert (len(got), parity.sha256(got)) == (case["bytes"], case["sha256"])
