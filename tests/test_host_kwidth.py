"""CPU: the pass-2 templates (abb_walk.cuh through tests/host_walk), `abyss-bloom graph` (tests/host_bloom_graph) and `abyss-bloom
trim` (tests/host_trim) at every k-mer width the kernels are compiled for, up to k = 192, against the unmodified reference
(tests/golden/kwidth_cases.json, tests/golden/make_golden_kwidth.py).  The harnesses instantiate the same Kmer<KW> templates
the CUDA kernels do, so a template that is wrong only for four or six words fails here without a GPU."""
import json
import os
import re

import pytest

import parity
from make_golden_kwidth import TRIM_FILTERS, write_graph_inputs, write_trim_inputs

CASES = json.load(open(os.path.join(parity.GOLD, "kwidth_cases.json")))
ASM = CASES["assembler"]
host_walk = parity.harness("host_walk", "tests/host_walk/host_walk.cpp", parity.ORACLE)
host_bloom_graph = parity.harness("host_bloom_graph", "tests/host_bloom_graph/host_bloom_graph.cpp", parity.ORACLE)
host_konnector = parity.harness("host_konnector", "tests/host_konnector/host_konnector.cpp")
host_trim = parity.harness("host_trim", "tests/host_trim/host_trim.cpp")


def kw(k):
    return {1: 1, 2: 2, 3: 3, 4: 4}.get((2 * k + 63) // 64, 6)


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


# the assembler builds no tiles for a spaced seed (abb_assemble.cu: tiles_on), so those cases run vertex by vertex only
WALKS = [(c, t) for c in ASM for t in (False, True) if not (t and c["opt"])]


@pytest.mark.parametrize("case,tiles", WALKS, ids=[c["name"] + ("-tiles" if t else "-vertex") for c, t in WALKS])
def test_assembler(host_walk, tmp_path, case, tiles):
    parity.check_host_assembler(host_walk, case, tmp_path, tiles)


@pytest.fixture(scope="module")
def graph_work(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("kwg"))
    write_graph_inputs(d)  # the harness rebuilds each filter from the recipe in the case's command line
    return d


@pytest.mark.parametrize("case", CASES["graph"], ids=[c["name"] for c in CASES["graph"]])
def test_bloom_graph(host_bloom_graph, graph_work, case):
    parity.check_host_bloom_graph(host_bloom_graph, case, graph_work, os.path.join(parity.GOLD, f"kwidth_{case['name']}.dot.gz"))


@pytest.fixture(scope="module")
def trim_work(tmp_path_factory, host_konnector):
    d = str(tmp_path_factory.mktemp("kwt"))
    write_trim_inputs(d)
    for f in TRIM_FILTERS:
        parity.run(host_konnector, *f["harness"], cwd=d)
    return d


@pytest.mark.parametrize("case", CASES["trim"], ids=[c["name"] for c in CASES["trim"]])
def test_trim(host_trim, trim_work, case):
    parity.check_host_trim(host_trim, case, trim_work)
