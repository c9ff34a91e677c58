"""CPU: the GraphViz dump `abyss-bloom-dbg -g` -- the product's traversal (abyss_b200/host/graph_dump.h) and the out-edge walk
the CUDA kernel runs (successors_chain, abyss_b200/csrc/abb_graph.cuh), driven by the single-thread harness tests/host_graph
on an oracle-built filter -- writes the bytes of the unmodified reference's -g file (tests/golden/make_golden_graph.py)."""
import json
import os

import pytest

import parity
from make_golden_graph import write_reads

CASES = json.load(open(os.path.join(parity.GOLD, "graph_cases.json")))
harness = parity.harness("host_graph", "tests/host_graph/host_graph.cpp", parity.ORACLE)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_graph_dump(harness, tmp_path, case):
    c = case
    fq = str(tmp_path / "r.fq")
    write_reads(c, fq)
    r = parity.run(harness, c["k"], c["kc"], c["H"], c["counters"], fq)
    parity.check_dump(r.stdout, c, os.path.join(parity.GOLD, c["name"] + ".dot.gz"))
