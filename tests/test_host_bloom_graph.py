"""CPU: `abyss-bloom graph` -- the product's traversal (abyss_b200/host/bloom_graph.h) and the per-lane neighbour probes the CUDA
kernel runs (kmer_hash_part, nbr_lane, nbr_mask of abyss_b200/csrc/abb_graph.cuh), driven by the single-thread harness
tests/host_bloom_graph on filters the C oracle rebuilds -- writes the bytes of the unmodified reference's dump on every case of
tests/golden/bloom_graph_cases.json (tests/golden/make_golden_bloom_graph.py) that prints one."""
import json
import os

import pytest

import parity
from make_golden_bloom_graph import RECIPES, write_inputs

CASES = [c for c in json.load(open(os.path.join(parity.GOLD, "bloom_graph_cases.json"))) if c["harness"]]
host_bloom_graph = parity.harness("host_bloom_graph", "tests/host_bloom_graph/host_bloom_graph.cpp", parity.ORACLE)


def harness_args(args):
    """the command line of `abyss-bloom graph` as the harness takes it: K DEPTH FILTER, then -R / -f / -a / -A pairs"""
    k, depth, rest, pos = None, None, [], []
    it = iter(args[1:])
    long = {"--node-attr": "-a", "--fasta-attr": "-a", "--bloom-attr": "-A", "--root": "-R", "--root-fasta": "-f", "--depth": "-d"}
    for a in it:
        if a == "-v":
            continue
        if a.startswith("--"):
            name, _, val = a.partition("=")
            opt, val = long[name], val or next(it)
        elif a.startswith("-"):
            opt, val = a[:2], a[2:] or next(it)
        else:
            pos.append(a)
            continue
        if opt == "-k":
            k = val
        elif opt == "-d":
            depth = val
        else:
            rest += [opt, ",".join(map(str, RECIPES[val.split(":", 1)[1]])) if opt == "-A" else val]
            if opt == "-A":
                rest[-1] = val.split(":", 1)[0] + ":" + rest[-1]
    return [k, depth or k, ",".join(map(str, RECIPES[pos[0]]))] + rest


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("bg"))
    write_inputs(d, large=any(c["name"] == "large" for c in CASES))
    return d


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_bloom_graph_dump(host_bloom_graph, work, case):
    r = parity.run(host_bloom_graph, *harness_args(case["args"]), cwd=work)
    parity.check_dump(r.stdout, case, os.path.join(parity.GOLD, f"bloom_graph_{case['name']}.dot.gz"))


def test_harness_args():
    assert harness_args(["graph", "-v", "-k25", "-d", "3", "-R", "ACGT", "--node-attr=c:x.fa", "-A", "s:sub25_H1.bloom", "g25_H2.bloom"]) == [
        "25", "3", "2,1,2097152,g.fq", "-R", "ACGT", "-a", "c:x.fa", "-A", "s:1,1,2097152,sub.fq"]
