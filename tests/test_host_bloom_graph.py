"""CPU: `abyss-bloom graph` -- the product's traversal (abyss_b200/host/bloom_graph.h) and the per-lane neighbour probes the CUDA
kernel runs (kmer_hash_part, nbr_lane, nbr_mask of abyss_b200/csrc/abb_graph.cuh), driven by the single-thread harness
tests/host_bloom_graph on filters the C oracle rebuilds -- writes the bytes of the unmodified reference's dump on every case of
tests/golden/bloom_graph_cases.json (tests/golden/make_golden_bloom_graph.py) that prints one."""
import gzip
import hashlib
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, GOLD)
from make_golden_bloom_graph import RECIPES, write_inputs  # noqa: E402

CASES = [c for c in json.load(open(os.path.join(GOLD, "bloom_graph_cases.json"))) if c["harness"]]


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
    d = tmp_path_factory.mktemp("bg")
    exe = str(d / "host_bloom_graph")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wno-unknown-pragmas", "-pthread", "-o", exe,
                    os.path.join(ROOT, "tests", "host_bloom_graph", "host_bloom_graph.cpp"), os.path.join(ROOT, "oracle", "abyss_oracle.c")],
                   check=True, capture_output=True)
    write_inputs(str(d), large=any(c["name"] == "large" for c in CASES))
    return str(d), exe


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_bloom_graph_dump(work, case):
    d, exe = work
    r = subprocess.run([exe, *harness_args(case["args"])], cwd=d, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert (len(r.stdout), r.stdout.count(b"\n")) == (case["bytes"], case["lines"])
    full = os.path.join(GOLD, f"bloom_graph_{case['name']}.dot.gz")
    if os.path.exists(full):
        assert r.stdout == gzip.open(full, "rb").read()
    assert hashlib.sha256(r.stdout).hexdigest() == case["sha256"]


def test_harness_args():
    assert harness_args(["graph", "-v", "-k25", "-d", "3", "-R", "ACGT", "--node-attr=c:x.fa", "-A", "s:sub25_H1.bloom", "g25_H2.bloom"]) == [
        "25", "3", "2,1,2097152,g.fq", "-R", "ACGT", "-a", "c:x.fa", "-A", "s:1,1,2097152,sub.fq"]
