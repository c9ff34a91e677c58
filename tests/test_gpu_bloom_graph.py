"""GPU: `abyss-bloom graph` over libabyssb200 prints the stdout, stderr and exit status of the unmodified reference on every case of
tests/golden/bloom_graph_cases.json (tests/golden/make_golden_bloom_graph.py), on filters our own `abyss-bloom build -t
rolling-hash` makes, and refuses as documented where the reference asserts; abb_graph_neighbors agrees with the C oracle's
bit-filter contains() on random and read-derived k-mers, with and without attribute filters, across its internal pieces."""
import gzip
import hashlib
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
EXE = os.path.join(ROOT, "abyss_b200", "lib", "abyss-bloom")
sys.path.insert(0, GOLD)
from make_golden_bloom_graph import FILTERS, LARGE_FILTERS, OTHER_FILTERS, rc, write_inputs  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "bloom_graph_cases.json")))
LARGE = any(c["name"] == "large" for c in CASES)


def _run(d, args):
    return subprocess.run([EXE, *args], cwd=d, capture_output=True)


@pytest.fixture(scope="module")
def work(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("bloom_graph"))
    write_inputs(d, LARGE)
    for f in [x["args"] for x in FILTERS + (LARGE_FILTERS if LARGE else [])] + OTHER_FILTERS:
        r = _run(d, f)
        assert r.returncode == 0, r.stderr.decode()
    return d


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_graph_cli(work, case):
    r = _run(work, case["args"])
    assert r.returncode == case["rc"], r.stderr.decode()
    assert r.stderr.decode() == case["stderr"]
    assert (len(r.stdout), r.stdout.count(b"\n")) == (case["bytes"], case["lines"])
    full = os.path.join(GOLD, f"bloom_graph_{case['name']}.dot.gz")
    if os.path.exists(full):
        assert r.stdout == gzip.open(full, "rb").read()
    assert hashlib.sha256(r.stdout).hexdigest() == case["sha256"]


def _bits(oracle, k, H, mbits, seqs):
    bits = np.zeros(mbits // 8, dtype=np.uint8)
    for s in seqs:
        oracle.bf_load(bits, [s.encode()], k, H)
    return bits


def _canonical(oracle, kmer, k):
    return int(oracle.hash_seq(kmer, k, 1)[0][0, 0])


def _oracle_contains(oracle, bits, k, H, kmer):
    h = np.ascontiguousarray(oracle.hash_seq(kmer, k, H)[0][0])
    return oracle.lib.abo_bf_contains(bits.ctypes.data, bits.size * 8, h.ctypes.data, H)


@pytest.mark.parametrize("k,H,n_attr,n", [(25, 2, 0, 3000), (32, 4, 3, 2000), (64, 3, 32, 1500), (31, 1, 2, 150000), (25, 5, 2, 2000),
                                         (33, 6, 4, 1500), (27, 7, 1, 1500), (29, 8, 3, 1500), (40, 20, 5, 800), (25, 32, 2, 400)])
def test_graph_neighbors_against_the_oracle(abb, oracle, k, H, n_attr, n):
    rng = random.Random(k * 100 + n_attr)
    genome = "".join(rng.choice("ACGT") for _ in range(4000))
    mbits = 1 << 16
    g = _bits(oracle, k, H, mbits, [genome])
    # attribute filter 0 has as many hashes as the graph (the most probes a lane makes), the others fewer
    attr_specs = [(H if a == 0 else 1 + a % H, mbits * (1 + a % 3), genome[a * 100:a * 100 + 400]) for a in range(n_attr)]
    attr_bits = [_bits(oracle, k, h, m, [s]) for h, m, s in attr_specs]
    fg = abb.Filter.bits(mbits, H, k)
    fg.upload(g)
    fa = []
    for (h, m, _), b in zip(attr_specs, attr_bits):
        f = abb.Filter.bits(m, h, k)
        f.upload(b)
        fa.append(f)
    # read-derived k-mers (in the graph, mostly), their reverse complements, lower case, and random ones
    kmers = []
    while len(kmers) < n:
        i = rng.randrange(len(genome) - k)
        s = genome[i:i + k]
        kmers.append([s, rc(s), s.lower(), "".join(rng.choice("ACGT") for _ in range(k))][len(kmers) % 4])
    got = abb.graph_neighbors(fg, kmers, fa)
    check = range(n) if n <= 3000 else sorted(rng.sample(range(n), 3000)) + list(range(n - 50, n))
    for i in check:
        u = kmers[i].upper()
        nb = [u[1:] + b for b in "ACGT"] + [b + u[:-1] for b in "ACGT"]
        o = got[i]
        assert o["self"] == _canonical(oracle, u, k)
        assert o["hash"] == [_canonical(oracle, v, k) for v in nb], i
        assert o["mask"] == sum(_oracle_contains(oracle, g, k, H, v) << j for j, v in enumerate(nb)), i
        assert o["attr"] == sum(_oracle_contains(oracle, b, k, h, u) << a for a, ((h, _, _), b) in enumerate(zip(attr_specs, attr_bits))), i
    for f in fa + [fg]:
        f.close()


def test_graph_neighbors_refusals(abb):
    g = abb.Filter.bits(1 << 16, 2, 25)
    ok = abb.graph_neighbors(g, ["A" * 25], [])
    assert ok[0]["mask"] == 0
    for bad_graph in (abb.Filter.counting(1 << 16, 2, 25), abb.Filter.bits(1 << 16, 2, 25, mask="1" * 12 + "0" + "1" * 12)):
        with pytest.raises(abb.AbbError) as e:
            abb.graph_neighbors(bad_graph, ["A" * 25])
        assert e.value.code == abb.ABB_ESTATE
        bad_graph.close()
    for bad_attr in (abb.Filter.bits(1 << 16, 3, 25), abb.Filter.counting(1 << 16, 1, 25)):
        with pytest.raises(abb.AbbError) as e:
            abb.graph_neighbors(g, ["A" * 25], [bad_attr])
        assert e.value.code == abb.ABB_ESTATE
        bad_attr.close()
    g.close()
