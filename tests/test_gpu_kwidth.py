"""GPU: pass 1 and pass 2 at every k-mer width the kernels are compiled for (Kmer<KW>, KW = 1, 2, 3, 4 and 6 words, k up to
192) against the unmodified reference (tests/golden/kwidth_cases.json, tests/golden/make_golden_kwidth.py): the assembler
through the C ABI in one batch and in batches of 997 reads, with and without tiles, and through abyss-bloom-dbg (FASTA, read
log, -T trace, counters); the -g dump and the -C/-R coverage track; `abyss-bloom graph` and `abyss-bloom trim`; and the masked
K1 hashes against the C oracle."""
import json
import os

import numpy as np
import pytest

import parity
from make_golden_kwidth import GRAPH_FILTERS, TRIM_FILTERS, write_graph_inputs, write_trim_inputs

pytestmark = pytest.mark.gpu
CASES = json.load(open(os.path.join(parity.GOLD, "kwidth_cases.json")))
ASM = CASES["assembler"]


@pytest.mark.parametrize("case", ASM, ids=[c["name"] for c in ASM])
def test_assembler_c_abi(abb, monkeypatch, case):
    parity.check_assembler_c_abi(case, monkeypatch)


@pytest.mark.parametrize("case", ASM, ids=[c["name"] for c in ASM])
def test_assembler_cli(abb, tmp_path, case):
    parity.check_assembler_cli(case, tmp_path)


@pytest.mark.parametrize("case", CASES["dbg_graph"], ids=[c["name"] for c in CASES["dbg_graph"]])
def test_graphviz_dump(abb, tmp_path, case):
    parity.check_dbg_graph(case, tmp_path)


@pytest.mark.parametrize("case", CASES["covtrack"], ids=[c["name"] for c in CASES["covtrack"]])
def test_coverage_track(abb, tmp_path, case):
    parity.check_coverage_track(case, tmp_path)


@pytest.fixture(scope="module")
def graph_work(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("kwg"))
    write_graph_inputs(d)
    parity.build_filters(GRAPH_FILTERS.values(), d)
    return d


@pytest.mark.parametrize("case", CASES["graph"], ids=[c["name"] for c in CASES["graph"]])
def test_bloom_graph_cli(graph_work, case):
    parity.check_bloom_graph_cli(case, graph_work, os.path.join(parity.GOLD, f"kwidth_{case['name']}.dot.gz"))


@pytest.fixture(scope="module")
def trim_work(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("kwt"))
    write_trim_inputs(d)
    parity.build_filters(TRIM_FILTERS, d)
    return d


@pytest.mark.parametrize("case", CASES["trim"], ids=[c["name"] for c in CASES["trim"]])
def test_trim_cli(trim_work, case):
    parity.check_trim_cli(case, trim_work)


def _masks(k):
    """a symmetric seed (two k-mers of k / 3 at the ends) and an asymmetric one (a '0' every 7th column from 3 on)"""
    third = k // 3
    sym = "1" * third + "0" * (k - 2 * third) + "1" * third
    asym = "".join("0" if i % 7 == 3 else "1" for i in range(k))
    assert sym == sym[::-1] and asym != asym[::-1] and asym[0] == asym[-1] == "1"
    return {"symmetric": sym, "asymmetric": asym}


@pytest.mark.parametrize("kind", ["symmetric", "asymmetric"])
@pytest.mark.parametrize("k", [97, 128, 129, 160, 192])
def test_masked_hash_reads_vs_oracle(abb, oracle, k, kind):
    # the masked K1 (k_hash_reads_masked) at four and six words: canonical hash and valid windows of every read, with N, lower
    # case, reads shorter than k and one longer than a staging buffer
    mask = _masks(k)[kind]
    rng = np.random.default_rng(k * 2 + len(kind))
    seqs = []
    for i in range(80):
        L = int(rng.integers(0, 900))
        s = rng.choice(list("ACGT"), size=L)
        if i % 3 == 0 and L:
            s[rng.integers(0, L, size=max(1, L // 150))] = "N"
        if i % 5 == 0:
            s = np.char.lower(s)
        seqs.append("".join(s))
    seqs += ["", "A" * (k - 1), "ACGT" * 3000]
    h0, valid, slot_offs = abb.hash_reads(k, seqs, mask)
    for i, s in enumerate(seqs):
        a, b = int(slot_offs[i]), int(slot_offs[i + 1])
        v = valid[a:b].astype(bool)
        want, pos = oracle.hash_seq(s, k, 1, mask)
        assert np.nonzero(v)[0].tolist() == pos.tolist(), i
        assert (h0[a:b][v] == want[:, 0]).all(), i
