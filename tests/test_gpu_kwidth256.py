"""GPU: k = 193..256 (Kmer<8> in pass 2, the 512-entry K1 ring above k = 224, eight-word Konnector k-mers) against the
unmodified reference built with MAX_KMER = 256 (tests/golden/kwidth256_cases.json, tests/golden/make_golden_kwidth256.py): the
assembler through the C ABI in one batch and in batches of 997 reads, with and without tiles, and through abyss-bloom-dbg; the
-g dump and the -C/-R coverage track; `abyss-bloom graph`, Konnector filters and `trim`; AdjList in every output format; the
K1 hashes against the C oracle; and k = 257 refused."""
import json
import os
import subprocess

import numpy as np
import pytest

import overlap_cases as oc
import parity
from make_golden_kwidth import write_fastq, write_graph_inputs, write_trim_inputs
from make_golden_kwidth256 import GRAPH_FILTERS, adjlist_input

pytestmark = pytest.mark.gpu
BIN = parity.BIN
CASES = json.load(open(os.path.join(parity.GOLD, "kwidth256_cases.json")))
ASM = CASES["assembler"]
ENV = dict(os.environ, ABYSS_MAX_KMER="256")  # the command-line programs' MAX_KMER (192 without it)


@pytest.fixture(autouse=True)
def max_kmer_256(abb):
    """MAX_KMER = 256 for the C ABI, as ABYSS_MAX_KMER=256 is for the programs; back to the default afterwards"""
    abb.set_max_kmer(256)
    yield
    abb.set_max_kmer(192)


@pytest.mark.parametrize("case", ASM, ids=[c["name"] for c in ASM])
def test_assembler_c_abi(abb, monkeypatch, case):
    parity.check_assembler_c_abi(case, monkeypatch)


@pytest.mark.parametrize("case", ASM, ids=[c["name"] for c in ASM])
def test_assembler_cli(abb, tmp_path, case):
    parity.check_assembler_cli(case, tmp_path, env=ENV)


@pytest.mark.parametrize("case", CASES["dbg_graph"], ids=[c["name"] for c in CASES["dbg_graph"]])
def test_graphviz_dump(abb, tmp_path, case):
    parity.check_dbg_graph(case, tmp_path, ENV)


@pytest.mark.parametrize("case", CASES["covtrack"], ids=[c["name"] for c in CASES["covtrack"]])
def test_coverage_track(abb, tmp_path, case):
    parity.check_coverage_track(case, tmp_path, ENV)


@pytest.fixture(scope="module")
def graph_work(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("kwg256"))
    write_graph_inputs(d)
    parity.build_filters(GRAPH_FILTERS.values(), d, ENV)
    return d


@pytest.mark.parametrize("case", CASES["graph"], ids=[c["name"] for c in CASES["graph"]])
def test_bloom_graph_cli(graph_work, case):
    parity.check_bloom_graph_cli(case, graph_work, os.path.join(parity.GOLD, f"kwidth256_{case['name']}.dot.gz"), ENV)


@pytest.fixture(scope="module")
def konnector_work(tmp_path_factory, abb):
    """every Konnector case in file order (later cases read the files earlier ones wrote)"""
    d = str(tmp_path_factory.mktemp("kwk256"))
    write_trim_inputs(d)
    out = {}
    for c in CASES["konnector"]:
        r = parity.abyss_bloom(*c["args"], cwd=d, env=ENV)
        rec = {"rc": r.returncode, "stdout_md5": parity.md5(r.stdout), "stderr": r.stderr.decode()}
        if "file" in c and os.path.exists(os.path.join(d, c["file"])):
            rec["sha256"] = parity.sha256(open(os.path.join(d, c["file"]), "rb").read())
        out[c["name"]] = rec
    return d, out


@pytest.mark.parametrize("case", CASES["konnector"], ids=[c["name"] for c in CASES["konnector"]])
def test_konnector_cli(konnector_work, case):
    got = konnector_work[1][case["name"]]
    assert got["rc"] == case["rc"], got["stderr"]
    assert got["stderr"] == case["stderr"]
    assert got["stdout_md5"] == case["stdout_md5"]
    if "sha256" in case:
        assert got["sha256"] == case["sha256"]


@pytest.mark.parametrize("case", CASES["trim"], ids=[c["name"] for c in CASES["trim"]])
def test_trim_cli(konnector_work, case):
    parity.check_trim_cli(case, konnector_work[0], ENV)


@pytest.mark.parametrize("case", CASES["adjlist"], ids=[c["name"] for c in CASES["adjlist"]])
def test_adjlist_cli(abb, tmp_path, case):
    t = adjlist_input(case)
    fa, exe = str(tmp_path / "in.fa"), os.path.join(BIN, "AdjList")
    oc.write_fasta(t, fa)
    r = subprocess.run([exe] + oc.command_args(t, fa), capture_output=True, env=ENV)
    assert r.returncode == 0, r.stderr.decode()
    got = oc.normalise(r.stdout, exe).replace(fa.encode(), b"IN.fa")
    assert (len(got), parity.sha256(got)) == (case["bytes"], case["sha256"])


def _reads(k):
    """reads with N, lower case, reads shorter than k, several that cross a 32-base boundary of the ring, and one longer
    than a staging buffer"""
    rng = np.random.default_rng(k)
    seqs = []
    for i in range(120):
        L = int(rng.integers(0, 1200))
        s = rng.choice(list("ACGT"), size=L)
        if i % 3 == 0 and L:
            s[rng.integers(0, L, size=max(1, L // 150))] = "N"
        if i % 5 == 0:
            s = np.char.lower(s)
        seqs.append("".join(s))
    return seqs + ["", "A" * (k - 1), "C" * k, "ACGT" * 3000]


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("k", [224, 225, 240, 256])
def test_hash_reads_vs_oracle(abb, oracle, k, masked):
    # the unmasked K1 with the 256-entry ring (k = 224) and the 512-entry one (k >= 225), and the masked K1
    mask = "".join("0" if i % 7 == 3 else "1" for i in range(k)) if masked else ""
    seqs = _reads(k)
    h0, valid, slot_offs = abb.hash_reads(k, seqs, mask)
    for i, s in enumerate(seqs):
        a, b = int(slot_offs[i]), int(slot_offs[i + 1])
        assert b - a == max(0, len(s) - k + 1), i
        v = valid[a:b].astype(bool)
        want, pos = oracle.hash_seq(s, k, 1, mask)
        assert np.nonzero(v)[0].tolist() == pos.tolist(), i
        assert (h0[a:b][v] == want[:, 0]).all(), i


def test_max_kmer_setting(abb):
    # 192 until it is raised, like the reference's default MAX_KMER; any value up to 256 after
    abb.set_max_kmer(192)
    assert abb.max_kmer() == 192
    with pytest.raises(abb.AbbError) as e:
        abb.Filter.counting(4096, 4, 193, 2)
    assert e.value.code == abb.ABB_EINVAL and "1..192" in str(e.value)
    with pytest.raises(abb.AbbError) as e:
        abb.Filter.konnector(1 << 16, 193)
    assert e.value.code == abb.ABB_EINVAL
    abb.Filter.counting(4096, 4, 192, 2).close()
    abb.set_max_kmer(224)
    abb.Filter.counting(4096, 4, 224, 2).close()
    with pytest.raises(abb.AbbError):
        abb.hash_reads(225, ["A" * 300], "")
    for bad in (0, 257):
        with pytest.raises(abb.AbbError) as e:
            abb.set_max_kmer(bad)
        assert e.value.code == abb.ABB_EINVAL
    assert abb.max_kmer() == 224
    abb.set_max_kmer(256)
    abb.Filter.counting(4096, 4, 256, 2).close()
    abb.Filter.konnector(1 << 16, 256).close()


def test_k257_refused_by_the_abi(abb):
    with pytest.raises(abb.AbbError) as e:
        abb.Filter.counting(1 << 16, 4, 257, 2)
    assert e.value.code == abb.ABB_EINVAL
    with pytest.raises(abb.AbbError) as e:
        abb.hash_reads(257, ["A" * 300], "")
    assert e.value.code == abb.ABB_EINVAL


def test_k257_refused_by_the_cli(abb, tmp_path):
    fq = str(tmp_path / "r.fq")
    write_fastq([("r0", "ACGT" * 80)], fq)
    dbg = os.path.join(BIN, "abyss-bloom-dbg")
    r = subprocess.run([dbg, "-k257", "-b1M", "-H4", "-o", os.devnull, fq], capture_output=True, text=True, env=ENV)
    assert r.returncode != 0
    assert "must be <= 256" in r.stderr
    # without ABYSS_MAX_KMER the programs keep the default MAX_KMER of 192
    env = {x: v for x, v in os.environ.items() if x != "ABYSS_MAX_KMER"}
    r = subprocess.run([dbg, "-k193", "-b1M", "-H4", "-o", os.devnull, fq], capture_output=True, text=True, env=env)
    assert r.returncode != 0
    assert "must be <= 192" in r.stderr
    assert "[<=192]" in subprocess.run([dbg, "--help"], capture_output=True, text=True, env=env).stdout
    assert "[<=256]" in subprocess.run([dbg, "--help"], capture_output=True, text=True, env=ENV).stdout
    for bad in ("257", "0", "x"):
        r = subprocess.run([dbg, "-k25", "-b1M", "-H4", "-o", os.devnull, fq], capture_output=True, text=True,
                           env=dict(env, ABYSS_MAX_KMER=bad))
        assert r.returncode != 0 and "ABYSS_MAX_KMER" in r.stderr
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), "build", "-k193", "-b64K", str(tmp_path / "o.bloom"), fq], capture_output=True,
                       text=True, env=env)
    assert r.returncode != 0
