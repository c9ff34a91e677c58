"""GPU: k = 193..256 (Kmer<8> in pass 2, the 512-entry K1 ring above k = 224, eight-word Konnector k-mers) against the
unmodified reference built with MAX_KMER = 256 (tests/golden/kwidth256_cases.json, tests/golden/make_golden_kwidth256.py): the
assembler through the C ABI in one batch and in batches of 997 reads, with and without tiles, and through abyss-bloom-dbg; the
-g dump and the -C/-R coverage track; `abyss-bloom graph`, Konnector filters and `trim`; AdjList in every output format; the
K1 hashes against the C oracle; and k = 257 refused."""
import gzip
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "abyss_b200", "lib")
sys.path.insert(0, GOLD)
from make_golden_kwidth import blank_trace, raw_reads, reader_view, write_fastq, write_graph_inputs, write_trim_inputs  # noqa: E402
from make_golden_kwidth256 import GRAPH_FILTERS, adjlist_input  # noqa: E402
import overlap_cases as oc  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "kwidth256_cases.json")))
ASM = CASES["assembler"]
ENV = dict(os.environ, ABYSS_MAX_KMER="256")  # the command-line programs' MAX_KMER (192 without it)


@pytest.fixture(autouse=True)
def max_kmer_256(abb):
    """MAX_KMER = 256 for the C ABI, as ABYSS_MAX_KMER=256 is for the programs; back to the default afterwards"""
    abb.set_max_kmer(256)
    yield
    abb.set_max_kmer(192)


def md5(data):
    return hashlib.md5(data).hexdigest()


def sha256(data):
    return hashlib.sha256(data).hexdigest()


def _read_log(ids, codes):
    from abyss_b200.capi import READ_CODES
    return "read_id\tresult\n" + "".join(f"{i}\t{READ_CODES[c]}\n" for i, c in zip(ids, codes))


@pytest.mark.parametrize("case", ASM, ids=[c["name"] for c in ASM])
def test_assembler_c_abi(abb, monkeypatch, case):
    from abyss_b200.capi import Filter, bloom_dbg
    ids, seqs = map(list, zip(*reader_view(raw_reads(case["reads"]))))
    mask = case.get("mask", "")
    if "counters_sha256" in case:
        f = Filter.counting(case["counters"], case["H"], case["k"], case["kc"])
        f.insert_reads(seqs)
        assert sha256(f.download().tobytes()) == case["counters_sha256"]
        f.close()
    for batch in (None, 997):
        fasta, codes = bloom_dbg(ids, seqs, case["k"], case["kc"], case["H"], counters=case["counters"], batch_reads=batch,
                                 read_log=True, mask=mask)
        assert fasta.count(">") == case["n_contigs"], batch
        assert md5(fasta.encode()) == case["fasta_md5"], batch
        assert md5(_read_log(ids, codes).encode()) == case["readlog_md5"], batch
    monkeypatch.setenv("ABB_NO_TILES", "1")
    fasta, _ = bloom_dbg(ids, seqs, case["k"], case["kc"], case["H"], counters=case["counters"], mask=mask)
    assert md5(fasta.encode()) == case["fasta_md5"], "ABB_NO_TILES=1"


@pytest.mark.parametrize("case", ASM, ids=[c["name"] for c in ASM])
def test_assembler_cli(abb, tmp_path, case):
    fq, fa, log, tr, bf = (str(tmp_path / x) for x in ("reads.fq", "out.fa", "read.log", "trace.tsv", "c.bloom"))
    write_fastq(raw_reads(case["reads"]), fq)
    opt = [case["opt"]] if case["opt"] else []
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"-k{case['k']}", *opt, f"--kc={case['kc']}", f"-b{case['b']}",
                        f"-H{case['H']}", "-j1", f"--read-log={log}", "-T", tr, "-o", fa, fq], capture_output=True, env=ENV, text=True)
    assert r.returncode == 0, r.stderr
    assert md5(open(fa, "rb").read()) == case["fasta_md5"]
    assert md5(open(log, "rb").read()) == case["readlog_md5"]
    assert sha256(blank_trace(open(tr).read()).encode()) == case["trace_sha256"]
    if "counters_sha256" in case:
        r = subprocess.run([os.path.join(BIN, "abyss-bloom"), "build", "-k", str(case["k"]), "-t", "counting", f"-b{case['counters']}",
                            f"-H{case['H']}", bf, fq], capture_output=True, env=ENV, text=True)
        assert r.returncode == 0, r.stderr
        blob = open(bf, "rb").read()
        assert sha256(blob[blob.index(b"[HeaderEnd]\n") + 12:]) == case["counters_sha256"]


@pytest.mark.parametrize("case", CASES["dbg_graph"], ids=[c["name"] for c in CASES["dbg_graph"]])
def test_graphviz_dump(abb, tmp_path, case):
    fq, dot = str(tmp_path / "reads.fq"), str(tmp_path / "g.dot")
    write_fastq(raw_reads(case["reads"]), fq)
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"-k{case['k']}", f"--kc={case['kc']}", f"-b{case['b']}", f"-H{case['H']}",
                        "-g", dot, "--batch-reads=700", "-o", os.devnull, fq], capture_output=True, env=ENV, text=True)
    assert r.returncode == 0, r.stderr
    data = open(dot, "rb").read()
    assert (len(data), data.count(b"\n")) == (case["bytes"], case["lines"])
    assert sha256(data) == case["sha256"]


@pytest.mark.parametrize("case", CASES["covtrack"], ids=[c["name"] for c in CASES["covtrack"]])
def test_coverage_track(abb, tmp_path, case):
    from abyss_b200.synth import ReadSet
    from make_golden_covtrack import ref_fasta
    fq, ref, wig = str(tmp_path / "reads.fq"), str(tmp_path / "ref.fa"), str(tmp_path / "cov.wig")
    s = case["reads"]
    write_fastq(raw_reads(s), fq)
    ref_fasta(ReadSet.from_coverage(s["seed"], s["genome"], s["cov"], s["L"], s["err"]), ref)
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"-k{case['k']}", f"--kc={case['kc']}", f"-b{case['b']}", f"-H{case['H']}",
                        "-C", wig, "-R", ref, "-o", os.devnull, fq], capture_output=True, env=ENV, text=True)
    assert r.returncode == 0, r.stderr
    data = open(wig, "rb").read()
    assert (len(data), data.count(b"\n")) == (case["bytes"], case["lines"])
    assert sha256(data) == case["sha256"]


@pytest.fixture(scope="module")
def graph_work(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("kwg256"))
    write_graph_inputs(d)
    for f in GRAPH_FILTERS.values():
        r = subprocess.run([os.path.join(BIN, "abyss-bloom"), *f["args"]], cwd=d, capture_output=True, env=ENV)
        assert r.returncode == 0, r.stderr.decode()
    return d


@pytest.mark.parametrize("case", CASES["graph"], ids=[c["name"] for c in CASES["graph"]])
def test_bloom_graph_cli(graph_work, case):
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), *case["args"]], cwd=graph_work, capture_output=True, env=ENV)
    assert r.returncode == case["rc"], r.stderr.decode()
    assert r.stderr.decode() == case["stderr"]
    assert (len(r.stdout), r.stdout.count(b"\n")) == (case["bytes"], case["lines"])
    assert r.stdout == gzip.open(os.path.join(GOLD, f"kwidth256_{case['name']}.dot.gz"), "rb").read()


@pytest.fixture(scope="module")
def konnector_work(tmp_path_factory, abb):
    """every Konnector case in file order (later cases read the files earlier ones wrote)"""
    d = str(tmp_path_factory.mktemp("kwk256"))
    write_trim_inputs(d)
    out = {}
    for c in CASES["konnector"]:
        r = subprocess.run([os.path.join(BIN, "abyss-bloom"), *c["args"]], cwd=d, capture_output=True, env=ENV)
        rec = {"rc": r.returncode, "stdout_md5": md5(r.stdout), "stderr": r.stderr.decode()}
        if "file" in c and os.path.exists(os.path.join(d, c["file"])):
            rec["sha256"] = sha256(open(os.path.join(d, c["file"]), "rb").read())
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
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), *case["args"]], cwd=konnector_work[0], capture_output=True, env=ENV)
    assert r.returncode == case["rc"], r.stderr.decode()
    assert r.stderr.decode() == case["stderr"]
    assert md5(r.stdout) == case["stdout_md5"]


@pytest.mark.parametrize("case", CASES["adjlist"], ids=[c["name"] for c in CASES["adjlist"]])
def test_adjlist_cli(abb, tmp_path, case):
    t = adjlist_input(case)
    fa, exe = str(tmp_path / "in.fa"), os.path.join(BIN, "AdjList")
    oc.write_fasta(t, fa)
    r = subprocess.run([exe] + oc.command_args(t, fa), capture_output=True, env=ENV)
    assert r.returncode == 0, r.stderr.decode()
    got = oc.normalise(r.stdout, exe).replace(fa.encode(), b"IN.fa")
    assert (len(got), sha256(got)) == (case["bytes"], case["sha256"])


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
