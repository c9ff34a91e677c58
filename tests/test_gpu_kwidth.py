"""GPU: pass 1 and pass 2 at every k-mer width the kernels are compiled for (Kmer<KW>, KW = 1, 2, 3, 4 and 6 words, k up to
192) against the unmodified reference (tests/golden/kwidth_cases.json, tests/golden/make_golden_kwidth.py): the assembler
through the C ABI in one batch and in batches of 997 reads, with and without tiles, and through abyss-bloom-dbg (FASTA, read
log, -T trace, counters); the -g dump and the -C/-R coverage track; `abyss-bloom graph` and `abyss-bloom trim`; and the masked
K1 hashes against the C oracle."""
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
from make_golden_kwidth import (GRAPH_FILTERS, TRIM_FILTERS, blank_trace, raw_reads, reader_view, write_fastq,  # noqa: E402
                                write_graph_inputs, write_trim_inputs)

CASES = json.load(open(os.path.join(GOLD, "kwidth_cases.json")))
ASM = CASES["assembler"]


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
                        f"-H{case['H']}", "-j1", f"--read-log={log}", "-T", tr, "-o", fa, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert md5(open(fa, "rb").read()) == case["fasta_md5"]
    assert md5(open(log, "rb").read()) == case["readlog_md5"]
    assert sha256(blank_trace(open(tr).read()).encode()) == case["trace_sha256"]
    if "counters_sha256" in case:
        r = subprocess.run([os.path.join(BIN, "abyss-bloom"), "build", "-k", str(case["k"]), "-t", "counting", f"-b{case['counters']}",
                            f"-H{case['H']}", bf, fq], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        blob = open(bf, "rb").read()
        assert sha256(blob[blob.index(b"[HeaderEnd]\n") + 12:]) == case["counters_sha256"]


@pytest.mark.parametrize("case", CASES["dbg_graph"], ids=[c["name"] for c in CASES["dbg_graph"]])
def test_graphviz_dump(abb, tmp_path, case):
    fq, dot = str(tmp_path / "reads.fq"), str(tmp_path / "g.dot")
    write_fastq(raw_reads(case["reads"]), fq)
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"-k{case['k']}", f"--kc={case['kc']}", f"-b{case['b']}", f"-H{case['H']}",
                        "-g", dot, "--batch-reads=700", "-o", os.devnull, fq], capture_output=True, text=True)
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
                        "-C", wig, "-R", ref, "-o", os.devnull, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    data = open(wig, "rb").read()
    assert (len(data), data.count(b"\n")) == (case["bytes"], case["lines"])
    assert sha256(data) == case["sha256"]


@pytest.fixture(scope="module")
def graph_work(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("kwg"))
    write_graph_inputs(d)
    for f in GRAPH_FILTERS.values():
        r = subprocess.run([os.path.join(BIN, "abyss-bloom"), *f["args"]], cwd=d, capture_output=True)
        assert r.returncode == 0, r.stderr.decode()
    return d


@pytest.mark.parametrize("case", CASES["graph"], ids=[c["name"] for c in CASES["graph"]])
def test_bloom_graph_cli(graph_work, case):
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), *case["args"]], cwd=graph_work, capture_output=True)
    assert r.returncode == case["rc"], r.stderr.decode()
    assert r.stderr.decode() == case["stderr"]
    assert (len(r.stdout), r.stdout.count(b"\n")) == (case["bytes"], case["lines"])
    assert r.stdout == gzip.open(os.path.join(GOLD, f"kwidth_{case['name']}.dot.gz"), "rb").read()


@pytest.fixture(scope="module")
def trim_work(tmp_path_factory, abb):
    d = str(tmp_path_factory.mktemp("kwt"))
    write_trim_inputs(d)
    for f in TRIM_FILTERS:
        r = subprocess.run([os.path.join(BIN, "abyss-bloom"), *f["args"]], cwd=d, capture_output=True)
        assert r.returncode == 0, r.stderr.decode()
    return d


@pytest.mark.parametrize("case", CASES["trim"], ids=[c["name"] for c in CASES["trim"]])
def test_trim_cli(trim_work, case):
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), *case["args"]], cwd=trim_work, capture_output=True)
    assert r.returncode == case["rc"], r.stderr.decode()
    assert r.stderr.decode() == case["stderr"]
    assert md5(r.stdout) == case["stdout_md5"]


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
