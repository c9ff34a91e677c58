"""GPU: pass 2 on long reads of 5 to 80 kbp against the unmodified reference (tests/golden/longread_cases.json,
tests/golden/make_golden_longreads.py): through the C ABI in one batch, in batches of 7 reads and without tiles, and through
abyss-bloom-dbg (FASTA, read log, -T trace, counters).  The cases reach what short reads never do: the whole-grid replay of
unitigs of 2^15 k-mers and more in K5, the read-level loops of K2, K3 and K5 past 1 024 k-mers, and the rerun of K4 when its
record buffer overflows.  abb_assembly_stats shows that the round structure those paths need was reached."""
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
from make_golden_kwidth import blank_trace  # noqa: E402
from make_golden_longreads import raw_reads, write_fasta, write_fastq  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "longread_cases.json")))
BY_NAME = {c["name"]: c for c in CASES}


def md5(data):
    return hashlib.md5(data).hexdigest()


def sha256(data):
    return hashlib.sha256(data).hexdigest()


def _read_log(ids, codes):
    from abyss_b200.capi import READ_CODES
    return "read_id\tresult\n" + "".join(f"{i}\t{READ_CODES[c]}\n" for i, c in zip(ids, codes))


def _assemble(case, ids, seqs, batch=None):
    """abyss-bloom-dbg through the C ABI (capi.bloom_dbg), keeping the assembler's statistics: (fasta, read codes, stats)"""
    from abyss_b200.capi import Assembler, Filter, pack_reads
    bases, offs = pack_reads(seqs)
    f = Filter.counting(case["counters"], case["H"], case["k"], case["kc"])
    f.insert_reads((bases, offs))
    a = Assembler(f, read_log=True)
    out, codes = [], []
    step = batch or len(seqs)
    for lo in range(0, len(seqs), step):
        hi = min(len(seqs), lo + step)
        sub = (bases[int(offs[lo]):int(offs[hi])], (offs[lo:hi + 1] - offs[lo]).astype(np.uint64))
        for seed, seq, cov in a.process_reads(sub):
            out.append(f">{len(out)} {len(seq)} {cov} read:{ids[seed]}\n{seq}\n")
        codes.append(a.read_results())
    st = a.stats()
    a.close()
    f.close()
    return "".join(out), np.concatenate(codes), st


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_assembler_c_abi(abb, monkeypatch, case):
    ids, seqs = map(list, zip(*raw_reads(case["reads"])))
    f = abb.Filter.counting(case["counters"], case["H"], case["k"], case["kc"])
    f.insert_reads(seqs)
    assert sha256(f.download().tobytes()) == case["counters_sha256"]
    f.close()
    for batch in (None, 7):
        fasta, codes, st = _assemble(case, ids, seqs, batch)
        assert fasta.count(">") == case["n_contigs"], batch
        assert md5(fasta.encode()) == case["fasta_md5"], batch
        assert md5(_read_log(ids, codes).encode()) == case["readlog_md5"], batch
        if batch is None and case["name"] == "lr_dense_k64":
            # every candidate in one round, and more records than the first K4 record buffer holds: it was rerun
            assert st.rounds == 1, (st.rounds, st.speculated_reads)
            assert st.contigs_tried > max(8 * st.speculated_reads, 4096), (st.contigs_tried, st.speculated_reads)
        if batch is None and case["name"].startswith("lr_repeats"):
            # speculated reads of more than 1 024 k-mers that the replay found covered
            assert st.wasted_reads > 0
    monkeypatch.setenv("ABB_NO_TILES", "1")
    fasta, codes, _ = _assemble(case, ids, seqs)
    assert md5(fasta.encode()) == case["fasta_md5"], "ABB_NO_TILES=1"
    assert md5(_read_log(ids, codes).encode()) == case["readlog_md5"], "ABB_NO_TILES=1"


def _cli(case, reads, tmp_path):
    fa, log, tr = (str(tmp_path / x) for x in ("out.fa", "read.log", "trace.tsv"))
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"-k{case['k']}", f"--kc={case['kc']}", f"-b{case['b']}", f"-H{case['H']}",
                        "-j1", f"--read-log={log}", "-T", tr, "-o", fa, reads], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return open(fa, "rb").read(), open(log, "rb").read(), open(tr).read()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_assembler_cli(abb, tmp_path, case):
    fq, bf = str(tmp_path / "reads.fq"), str(tmp_path / "c.bloom")
    write_fastq(raw_reads(case["reads"]), fq)
    fasta, log, trace = _cli(case, fq, tmp_path)
    assert md5(fasta) == case["fasta_md5"]
    assert md5(log) == case["readlog_md5"]
    assert sha256(blank_trace(trace).encode()) == case["trace_sha256"]
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), "build", "-k", str(case["k"]), "-t", "counting", f"-b{case['counters']}",
                        f"-H{case['H']}", bf, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    blob = open(bf, "rb").read()
    assert sha256(blob[blob.index(b"[HeaderEnd]\n") + 12:]) == case["counters_sha256"]


def test_assembler_cli_wrapped_fasta(abb, tmp_path):
    """the same long reads as FASTA records wrapped at 60 columns give the same bytes"""
    case = BY_NAME["lr_repeats_k64"]
    fa = str(tmp_path / "reads.fa")
    write_fasta(raw_reads(case["reads"]), fa)
    fasta, log, trace = _cli(case, fa, tmp_path)
    assert md5(fasta) == case["fasta_md5"]
    assert md5(log) == case["readlog_md5"]
    assert sha256(blank_trace(trace).encode()) == case["trace_sha256"]
