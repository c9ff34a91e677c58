"""CPU: the overlap-graph join logic (abyss_b200/csrc/abb_overlap.cuh -- the SAME per-item functions the CUDA kernels
call) and the product's AdjList command line and graph writers (abyss_b200/host/adjlist_main.h), run by the
single-thread harness tests/host_overlap, against the unmodified reference AdjList: committed goldens
(tests/golden/make_golden_overlap.py, tests/golden/make_golden_ref_live.py)."""
import gzip
import json
import os
import subprocess

import pytest

import overlap_cases as oc
import parity
import ref_golden

GOLD = parity.GOLD
harness = parity.harness("AdjList", "tests/host_overlap/host_overlap.cpp")


def run_case(exe, case, tmp_path):
    fa = str(tmp_path / (case["name"] + ".fa"))
    oc.write_fasta(case, fa)
    r = subprocess.run([exe] + oc.command_args(case, fa), capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    return oc.normalise(r.stdout, exe).replace(fa.encode(), b"IN.fa")


def test_goldens(harness, tmp_path):
    want = json.load(open(os.path.join(GOLD, "overlap_cases.json")))
    cases = oc.all_cases()
    assert sorted(c["name"] for c in cases) == sorted(want)
    for c in cases:
        got = run_case(harness, c, tmp_path)
        assert len(got) == want[c["name"]]["bytes"], c["name"]
        assert parity.sha256(got) == want[c["name"]]["sha256"], c["name"]
        full = os.path.join(GOLD, "overlap_" + c["name"] + ".txt")
        if os.path.exists(full):
            assert got == open(full, "rb").read()


def live_cases():
    return [oc.fuzz_case(seed) for seed in range(1000, 1120)]


def test_live_against_reference(harness, tmp_path):
    want = ref_golden.load("adjlist")
    for c in live_cases():
        got = run_case(harness, c, tmp_path)
        assert ref_golden.matches(got, want[c["name"]]), (c["name"], c["k"], c["m"], c["args"])


def test_errors(harness, tmp_path):
    fa = str(tmp_path / "n.fa")
    open(fa, "w").write(">0 12 3\nACGTNACGTACG\n>1 12 3\nACGTACGTACGA\n")
    r = subprocess.run([harness, "-k6", fa], capture_output=True, text=True)
    assert r.returncode != 0 and "nucleotide" in r.stderr  # the reference's Kmer constructor aborts on the N
    open(fa, "w").write(">0\nACGT\n")
    r = subprocess.run([harness, "-k6", fa], capture_output=True, text=True)
    assert r.returncode != 0 and "not longer than k-1" in r.stderr
    open(fa, "w").write(">a\nACGTACGTAA\n>a\nACGTACGTAC\n")
    r = subprocess.run([harness, "-k6", fa], capture_output=True, text=True)
    assert r.returncode != 0 and "duplicate ID" in r.stderr
    r = subprocess.run([harness, fa], capture_output=True, text=True)
    assert r.returncode != 0 and "missing -k,--kmer option" in r.stderr


REAL_UNITIG_SETS = [(32, 0, "--adj"), (32, 20, "--dot"), (48, 30, "--gfa1"), (64, 50, "--gfa2"), (96, 50, "--sam"), (40, 25, "--asqg")]


@pytest.mark.parametrize("k,m,fmt", REAL_UNITIG_SETS)
def test_real_unitig_sets(harness, tmp_path, k, m, fmt):
    # the pipeline of bin/abyss-pe on config 1 (SURVEY.md 8d: 53 333 x 150 bp reads of a 200 kbp genome): the reference's own
    # unitig FASTA (tips, branches, blunt ends from coverage gaps; tests/golden/unitigs_cfg1_k*.fa.gz) into AdjList
    fa = str(tmp_path / "unitigs-1.fa")
    with gzip.open(os.path.join(GOLD, f"unitigs_cfg1_k{k}.fa.gz")) as src, open(fa, "wb") as dst:
        dst.write(src.read())
    n = sum(1 for line in open(fa) if line.startswith(">"))
    assert n > 10
    b = subprocess.run([harness, f"-k{k}", f"-m{m}", fmt, fa], capture_output=True)
    assert b.returncode == 0, b.stderr.decode()
    got = oc.normalise(b.stdout, harness).replace(fa.encode(), b"IN.fa")
    assert len(got) > 0
    assert ref_golden.matches(got, ref_golden.load("real_unitigs")[f"k{k}_m{m}_{fmt[2:]}"])


def alias_runs(d):
    """(arguments, standard input) of the runs of test_option_aliases_and_stdin, input files written under d"""
    c = oc.tiled_case(21, 20000, 31, 20)
    half = len(c["records"]) // 2
    a_fa, b_fa = os.path.join(d, "a.fa"), os.path.join(d, "b.fa")
    oc.write_fasta(dict(c, records=c["records"][:half]), a_fa)
    oc.write_fasta(dict(c, records=c["records"][half:]), b_fa)
    both = (open(a_fa).read() + open(b_fa).read()).encode()
    return [(["--kmer=31", "--min-overlap=20", "--gv", a_fa, b_fa], None), (["-k31", "-m0", "--gfa", a_fa, b_fa], None),
            (["-k", "31", "-m", "25", "--SS", "--adj"], both), (["-k31", "--no-SS", "--asqg", "-"], both)]


def test_option_aliases_and_stdin(harness, tmp_path):
    # --gv = --dot, --gfa = --gfa1, -m0 = k-1, long options, several input files, contigs on standard input
    want = ref_golden.load("adjlist_aliases")
    runs = alias_runs(str(tmp_path))
    assert len(runs) == len(want)
    for (args, stdin), w in zip(runs, want):
        got = subprocess.run([harness] + args, input=stdin, capture_output=True)
        assert got.returncode == 0, got.stderr.decode()
        assert ref_golden.matches(got.stdout.replace(str(tmp_path).encode(), b"TMP"), w), args
