"""GPU: the C++ command-line programs (abyss-bloom-dbg, abyss-bloom build) over libabyssb200 produce
the same bytes as the unmodified reference binaries (committed goldens)."""
import hashlib
import json
import os
import subprocess

import pytest

import parity
from abyss_b200.synth import ReadSet

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "abyss_b200", "lib")


@pytest.fixture(scope="module")
def cases(tmp_path_factory, abb):
    d = tmp_path_factory.mktemp("cli")
    out = {}
    for c in json.load(open(os.path.join(ROOT, "tests", "golden", "e2e_cases.json"))):
        rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
        fq = str(d / (c["name"] + ".fq"))
        rs.write_fastq(fq)
        out[c["name"]] = (c, fq, d)
    return out


@pytest.mark.parametrize("name", ["e2e_g20k_k32", "e2e_g30k_k64", "e2e_g10k_k25_small"])
def test_abyss_bloom_dbg_cli(cases, tmp_path, name):
    c, fq, _ = cases[name]
    fasta, log, _ = parity.bloom_dbg_cli(c, fq, tmp_path, "--batch-reads=1500")
    assert fasta == open(os.path.join(parity.GOLD, name + ".fa"), "rb").read()
    assert log == open(os.path.join(parity.GOLD, name + ".readlog.tsv"), "rb").read()


@pytest.mark.parametrize("name", ["e2e_g20k_k32", "e2e_g30k_k64", "e2e_g10k_k25_small"])
def test_trace_file_identical_to_reference(cases, tmp_path, name):
    # -T FILE: one ContigRecord row per contig handed to outputContig (seed k-mer, both extension lengths and result
    # codes, redundancy, contig id) -- the K4 parity channel SURVEY.md 7-9 names.  The reference leaves `length`
    # uninitialised for redundant rows; the golden generator and this test blank that cell.
    import gzip
    c, fq, _ = cases[name]
    _, _, trace = parity.bloom_dbg_cli(c, fq, tmp_path, "--batch-reads=1500")
    g = os.path.join(parity.GOLD, name + ".trace.tsv")
    want = gzip.open(g + ".gz", "rt").read() if os.path.exists(g + ".gz") else open(g).read()
    assert parity.blank_trace(trace) == want


def test_checkpoints(cases):
    # --checkpoint=N: PREFIX.dbg.bloom / .visited.bloom / .counters.tsv / .contigs.fa byte-identical to the files the
    # reference's createCheckpoint writes (BloomDBG/Checkpoint.h:31-127; goldens from tests/golden/make_golden_checkpoint.py),
    # and a run that finds them resumes there and ends with the FASTA of the uninterrupted run.  (The reference's own
    # resume path is broken in 2.3.10 -- it emits 35 000 k-length contigs on this input -- so resume is checked against
    # the uninterrupted output, which is what resumeFromCheckpoint is meant to reproduce.)
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "checkpoint_case.json")))
    c, fq, d = cases[g["case"]]
    pfx = str(d / "ck")
    fa = str(d / "ck_out.fa")
    cmd = [os.path.join(BIN, "abyss-bloom-dbg"), f"-k{c['k']}", f"--kc={c['kc']}", f"-b{c['b']}", f"-H{c['H']}",
           f"--checkpoint={g['reads_per_checkpoint']}", "--keep-checkpoint", f"--checkpoint-prefix={pfx}", "-o", fa, fq]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    golden_fa = open(os.path.join(ROOT, "tests", "golden", g["case"] + ".fa")).read()
    assert open(fa).read() == golden_fa
    sha = lambda p: hashlib.sha256(open(p, "rb").read()).hexdigest()
    assert open(pfx + ".counters.tsv").read() == g["counters_tsv"]
    assert sha(pfx + ".dbg.bloom") == g["dbg_bloom_sha256"]
    assert sha(pfx + ".visited.bloom") == g["visited_bloom_sha256"]
    assert sha(pfx + ".contigs.fa") == g["contigs_fa_sha256"]
    # resume from the state after 3000 of the 4000 reads
    fa2 = str(d / "ck_resumed.fa")
    r = subprocess.run(cmd[:-3] + ["-v", "-o", fa2, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "Resuming from last checkpoint" in r.stderr and "Advancing to read index 3000" in r.stderr
    assert open(fa2).read() == golden_fa
    # without --keep-checkpoint the files are removed at the end (removeCheckpointData)
    cmd3 = [x for x in cmd if x != "--keep-checkpoint"]
    r = subprocess.run(cmd3, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert not os.path.exists(pfx + ".dbg.bloom") and not os.path.exists(pfx + ".counters.tsv")


def test_abyss_bloom_build_and_prebuilt(cases):
    c, fq, d = cases["e2e_g20k_k32"]
    bf = str(d / "counting.bloom")
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), "build", "-k", str(c["k"]), "-t", "counting", f"-b{c['counters']}",
                        f"-H{c['H']}", bf, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert hashlib.sha256(open(bf, "rb").read()).hexdigest() == c["counting_file_sha256"]
    # -i FILE: prebuiltBloomAssembly gives the same unitigs as the de novo run
    fa = str(d / "prebuilt.fa")
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"--kc={c['kc']}", "-i", bf, "-o", fa, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert open(fa).read() == open(os.path.join(ROOT, "tests", "golden", "e2e_g20k_k32.fa")).read()
    # abyss-bloom info on both file formats: size / popcount / FPR lines (printBloomStats, bloom.cc:433-441)
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), "info", bf], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert f"Bloom size (bits): {c['counters']}" in r.stderr and f"Bloom popcount (bits): {c['counters_nonzero']}" in r.stderr
    # rolling-hash cascading filter, 2 levels: file identical to the reference's
    rh = str(d / "rh.bloom")
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), "build", "-k", str(c["k"]), "-t", "rolling-hash", "-l", "2", f"-H{c['H']}",
                        f"-b{c['rolling_hash_l2_b']}", rh, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert hashlib.sha256(open(rh, "rb").read()).hexdigest() == c["rolling_hash_l2_file_sha256"]


def test_rolling_hash_levels_not_multiple_of_16_bytes(cases):
    # -b 1000 over two levels: each level rounds up to 504 bytes, not a multiple of 16, and -v reports the population of
    # the last one; file identical to the reference's (tests/golden/make_golden_hashnum.py)
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "hashnum_cases.json")))["rolling_hash"]
    c, fq, d = cases[g["reads"]]
    rh = str(d / "rh_b1000.bloom")
    r = subprocess.run([os.path.join(BIN, "abyss-bloom"), "build", "-k", str(c["k"]), "-t", "rolling-hash", "-l", str(g["levels"]),
                        f"-H{g['H']}", f"-b{g['b']}", "-v", rh, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    blob = open(rh, "rb").read()
    assert len(blob) == g["file_bytes"]
    assert hashlib.sha256(blob).hexdigest() == g["file_sha256"]


def test_cli_errors(cases):
    c, fq, d = cases["e2e_g20k_k32"]
    exe = os.path.join(BIN, "abyss-bloom-dbg")
    r = subprocess.run([exe, "-k32", fq], capture_output=True, text=True)
    assert r.returncode != 0 and "missing mandatory option `-b'" in r.stderr
    r = subprocess.run([exe, "-b1M", fq], capture_output=True, text=True)
    assert r.returncode != 0 and "missing mandatory option `-k'" in r.stderr
    r = subprocess.run([exe, "-b1M", "-k32"], capture_output=True, text=True)
    assert r.returncode != 0 and "missing input file arguments" in r.stderr


@pytest.mark.parametrize("name", ["mask_g20k_K20", "mask_g20k_qr11", "mask_g10k_K5"])
def test_abyss_bloom_dbg_cli_spaced_seed(cases, name):
    # -K / --qr-seed through the option parser (bloom-dbg.cc:420-460, initGlobals :215-233)
    mc = {c["name"]: c for c in json.load(open(os.path.join(ROOT, "tests", "golden", "mask_cases.json")))}[name]
    _, fq, d = cases[mc["reads"]]
    fa = str(d / (name + ".fa"))
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"-k{mc['k']}", mc["opt"], f"--kc={mc['kc']}", f"-b{mc['b']}", f"-H{mc['H']}",
                        "-v", "-o", fa, fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert f"Using spaced seed {mc['mask']}" in r.stderr
    assert open(fa).read() == open(os.path.join(ROOT, "tests", "golden", name + ".fa")).read()
    # the same pattern given literally with -s
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"-k{mc['k']}", "-s", mc["mask"], f"--kc={mc['kc']}", f"-b{mc['b']}",
                        f"-H{mc['H']}", fq], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stdout == open(os.path.join(ROOT, "tests", "golden", name + ".fa")).read()


def test_abyss_bloom_dbg_cli_bad_seed(cases):
    _, fq, _ = cases["e2e_g20k_k32"]
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), "-k32", "--qr-seed=16", "-b1M", fq], capture_output=True, text=True)
    assert r.returncode != 0 and "spaced seed must begin and end with '1's" in r.stderr  # the reference's message for this k


def test_coverage_track(cases, tmp_path):
    # -C FILE -R REF: the 0/1 "k-mer is solid" WIG track over a reference (writeCovTrack, bloom-dbg.h:1280-1334), one GPU query
    # per batch of reference records (abb_contains_reads); golden = the unmodified reference (make_golden_covtrack.py)
    from make_golden_covtrack import ref_fasta
    c, fq, d = cases["e2e_g20k_k32"]
    rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
    ref = str(tmp_path / "ref.fa")
    ref_fasta(rs, ref)
    wig = str(tmp_path / "cov.wig")
    parity.bloom_dbg_cli(c, fq, tmp_path, "-C", wig, "-R", ref)
    assert open(wig).read() == open(os.path.join(ROOT, "tests", "golden", "covtrack_g20k_k32.wig")).read()
    # -C without -R is a usage error, as in the reference (bloom-dbg.cc:512-515)
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), "-k32", "-b1M", "-C", wig, fq], capture_output=True, text=True)
    assert r.returncode != 0 and "you must specify a reference" in r.stderr


def test_graphviz_dump(tmp_path, abb):
    # -g FILE: the breadth-first GraphViz dump of the Bloom filter de Bruijn graph (outputGraph, bloom-dbg.h:1171-1242): the
    # traversal order is the reference's, the Bloom lookups are GPU batches (abb_contains_reads, abb_successors); goldens from
    # the unmodified reference (make_golden_graph.py)
    from make_golden_graph import write_reads
    for c in json.load(open(os.path.join(parity.GOLD, "graph_cases.json"))):
        fq = str(tmp_path / (c["name"] + ".fq"))
        write_reads(c, fq)
        dot = str(tmp_path / (c["name"] + ".dot"))
        parity.bloom_dbg_cli(c, fq, tmp_path, "-g", dot, "--batch-reads=700")
        parity.check_dump(open(dot, "rb").read(), c, os.path.join(parity.GOLD, c["name"] + ".dot.gz"))
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), "-k21", "-K5", "-b64k", "-g", dot, fq], capture_output=True, text=True)
    assert r.returncode != 0 and "spaced seed" in r.stderr


def test_successors_c_abi(abb):
    # abb_successors against a filter that holds exactly the k-mers of one sequence: every vertex has one out-edge, the
    # chain runs to max_chain and reproduces the sequence; the canonical hashes equal those of abb_hash_reads
    import ctypes as C
    import numpy as np
    rng = np.random.default_rng(5)
    k = 31
    seq = "".join("ACGT"[i] for i in rng.integers(0, 4, 400))
    f = abb.Filter.counting(1 << 22, 4, k, 1)
    f.insert_reads([seq])
    h0, valid, _ = abb.hash_reads(k, [seq])
    lib = abb.load()
    info = (abb.SuccInfo * 64)()
    ln = (C.c_uint * 1)()
    self_h = (C.c_uint64 * 1)()
    km = seq[:k].encode()
    abb.check(lib.abb_successors(f.handle, km, 1, 64, info, ln, self_h))
    assert self_h[0] == int(h0[0]) and ln[0] == 64
    for s in range(64):
        b = "ACGT".index(seq[k + s])
        assert info[s].mask == 1 << b, (s, info[s].mask)
        assert info[s].hash[b] == int(h0[s + 1])
    # a k-mer the filter has never seen: no out-edges (up to false positives, none at this load), chain length 1
    abb.check(lib.abb_successors(f.handle, b"A" * k, 1, 64, info, ln, self_h))
    assert ln[0] == 1 and info[0].mask == 0
    f.close()
