"""CPU: the pass-2 graph logic (abyss_b200/csrc/abb_walk.cuh -- the SAME templates the CUDA kernels instantiate) run by
the single-lane host harness tests/host_walk against the reference's golden unitigs: plain k-mers with and without
tiles, spaced seeds (-K / --qr-seed patterns, 'N' columns of short paths, the full-k-mer orientation rule of
RollingBloomDBGVertex::compare), hairpins and tandem repeats.  The GPU tests check the kernels; this one lets the
traversal logic be verified on a machine without a GPU."""
import gzip
import json
import os
import re
import subprocess

import pytest

from abyss_b200.synth import ReadSet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def host_walk(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("hw") / "host_walk")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wno-unknown-pragmas", "-o", exe, os.path.join(ROOT, "tests", "host_walk", "host_walk.cpp"),
                    os.path.join(ROOT, "oracle", "abyss_oracle.c")], check=True, capture_output=True)
    return exe


def _reads(tmp_path, reads):
    if reads.endswith(".gz"):
        out = tmp_path / reads[:-3]
        out.write_bytes(gzip.open(os.path.join(GOLD, reads), "rb").read())
        return str(out)
    c = {c["name"]: c for c in json.load(open(os.path.join(GOLD, "e2e_cases.json")))}[reads]
    rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
    out = str(tmp_path / (reads + ".fq"))
    rs.write_fastq(out)
    return out


def _run(exe, k, kc, H, counters, trim, reads, mask="", tiles=False):
    env = dict(os.environ, HOST_WALK_MASK=mask)
    env.pop("HOST_WALK_TILES", None)
    if tiles:
        env["HOST_WALK_TILES"] = "1"
    r = subprocess.run([exe, str(k), str(kc), str(H), str(counters), str(trim), reads], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    return r.stdout


@pytest.mark.parametrize("tiles", [False, True])
def test_plain_kmers(host_walk, tmp_path, tiles):
    c = {c["name"]: c for c in json.load(open(os.path.join(GOLD, "e2e_cases.json")))}["e2e_g10k_k25_small"]
    got = _run(host_walk, c["k"], c["kc"], c["H"], c["counters"], c["k"], _reads(tmp_path, c["name"]), tiles=tiles)
    assert got == open(os.path.join(GOLD, c["name"] + ".fa")).read()


MASK_CASES = json.load(open(os.path.join(GOLD, "mask_cases.json")))


@pytest.mark.parametrize("case", [c for c in MASK_CASES if c["name"] in
                                  ("mask_g20k_qr11", "mask_g10k_K5", "mask_tandem_qr15", "mask_hairpin_K10", "mask_circ_qr17")],
                         ids=lambda c: c["name"])
def test_spaced_seeds(host_walk, tmp_path, case):
    got = _run(host_walk, case["k"], case["kc"], case["H"], case["counters"], case["k"], _reads(tmp_path, case["reads"]),
               mask=case["mask"])
    want = open(os.path.join(GOLD, case["name"] + ".fa")).read()
    assert got.count(">") == case["n_contigs"]
    assert got == want


def test_marker_set_full(host_walk):
    # marker_set_insert (abb_walk.cuh, the insert of k_find_markers) on 64-, 128- and 4096-entry sets filled past capacity:
    # a full set answers "no room" instead of probing forever, no key is ever fresh twice, and keys stored earlier are found
    r = subprocess.run([host_walk, "markerset"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("cap 64 fresh 64 no_room 192 refound 64 twice 0\n")


def _cyc_reads(tmp_path, case):
    b = case["b"]
    n = int(b / 1.125 + 0.5)  # counters_for_budget
    return _reads(tmp_path, case["reads"]), n if n % 64 == 0 else n + 64 - n % 64


@pytest.mark.parametrize("name", ["e2e_g10k_k25_small", "cyc_circ_k25"])
@pytest.mark.parametrize("seed", [1, 7])
def test_dropped_tiles_same_output(host_walk, tmp_path, name, seed):
    # what a full tile store leaves behind: markers missing one of their four tiles, markers missing all four.  Walks pass
    # them vertex by vertex and the unitigs stay the reference's
    if name.startswith("cyc_"):
        c = {c["name"]: c for c in json.load(open(os.path.join(GOLD, "cyc_cases.json")))}[name]
        reads, counters = _cyc_reads(tmp_path, c)
        trim = c["trim"]
    else:
        c = {c["name"]: c for c in json.load(open(os.path.join(GOLD, "e2e_cases.json")))}[name]
        reads, counters, trim = _reads(tmp_path, name), c["counters"], c["k"]
    env = dict(os.environ, HOST_WALK_MASK="", HOST_WALK_TILES="1", HOST_WALK_DROP_TILES=str(seed))
    r = subprocess.run([host_walk, str(c["k"]), str(c["kc"]), str(c["H"]), str(counters), str(trim), reads], capture_output=True,
                       text=True, env=env)
    assert r.returncode == 0, r.stderr
    m = re.search(r"(\d+) dropped \((\d+) markers lost one tile, (\d+) all four\)", r.stderr)
    assert m and int(m.group(2)) > 0 and int(m.group(3)) > 0, r.stderr
    assert r.stdout == open(os.path.join(GOLD, name + ".fa")).read()
