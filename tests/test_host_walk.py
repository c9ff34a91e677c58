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

import parity
from abyss_b200.synth import ReadSet

GOLD = parity.GOLD
host_walk = parity.harness("host_walk", "tests/host_walk/host_walk.cpp", parity.ORACLE)


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


@pytest.mark.parametrize("tiles", [False, True])
def test_plain_kmers(host_walk, tmp_path, tiles):
    c = {c["name"]: c for c in json.load(open(os.path.join(GOLD, "e2e_cases.json")))}["e2e_g10k_k25_small"]
    got, _, _ = parity.run_host_walk(host_walk, c, _reads(tmp_path, c["name"]), tiles=tiles)
    assert got == open(os.path.join(GOLD, c["name"] + ".fa"), "rb").read()


MASK_CASES = json.load(open(os.path.join(GOLD, "mask_cases.json")))


@pytest.mark.parametrize("case", [c for c in MASK_CASES if c["name"] in
                                  ("mask_g20k_qr11", "mask_g10k_K5", "mask_tandem_qr15", "mask_hairpin_K10", "mask_circ_qr17")],
                         ids=lambda c: c["name"])
def test_spaced_seeds(host_walk, tmp_path, case):
    got, _, _ = parity.run_host_walk(host_walk, case, _reads(tmp_path, case["reads"]))
    want = open(os.path.join(GOLD, case["name"] + ".fa"), "rb").read()
    assert got.count(b">") == case["n_contigs"]
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
    fasta, _, err = parity.run_host_walk(host_walk, dict(c, counters=counters, trim=trim), reads, drop=seed)
    m = re.search(r"(\d+) dropped \((\d+) markers lost one tile, (\d+) all four\)", err)
    assert m and int(m.group(2)) > 0 and int(m.group(3)) > 0, err
    assert fasta == open(os.path.join(GOLD, name + ".fa"), "rb").read()
