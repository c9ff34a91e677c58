"""CPU: pass-2 tiles under a spaced seed (-K, --qr-seed), through the single-lane harness tests/host_walk/host_walk_spaced.cpp,
which instantiates the same abb_walk.cuh templates as the kernels and enumerates markers as k_find_markers does.  Markers and tiles are named by the full k-mer (tile_key), so splicing them must
give the reference's bytes on every spaced-seed golden: the short-read, circular, hairpin and tandem cases of
mask_cases.json, the k = 128 to 192 cases of kwidth_cases.json and the larger cases of spaced_tiles_cases.json
(tests/golden/make_golden_spaced_tiles.py), including a don't-care adversary on which tiles named by the vertex identity
would splice the wrong continuation.  Dropping a seeded subset of the tiles, as a full tile store does, changes nothing.
The 1 M-read case sp_m1_k80_K32 takes the single-lane harness minutes; it runs on the GPU only
(tests/test_gpu_spaced_seed_tiles.py)."""
import gzip
import json
import os
import re

import pytest

import parity  # first: it puts tests/golden on the path
import make_golden_kwidth as kwidth
import make_golden_spaced_tiles as spaced
from abyss_b200.synth import ReadSet
from parity import md5

GOLD = parity.GOLD

MASK = json.load(open(os.path.join(GOLD, "mask_cases.json")))
KWIDTH = [c for c in json.load(open(os.path.join(GOLD, "kwidth_cases.json")))["assembler"] if c["opt"]]
SPACED = [c for c in json.load(open(os.path.join(GOLD, "spaced_tiles_cases.json"))) if c["name"] != "sp_m1_k80_K32"]
E2E = {c["name"]: c for c in json.load(open(os.path.join(GOLD, "e2e_cases.json")))}
host_walk = parity.harness("host_walk_spaced", "tests/host_walk/host_walk_spaced.cpp", parity.ORACLE)


def _write_reads(tmp_path, suite, case):
    """the case's reads as a FASTQ/FASTA file, and the golden FASTA bytes, md5 of the golden read log (or None)"""
    out = str(tmp_path / "reads.fq")
    if suite == "mask":
        if case["reads"].endswith(".gz"):
            out = str(tmp_path / case["reads"][:-3])
            open(out, "wb").write(gzip.open(os.path.join(GOLD, case["reads"]), "rb").read())
        else:
            e = E2E[case["reads"]]
            ReadSet.from_coverage(e["seed"], e["genome"], e["cov"], e["L"], e["err"]).write_fastq(out)
        fa = open(os.path.join(GOLD, case["name"] + ".fa"), "rb").read()
        log = os.path.join(GOLD, case["name"] + ".readlog.tsv")
        return out, md5(fa), md5(open(log, "rb").read()) if case.get("readlog") else None
    if suite == "kwidth":
        kwidth.write_fastq(kwidth.reader_view(kwidth.raw_reads(case["reads"])), out)
    else:
        kwidth.write_fastq(spaced.raw_reads(case["reads"]), out)
    return out, case["fasta_md5"], case["readlog_md5"]


def _walk(exe, tmp_path, case, reads, drop=None):
    log = str(tmp_path / "read.log")
    r = parity.run(exe, case["k"], case["kc"], case["H"], case["counters"], case.get("trim", case["k"]), case["mask"], reads, log,
                   *([] if drop is None else [drop]))
    err = r.stderr.decode()
    m = re.search(r"(\d+) tiles from (\d+) markers.*\n.*?(\d+) tile splices, (\d+) serial fallbacks", err)
    assert m, err
    return r.stdout, open(log, "rb").read(), dict(tiles=int(m.group(1)), markers=int(m.group(2)), splices=int(m.group(3))), err


def _longest_kmers(fasta, k):
    return max((len(l) - k + 1 for l in fasta.decode().splitlines() if l and l[0] != ">"), default=0)


CASES = [("mask", c) for c in MASK] + [("kwidth", c) for c in KWIDTH] + [("spaced", c) for c in SPACED]
IDS = [c["name"] for _, c in CASES]


@pytest.mark.parametrize("suite,case", CASES, ids=IDS)
def test_tiles_under_mask(host_walk, tmp_path, suite, case):
    reads, fasta_md5, log_md5 = _write_reads(tmp_path, suite, case)
    fasta, log, st, err = _walk(host_walk, tmp_path, case, reads)
    assert md5(fasta) == fasta_md5
    if log_md5:
        assert md5(log) == log_md5
    assert st["markers"] > 0 and st["tiles"] > 0, err
    # a unitig of 1 000 k-mers passes about four markers: tiles must have been spliced
    if _longest_kmers(fasta, case["k"]) >= 1000:
        assert st["splices"] > 0, err
    if suite == "spaced" and case["name"].startswith(("sp_cfg1", "sp_lr")):
        assert st["markers"] >= 1000, err  # the tile store does real work


@pytest.mark.parametrize("suite,case", [x for x in CASES if x[0] != "kwidth"], ids=[c["name"] for s, c in CASES if s != "kwidth"])
def test_dropped_tiles_under_mask(host_walk, tmp_path, suite, case):
    # what a full tile store leaves behind under a mask: markers missing one or all four tiles are passed vertex by vertex
    reads, fasta_md5, _ = _write_reads(tmp_path, suite, case)
    fasta, _, _, err = _walk(host_walk, tmp_path, case, reads, drop=5)
    m = re.search(r"(\d+) dropped \((\d+) markers lost one tile, (\d+) all four\)", err)
    assert m and int(m.group(1)) > 0, err
    assert md5(fasta) == fasta_md5


def test_adversary_shares_identity_not_key():
    # the adversary's two k-mers are one vertex to the reference and a marker by identity, but they are different full k-mers
    c = {c["name"]: c for c in SPACED}["sp_adversary_k64_K24"]
    _, x, x2 = spaced.adversary_genome(c["reads"])
    assert x != x2
    assert spaced.identity(x, c["mask"]) == spaced.identity(x2, c["mask"])
    assert spaced.identity(x, c["mask"]) & spaced.MARKER_MASK == 0
    assert c["pre"]["x_in"] >= 1 and c["pre"]["x2_in"] >= 1
