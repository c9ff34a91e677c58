"""GPU: pass-2 tiles under a spaced seed (-K, --qr-seed, -s).  Markers are enumerated by the canonical hash of the full k-mer
(k_find_markers over an unmasked K1 pass), tiles are named by it (tile_key, abb_walk.cuh), and the walks splice them: every
case must give the unmodified reference's bytes (tests/golden/spaced_tiles_cases.json, make_golden_spaced_tiles.py, and the
spaced-seed cases of mask_cases.json), with tiles built and spliced, with ABB_NO_TILES=1, through the C ABI and through
abyss-bloom-dbg, and with a tile store that fills up."""
import json
import os

import pytest

import parity
from make_golden_spaced_tiles import raw_reads

pytestmark = pytest.mark.gpu
GOLD = parity.GOLD
SPACED = json.load(open(os.path.join(GOLD, "spaced_tiles_cases.json")))
BY_NAME = {c["name"]: c for c in SPACED}
MASK = json.load(open(os.path.join(GOLD, "mask_cases.json")))


def _run(case, ids, seqs):
    """(fasta, read log, stats) of the reads through the C ABI on a fresh filter and assembler"""
    fasta, codes, st = parity.assemble(case, ids, seqs)
    return fasta, parity.read_log(ids, codes), st


@pytest.mark.parametrize("case", SPACED, ids=[c["name"] for c in SPACED])
def test_c_abi(abb, monkeypatch, case):
    ids, seqs = map(list, zip(*raw_reads(case["reads"])))
    fasta, log, st = _run(case, ids, seqs)
    parity.check_unitigs(case, fasta, log)
    # tiles were built under the mask and walks spliced them
    assert st.markers > 0 and st.tiles > 0, (st.markers, st.tiles)
    assert (st.untiled_markers, st.dropped_tiles) == (0, 0)
    monkeypatch.setenv("ABB_NO_TILES", "1")
    fasta, log, st = _run(case, ids, seqs)
    parity.check_unitigs(case, fasta, log)
    assert st.markers == 0 and st.tiles == 0


CLI = [(c, [c["opt"]]) for c in SPACED] + [(BY_NAME["sp_cfg1_k80_K32"], ["-s", BY_NAME["sp_cfg1_k80_K32"]["mask"]])]


@pytest.mark.parametrize("case,opt", CLI, ids=[c["name"] + ("-s" if o[0] == "-s" else "") for c, o in CLI])
def test_cli(abb, tmp_path, case, opt):
    parity.check_assembler_cli(case, tmp_path, raw_reads(case["reads"]), opt)


def _mask_reads(case):
    import gzip
    from abyss_b200.synth import ReadSet
    if case["reads"].endswith(".gz"):
        ids, seqs = [], []
        with gzip.open(os.path.join(GOLD, case["reads"]), "rt") as f:
            for line in f:
                (ids if line[0] == ">" else seqs).append(line[1:].strip() if line[0] == ">" else line.strip())
        return ids, seqs
    c = {c["name"]: c for c in json.load(open(os.path.join(GOLD, "e2e_cases.json")))}[case["reads"]]
    rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
    return [rs.read_id(i) for i in range(rs.n)], [a.tobytes().decode() for a in rs.ascii(0, rs.n)]


@pytest.mark.parametrize("case", MASK, ids=[c["name"] for c in MASK])
def test_mask_cases_build_tiles(abb, case):
    # the short-read, circular, hairpin and tandem spaced-seed cases: tiles are built; where a splice would skip an ER_CYCLE
    # the repeat check sends the read back to the vertex-by-vertex walk, and the bytes stay the reference's
    ids, seqs = _mask_reads(case)
    fasta, log, st = _run(case, ids, seqs)
    assert fasta == open(os.path.join(GOLD, case["name"] + ".fa")).read()
    if case.get("readlog"):
        assert log == open(os.path.join(GOLD, case["name"] + ".readlog.tsv")).read()
    assert st.markers > 0 and st.tiles > 0


def test_full_tile_store_under_mask(abb):
    # abb_assembler_reset keeps the tile store sized for the first, small assembly; the 5 Mbp genome of sp_m1_k80_K32 then has
    # more new markers than the store's marker list holds (about 19 500 against 16 384) and more tile bytes than its pool, so
    # markers go untiled and tiles are dropped, and those markers are walked vertex by vertex with the same bytes
    from abyss_b200.capi import Assembler, Filter, pack_reads
    from abyss_b200.synth import ReadSet
    case = BY_NAME["sp_m1_k80_K32"]
    ids, seqs = map(list, zip(*raw_reads(case["reads"])))
    f = Filter.counting(case["counters"], case["H"], case["k"], case["kc"], mask=case["mask"])
    a = Assembler(f, read_log=True)
    rs = ReadSet(7, 4000, 800, 150, 0.0)
    small = pack_reads([x.tobytes().decode() for x in rs.ascii(0, rs.n)])
    f.insert_reads(small)
    a.assemble([rs.read_id(i) for i in range(rs.n)], small)
    assert a.stats().markers > 0  # the first assembly sized the store
    f.clear()
    a.reset()
    reads = pack_reads(seqs)
    f.insert_reads(reads)
    fasta, codes = a.assemble(ids, reads)
    st = a.stats()
    a.close()
    f.close()
    parity.check_unitigs(case, fasta, parity.read_log(ids, codes))
    assert st.untiled_markers > 0 and st.dropped_tiles > 0, (st.markers, st.tiles, st.dropped_tiles, st.untiled_markers)
