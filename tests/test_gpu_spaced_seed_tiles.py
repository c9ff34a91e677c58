"""GPU: pass-2 tiles under a spaced seed (-K, --qr-seed, -s).  Markers are enumerated by the canonical hash of the full k-mer
(k_find_markers over an unmasked K1 pass), tiles are named by it (tile_key, abb_walk.cuh), and the walks splice them: every
case must give the unmodified reference's bytes (tests/golden/spaced_tiles_cases.json, make_golden_spaced_tiles.py, and the
spaced-seed cases of mask_cases.json), with tiles built and spliced, with ABB_NO_TILES=1, through the C ABI and through
abyss-bloom-dbg, and with a tile store that fills up."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "abyss_b200", "lib")
sys.path.insert(0, GOLD)
from make_golden_kwidth import blank_trace, write_fastq  # noqa: E402
from make_golden_spaced_tiles import raw_reads  # noqa: E402

SPACED = json.load(open(os.path.join(GOLD, "spaced_tiles_cases.json")))
BY_NAME = {c["name"]: c for c in SPACED}
MASK = json.load(open(os.path.join(GOLD, "mask_cases.json")))


def md5(data):
    return hashlib.md5(data).hexdigest()


def sha256(data):
    return hashlib.sha256(data).hexdigest()


def _read_log(ids, codes):
    from abyss_b200.capi import READ_CODES
    return "read_id\tresult\n" + "".join(f"{i}\t{READ_CODES[c]}\n" for i, c in zip(ids, codes))


def _assemble(a, ids, bases, offs):
    out = []
    for seed, seq, cov in a.process_reads((bases, offs)):
        out.append(f">{len(out)} {len(seq)} {cov} read:{ids[seed]}\n{seq}\n")
    return "".join(out), _read_log(ids, a.read_results())


def _run(case, ids, seqs):
    """(fasta, read log, stats) of the reads through the C ABI on a fresh filter and assembler"""
    from abyss_b200.capi import Assembler, Filter, pack_reads
    bases, offs = pack_reads(seqs)
    f = Filter.counting(case["counters"], case["H"], case["k"], case["kc"], mask=case["mask"])
    f.insert_reads((bases, offs))
    a = Assembler(f, read_log=True)
    fasta, log = _assemble(a, ids, bases, offs)
    st = a.stats()
    a.close()
    f.close()
    return fasta, log, st


@pytest.mark.parametrize("case", SPACED, ids=[c["name"] for c in SPACED])
def test_c_abi(abb, monkeypatch, case):
    ids, seqs = map(list, zip(*raw_reads(case["reads"])))
    fasta, log, st = _run(case, ids, seqs)
    assert fasta.count(">") == case["n_contigs"]
    assert md5(fasta.encode()) == case["fasta_md5"]
    assert md5(log.encode()) == case["readlog_md5"]
    # tiles were built under the mask and walks spliced them
    assert st.markers > 0 and st.tiles > 0, (st.markers, st.tiles)
    assert (st.untiled_markers, st.dropped_tiles) == (0, 0)
    monkeypatch.setenv("ABB_NO_TILES", "1")
    fasta, log, st = _run(case, ids, seqs)
    assert md5(fasta.encode()) == case["fasta_md5"], "ABB_NO_TILES=1"
    assert md5(log.encode()) == case["readlog_md5"], "ABB_NO_TILES=1"
    assert st.markers == 0 and st.tiles == 0


def _cli(case, opt, reads, tmp_path):
    fa, log, tr = (str(tmp_path / x) for x in ("out.fa", "read.log", "trace.tsv"))
    r = subprocess.run([os.path.join(BIN, "abyss-bloom-dbg"), f"-k{case['k']}", *opt, f"--kc={case['kc']}", f"-b{case['b']}",
                        f"-H{case['H']}", "-j1", f"--read-log={log}", "-T", tr, "-o", fa, reads], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return open(fa, "rb").read(), open(log, "rb").read(), open(tr).read()


CLI = [(c, [c["opt"]]) for c in SPACED] + [(BY_NAME["sp_cfg1_k80_K32"], ["-s", BY_NAME["sp_cfg1_k80_K32"]["mask"]])]


@pytest.mark.parametrize("case,opt", CLI, ids=[c["name"] + ("-s" if o[0] == "-s" else "") for c, o in CLI])
def test_cli(abb, tmp_path, case, opt):
    fq = str(tmp_path / "reads.fq")
    write_fastq(raw_reads(case["reads"]), fq)
    fasta, log, trace = _cli(case, opt, fq, tmp_path)
    assert md5(fasta) == case["fasta_md5"]
    assert md5(log) == case["readlog_md5"]
    assert sha256(blank_trace(trace).encode()) == case["trace_sha256"]


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
    _assemble(a, [rs.read_id(i) for i in range(rs.n)], *small)
    assert a.stats().markers > 0  # the first assembly sized the store
    f.clear()
    a.reset()
    bases, offs = pack_reads(seqs)
    f.insert_reads((bases, offs))
    fasta, log = _assemble(a, ids, bases, offs)
    st = a.stats()
    a.close()
    f.close()
    assert md5(fasta.encode()) == case["fasta_md5"]
    assert md5(log.encode()) == case["readlog_md5"]
    assert st.untiled_markers > 0 and st.dropped_tiles > 0, (st.markers, st.tiles, st.dropped_tiles, st.untiled_markers)
