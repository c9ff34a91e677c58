"""GPU parity for pass 2 when its bounded tile scratch fills up: the marker set, the new-marker list, the tile records and
pool, and K4's record buffer.  Whatever does not fit gets no tiles and is walked vertex by vertex, so the unitigs must still
be the reference's -j1 output byte for byte (tests/golden/make_golden_pass2_capacity.py, pass2_capacity.json), and the two
counters of abb_assembly_stats say that the full-store paths ran.

  g12m_k64         1.6 M reads of a 12 Mbp genome: on a fresh handle nothing overflows (one batch and 200 000-read
                   batches); on a handle whose tile store was sized by a small first assembly the marker set, the
                   new-marker list and the tile records all fill up.
  overload_k25_H1  a far too small filter: half of all counters reach kc, so the marker set of a fresh handle overflows
                   and every read yields many short unitigs."""
import json
import os

import numpy as np
import pytest

import parity
from abyss_b200.synth import ReadSet

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {c["name"]: c for c in json.load(open(os.path.join(ROOT, "tests", "golden", "pass2_capacity.json")))}


def reads_of(c, parts):
    """(ids, (bases, offsets)) of the reads of `parts` in file order, as the golden script writes them"""
    from abyss_b200.capi import fixed_length_reads
    ids, arrays = [], []
    for p in parts:
        rs = ReadSet(p["seed"], p["genome"], p["n_reads"], c["L"], c["err"])
        ids += [f"{p['prefix']}{i}" for i in range(rs.n)]
        arrays.append(rs.ascii(0, rs.n))
    return ids, fixed_length_reads(np.concatenate(arrays))


def check_golden(c, fasta, codes, ids):
    parity.check_unitigs(c, fasta, parity.read_log(ids, codes))
    lens = [len(s) for s in fasta.split("\n")[1::2]]
    assert (sum(lens), max(lens)) == (c["bases"], c["longest"])


@pytest.fixture(scope="module")
def g12m():
    c = CASES["g12m_k64"]
    return c, reads_of(c, c["parts"])


@pytest.mark.parametrize("batch", [None, 200_000])
def test_g12m_fresh_handle(abb, g12m, batch):
    # the store sized from this filter holds every marker and tile: nothing is left untiled, also across batch boundaries
    c, (ids, reads) = g12m
    fasta, codes, st = parity.assemble(c, ids, reads, batch)
    check_golden(c, fasta, codes, ids)
    assert st.markers > 0 and st.tiles > 0
    assert (st.untiled_markers, st.dropped_tiles) == (0, 0)


def test_g12m_reused_handle_overflows_tile_store(abb, g12m):
    # abb_assembler_reset keeps the tile store sized for a 10 kbp genome (a 32 768-entry marker set); the 12 Mbp genome has
    # more distinct solid markers than that, so the set fills up, the new-marker list is cut and the tile records run out
    from abyss_b200.capi import Filter, Assembler
    c, (ids, reads) = g12m
    assert c["solid_markers"] > c["mset_reset"]
    f = Filter.counting(c["counters"], c["H"], c["k"], c["kc"])
    a = Assembler(f, read_log=True)
    first_ids, first = reads_of(c, [c["first"]])
    f.insert_reads(first)
    a.assemble(first_ids, first)
    assert a.stats().markers > 0  # the first assembly sized the store
    f.clear()
    a.reset()
    f.insert_reads(reads)
    fasta, codes = a.assemble(ids, reads)
    st = a.stats()
    a.close()
    f.close()
    check_golden(c, fasta, codes, ids)
    assert st.untiled_markers > 0 and st.dropped_tiles > 0


def test_overload_filter(abb, tmp_path):
    # -k25 -H1 -b256k over 213 333 reads: half of all counters reach kc, so about 53 000 distinct solid markers meet a
    # 32 768-entry marker set.  Through the C ABI and once through abyss-bloom-dbg
    from abyss_b200.capi import Filter, Assembler
    c = CASES["overload_k25_H1"]
    assert c["solid_markers"] > c["mset_fresh"]
    ids, reads = reads_of(c, c["parts"])
    f = Filter.counting(c["counters"], c["H"], c["k"], c["kc"])
    f.insert_reads(reads)
    assert parity.sha256(f.download().tobytes()) == c["counters_sha256"]
    a = Assembler(f, read_log=True)
    fasta, codes = a.assemble(ids, reads)
    st = a.stats()
    a.close()
    f.close()
    check_golden(c, fasta, codes, ids)
    assert st.untiled_markers > 0
    # no counter sees a single round: many more unitigs than 8 per speculated read is what makes K4 outgrow its record
    # buffer of max(8 * reads, 4096) records and run again (run_extend)
    assert st.contigs_tried > 8 * st.speculated_reads and st.contigs_tried > 4096
    fq = str(tmp_path / "reads.fq")
    bases, offs = reads
    with open(fq, "wb") as out:
        for i, rid in enumerate(ids):
            s = bases[int(offs[i]):int(offs[i + 1])].tobytes()
            out.write(b"@" + rid.encode() + b"\n" + s + b"\n+\n" + b"I" * len(s) + b"\n")
    fasta, log, _ = parity.bloom_dbg_cli(c, fq, tmp_path)
    parity.check_unitigs(c, fasta, log)
