"""GPU parity for pass 2 (classify, visited, extend, replay) through the C ABI: the unitig FASTA
must equal the reference's -j1 output byte for byte (committed goldens from the unmodified
reference, tests/golden/make_golden.py), and the per-read outcome log must match --read-log."""
import json
import os

import pytest

import parity
from abyss_b200.synth import ReadSet

pytestmark = pytest.mark.gpu


def load_case(golden_dir, name):
    cases = {c["name"]: c for c in json.load(open(os.path.join(golden_dir, "e2e_cases.json")))}
    c = cases[name]
    rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
    return c, rs


@pytest.mark.parametrize("name", ["e2e_g20k_k32", "e2e_g30k_k64", "e2e_g10k_k25_small"])
@pytest.mark.parametrize("batch", [None, 997])
def test_fasta_identical_to_reference(abb, golden_dir, name, batch):
    from abyss_b200.capi import fixed_length_reads, bloom_dbg
    c, rs = load_case(golden_dir, name)
    ids = [rs.read_id(i) for i in range(rs.n)]
    fasta, codes = bloom_dbg(ids, fixed_length_reads(rs.ascii(0, rs.n)), c["k"], c["kc"], c["H"], counters=c["counters"],
                             batch_reads=batch, read_log=True)
    want = open(os.path.join(golden_dir, name + ".fa")).read()
    assert fasta.count(">") == c["n_contigs"]
    assert fasta == want
    assert parity.read_log(ids, codes) == open(os.path.join(golden_dir, name + ".readlog.tsv")).read()


def test_mixed_reads_edge_cases(abb, golden_dir):
    # short reads, reads with N, lower case, empty batch mixed in: must not disturb the others
    from abyss_b200.capi import bloom_dbg, READ_CODES
    c, rs = load_case(golden_dir, "e2e_g20k_k32")
    seqs = [a.tobytes().decode() for a in rs.ascii(0, 600)]
    seqs[10] = seqs[10][:20]
    seqs[11] = seqs[11][:70] + "N" + seqs[11][71:]
    seqs[12] = ""
    seqs[13] = seqs[13].lower()
    ids = [f"q{i}" for i in range(len(seqs))]
    fasta, codes = bloom_dbg(ids, seqs, 32, 2, 4, counters=c["counters"], read_log=True)
    assert READ_CODES[codes[10]] == "SHORTER_THAN_K"
    assert READ_CODES[codes[11]] == "NON_ACGT"
    assert READ_CODES[codes[12]] == "SHORTER_THAN_K"
    assert codes.max() <= 5


def _read_fasta_gz(path):
    import gzip
    ids, seqs = [], []
    with gzip.open(path, "rt") as f:
        for line in f:
            (ids if line[0] == ">" else seqs).append(line[1:].strip() if line[0] == ">" else line.strip())
    return ids, seqs


@pytest.mark.parametrize("case", json.load(open(os.path.join(os.path.dirname(__file__), "golden", "cyc_cases.json"))),
                         ids=lambda c: c["name"])
def test_cycles_hairpins_tandems(abb, golden_dir, case):
    # circular plasmids, palindromic hairpins and tandem repeats: ER_CYCLE paths, the tile splice's
    # repeat check and the vertex-by-vertex fallback must all reproduce the reference
    from abyss_b200.capi import bloom_dbg
    ids, seqs = _read_fasta_gz(os.path.join(golden_dir, case["reads"]))
    fasta, _ = bloom_dbg(ids, seqs, case["k"], case["kc"], case["H"], bloom_size=case["b"], trim=case["trim"])
    assert fasta == open(os.path.join(golden_dir, case["name"] + ".fa")).read()


MASK_CASES = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "mask_cases.json")))


@pytest.mark.parametrize("case", MASK_CASES, ids=lambda c: c["name"])
def test_spaced_seeds_identical_to_reference(abb, golden_dir, case):
    # -K / --qr-seed / -s: the spaced seed changes the hash (pass 1 and every Bloom probe), vertex identity
    # (RollingBloomDBGVertex::compare orients by the full k-mer) and pathToSeq ('N' where no vertex writes a column)
    from abyss_b200.capi import bloom_dbg, fixed_length_reads, kmer_pair_seed, qr_seed_pair
    if case["opt"].startswith("-K"):
        assert kmer_pair_seed(case["k"], int(case["opt"][2:])) == case["mask"]
    else:
        assert qr_seed_pair(case["k"], int(case["opt"].split("=")[1])) == case["mask"]
    if case["reads"].endswith(".gz"):
        ids, seqs = _read_fasta_gz(os.path.join(golden_dir, case["reads"]))
    else:
        _, rs = load_case(golden_dir, case["reads"])
        ids = [rs.read_id(i) for i in range(rs.n)]
        seqs = fixed_length_reads(rs.ascii(0, rs.n))
    fasta, codes = bloom_dbg(ids, seqs, case["k"], case["kc"], case["H"], counters=case["counters"], mask=case["mask"],
                             read_log=True)
    want = open(os.path.join(golden_dir, case["name"] + ".fa")).read()
    assert fasta.count(">") == case["n_contigs"]
    assert fasta == want
    if case.get("readlog"):
        assert parity.read_log(ids, codes) == open(os.path.join(golden_dir, case["name"] + ".readlog.tsv")).read()


def test_spaced_seed_validation(abb):
    from abyss_b200.capi import Filter, Assembler, AbbError
    for bad in ("0" + "1" * 30 + "0", "1" * 20 + "0" * 11 + "1"):  # must begin/end with '1'; must be symmetric
        f = Filter.counting(4096, 4, 32, 2, mask=bad)
        with pytest.raises(AbbError):
            Assembler(f)
        f.close()


def test_tiles_on_off_same_output(abb, golden_dir, monkeypatch):
    from abyss_b200.capi import fixed_length_reads, bloom_dbg
    c, rs = load_case(golden_dir, "e2e_g20k_k32")
    ids = [rs.read_id(i) for i in range(rs.n)]
    reads = fixed_length_reads(rs.ascii(0, rs.n))
    on, _ = bloom_dbg(ids, reads, c["k"], c["kc"], c["H"], counters=c["counters"])
    monkeypatch.setenv("ABB_NO_TILES", "1")
    off, _ = bloom_dbg(ids, reads, c["k"], c["kc"], c["H"], counters=c["counters"])
    assert on == off == open(os.path.join(golden_dir, "e2e_g20k_k32.fa")).read()


def test_assembler_reset_reuses_handle(abb, golden_dir):
    # abb_assembler_reset: a second assembly on the same handles gives the same bytes
    from abyss_b200.capi import fixed_length_reads, Filter, Assembler
    c, rs = load_case(golden_dir, "e2e_g20k_k32")
    ids = [rs.read_id(i) for i in range(rs.n)]
    reads = fixed_length_reads(rs.ascii(0, rs.n))
    f = Filter.counting(c["counters"], c["H"], c["k"], c["kc"])
    a = Assembler(f)
    outs = []
    for _ in range(2):
        f.clear()
        a.reset()
        f.insert_reads(reads)
        outs.append(a.assemble(ids, reads)[0])
    a.close()
    f.close()
    assert outs[0] == outs[1] == open(os.path.join(golden_dir, "e2e_g20k_k32.fa")).read()


HASHNUM = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hashnum_cases.json")))


@pytest.mark.parametrize("case", HASHNUM["dbg"], ids=lambda c: c["name"])
def test_hash_counts_identical_to_reference(abb, golden_dir, tmp_path, case):
    # H = 1, 2, 5, 8, 9: the MAXH = 4 kernels with lanes that have nothing to probe, and the MAXH = 8 and 32 kernels.  Counters,
    # FASTA and read log against the reference's -j1 run (tests/golden/make_golden_hashnum.py), through the C ABI as one batch
    # and in batches of 997 reads, and through abyss-bloom-dbg
    from abyss_b200.capi import fixed_length_reads, bloom_dbg, Filter
    c, rs = load_case(golden_dir, case["reads"])
    H = case["H"]
    ids = [rs.read_id(i) for i in range(rs.n)]
    reads = fixed_length_reads(rs.ascii(0, rs.n))
    f = Filter.counting(c["counters"], H, c["k"], c["kc"])
    f.insert_reads(reads)
    assert parity.sha256(f.download().tobytes()) == case["counters_sha256"]
    f.close()
    for batch in (None, 997):
        fasta, codes = bloom_dbg(ids, reads, c["k"], c["kc"], H, counters=c["counters"], batch_reads=batch, read_log=True)
        parity.check_unitigs(case, fasta, parity.read_log(ids, codes))
    fq = str(tmp_path / "reads.fq")
    rs.write_fastq(fq)
    fasta, log, _ = parity.bloom_dbg_cli(dict(c, H=H), fq, tmp_path)
    parity.check_unitigs(case, fasta, log)
