"""GPU: pass 2 on long reads of 5 to 80 kbp against the unmodified reference (tests/golden/longread_cases.json,
tests/golden/make_golden_longreads.py): through the C ABI in one batch, in batches of 7 reads and without tiles, and through
abyss-bloom-dbg (FASTA, read log, -T trace, counters).  The cases reach what short reads never do: the whole-grid replay of
unitigs of 2^15 k-mers and more in K5, the read-level loops of K2, K3 and K5 past 1 024 k-mers, and the rerun of K4 when its
record buffer overflows.  abb_assembly_stats shows that the round structure those paths need was reached."""
import json
import os

import pytest

import parity
from make_golden_longreads import raw_reads, write_fasta

pytestmark = pytest.mark.gpu
CASES = json.load(open(os.path.join(parity.GOLD, "longread_cases.json")))
BY_NAME = {c["name"]: c for c in CASES}


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_assembler_c_abi(abb, monkeypatch, case):
    st = parity.check_assembler_c_abi(case, monkeypatch, list(map(list, zip(*raw_reads(case["reads"])))), batch=7)
    if case["name"] == "lr_dense_k64":
        # every candidate in one round, and more records than the first K4 record buffer holds: it was rerun
        assert st.rounds == 1, (st.rounds, st.speculated_reads)
        assert st.contigs_tried > max(8 * st.speculated_reads, 4096), (st.contigs_tried, st.speculated_reads)
    if case["name"].startswith("lr_repeats"):
        # speculated reads of more than 1 024 k-mers that the replay found covered
        assert st.wasted_reads > 0


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_assembler_cli(abb, tmp_path, case):
    parity.check_assembler_cli(case, tmp_path, raw_reads(case["reads"]))


def test_assembler_cli_wrapped_fasta(abb, tmp_path):
    """the same long reads as FASTA records wrapped at 60 columns give the same bytes"""
    case = BY_NAME["lr_repeats_k64"]
    fa = str(tmp_path / "reads.fa")
    write_fasta(raw_reads(case["reads"]), fa)
    parity.check_unitigs(case, *parity.bloom_dbg_cli(case, fa, tmp_path))
