"""CPU: the arithmetic helpers shared by host and device code (exact modulo, split rotations, ntHash
rolls, 2-bit k-mers) against the oracle, and the CLI's FASTA/FASTQ reader semantics
(DataLayer/FastaReader.cpp:130-421: Casava chastity filter, masked-end trimming, case folding, quality trim)."""
import subprocess

import parity

host_arith = parity.harness("host_arith", "tests/host_arith/host_arith.cpp", parity.ORACLE)


def test_host_arith_and_reader(host_arith, tmp_path):
    fq = tmp_path / "in.fq"
    fq.write_text(
        "# a comment line\n"
        "@read1 1:N:0:ACGT\nacgtACGTNNacgt\n+\nIIIIIIIIIIIIII\n"       # Casava, chaste; masked ends trimmed; /1 appended (ids longer than 2)
        "@r2 2:Y:0:ACGT\nACGTACGT\n+\nIIIIIIII\n"                       # unchaste: dropped
        "@r3/1\nACGTacgtAC\n+\n##IIIIII##\n"                            # quality trim at q>=3 removes '#' (q=2) ends
        ">f1 some comment\nACGT\nACGT\nAC\n"                            # multi-line FASTA
        ">f2\nacgt\n")                                                  # all masked -> empty read
    r = subprocess.run([host_arith, str(fq), "3"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.strip().split("\n")
    assert lines[-1] == "HOST_ARITH_OK"
    assert lines[:-1] == ["read1/1\tACGTNN", "r3/1\tGTACGT", "f1\tACGTACGTAC", "f2\t"]
