"""CPU: `abyss-bloom trim` (the Konnector vertex, kon_left_trim and the walk templates of abb_walk.cuh, the reader's comments
and qualities, the record writer), run on one thread by tests/host_trim, prints the bytes of the unmodified reference's
`abyss-bloom trim` on every case of tests/golden/trim_cases.json that has a harness entry; the filters are built by
tests/host_konnector, whose files are the reference's (tests/test_host_konnector.py).  On the hand-made graphs the trim
lengths are also compared read by read with the ones the reference's output shows.  Case trim_quality runs the reader's -q
through trim and expects what the reference prints for the file cut beforehand."""
import json
import os
import re
import subprocess

import pytest

import parity
from make_golden_trim import FILTERS, fastq_records, write_inputs

CASES = [c for c in json.load(open(os.path.join(parity.GOLD, "trim_cases.json"))) if "harness" in c]
EXITS = ("end_no_vertex", "end_tip", "first_not_tip", "fork")
host_konnector = parity.harness("host_konnector", "tests/host_konnector/host_konnector.cpp")
host_trim = parity.harness("host_trim", "tests/host_trim/host_trim.cpp")


@pytest.fixture(scope="module")
def work(tmp_path_factory, host_konnector, host_trim):
    d = tmp_path_factory.mktemp("ht")
    write_inputs(str(d))
    for f in FILTERS:
        parity.run(host_konnector, *f["harness"], cwd=d)
    out = {}
    for c in CASES:
        r = parity.run(host_trim, c["harness"][0], "--lengths", "len.txt", *c["harness"][1:], cwd=d)
        out[c["name"]] = (parity.md5(r.stdout), r.stderr.decode(), open(d / "len.txt").read().splitlines(), r.stdout)
    out["dir"], out["exe"] = d, host_trim
    return out


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_trimmed_reads(work, case):
    md5, err, lengths, _ = work[case["name"]]
    if "lengths" in case:  # first, so that a failure names the read and the end
        ids = [i for i, _, _ in fastq_records(str(work["dir"] / case["harness"][-1]))]
        got = {i: l.split() for i, l in zip(ids, lengths)}
        for i, (left, right) in case["lengths"].items():
            assert got[i] == [str(left), str(right)], f"read {i}: (left, right) = {got[i]}, the reference shows {left, right}"
    assert md5 == case["stdout_md5"]
    m = re.search(r"min length threshold for true branches \(k-mers\): (\d+)", case["stderr"])
    if m:
        assert f"minBranchLen {m.group(1)} " in err


def test_trimmed_fasta_record(work):
    # A FASTA record has no quality string; the reference aborts when it cuts one on the left, this program writes the cut
    # record.  Expected: the reference's FASTQ output of the same reads without its quality lines.
    d = work["dir"]
    with open(d / "H25.fa", "w") as f:
        for i, s, _ in fastq_records(str(d / "H25.fq")):
            f.write(f">{i}\n{s}\n")
    fq = work["hand_g25"][3].decode().split("\n")
    want = "".join(f">{fq[i][1:]}\n{fq[i + 1]}\n" for i in range(0, len(fq) - 3, 4))
    assert any(v[0] > 0 for v in {c["name"]: c for c in CASES}["hand_g25"]["lengths"].values())  # some record is cut on the left
    r = subprocess.run([work["exe"], "25", "g25.bloom", "H25.fa"], cwd=str(d), capture_output=True)
    assert r.returncode == 0 and r.stdout.decode() == want


def test_every_exit_of_the_scan_is_taken(work):
    total = dict.fromkeys(EXITS, 0)
    runs = [v for k, v in work.items() if k not in ("dir", "exe")]
    for _, err, _, _ in runs:
        for e in EXITS:
            total[e] += int(re.search(e + r" (\d+)", err).group(1))
    assert all(total[e] > 0 for e in EXITS), total
    # the branch length thresholds the cases are there for
    seen = {int(re.search(r"minBranchLen (\d+)", err).group(1)) for _, err, _, _ in runs}
    assert {0, 1, 2, 4} <= seen and max(seen) >= 8
