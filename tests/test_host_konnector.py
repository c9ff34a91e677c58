"""CPU: the Konnector kernels' arithmetic (abyss_b200/csrc/abb_konnector.cuh: rolling canonical k-mer, CityHash64WithSeed,
level walk, windows, copyBits), run single-threaded by tests/host_konnector, writes the bytes of the unmodified reference's
`abyss-bloom build -t konnector`, `union` and `intersect` files (tests/golden/make_golden_konnector.py).  The hash cases
cover k = 1..192, i.e. every CityHash length branch, with seeds 0, 1 and one above 2^32."""
import json
import os

import pytest

import parity
from make_golden_konnector import write_reads

CASES = [c for c in json.load(open(os.path.join(parity.GOLD, "konnector_cases.json"))) if "harness" in c]
host_konnector = parity.harness("host_konnector", "tests/host_konnector/host_konnector.cpp")


@pytest.fixture(scope="module")
def work(tmp_path_factory, host_konnector):
    d = tmp_path_factory.mktemp("hk")
    write_reads(str(d))
    # the harness cases run in file order: the union cases read the window files built before them
    out = {}
    for c in CASES:
        parity.run(host_konnector, *c["harness"], cwd=d)
        out[c["name"]] = parity.sha256(open(d / c["file"], "rb").read())
    return out


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_konnector_file(work, case):
    assert work[case["name"]] == case["sha256"]


def test_union_of_windows_is_the_reference_union(work):
    # The reference's copyBits shifts `char` bytes, so a window that starts inside a byte ORs ones into the bits before each
    # source byte whose top bit is set: the union of the -w windows is the reference's union, not the unwindowed filter.
    by = {c["name"]: c for c in CASES}
    assert work["union_windows"] == by["union_windows"]["sha256"]
    assert by["union_windows"]["sha256"] != by["full_l3"]["sha256"]
