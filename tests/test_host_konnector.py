"""CPU: the Konnector kernels' arithmetic (abyss_b200/csrc/abb_konnector.cuh: rolling canonical k-mer, CityHash64WithSeed,
level walk, windows, copyBits), run single-threaded by tests/host_konnector, writes the bytes of the unmodified reference's
`abyss-bloom build -t konnector`, `union` and `intersect` files (tests/golden/make_golden_konnector.py).  The hash cases
cover k = 1..192, i.e. every CityHash length branch, with seeds 0, 1 and one above 2^32."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, GOLD)
from make_golden_konnector import write_reads  # noqa: E402

CASES = [c for c in json.load(open(os.path.join(GOLD, "konnector_cases.json"))) if "harness" in c]


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    d = tmp_path_factory.mktemp("hk")
    exe = str(d / "host_konnector")
    subprocess.run(["g++", "-std=c++17", "-O2", "-pthread", "-o", exe, os.path.join(ROOT, "tests", "host_konnector", "host_konnector.cpp")],
                   check=True, capture_output=True)
    write_reads(str(d))
    # the harness cases run in file order: the union cases read the window files built before them
    out = {}
    for c in CASES:
        r = subprocess.run([exe, *map(str, c["harness"])], cwd=str(d), capture_output=True)
        assert r.returncode == 0, r.stderr.decode()
        out[c["name"]] = hashlib.sha256(open(d / c["file"], "rb").read()).hexdigest()
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
