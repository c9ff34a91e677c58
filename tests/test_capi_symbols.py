"""CPU-only: the C-ABI library builds (nvcc cross-compiles), loads, and exports every symbol that
include/abyss_b200.h declares; without a GPU every compute entry point fails loudly (no fallback)."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "abyss_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(abb_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(abb):
    lib = abb.load()
    names = declared_symbols()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/abyss_b200.h but not exported"
        assert n in abb.SIGNATURES, f"{n} has no ctypes signature in abyss_b200/capi.py"
    assert lib.abb_version() == 101


def test_no_cpu_fallback(abb):
    import torch
    if torch.cuda.is_available():
        return  # the gpu suite covers the working path
    lib = abb.load()
    assert lib.abb_device_count() < 0 or lib.abb_device_count() == 0
    try:
        abb.Filter.counting(1024, 4, 20)
    except abb.AbbError as e:
        assert e.code == abb.ABB_ENODEV
        assert "no CPU fallback" in str(e)
    else:
        raise AssertionError("filter creation must fail without a CUDA device")
    try:
        abb.hash_reads(5, ["ACGTACGT"])
    except abb.AbbError as e:
        assert e.code == abb.ABB_ENODEV
    else:
        raise AssertionError("hash_reads must fail without a CUDA device")


def test_hash_reads_refuses_malformed_batch(abb):
    # the read batch is checked on the host before any CUDA call, so a malformed one is ABB_EINVAL with or without a device
    import ctypes as C
    lib = abb.load()
    bases = np.frombuffer(b"ACGTACGTAC", dtype=np.uint8).copy()
    offs, shifted = np.array([0, 10], dtype=np.uint64), np.array([1, 10], dtype=np.uint64)
    h0, valid, n = np.zeros(16, dtype=np.uint64), np.zeros(16, dtype=np.uint8), C.c_uint64(7)

    def run(b, o):
        return lib.abb_hash_reads(5, b"", b, o, 1, h0.ctypes.data, valid.ctypes.data, C.byref(n), 0)

    assert run(None, offs.ctypes.data) == abb.ABB_EINVAL
    assert "NULL read buffers" in lib.abb_last_error().decode()
    assert run(bases.ctypes.data, None) == abb.ABB_EINVAL
    assert run(bases.ctypes.data, shifted.ctypes.data) == abb.ABB_EINVAL
    assert "offsets[0] must be 0" in lib.abb_last_error().decode()
    assert n.value == 0


def test_header_is_plain_c(tmp_path):
    # the boundary is a C ABI: include/abyss_b200.h compiles as C99 (no C++, no torch or CUDA types) and a C program links against
    # the library using nothing but that header
    import subprocess
    src = tmp_path / "use_abi.c"
    src.write_text(
        '#include "abyss_b200.h"\n'
        "#include <stdio.h>\n"
        "int main(void) {\n"
        "    abb_filter* f = NULL; abb_overlap* o = NULL; abb_succ_info s; abb_overlap_edge e; abb_assembly_params p = {0, 0, 0, 0};\n"
        "    (void)s; (void)e; (void)p;\n"
        "    printf(\"%d\\n\", abb_version());\n"
        "    if (abb_device_count() <= 0) {\n"
        "        int rc = abb_filter_create(&f, ABB_COUNTING, 1024, 4, 20, 2, \"\", 0);\n"
        "        int rc2 = abb_overlap_create(&o, 0);\n"
        "        printf(\"%d %d %s\\n\", rc, rc2, abb_last_error());\n"
        "    }\n"
        "    return 0;\n"
        "}\n")
    exe = tmp_path / "use_abi"
    lib = os.path.join(ROOT, "abyss_b200", "lib")
    subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", str(exe), str(src),
                    "-L" + lib, "-labyssb200", "-Wl,-rpath," + lib], check=True, capture_output=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.split("\n")
    assert lines[0] == "101"
    import torch
    if not torch.cuda.is_available():
        assert lines[1].startswith("-2 -2 ") and "no CPU fallback" in lines[1]  # ABB_ENODEV from both entry points


def test_assembly_stats_mirror_matches_header(tmp_path, abb):
    # capi.AssemblyStats mirrors abb_assembly_stats field by field: a field added to one and not the other shifts every later
    # field, so the size and the offset of every field must agree with what a C compiler makes of the header
    import ctypes
    import subprocess
    fields = [f for f, _ in abb.AssemblyStats._fields_]
    src = tmp_path / "stats_layout.c"
    src.write_text('#include "abyss_b200.h"\n#include <stddef.h>\n#include <stdio.h>\nint main(void) {\n'
                   '    printf("%zu\\n", sizeof(abb_assembly_stats));\n'
                   + "".join(f'    printf("%zu\\n", offsetof(abb_assembly_stats, {f}));\n' for f in fields)
                   + "    return 0;\n}\n")
    exe = tmp_path / "stats_layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True,
                   capture_output=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got[0] == ctypes.sizeof(abb.AssemblyStats)
    assert got[1:] == [getattr(abb.AssemblyStats, f).offset for f in fields]
    assert fields[-2:] == ["untiled_markers", "dropped_tiles"]


def test_bench_derived_rooflines():
    # bench.py's pass-2 roofline entries are plain arithmetic on counters the run reports: checked here on phase times and
    # counters of the shape of the bench workload (the genome assembled once), and never allowed to raise
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    phases_ms, bases_assembled = {"classify": 700.0, "tiles": 700.0}, 187_500_000
    r = bench.pass2_rooflines(phases_ms, 20_000_000, bases_assembled, 3350.0)
    assert len(r) == 2 and all(0 < x["frac"] < 1 for x in r)
    tiles = [x for x in r if x["kernel"].startswith("k_make_tiles")][0]
    assert abs(tiles["alg_bytes"] - 4 * bases_assembled * 1024) < 1
    assert bench.pass2_rooflines({}, 0, 0, 3350.0) == []
    assert "error" in bench.pass2_rooflines(None, 1, 1, 1.0)[0]
