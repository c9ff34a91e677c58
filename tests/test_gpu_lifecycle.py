"""GPU: every handle kind gives its device memory back.  Several create -> use -> destroy cycles of each handle in one
process leave the device's free memory where it was, and a filter too large for the device fails with ABB_ENOMEM,
leaves nothing behind and does not disturb the next filter."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from abyss_b200.synth import ReadSet

pytestmark = pytest.mark.gpu

GiB = 1 << 30
FILTER_BYTES = 4 * GiB  # each filter of a cycle; the assembler's unitig arena is 4 GiB as well
CYCLES = 3
MARGIN = 4 * GiB  # free memory is device wide, and other processes on the GPU move it too: one leak per cycle is 12 GiB


def _free_bytes():
    import torch
    torch.cuda.synchronize(0)
    return torch.cuda.mem_get_info(0)[0]


@pytest.fixture(scope="module")
def case(golden_dir):
    c = {x["name"]: x for x in json.load(open(os.path.join(golden_dir, "e2e_cases.json")))}["e2e_g20k_k32"]
    return c, ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])


def _cycle(abb, c, rs):
    lib = abb.load()
    k, H = c["k"], c["H"]
    reads = abb.fixed_length_reads(rs.ascii(0, rs.n))
    bases, offs = reads
    # counting filter and assembler: pass 1 with the profiling events, pass 2 with tiles (tile store and unitig arena)
    f = abb.Filter.counting(FILTER_BYTES, H, k, c["kc"])
    f.set_profiling(True)
    assert f.insert_reads(reads) > 0
    a = abb.Assembler(f)
    unitigs = [s for _, s, _ in a.process_reads(reads)]
    assert unitigs
    a.close()
    f.close()
    # bit filter and the one-shot queries
    b = abb.Filter.bits(8 * FILTER_BYTES, H, k)
    b.insert_reads(reads)
    slots = int(offs[-1]) - rs.n * (k - 1)
    flag, valid, n = np.zeros(slots, np.uint8), np.zeros(slots, np.uint8), C.c_uint64(0)
    abb.check(lib.abb_contains_reads(b.handle, abb._ptr(bases), abb._ptr(offs), rs.n, abb._ptr(flag), abb._ptr(valid), slots,
                                     C.byref(n)))
    assert n.value == slots and valid.any() and flag[valid == 1].all()
    assert len(abb.successors(b, [unitigs[0][:k]])) == 1
    assert len(abb.hash_reads(k, reads)[0]) == slots
    b.close()
    cf = abb.Filter.cascading(8 * FILTER_BYTES // 2, H, 2, k)
    cf.insert_reads(reads)
    cf.close()
    kf = abb.Filter.konnector(8 * FILTER_BYTES, 25)
    assert kf.insert_reads(reads) > 0
    kf.close()
    abb.overlap_graph(unitigs, k)


def test_handles_give_their_memory_back(abb, case):
    _cycle(abb, *case)  # module loading and the runtime's own first allocations happen once per process
    before = _free_bytes()
    for _ in range(CYCLES):
        _cycle(abb, *case)
    lost = before - _free_bytes()
    assert lost < MARGIN, f"{lost / GiB:.1f} GiB less free device memory after {CYCLES} cycles"


def test_filter_too_large_for_the_device(abb, case):
    import torch
    lib = abb.load()
    bits = 16 * torch.cuda.mem_get_info(0)[1]  # twice the device's memory
    before = _free_bytes()
    h = C.c_void_p()
    assert lib.abb_konnector_create(C.byref(h), bits, 25, 1, 0, 0, bits - 1, 0) == abb.ABB_ENOMEM
    assert not h.value
    assert abs(_free_bytes() - before) < MARGIN
    # the failed allocation is not reported again by the next filter's calls
    f = abb.Filter.konnector(1 << 24, 25)
    assert f.insert_reads(abb.fixed_length_reads(case[1].ascii(0, 100))) > 0
    f.close()
