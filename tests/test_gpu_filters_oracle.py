"""Differential matrix: every Bloom filter kind against the sequential oracle (oracle/abyss_oracle.c), through the C ABI.

Each case compares the whole downloaded filter with the oracle.  The matrix covers the configurations the kernels are
instantiated for and the places where they change behaviour: every MAXH instantiation (H <= 4, <= 8, <= 32), dense filters
whose counters saturate and whose slots carry across windows and drain in the middle of a call, bit and cascading levels
of every size modulo 16 bytes, window sizes and call splits, chunk and copy-piece boundaries of one large call, and
positions that need 33 bits."""
import ctypes as C

import numpy as np
import pytest

from abyss_b200.synth import ReadSet, edge_mutate

pytestmark = pytest.mark.gpu

HS = [1, 2, 3, 4, 5, 7, 8, 9, 16, 31, 32]
POP8 = np.array([bin(i).count("1") for i in range(256)], dtype=np.uint64)


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def reads(seed, genome, n, L, err=0.01):
    rs = ReadSet(seed, genome, n, L, err)
    return [a.tobytes().decode() for a in rs.ascii(0, n)]


def edgy(seqs):
    """N, lower case and reads shorter than k at fixed places (synth.edge_mutate), plus empty reads"""
    out = edge_mutate(seqs, every_n=7, every_lc=11, every_short=13)
    out[2:2] = ["", "ACGT", "N" * 60, "acgtACGTnnACGTacgt" * 6]
    return out


def slot_offsets(seqs, k):
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    so = np.zeros(len(seqs) + 1, dtype=np.uint64)
    so[1:] = np.cumsum(np.maximum(lens - k + 1, 0))
    return so


def oracle_slots(oracle, seqs, k, H, mask=""):
    """(slot index, H hashes) of every k-mer RollingHashIterator yields, slot = window start in the batch"""
    so = slot_offsets(seqs, k)
    idx, hs = [], []
    for i, s in enumerate(seqs):
        h, pos = oracle.hash_seq(s, k, H, mask)
        idx.append(so[i] + pos.astype(np.uint64))
        hs.append(h)
    return np.concatenate(idx).astype(np.int64), np.concatenate(hs).reshape(-1, H), int(so[-1])


def bf_insert(oracle, bits, mbits, rows):
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    for r in rows:
        oracle.lib.abo_bf_insert(bits.ctypes.data, mbits, r.ctypes.data, rows.shape[1])


def bf_contains(oracle, bits, mbits, rows):
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    return np.array([oracle.lib.abo_bf_contains(bits.ctypes.data, mbits, r.ctypes.data, rows.shape[1]) for r in rows], dtype=bool)


def casc_insert(oracle, levels, mbits, L, rows):
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    for r in rows:
        oracle.lib.abo_casc_insert(levels.ctypes.data, mbits, L, r.ctypes.data, rows.shape[1])


def contains_reads(abb, f, seqs):
    """abb_contains_reads: per-slot membership and validity"""
    bases, offs = seqs if isinstance(seqs, tuple) else abb.pack_reads(seqs)
    k = f.getKmerSize()
    lens = np.diff(offs).astype(np.int64)
    total = int(np.maximum(lens - k + 1, 0).sum())
    flag = np.full(total, 7, dtype=np.uint8)
    valid = np.full(total, 7, dtype=np.uint8)
    n = C.c_uint64(0)
    abb.check(abb.load().abb_contains_reads(f.handle, abb._ptr(bases), abb._ptr(offs), len(offs) - 1, abb._ptr(flag),
                                            abb._ptr(valid), total, C.byref(n)))
    assert n.value == total
    return flag, valid


def bits_of(level, mbits, rows):
    """contains() of one bit level for hash rows, in numpy"""
    p = rows % np.uint64(mbits)
    return ((level[(p >> np.uint64(3)).astype(np.int64)] >> (p & np.uint64(7)).astype(np.uint8)) & 1).all(axis=1)


def assert_same(got, exp, what):
    if not np.array_equal(got, exp):
        d = np.flatnonzero(got != exp)
        raise AssertionError(f"{what}: {d.size} bytes differ, first at {d[0]}: got {got[d[0]]}, oracle {exp[d[0]]}")


# ---------------------------------------------------------------------------------------------------------------------
# 1. counting, reads path, every MAXH
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", HS)
def test_counting_reads_sparse(abb, oracle, H):
    k = 25
    seqs = edgy(reads(100 + H, 20000, 700, 100))
    slots = int(slot_offsets(seqs, k)[-1])
    # CountingBloomFilter pads the size to a multiple of 8 counters (CountingBloomFilter.hpp:40-49)
    f = abb.Filter.counting(20 * slots + 8 * H + 3, H, k)
    m = f.size()
    assert m == 20 * slots + 8 * H + 8
    exp = np.zeros(m, dtype=np.uint8)
    n_exp = oracle.cbf_load(exp, seqs, k, H)
    assert f.insert_reads(seqs) == n_exp
    assert_same(f.download(), exp, f"sparse H={H}")
    f.close()


@pytest.mark.parametrize("H,mask", [(h, "") for h in HS] + [(9, "1111111111" + "00000" + "1111111111")])
def test_counting_reads_dense_saturating(abb, oracle, H, mask):
    # a few hundred counters and every read many times: nearly every slot conflicts, most windows carry more slots than a
    # window serves, so the kernel stops for drains in the middle of each call, and counters reach 255
    k, m = 25, 512
    base = edgy(reads(200 + H, 4000, 150, 100))
    calls = [base * 16, base[:60] * 10, base * 16]
    exp = np.zeros(m, dtype=np.uint8)
    f = abb.Filter.counting(m, H, k, mask=mask)
    for seqs in calls:
        n_exp = oracle.cbf_load(exp, seqs, k, H, mask)
        assert f.insert_reads(seqs) == n_exp
    assert_same(f.download(), exp, f"dense H={H} mask={mask!r}")
    assert (exp == 255).any(), "the case no longer saturates counters"
    st = f.stats()
    assert st.deferred > 0, "no slot was carried"
    assert st.drains > len(calls), f"{st.drains} drains in {len(calls)} calls: none happened in the middle of a call"
    f.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. counting, literal hashes, every MAXH
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", HS)
def test_counting_literal(abb, oracle, H):
    rng = np.random.default_rng(1000 + H)
    m = 4001 * 8
    rows = rng.integers(0, 2**64, size=(12000, H), dtype=np.uint64)
    rows[3000:4000] = rows[:1000]                      # repeated rows
    rows[5000:5200, H - 1] = rows[5000:5200, 0]        # duplicate positions inside one row
    rows[5200:5300, :] = rows[5200:5300, :1]           # every position of the row the same
    # rows forced onto eight counters (plus multiples of m: the same positions through the modulo), so that carries chain
    # from window to window and counters saturate
    hot = rng.integers(0, 8, size=(3000, H), dtype=np.uint64) + np.uint64(m) * rng.integers(0, 1 << 40, size=(3000, H), dtype=np.uint64)
    rows[7000:10000] = hot
    exp = np.zeros(m, dtype=np.uint8)
    oracle.cbf_insert_hashes(exp, rows)
    f = abb.Filter.counting(m, H, 31, threshold=1)
    f.set_window(1024)
    f.insert(rows)
    assert_same(f.download(), exp, f"literal H={H}")
    assert (exp[:8] == 255).any()
    assert f.stats().deferred > 0
    q = rng.integers(0, 2**64, size=(4000, H), dtype=np.uint64)
    q[:1500] = rows[::8][:1500]
    q[1500:1600] = hot[:100]
    mn = oracle.cbf_min_hashes(exp, q)
    assert (f.minCount(q) == mn).all()
    for t in (1, 2, 3):
        f.set_threshold(t)
        assert (f.contains(q) == (mn >= t)).all(), t
        assert f.popcounts() == (np.count_nonzero(exp), np.count_nonzero(exp >= t)), t
    f.close()


@pytest.mark.parametrize("H", [h for h in HS if h > 4])
def test_counting_literal_conflict_past_fourth_hash(abb, oracle, H):
    # pairs of rows in one window that share only their positions 4..H-1; the second row's first four counters are already
    # 1, so in file order it finds its minimum 1 after the first row and raises every counter to 2.  Applied side by side,
    # it would read 0 at the shared counters and leave them at 1: the window must see conflicts on every position.
    rng = np.random.default_rng(3000 + H)
    m = (1 << 22) + 8
    n = 2000
    a = rng.integers(0, m, size=(n, H), dtype=np.uint64)
    b = rng.integers(0, m, size=(n, H), dtype=np.uint64)
    b[:, 4:] = a[:, 4:]
    pre = rng.integers(0, m, size=(n, H), dtype=np.uint64)
    pre[:, :4] = b[:, :4]
    pairs = np.stack([a, b], axis=1).reshape(-1, H)
    exp = np.zeros(m, dtype=np.uint8)
    f = abb.Filter.counting(m, H, 31)
    for rows in (pre, pairs):
        oracle.cbf_insert_hashes(exp, rows)
        f.insert(rows)
    shared = a[:, 4:].astype(np.int64)
    assert (exp[shared] >= 2).mean() > 0.9, "the case no longer depends on conflicts past the fourth position"
    assert_same(f.download(), exp, f"H={H}")
    assert f.stats().deferred > 0
    f.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. bit and cascading filters, every MAXH, every level size modulo 16 bytes
# ---------------------------------------------------------------------------------------------------------------------
LEVEL_BYTES = [1001, 1002, 1003, 1000, 1024]  # = 9, 10, 11, 8, 0 (mod 16)


@pytest.mark.parametrize("H", HS)
def test_bits_and_cascading(abb, oracle, H):
    k = 21
    rng = np.random.default_rng(2000 + H)
    seqs = edgy(reads(300 + H, 3000, 60, 60))
    seqs = seqs + seqs[:30] + seqs[:10]
    lit = rng.integers(0, 2**64, size=(400, H), dtype=np.uint64)
    lit[200:300] = lit[:100]
    for nbytes in LEVEL_BYTES:
        mbits = 8 * nbytes
        for L in (0, 1, 2, 3, 5):  # 0: a plain bit filter
            levels = max(L, 1)
            exp = np.zeros(levels * nbytes, dtype=np.uint8)
            if L == 0:
                n_exp = oracle.bf_load(exp, seqs, k, H)
                f = abb.Filter.bits(mbits, H, k)
            else:
                n_exp = oracle.casc_load(exp, mbits, L, seqs, k, H)
                f = abb.Filter.cascading(mbits, H, L, k)
            what = f"H={H} bytes={nbytes} L={L}"
            assert f.insert_reads(seqs) == n_exp, what
            if L == 0:
                bf_insert(oracle, exp, mbits, lit)
            else:
                casc_insert(oracle, exp, mbits, L, lit)
            f.insert(lit)
            exp = exp.reshape(levels, nbytes)
            for lv in range(levels):
                assert_same(f.download(lv), exp[lv], f"{what} level {lv}")
            last = exp[-1]
            q = np.concatenate([lit[:150], rng.integers(0, 2**64, size=(150, H), dtype=np.uint64)])
            want = bf_contains(oracle, last, mbits, q)
            assert (f.contains(q) == want).all(), what
            assert f.popCount() == int(POP8[last].sum()), what
            # upload into one level and read every level back: the neighbours must be untouched
            lv = levels // 2
            junk = rng.integers(0, 256, size=nbytes, dtype=np.uint8)
            f.upload(junk, lv)
            for j in range(levels):
                assert_same(f.download(j), junk if j == lv else exp[j], f"{what} after upload to level {lv}: level {j}")
            f.clear()
            assert f.popCount() == 0 and not f.download(0).any()
            f.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. window sizes and call splitting
# ---------------------------------------------------------------------------------------------------------------------
def reads_with_slots(rng, n_slots, k, L=1000):
    """random reads of length L (and one shorter) with exactly n_slots k-mer slots; each read starts with a 12-base unit
    repeated five times, so that every window of at least 13 slots holds the same k-mer twice"""
    per = L - k + 1
    n_full, rest = divmod(n_slots, per)
    lut = np.frombuffer(b"ACGT", dtype=np.uint8)
    codes = [rng.integers(0, 4, size=L, dtype=np.uint8) for _ in range(n_full)]
    if rest:
        codes.append(rng.integers(0, 4, size=rest + k - 1, dtype=np.uint8))
    for c in codes:
        n = min(60, c.size)
        c[:n] = np.tile(c[:12], 5)[:n]
    return [lut[c].tobytes().decode() for c in codes]


@pytest.mark.parametrize("W", [32, 33, 4096, 1 << 17, (1 << 20) - 64])
def test_window_sizes(abb, oracle, W):
    k, H, m = 25, 4, 4096
    rng = np.random.default_rng(W)
    mult = 2 if W > 4096 else 3
    for n_slots in (mult * W, mult * W + 1, mult * W - 1, W - 5 if W > 32 else 7):
        seqs = reads_with_slots(rng, n_slots, k)
        assert int(slot_offsets(seqs, k)[-1]) == n_slots
        exp = np.zeros(m, dtype=np.uint8)
        n_exp = oracle.cbf_load(exp, seqs, k, H)
        f = abb.Filter.counting(m, H, k)
        f.set_window(W)
        assert f.insert_reads(seqs) == n_exp == n_slots
        assert_same(f.download(), exp, f"W={W} slots={n_slots}")
        if n_slots >= W:
            assert f.stats().deferred > 0
        f.close()


@pytest.mark.parametrize("n_calls", [1, 3, 17])
def test_call_splitting(abb, oracle, n_calls):
    # the same reads in 1, 3 or 17 calls with a literal insert after the first: one oracle pass in file order
    k, H, m = 25, 5, 3000
    seqs = edgy(reads(77, 6000, 900, 120))
    rng = np.random.default_rng(77)
    lit = rng.integers(0, 2**64, size=(3000, H), dtype=np.uint64)
    lit[1000:2000] = lit[:1000]
    cuts = np.linspace(0, len(seqs), n_calls + 1).astype(int)
    exp = np.zeros(m, dtype=np.uint8)
    f = abb.Filter.counting(m, H, k)
    f.set_window(2048)
    for c in range(n_calls):
        part = seqs[cuts[c]:cuts[c + 1]]
        assert f.insert_reads(part) == oracle.cbf_load(exp, part, k, H)
        if c == 0:
            oracle.cbf_insert_hashes(exp, lit)
            f.insert(lit)
    assert_same(f.download(), exp, f"{n_calls} calls")
    f.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. abb_contains_reads
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 4, 9])
def test_contains_reads(abb, oracle, H):
    k = 27
    built = edgy(reads(400 + H, 8000, 400, 100))
    query = edgy(built[:150] + reads(401 + H, 8000, 150, 100) + ["ACGT" * 5, "N" * 40, "acgtn" * 30])
    idx, rows, total = oracle_slots(oracle, query, k, H)
    exp_valid = np.zeros(total, dtype=np.uint8)
    exp_valid[idx] = 1
    # counting
    m = 50000
    exp = np.zeros(m, dtype=np.uint8)
    oracle.cbf_load(exp, built + built[:100] * 2, k, H)
    f = abb.Filter.counting(m, H, k)
    f.insert_reads(built + built[:100] * 2)
    assert_same(f.download(), exp, "counting")
    mn = exp[(rows % np.uint64(m)).astype(np.int64)].min(axis=1)
    assert (mn >= 3).any() and (mn == 0).any()
    for t in (0, 1, 3):
        f.set_threshold(t)
        flag, valid = contains_reads(abb, f, query)
        assert (valid == exp_valid).all(), t
        want = np.zeros(total, dtype=np.uint8)
        want[idx] = mn >= t
        assert (flag == want).all(), t
    f.close()
    # bit and cascading (last level)
    mbits = 8 * 1003
    for L in (0, 3):
        levels = max(L, 1)
        exp = np.zeros(levels * (mbits // 8), dtype=np.uint8)
        ins = built[:10] if L == 0 else built[:10] + built[:5] + built[:2]
        if L == 0:
            oracle.bf_load(exp, ins, k, H)
            f = abb.Filter.bits(mbits, H, k)
        else:
            oracle.casc_load(exp, mbits, L, ins, k, H)
            f = abb.Filter.cascading(mbits, H, L, k)
        f.insert_reads(ins)
        flag, valid = contains_reads(abb, f, query)
        assert (valid == exp_valid).all(), L
        want = np.zeros(total, dtype=np.uint8)
        want[idx] = bits_of(exp[-(mbits // 8):], mbits, rows)
        assert want.any() and not want[idx].all()
        assert (flag == want).all(), L
        f.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. chunk and copy-piece boundaries of one large call
# ---------------------------------------------------------------------------------------------------------------------
CHUNK_SLOTS = 1 << 27  # abb_api.cu kChunkSlots
PIECE_BYTES = 256 << 20  # abb_insert_reads kPiece


def chunk_bounds(so, cap):
    """the reads at which abb_api.cu k_chunk_bounds cuts one call"""
    bounds, r, n = [0], 0, len(so) - 1
    while r < n:
        r = max(r + 1, int(np.searchsorted(so, so[r] + cap, side="right")) - 1)
        bounds.append(min(r, n))
    return bounds


class Layout:
    """reads of one call as (offset, length, kind) with kind 'N' (all-N padding), 'r' (real) or 's' (shorter than k)"""

    def __init__(self, k):
        self.k, self.items, self.byte, self.slot = k, [], 0, 0

    def add(self, n, kind):
        self.items.append((self.byte, n, kind))
        self.byte += n
        self.slot += max(0, n - self.k + 1)

    def pad_to_slot(self, s):
        gap = s - self.slot
        assert gap > 1000, gap
        self.add(gap + self.k - 1, "N")

    def pad_to_byte(self, b):
        gap = b - self.byte
        assert gap > 1000, gap
        self.add(gap, "N")


def big_call(k, real_len=150, around=6):
    lay = Layout(k)
    for _ in range(20000):  # 480 kB of reads shorter than k: keeps slot and byte boundaries apart
        lay.add(k - 1, "s")
    n_chunks = 4
    events = [("slot", c * CHUNK_SLOTS) for c in range(1, n_chunks + 1)] + [("byte", p * PIECE_BYTES) for p in (1, 2)]
    est = lambda e: e[1] + 20000 * (k - 1) if e[0] == "slot" else e[1]  # noqa: E731
    per = real_len - k + 1
    for kind, at in sorted(events, key=est):
        if kind == "slot":
            lay.pad_to_slot(at - around * per)
            for _ in range(2 * around):
                lay.add(real_len, "r")
        elif at == PIECE_BYTES:
            lay.pad_to_byte(at - around * real_len)
            for _ in range(2 * around):
                lay.add(real_len, "r")
        else:  # one read across the boundary
            lay.pad_to_byte(at - around * real_len - real_len // 2)
            for _ in range(2 * around + 1):
                lay.add(real_len, "r")
    lay.pad_to_slot(lay.slot + CHUNK_SLOTS // 3)
    for _ in range(around):
        lay.add(real_len, "r")
    return lay


def test_chunk_and_copy_boundaries(abb, oracle):
    import torch
    k, H, m = 25, 4, 65536
    lay = big_call(k)
    n_bases = lay.byte
    offs = np.zeros(len(lay.items) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([n for _, n, _ in lay.items])
    lens = np.diff(offs).astype(np.int64)
    so = np.zeros(len(lens) + 1, dtype=np.uint64)
    so[1:] = np.cumsum(np.maximum(lens - k + 1, 0))
    assert int(so[-1]) == lay.slot
    # what the call must reach: more than two chunks and more than two copy pieces, real reads on both sides of every
    # chunk boundary and every piece boundary, one real read across a piece boundary
    bounds = chunk_bounds(so, CHUNK_SLOTS)
    assert len(bounds) - 1 > 2 and n_bases > 2 * PIECE_BYTES
    kinds = [kd for _, _, kd in lay.items]
    for b in bounds[1:-1]:
        assert kinds[b - 1] == "r" and kinds[b] == "r", b
    starts = np.array([o for o, _, _ in lay.items], dtype=np.int64)
    for p in (1, 2):
        i = int(np.searchsorted(starts, p * PIECE_BYTES, side="right")) - 1
        assert kinds[i] == "r" and kinds[i - 1] == "r" and kinds[i + 1] == "r", p
    assert any(o < 2 * PIECE_BYTES < o + n for o, n, kd in lay.items if kd == "r")
    # real reads: a few distinct reads, each used several times, so that slots carry up to the end of each chunk
    src = reads(5150, 3000, 40, 150)
    real = []

    def fill(buf):
        nonlocal real
        buf[:] = ord("N")
        real = []
        j = 0
        for o, n, kd in lay.items:
            if kd == "r":
                s = src[j % len(src)] if j % 3 else src[(j // 3) % 5]
                buf[o:o + n] = np.frombuffer(s.encode(), dtype=np.uint8)
                real.append(s)
                j += 1
            elif kd == "s":
                buf[o:o + n] = ord("A")

    exp = np.zeros(m, dtype=np.uint8)
    # all-N reads have no k-mer and reads shorter than k none either (RollingHashIterator.h:37-56): the oracle sees the
    # real reads only, in file order
    pinned = torch.empty(n_bases, dtype=torch.uint8, pin_memory=True)
    bases_np = pinned.numpy()
    fill(bases_np)
    n_exp = oracle.cbf_load(exp, real, k, H)
    assert n_exp > 0
    for run in ("pinned", "pageable"):
        buf = bases_np
        if run == "pageable":
            del bases_np, pinned
            buf = np.empty(n_bases, dtype=np.uint8)
            fill(buf)
        f = abb.Filter.counting(m, H, k)
        assert f.insert_reads((buf, offs)) == n_exp, run
        assert_same(f.download(), exp, run)
        st = f.stats()
        assert st.slots == lay.slot and st.deferred > 0, run
        f.close()
        del buf


# ---------------------------------------------------------------------------------------------------------------------
# 7. positions of 33 bits
# ---------------------------------------------------------------------------------------------------------------------
def host_free_bytes():
    with open("/proc/meminfo") as fh:
        for line in fh:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def need_memory(device_bytes, host_bytes):
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < device_bytes:
        pytest.skip(f"needs {device_bytes / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    if host_free_bytes() < host_bytes:
        pytest.skip(f"needs {host_bytes / 2**30:.1f} GiB of free host memory, {host_free_bytes() / 2**30:.1f} GiB free")


def test_counting_33bit_positions(abb, oracle):
    k, H = 32, 4
    m = 5 * 2**30 + 8
    need_memory(m + 3 * 2**30, 2 * m + 2**30)
    seqs = edgy(reads(3333, 200000, 12000, 150))
    exp = np.zeros(m, dtype=np.uint8)
    n_exp = oracle.cbf_load(exp, seqs, k, H)
    rng = np.random.default_rng(33)
    # literal rows whose positions sit around 2^32 and at m - 1 (a hash below m is its own position), repeated so that
    # they carry and drain
    band = rng.integers(2**32 - 2**16, 2**32 + 2**16, size=(2000, H), dtype=np.uint64)
    band[::50, 0] = m - 1
    band[1::50, :] = m - 1
    band[2::50, :] = 2**32 - 1
    band[3::50, :] = 2**32
    lit = np.concatenate([band] * 6)
    oracle.cbf_insert_hashes(exp, lit)
    f = abb.Filter.counting(m, H, k, threshold=2)
    assert f.insert_reads(seqs) == n_exp
    f.stats(reset=True)
    f.insert(lit)
    assert f.stats().deferred > 0
    got = f.download()
    nz = np.flatnonzero(exp)
    assert np.array_equal(np.flatnonzero(got), nz)
    assert np.array_equal(got[nz], exp[nz])
    high = np.count_nonzero(nz >= 2**32)
    assert high > 0.1 * nz.size and exp[m - 1] > 0, "the case no longer touches positions of 33 bits"
    del got
    idx, rows, total = oracle_slots(oracle, seqs[:3000], k, H)
    q = np.concatenate([band, rows[:5000], rng.integers(0, 2**64, size=(2000, H), dtype=np.uint64)])
    mn = exp[(q % np.uint64(m)).astype(np.int64)].min(axis=1)
    assert (f.minCount(q) == mn).all()
    assert (f.contains(q) == (mn >= 2)).all()
    flag, valid = contains_reads(abb, f, seqs[:3000])
    want = np.zeros(total, dtype=np.uint8)
    want[idx] = exp[(rows % np.uint64(m)).astype(np.int64)].min(axis=1) >= 2
    assert valid.sum() == idx.size and (flag == want).all()
    assert f.popcounts() == (nz.size, int(np.count_nonzero(exp[nz] >= 2)))
    f.close()


def test_cascading_33bit_positions(abb, oracle):
    k, H, L = 32, 3, 3
    mbits = 2**33 + 64
    nbytes = mbits // 8  # 1 GiB + 8: the levels start on the padded stride
    need_memory(L * nbytes + 2**30, 2 * L * nbytes + 2**30)
    seqs = edgy(reads(3334, 100000, 6000, 150))
    seqs = seqs + seqs[:2000] + seqs[:500]
    exp = np.zeros(L * nbytes, dtype=np.uint8)
    n_exp = oracle.casc_load(exp, mbits, L, seqs, k, H)
    rng = np.random.default_rng(34)
    lit = rng.integers(2**33 - 2**12, 2**33 + 64, size=(500, H), dtype=np.uint64)
    lit = np.concatenate([lit] * 4)
    casc_insert(oracle, exp, mbits, L, lit)
    f = abb.Filter.cascading(mbits, H, L, k)
    assert f.insert_reads(seqs) == n_exp
    f.insert(lit)
    exp = exp.reshape(L, nbytes)
    for lv in range(L):
        assert_same(f.download(lv), exp[lv], f"level {lv}")
    nz = np.flatnonzero(exp[0])
    assert np.count_nonzero(nz >= 2**32 // 8) > 0 and exp[L - 1].any(), "the case no longer reaches bits of 33 bits"
    last = exp[L - 1]
    lnz = np.flatnonzero(last)
    assert f.popCount() == int(POP8[last[lnz]].sum())
    idx, rows, total = oracle_slots(oracle, seqs[:1500], k, H)
    flag, valid = contains_reads(abb, f, seqs[:1500])
    want = np.zeros(total, dtype=np.uint8)
    want[idx] = bits_of(last, mbits, rows)
    assert want.any() and (flag == want).all()
    f.close()
