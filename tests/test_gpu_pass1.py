"""GPU parity for pass 1 (K1 hash_reads, K2 ordered insert) through the C ABI, against the oracle
and the committed reference fixtures.  Bit-exact: this is integer work."""
import hashlib
import json
import os

import numpy as np
import pytest

from abyss_b200.synth import ReadSet

pytestmark = pytest.mark.gpu


def edge_seqs(golden_dir):
    return open(os.path.join(golden_dir, "seqs_edge.txt")).read().split("\n")[:-1]


def seeded(seed, genome, n, L, err=0.01):
    rs = ReadSet(seed, genome, n, L, err)
    return [a.tobytes().decode() for a in rs.ascii(0, n)]


def gpu_hashes(abb, seqs, k, H, mask=""):
    """(seq idx, pos, H hashes) rows in the order RollingHashIterator yields them"""
    from abyss_b200.capi import pack_reads
    h0, valid, slot_offs = abb.hash_reads(k, seqs, mask)
    rows_seq, rows_pos, rows_h = [], [], []
    mult = [np.uint64((i ^ ((k * 0x90b45d39fb6da1fa) & 0xFFFFFFFFFFFFFFFF)) & 0xFFFFFFFFFFFFFFFF) for i in range(H)]
    for i in range(len(seqs)):
        a, b = int(slot_offs[i]), int(slot_offs[i + 1])
        v = valid[a:b].astype(bool)
        pos = np.nonzero(v)[0]
        h = h0[a:b][v]
        hs = [h]
        with np.errstate(over="ignore"):
            for j in range(1, H):
                t = h * mult[j]
                hs.append(t ^ (t >> np.uint64(27)))
        rows_seq += [i] * len(pos)
        rows_pos += pos.tolist()
        rows_h.append(np.stack(hs, axis=1) if len(pos) else np.zeros((0, H), dtype=np.uint64))
    return rows_seq, rows_pos, np.concatenate(rows_h)


@pytest.mark.parametrize("name", ["hashes_k5", "hashes_k20", "hashes_k32", "hashes_k64", "hashes_mask", "hashes_mask33"])
def test_hash_reads_vs_reference_fixture(abb, golden_dir, name):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    k, H, mask = int(g["k"]), int(g["H"]), str(g["mask"])
    seqs = edge_seqs(golden_dir) + seeded(12, 20000, 600, 150)[:40]
    rs, rp, rh = gpu_hashes(abb, seqs, k, H, mask)
    assert rs == g["seq"].tolist()
    assert rp == g["pos"].tolist()
    assert (rh == g["h"]).all()


@pytest.mark.parametrize("k", [1, 2, 31, 33, 63, 64, 65, 96, 160, 192])
def test_hash_reads_vs_oracle_many_k(abb, oracle, k):
    rng = np.random.default_rng(k)
    seqs = []
    for i in range(60):
        L = int(rng.integers(0, 700))
        s = rng.choice(list("ACGT"), size=L)
        if i % 3 == 0 and L:
            s[rng.integers(0, L, size=max(1, L // 50))] = "N"
        if i % 5 == 0:
            s = np.char.lower(s)
        seqs.append("".join(s))
    seqs += ["", "A", "ACGT" * 300]
    H = 4
    rs, rp, rh = gpu_hashes(abb, seqs, k, H)
    es, ep, eh = [], [], []
    for i, s in enumerate(seqs):
        h, pos = oracle.hash_seq(s, k, H)
        es += [i] * len(pos)
        ep += pos.tolist()
        eh.append(h)
    assert rs == es and rp == ep
    assert (rh == np.concatenate(eh)).all()


@pytest.mark.parametrize("mask", ["", "".join("0" if i % 7 == 3 else "1" for i in range(31))])
def test_hash_reads_dev_unaligned_bases(abb, mask):
    # device-resident reads at 0, 1, 7 and 15 bytes past an aligned address: the bulk copy that stages read blocks needs a
    # 16-byte aligned source, so the unaligned batches are hashed from global memory and must give the same windows
    import torch
    from abyss_b200.capi import pack_reads
    k = 31
    rng = np.random.default_rng(17)
    seqs = []
    for i in range(300):
        s = rng.choice(list("ACGT"), size=int(rng.integers(0, 400)))
        if i % 4 == 0 and len(s):
            s[rng.integers(0, len(s), size=max(1, len(s) // 40))] = "N"
        seqs.append("".join(s))
    seqs.insert(150, "".join(rng.choice(list("ACGT"), size=9000)))  # longer than a staging buffer
    h0_ref, valid_ref, slot_offs = abb.hash_reads(k, seqs, mask)
    total = int(slot_offs[-1])
    bases, offs = pack_reads(seqs)
    dev = torch.device("cuda", 0)
    buf = torch.zeros(len(bases) + 32, dtype=torch.uint8, device=dev)
    assert buf.data_ptr() % 16 == 0
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    f = abb.Filter.counting(4096, 4, k, mask=mask)
    for off in (0, 1, 7, 15):
        buf.zero_()
        buf[off:off + len(bases)] = torch.from_numpy(bases).to(dev)
        h0 = torch.full((total,), -1, dtype=torch.int64, device=dev)
        valid = torch.full((total,), 7, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize(dev)
        n = f.hash_reads_dev(buf.data_ptr() + off, d_offs.data_ptr(), len(seqs), h0.data_ptr(), valid.data_ptr(), total)
        assert n == total
        assert (h0.cpu().numpy().view(np.uint64) == h0_ref).all(), off
        assert (valid.cpu().numpy() == valid_ref).all(), off
    f.close()


def test_counting_fixtures(abb, golden_dir):
    reads60 = seeded(11, 3000, 1500, 60)
    reads150 = seeded(12, 20000, 600, 150)
    edge = edge_seqs(golden_dir)
    for name, seqs in (("count_m4096", edge + reads60), ("count_m65536_H3", reads150),
                       ("count_sat", [edge[9]] * 40 + reads60[:200])):
        g = np.load(os.path.join(golden_dir, name + ".npz"))
        f = abb.Filter.counting(int(g["m"]), int(g["H"]), int(g["k"]))
        f.insert_reads(seqs)
        got = f.download()
        assert (got == g["data"]).all(), f"{name}: {np.count_nonzero(got != g['data'])} counters differ"
        st = f.stats()
        assert st.deferred > 0  # tiny filters: the ordered path was exercised
        f.close()


@pytest.mark.parametrize("window", [32, 1000, 1 << 14])
def test_counting_window_sizes(abb, oracle, window):
    # result must not depend on the window size (only on file order)
    seqs = seeded(31, 5000, 3000, 80, err=0.02)
    k, H, m = 24, 4, 20000
    exp = np.zeros(m, dtype=np.uint8)
    oracle.cbf_load(exp, seqs, k, H)
    f = abb.Filter.counting(m, H, k)
    f.set_window(window)
    n = f.insert_reads(seqs)
    assert n == sum(max(0, len(s) - k + 1) for s in seqs)
    assert (f.download() == exp).all()
    f.close()


def test_counting_repeated_kmer_long_chain(abb, oracle):
    # one k-mer repeated thousands of times inside a window: exercises the bounded-round resolve
    # and its strict in-order tail; plus foreign k-mers interleaved on shared counters
    base = "ACGTTGCAAGCTAGCTAGGATCGATCGGATTACA"
    seqs = [base * 40] * 30 + seeded(5, 2000, 300, 90)
    k, H, m = 20, 4, 512
    exp = np.zeros(m, dtype=np.uint8)
    oracle.cbf_load(exp, seqs, k, H)
    f = abb.Filter.counting(m, H, k)
    f.insert_reads(seqs)
    assert (f.download() == exp).all()
    f.close()


def test_bits_and_cascading_fixtures(abb, golden_dir):
    reads60 = seeded(11, 3000, 1500, 60)
    edge = edge_seqs(golden_dir)
    g = np.load(os.path.join(golden_dir, "bits_m8192.npz"))
    f = abb.Filter.bits(int(g["m"]), int(g["H"]), int(g["k"]))
    f.insert_reads(edge + reads60)
    assert (f.download() == g["data"]).all()
    assert f.popCount() == int(np.unpackbits(g["data"]).sum())
    f.close()
    g = np.load(os.path.join(golden_dir, "casc_m8192_L3.npz"))
    L, m = int(g["L"]), int(g["m"])
    f = abb.Filter.cascading(m, int(g["H"]), L, int(g["k"]))
    f.insert_reads(edge + reads60 + reads60[:700])
    got = np.concatenate([f.download(l) for l in range(L)])
    assert (got == g["data"]).all()
    f.close()


def test_literal_hash_interface(abb, oracle):
    # the reference's `const uint64_t hashes[]` interface: insert / contains / minCount
    rng = np.random.default_rng(7)
    H, m = 5, 3001 * 8
    hashes = rng.integers(0, 2**64, size=(20000, H), dtype=np.uint64)
    hashes[5000:6000] = hashes[:1000]          # repeats
    hashes[7000:7100, 1] = hashes[7000:7100, 0]  # duplicate position inside one k-mer
    exp = np.zeros(m, dtype=np.uint8)
    oracle.cbf_insert_hashes(exp, hashes)
    f = abb.Filter.counting(m, H, 31, threshold=2)
    f.insert(hashes)
    assert (f.download() == exp).all()
    q = rng.integers(0, 2**64, size=(5000, H), dtype=np.uint64)
    q[:2500] = hashes[:2500]
    mn = oracle.cbf_min_hashes(exp, q)
    assert (f.minCount(q) == mn).all()
    assert (f.contains(q) == (mn >= 2)).all()
    nz, th = f.popcounts()
    assert nz == np.count_nonzero(exp) and th == np.count_nonzero(exp >= 2)
    f.close()


def test_thomas_cover_edge_cases(abb):
    # empty batch, reads shorter than k, all-N reads
    f = abb.Filter.counting(4096, 4, 25)
    assert f.insert_reads([]) == 0
    assert f.insert_reads(["", "ACGT", "N" * 100]) == 0
    assert f.popCount() == 0
    with pytest.raises(abb.AbbError):
        abb.Filter.bits(1001, 4, 25)  # BloomFilter.hpp:374-379: size must be a multiple of 8
    with pytest.raises(abb.AbbError):
        abb.Filter.counting(4096, 33, 25)  # MAX_HASHES
    with pytest.raises(abb.AbbError):
        abb.Filter.counting(4096, 4, 193)  # MAX_KMER
    f.close()


def test_e2e_counting_filter_sha(abb, golden_dir):
    # same counters as `abyss-bloom build -t counting` (reference, -j1) on the e2e read sets
    cases = json.load(open(os.path.join(golden_dir, "e2e_cases.json")))
    from abyss_b200.capi import fixed_length_reads
    for c in cases:
        rs = ReadSet.from_coverage(c["seed"], c["genome"], c["cov"], c["L"], c["err"])
        f = abb.Filter.counting(c["counters"], c["H"], c["k"], c["kc"])
        f.insert_reads(fixed_length_reads(rs.ascii(0, rs.n)))
        raw = f.download()
        assert hashlib.sha256(raw.tobytes()).hexdigest() == c["counters_sha256"], c["name"]
        assert f.popCount() == c["counters_nonzero"]
        f.close()


def test_large_roundtrip_properties(abb):
    # size-independent properties at a size the oracle would take minutes for:
    # (1) idempotent result under different window sizes, (2) every inserted k-mer has minCount >= 1,
    # (3) sum of counters <= H * n_kmers
    rs = ReadSet.from_coverage(99, 2_000_000, 20, 150, 0.005)
    from abyss_b200.capi import fixed_length_reads
    reads = fixed_length_reads(rs.ascii(0, rs.n))
    k, H, m = 64, 4, 50_000_000
    digests = []
    for w in (1 << 16, 1 << 19):
        f = abb.Filter.counting(m, H, k, 2)
        f.set_window(w)
        n = f.insert_reads(reads)
        assert n == rs.n * (150 - k + 1)
        raw = f.download()
        digests.append(hashlib.sha256(raw.tobytes()).hexdigest())
        assert int(raw.astype(np.uint64).sum()) <= H * n
        h0, valid, _ = abb.hash_reads(k, (reads[0][:150 * 2000], reads[1][:2001]))
        hh = [h0]
        mult = [np.uint64((i ^ ((k * 0x90b45d39fb6da1fa) & 0xFFFFFFFFFFFFFFFF)) & 0xFFFFFFFFFFFFFFFF) for i in range(H)]
        with np.errstate(over="ignore"):
            for j in range(1, H):
                t = h0 * mult[j]
                hh.append(t ^ (t >> np.uint64(27)))
        assert f.minCount(np.stack(hh, axis=1)).min() >= 1
        f.close()
    assert digests[0] == digests[1]


def test_reference_unit_test_vectors(abb):
    # Unittest/BloomDBG/CountingBloomFilterTest.cpp:9-46 (threshold semantics on the four 16-mers) and
    # Unittest/BloomDBG/RollingBloomDBGTest.cpp (X-graph CGACT,TGACT -> GACTC -> ACTCT,ACTCG; k=5, H=2):
    # the neighbours of every vertex as the extension kernels see them (shift + A,C,G,T + contains)
    a, b, c, d = "AGATGTGCTGCCGCCT", "TGGACAGCGTTACCTC", "TAATAACAGTCCCTAT", "GATCGTGGCGGGCGAT"
    f = abb.Filter.counting(1000, 1, 16, threshold=2)
    f.insert_reads([a, a, b])
    h0, valid, _ = abb.hash_reads(16, [a, b, c, d])
    assert valid.all()
    assert f.minCount(h0.reshape(-1, 1)).tolist() == [2, 1, 0, 0]
    assert f.contains(h0.reshape(-1, 1)).tolist() == [True, False, False, False]
    f.close()
    kmers = ["CGACT", "TGACT", "GACTC", "ACTCT", "ACTCG"]
    g = abb.Filter.counting(100000, 2, 5, threshold=1)
    g.insert_reads(kmers)
    edges = {"CGACT": ("", "C"), "TGACT": ("", "C"), "GACTC": ("CT", "GT"), "ACTCT": ("G", ""), "ACTCG": ("G", "")}
    for v, (ins, outs) in edges.items():
        cand = [x + v[:-1] for x in "ACGT"] + [v[1:] + x for x in "ACGT"]
        h, ok, _ = abb.hash_reads(5, cand)
        H = np.stack([h, (h * np.uint64(1 ^ ((5 * 0x90b45d39fb6da1fa) & (2**64 - 1))))], axis=1)
        H[:, 1] ^= H[:, 1] >> np.uint64(27)  # NTE64, nthash.hpp:337-342
        got = g.contains(H)
        want = [x in ins for x in "ACGT"] + [x in outs for x in "ACGT"]
        assert got.tolist() == want, v
    g.close()
