"""The ordered counting insert on filters larger than its conflict maps, against the sequential oracle.

Each of the insert's conflict maps has two halves: half A indexed by the position modulo its size, half B by a
multiplicative hash of the whole position.  A slot waits only when both halves say one of its positions was touched again.
These cases use literal hash rows below the filter size (a literal hash below m is its own position), so that the rows
choose exactly which positions alias in half A and which are truly shared."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

M = (1 << 27) + 8      # counters: four times the positions half A of a map can tell apart
ALIAS = 1 << 25        # positions that differ by a multiple of this share their half-A entry (and did in the one-index map)


def aliased_rows(rng, n_rows, H):
    """n_rows rows of H distinct positions each, no position in two rows, every position of row 2j sharing its position
    modulo ALIAS with the same column of row 2j + 1"""
    assert n_rows % 2 == 0
    base = rng.choice(ALIAS, size=n_rows // 2 * H, replace=False).astype(np.uint64).reshape(-1, H)
    hi = rng.integers(0, M // ALIAS, size=base.shape, dtype=np.uint64)
    step = rng.integers(1, M // ALIAS, size=base.shape, dtype=np.uint64)
    lo_row = base + np.uint64(ALIAS) * hi
    hi_row = base + np.uint64(ALIAS) * ((hi + step) % np.uint64(M // ALIAS))
    rows = np.stack([lo_row, hi_row], axis=1).reshape(-1, H)
    assert (rows < np.uint64(M)).all()
    return rows


def assert_same(got, exp, what):
    if not np.array_equal(got, exp):
        d = np.flatnonzero(got != exp)
        raise AssertionError(f"{what}: {d.size} bytes differ, first at {d[0]}: got {got[d[0]]}, oracle {exp[d[0]]}")


@pytest.mark.parametrize("H", [4, 8])
def test_aliases_of_the_position_index_do_not_carry(abb, oracle, H):
    # every position aliases a position of another row in half A, none is shared: half B tells them apart, so nearly
    # every row applies in its own window (a map indexed by the position alone carries every row).  Expected false
    # carries: H positions per row, each meeting one of the other n * H positions in half B: H^2 n / 2^24 = 0.4 %.
    rng = np.random.default_rng(4100 + H)
    rows = aliased_rows(rng, (1 << 16) // (H * H), H)
    assert np.unique(rows).size == rows.size
    exp = np.zeros(M, dtype=np.uint8)
    oracle.cbf_insert_hashes(exp, rows)
    f = abb.Filter.counting(M, H, 31)
    f.insert(rows)
    assert_same(f.download(), exp, f"H={H}")
    st = f.stats()
    assert st.deferred < len(rows) // 100, f"{st.deferred} of {len(rows)} rows carried"
    f.close()


@pytest.mark.parametrize("W", [0, 4096])
@pytest.mark.parametrize("H", [4, 5, 9])
def test_true_sharing_among_aliases(abb, oracle, H, W):
    # the aliasing rows above, plus rows that truly share counters: repeated rows, rows that share one position with an
    # aliasing row, and pairs that share only their positions 4..H-1 after rows that raised the second one's first four
    # counters (in file order the second row of a pair then raises every counter to 2).  The default window and a small
    # one, so that carries also chain from window to window.
    rng = np.random.default_rng(4200 + 10 * H + (W > 0))
    alias = aliased_rows(rng, 20000, H)
    rows = [alias]
    rows.append(alias[rng.integers(0, len(alias), size=2000)])                       # repeated rows
    share = rng.integers(0, M, size=(2000, H), dtype=np.uint64)
    share[:, rng.integers(0, H)] = alias[rng.integers(0, len(alias), size=2000), 0]   # one shared position
    rows.append(share)
    if H > 4:
        n = 2000
        a = rng.integers(0, M, size=(n, H), dtype=np.uint64)
        b = rng.integers(0, M, size=(n, H), dtype=np.uint64)
        b[:, 4:] = a[:, 4:]
        pre = rng.integers(0, M, size=(n, H), dtype=np.uint64)
        pre[:, :4] = b[:, :4]
        rows += [pre, np.stack([a, b], axis=1).reshape(-1, H)]
    rows = np.concatenate(rows)
    exp = np.zeros(M, dtype=np.uint8)
    oracle.cbf_insert_hashes(exp, rows)
    if H > 4:
        assert (exp[a[:, 4:].astype(np.int64)] >= 2).mean() > 0.9, "the case no longer depends on conflicts past the fourth position"
    f = abb.Filter.counting(M, H, 31)
    if W:
        f.set_window(W)
    f.insert(rows)
    assert_same(f.download(), exp, f"H={H} W={W}")
    assert f.stats().deferred > 0
    f.close()
