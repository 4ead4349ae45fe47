"""The 32-bit cost tile of the materialised first-fit pass (pm_kernels.cuh build_fast<.., FOLD>, which pm_build_argmin
runs), restated in numpy and held against the int64 tile it replaces.

The int64 element is (price << 32) | (w0 + column) when the worker meets the ask and 0x7FFFFFFF_FFFFFFFF when not.
The narrow element keeps only the high word — price, or 0x7FFFFFFF — formed as b * (0x7FFFFFFF - price) + price with
b = 1 for an infeasible pair; the reader adds the column back.  Read back a lane at a time — 4 consecutive columns per
128-bit load and S such loads per row, (least word, its first column) kept with a strict "<", the packed int64 formed
once per lane and row — the word tile gives the int64 fold's ask_best, ask_count and first_ask: the narrow element
loses nothing.  Only prices below 0x7FFFFFFF may take the narrow tile."""
import numpy as np
import pytest

U32, I64 = np.uint32, np.int64
SENTINEL = 0x7FFFFFFF
K_INF = 0x7FFFFFFFFFFFFFFF
NONE = 0xFFFFFFFF
S, LANES, CPL = 8, 32, 4          # the lane read-back: a warp slice is S * 128 columns
CTA_COLS = 1024                   # the build kernel's stripe: ld is a multiple of it


def ld_of(nw):
    return (nw + CTA_COLS - 1) // CTA_COLS * CTA_COLS


def wide_tile(feasible, price, w0):
    """int64 [T, ld]; padding columns (>= nw) are a null worker: infeasible."""
    T, nw = feasible.shape
    ld = ld_of(nw)
    hi = np.full((T, ld), SENTINEL, dtype=np.uint64)
    lo = np.full((T, ld), 0xFFFFFFFF, dtype=np.uint64)
    cols = np.arange(nw, dtype=np.uint64) + np.uint64(w0)
    hi[:, :nw] = np.where(feasible, price.astype(np.uint64)[None, :], SENTINEL)
    lo[:, :nw] = np.where(feasible, cols[None, :], 0xFFFFFFFF)
    return ((hi << np.uint64(32)) | lo).view(I64)


def narrow_tile(feasible, price):
    """uint32 [T, ld] as the build kernel forms it: one multiply-add per element, b = 1 when infeasible."""
    T, nw = feasible.shape
    out = np.full((T, ld_of(nw)), SENTINEL, dtype=U32)
    b = (~feasible).astype(U32)
    p = price.astype(U32)[None, :]
    with np.errstate(over="ignore"):
        out[:, :nw] = b * (U32(SENTINEL) - p) + p
    return out


def fold_wide(tile, t0, w0, nw):
    T = tile.shape[0]
    feas = tile != K_INF
    best = np.where(feas.any(1), tile.min(1), K_INF).astype(I64)
    count = feas.sum(1).astype(U32)
    rows = np.where(feas, np.arange(T, dtype=np.uint64)[:, None] + np.uint64(t0), NONE)
    first = rows.min(0).astype(U32)[:nw]
    return best, count, first


def fold_narrow(words, t0, w0, nw):
    """The kernel's decomposition: per lane (least word, first column) over its S*4 columns, packed, then min."""
    T, ld = words.shape
    slice_cols = S * LANES * CPL
    padded = np.full((T, (ld + slice_cols - 1) // slice_cols * slice_cols), SENTINEL, dtype=U32)   # col < ld guard
    padded[:, :ld] = words
    n_slices = padded.shape[1] // slice_cols
    # column of (slice, s, lane, j): slice * S*128 + s * 128 + lane * 4 + j
    v = padded.reshape(T, n_slices, S, LANES, CPL).transpose(0, 1, 3, 2, 4).reshape(T, n_slices, LANES, S * CPL)
    off = (np.arange(S)[:, None] * LANES * CPL + np.arange(CPL)[None, :]).reshape(-1)          # lane-relative, increasing
    best = np.full(T, K_INF, dtype=I64)
    count = (words != SENTINEL).sum(1).astype(U32)
    for t in range(T):
        for sl in range(n_slices):
            for lane in range(LANES):
                bw, bc = SENTINEL, 0
                for k, x in enumerate(v[t, sl, lane]):
                    if x < bw:                       # strict: the first of equal words is kept
                        bw, bc = int(x), int(off[k])
                if bw != SENTINEL:
                    col = sl * slice_cols + lane * CPL + bc
                    best[t] = min(best[t], (bw << 32) | (w0 + col))
    feas = words[:, :nw] != SENTINEL
    first = np.where(feas, np.arange(T, dtype=np.uint64)[:, None] + np.uint64(t0), NONE).min(0).astype(U32)
    return best, count, first


def narrow_allowed(prices):
    """The engine's width selection (pm_check_worker_ranges): every price below the sentinel."""
    return bool((np.asarray(prices, dtype=np.uint64) < SENTINEL).all())


def case(seed, T, nw, density, special=()):
    rng = np.random.default_rng(seed)
    feasible = rng.random((T, nw)) < density
    price = rng.integers(0, 2000, nw).astype(U32)
    price[rng.random(nw) < 0.2] = 0
    for i, p in enumerate(special):
        price[(i * 7919) % nw] = p
    dup = rng.integers(0, nw, nw // 4)
    price[dup] = price[dup[::-1]]                    # many equal prices: ties broken by the column
    return feasible, price


@pytest.mark.parametrize("T,nw,density,w0", [(37, 1, 0.5, 0), (19, 1023, 0.01, 0), (23, 1025, 0.3, 5000),
                                              (11, 4099, 0.001, 123_457), (7, 9000, 0.9, 1), (5, 300, 0.0, 77)])
def test_narrow_fold_equals_wide_fold(T, nw, density, w0):
    feasible, price = case(T * 131 + nw, T, nw, density, special=(0, 0x7FFFFFFE, 0x7FFFFFFE, 1))
    assert narrow_allowed(price)
    t0 = 4096
    wb, wc, wf = fold_wide(wide_tile(feasible, price, w0), t0, w0, nw)
    nb, nc, nf = fold_narrow(narrow_tile(feasible, price), t0, w0, nw)
    assert np.array_equal(nb, wb) and np.array_equal(nc, wc) and np.array_equal(nf, wf)


def test_narrow_word_is_the_wide_high_word():
    feasible, price = case(3, 13, 2100, 0.4, special=(0x7FFFFFFE, 0))
    wide = wide_tile(feasible, price, 999).view(np.uint64)
    assert np.array_equal((wide >> np.uint64(32)).astype(U32), narrow_tile(feasible, price))


def test_all_equal_prices_pick_the_first_column():
    T, nw = 3, 5000
    feasible = np.zeros((T, nw), dtype=bool)
    feasible[0, [4095, 17, 4096]] = True
    feasible[1, [1023, 1024]] = True
    feasible[2, -1] = True
    price = np.full(nw, 0x7FFFFFFE, dtype=U32)
    nb, nc, _ = fold_narrow(narrow_tile(feasible, price), 0, 10, nw)
    assert [int(x) & 0xFFFFFFFF for x in nb] == [10 + 17, 10 + 1023, 10 + nw - 1]
    assert nc.tolist() == [3, 2, 1]


@pytest.mark.parametrize("bad", [0x7FFFFFFF, 0x80000000, 0xFFFFFFFF])
def test_width_selection_rejects_prices_the_word_cannot_hold(bad):
    """At 0x7FFFFFFF a feasible worker reads as the sentinel; at >= 2^31 the int64 tile orders it first (signed).
    Either way the narrow fold would differ, so such a table keeps the int64 tile."""
    feasible, price = case(11, 9, 700, 0.5)
    assert narrow_allowed(price)
    price[42] = bad
    feasible[:, 42] = True
    assert not narrow_allowed(price)
    wide = fold_wide(wide_tile(feasible, price, 0), 0, 0, 700)
    narrow = fold_narrow(narrow_tile(feasible, price), 0, 0, 700)
    assert not all(np.array_equal(a, b) for a, b in zip(wide, narrow))
    price[42] = 0x7FFFFFFE
    assert narrow_allowed(price)
