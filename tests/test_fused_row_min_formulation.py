"""The fused first-fit pass's per-ask row minimum (pm_kernels.cuh pm_fused_eval<.., STATS = true>), restated in numpy
and held against the packed cost it must reproduce.

ask_best is the signed int64 least (price << 32) | worker over the workers that meet the ask, PM_COST_INF when none
does: the value pm_argmin reads off the materialised tile and the oracle computes.  The fused kernel never forms that
int64 per pair.  A CTA owns 1024 consecutive workers, a warp 128 of them and a lane the 4 consecutive workers
4l .. 4l+3 (k = 0..3).  Per row and warp:
  1. each lane takes the least price of its feasible workers read as int32, or INT32_MAX when it has none;
  2. a signed min reduction over the 32 lanes gives the warp's least price p;
  3. one ballot per k of "feasible and price == p" gives the lowest worker at that price, (ffs(ballot) - 1) * 4 + k;
  4. lane 0 merges (uint32(p) << 32) | worker into the row's shared int64 with a signed atomicMin, and the CTA merges
     its rows into ask_best the same way.
Reading the price as int32 is what keeps this equal to the int64 order for prices of 2^31 and above."""
import numpy as np
import pytest

U32, I32, U64, I64 = np.uint32, np.int32, np.uint64, np.int64
K_INF = 0x7FFFFFFFFFFFFFFF
NONE = 0xFFFFFFFF
WPT, LANES, WARPS = 4, 32, 8
CTA_COLS = WPT * LANES * WARPS    # 1024 workers per CTA stripe


def packed_min(feasible, price, w0):
    """The definition: min over feasible workers of the signed packed cost."""
    T, nw = feasible.shape
    cost = ((price.astype(U64) << U64(32)) | (np.arange(nw, dtype=U64) + U64(w0))).view(I64)
    return np.where(feasible, cost[None, :], I64(K_INF)).min(1, initial=K_INF).astype(I64), feasible.sum(1).astype(U32)


def fused_row_min(feasible, price, w0, lane_min=np.min, signed=True, with_price=True):
    """The kernel's decomposition.  `signed=False` (an unsigned price reduction) and `with_price=False` (the lowest
    feasible worker alone) are the two ways it can go wrong; the tests check that the cases tell them apart."""
    T, nw = feasible.shape
    n_cta = (nw + CTA_COLS - 1) // CTA_COLS
    f = np.zeros((T, n_cta * CTA_COLS), dtype=bool)
    f[:, :nw] = feasible
    pr = np.zeros(n_cta * CTA_COLS, dtype=U32)   # columns past the table: null workers, never feasible, price 0
    pr[:nw] = price
    f = f.reshape(T, n_cta, WARPS, LANES, WPT)
    pr = pr.reshape(1, n_cta, WARPS, LANES, WPT)
    if not with_price:
        pr = np.zeros_like(pr)
    key = pr.view(I32).astype(I64) if signed else pr.astype(I64)
    top = np.iinfo(I32).max if signed else 0xFFFFFFFF
    lane_least = lane_min(np.where(f, key, top), axis=4)                  # 1. [T, cta, warp, lane]
    p = lane_least.min(axis=3)                                             # 2. redux.sync min over the warp
    cnt = f.sum(axis=(3, 4)).astype(U32)                                   #    redux.sync add
    hit = f & (key == p[..., None, None])
    ballot = (hit.astype(U64) << np.arange(LANES, dtype=U64)[:, None]).sum(axis=3)   # 3. [T, cta, warp, k]
    lowest = ballot & (~ballot + U64(1))
    ffs = np.where(ballot != 0, np.log2(np.maximum(lowest, 1).astype(np.float64)).astype(I64) + 1, 0)
    off = np.where(ballot != 0, (ffs - 1) * WPT + np.arange(WPT), NONE).min(axis=3)
    warp_gw0 = (U64(w0) + (np.arange(n_cta, dtype=U64)[:, None] * CTA_COLS + np.arange(WARPS, dtype=U64) * 128))
    word = (p.astype(I64).astype(U64) & U64(0xFFFFFFFF)) << U64(32)
    cand = (word | (warp_gw0[None] + off.astype(U64))).view(I64)
    cand = np.where(cnt > 0, cand, I64(K_INF))                              # 4. lane 0 only when the warp saw one
    s_best = cand.min(axis=2)                                               #    signed atomicMin in shared memory
    return s_best.min(axis=1).astype(I64), cnt.sum(axis=(1, 2)).astype(U32)   # signed atomicMin into ask_best


EDGES = (0x7FFFFFFE, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF)


def prices(kind, nw, rng):
    if kind == "zero":
        return np.zeros(nw, dtype=U32)
    if kind == "equal":
        return np.full(nw, 123_457, dtype=U32)
    if kind == "ties":        # four price levels: several lanes of a warp hold the least
        return (100 + rng.integers(0, 4, nw)).astype(U32)
    if kind == "edges":       # the int32 boundary mixed with small prices
        p = rng.integers(0, 50, nw).astype(U32)
        at = rng.choice(nw, size=min(nw, 4 * len(EDGES) * max(1, nw // 500)), replace=False)
        p[at] = np.resize(np.array(EDGES, dtype=U32), len(at))
        return p
    raise ValueError(kind)


SHAPES = [(17, 1, 0.5, 0), (23, 127, 0.2, 0), (19, 1025, 0.05, 0), (13, 3000, 0.3, 5000), (11, 4099, 0.002, 123_457),
          (7, 2048, 0.95, 1)]


@pytest.mark.parametrize("T,nw,density,w0", SHAPES)
@pytest.mark.parametrize("kind", ["zero", "equal", "ties", "edges"])
def test_fused_row_min_equals_packed_min(T, nw, density, w0, kind):
    rng = np.random.default_rng(T * 1009 + nw)
    feasible = rng.random((T, nw)) < density
    price = prices(kind, nw, rng)
    got = fused_row_min(feasible, price, w0)
    want = packed_min(feasible, price, w0)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_no_feasible_worker_leaves_the_row_at_infinity():
    rng = np.random.default_rng(5)
    for kind in ("zero", "edges"):
        feasible = np.zeros((9, 2500), dtype=bool)
        feasible[3, 1700] = True
        best, cnt = fused_row_min(feasible, prices(kind, 2500, rng), 77)
        assert (best[np.arange(9) != 3] == K_INF).all() and cnt.tolist() == [0, 0, 0, 1, 0, 0, 0, 0, 0]
        assert int(best[3]) & 0xFFFFFFFF == 77 + 1700


def test_equal_prices_break_by_the_lowest_worker_across_lanes_warps_and_ctas():
    """All prices equal: the row minimum is the lowest feasible worker, wherever it sits in the CTA decomposition."""
    nw, w0 = 3000, 10
    feasible = np.zeros((5, nw), dtype=bool)
    feasible[0, [2047, 1030, 1029]] = True     # two CTAs, lanes 1 and 1 (k = 1 and 2) of one warp
    feasible[1, [127, 128]] = True              # the last worker of warp 0, the first of warp 1
    feasible[2, [6, 5, 4]] = True               # one lane, k = 0..2
    feasible[3, [1023, 2999]] = True
    feasible[4, [2999]] = True
    best, cnt = fused_row_min(feasible, np.full(nw, 0x80000000, dtype=U32), w0)
    assert [int(x) & 0xFFFFFFFF for x in best] == [w0 + 1029, w0 + 127, w0 + 4, w0 + 1023, w0 + 2999]
    assert (best < 0).all() and cnt.tolist() == [3, 2, 3, 2, 1]


def test_the_least_price_beats_a_lower_worker_and_2_31_orders_first():
    nw = 1100
    feasible = np.zeros((4, nw), dtype=bool)
    feasible[:, [3, 500, 1050]] = True
    price = np.full(nw, 7, dtype=U32)
    price[[3, 500, 1050]] = [9, 8, 8]
    rows = [price.copy() for _ in range(4)]
    rows[1][1050] = 0x80000000      # negative packed cost: the least
    rows[2][500] = 0xFFFFFFFF       # -1 as int32: below 8, above 0x80000000
    rows[3][3] = 0x7FFFFFFF         # the int32 maximum: the most expensive feasible worker
    want = [(8, 500), (0x80000000, 1050), (0xFFFFFFFF, 500), (8, 500)]
    for p, (wp, ww) in zip(rows, want):
        best, _ = fused_row_min(feasible[:1], p, 0)
        assert int(best[0]) == int(np.array([(wp << 32) | ww], dtype=U64).view(I64)[0])
        assert np.array_equal(best, packed_min(feasible[:1], p, 0)[0])


def test_the_cases_tell_the_wrong_reductions_apart():
    """An unsigned price reduction differs once a feasible price is >= 2^31; dropping the price differs on any
    nonzero price that is not every row's least."""
    rng = np.random.default_rng(11)
    T, nw, w0 = 29, 3000, 5000
    feasible = rng.random((T, nw)) < 0.2
    for kind, wrong in (("edges", dict(signed=False)), ("edges", dict(with_price=False)),
                        ("ties", dict(with_price=False))):
        price = prices(kind, nw, np.random.default_rng(3))
        want = packed_min(feasible, price, w0)[0]
        assert np.array_equal(fused_row_min(feasible, price, w0)[0], want)
        assert not np.array_equal(fused_row_min(feasible, price, w0, **wrong)[0], want), (kind, wrong)
