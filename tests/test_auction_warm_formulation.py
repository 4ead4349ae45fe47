"""The auction's warm start (PM_AUCTION_WARM, DESIGN 4) on the CPU: the release rule restated in numpy against the
sequential checker (tests/auction_warm_checker.py), its independence of order, and the guarantee a warm pass keeps —
within T * eps of the optimum of the current instance, the optimum itself with cost_scale = T + 1 — over random
histories of row writes, resizes, cap and floor changes and toggles.  Also: a warm pass repairs what eps-scaling
leaves behind."""
import numpy as np
import pytest

import auction_warm_checker as wc
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth

NONE = wc.NONE


def market(T, W, seed, floors=False):
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed, price="loguniform")
    a = synth.make_asks(T, "mixed", seed=synth.SEED_ASKS + seed)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    rng = np.random.default_rng(seed)
    cap = rng.integers(20, 120, T).astype(np.uint32)
    t = dict(wa=w.a, wb=w.b, asks=a.asks, opts=a.opts, bits=bits, words=words)
    rep = rng.integers(0, 4, W).astype(np.uint32) if floors else None
    fl = rng.integers(0, 3, T).astype(np.uint32) if floors else None
    return wc.Market(t, cap, rep, fl)


def lsa_optimum(price, cap, feasible, scale=1):
    """Minimum total cost (price * scale of the worker, or the outside option (cap + 1) * scale) over injective
    assignments of feasible pairs — scipy's Hungarian solver, an anchor outside this repository's code (restated from
    tests/test_oracle_auction.py)."""
    from scipy.optimize import linear_sum_assignment

    T, W = feasible.shape
    BIG = 1 << 40
    C = np.full((T, W + T), BIG, dtype=np.int64)
    ok = feasible & (price[None, :] <= cap[:, None])
    C[:, :W][ok] = np.broadcast_to(price[None, :].astype(np.int64) * scale, (T, W))[ok]
    C[np.arange(T), W + np.arange(T)] = (cap.astype(np.int64) + 1) * scale
    r, c = linear_sum_assignment(C)
    return int(C[r, c].sum())


def release_numpy(F, ap, S, price, assigned, n_kept, rows, asks):
    """Steps 1-3 as whole-array operations: the initial release, then the closure as a fixpoint over all raised
    workers at once (every still-assigned ask against every raised worker, until no ask is released)."""
    T, W = F.shape
    keep = min(n_kept, W)
    p = np.zeros(W, dtype=np.int64)
    p[:keep] = price[:keep]
    a = assigned.astype(np.int64)
    a[a == NONE] = -1
    rel = np.zeros(T, dtype=bool)
    rel |= a >= keep
    rows_mask = np.zeros(W, dtype=bool)
    rows_mask[[r for r in rows if r < W]] = True
    rows_mask[keep:] = True
    held = a >= 0
    rel |= held & rows_mask[np.where(held & (a < W), a, 0)] & (a < W)
    rel[list(asks)] = True
    rel &= held
    owned = np.zeros(W, dtype=bool)
    owned[a[held & ~rel]] = True
    raised = (~owned & (p != 0)) | rows_mask
    p[~owned] = 0
    a[rel] = -1
    apl = ap.astype(np.int64)
    while True:
        v = -(apl * S) - p
        hold = np.flatnonzero(a >= 0)
        vt = v[a[hold]]
        better = F[hold][:, raised] & ((v[raised] - 1)[None, :] > vt[:, None])
        hit = hold[better.any(axis=1)]
        if len(hit) == 0:
            break
        ws = a[hit]
        rel[hit] = True
        a[hit] = -1
        p[ws] = 0
        raised = np.zeros(W, dtype=bool)
        raised[ws] = True
    return p, np.flatnonzero(rel)


@pytest.mark.parametrize("T,W,seed", [(30, 120, 1), (60, 90, 2), (25, 400, 3)])
def test_checker_rounds_restate_the_oracle(T, W, seed):
    """The checker's rounds from an empty state are orc_soa_auction: assignment, prices and rounds, at two scales."""
    m = market(T, W, seed, floors=seed == 2)
    F = m.F()
    for S in (1, T + 1):
        a, p, n = wc.cold(F, m.wb["ext_ask_price"], m.cap, S)
        want, price, rounds = orc.soa_auction(m.wa, m.wb, m.asks, m.opts, m.bits, m.words, m.cap, cost_scale=S,
                                              reputation=m.reputation, min_reputation=m.floors)
        assert np.array_equal(a, want) and np.array_equal(p, price) and n == rounds


def run_history(m, rng, S, steps, check):
    a, p, _ = m.cold(S)
    m.store(p, a)
    for _ in range(steps):
        for _ in range(int(rng.integers(1, 3))):
            wc.random_step(m, rng)
        check(m)
        a, p, n, rel = m.warm(S)
        F = m.F()
        wc.check_feasible_injective(F, a)
        opt = lsa_optimum(m.wb["ext_ask_price"].astype(np.int64), m.cap, F)
        got = wc.total_cost(a, m.wb["ext_ask_price"], m.cap)
        T = len(m.asks)
        if S == 1:
            assert opt <= got <= opt + T, (opt, got)
        else:
            assert got == opt, (opt, got)
        assert np.all(p[np.setdiff1d(np.arange(m.n_workers), a[a != NONE])] == 0)   # unowned workers: price 0
        m.store(p, a)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("S_mode", ["unit", "exact"])
def test_release_restated_and_warm_results_optimal(seed, S_mode):
    T, W = 40, 150
    m = market(T, W, 10 + seed, floors=seed % 2 == 1)
    S = 1 if S_mode == "unit" else T + 1
    rng = np.random.default_rng(100 + seed)

    def check(m):
        F = m.F()
        ap = m.wb["ext_ask_price"]
        p, a, rel, R = wc.release(F, ap, S, m.price, m.assigned, m.n_kept, m.changed_rows(), m.changed_asks())
        p2, rel2 = release_numpy(F, ap, S, m.price, m.assigned, m.n_kept, m.changed_rows(), m.changed_asks())
        assert np.array_equal(rel, rel2) and np.array_equal(p, p2)
        # the least fixpoint does not depend on the order the raised workers are taken in
        for k in range(3):
            perm_rows = rng.permutation(m.changed_rows()).tolist()
            perm_asks = rng.permutation(m.changed_asks()).tolist()
            p3, _, rel3, _ = wc.release(F, ap, S, m.price, m.assigned, m.n_kept, perm_rows, perm_asks)
            assert np.array_equal(rel3, rel) and np.array_equal(p3, p)

    run_history(m, rng, S, 12, check)


def test_history_covers_every_kind_of_change():
    m = market(40, 150, 7, floors=True)
    rng = np.random.default_rng(7)
    a, p, _ = m.cold(1)
    m.store(p, a)
    seen = set()
    for _ in range(60):
        seen.add(wc.random_step(m, rng))
    assert seen == {"price", "flags", "spec", "resize", "caps", "floors", "toggle", "reputation"}


@pytest.mark.parametrize("seed", range(3))
def test_no_change_returns_the_stored_state(seed):
    m = market(50, 120, 20 + seed)
    a, p, _ = m.cold(1)
    m.store(p, a)
    a2, p2, n, rel = m.warm(1)
    assert np.array_equal(a2, a) and np.array_equal(p2, p) and len(rel) == 0
    assert n <= 1 and (n == 1) == bool((a == NONE).any())   # the unassigned asks withdraw again in round 1


@pytest.mark.parametrize("seed", range(3))
def test_warm_pass_repairs_an_eps_scaled_state(seed):
    """An eps_start = 64 pass leaves unowned workers at inflated prices and asks withdrawn at them: one warm pass with
    no changes resets those prices, releases what they disturb and meets the T * eps bound (the optimum with
    cost_scale = T + 1)."""
    T, W = 60, 200
    m = market(T, W, 30 + seed)
    F = m.F()
    ap = m.wb["ext_ask_price"].astype(np.int64)
    opt = lsa_optimum(ap, m.cap, F)
    for S in (1, T + 1):
        a, p, _ = orc.soa_auction(m.wa, m.wb, m.asks, m.opts, m.bits, m.words, m.cap, cost_scale=S, eps_start=64, eps_div=4)
        m.store(p, a)
        a2, p2, _, _ = m.warm(S)
        wc.check_feasible_injective(F, a2)
        got = wc.total_cost(a2, ap, m.cap)
        assert (opt <= got <= opt + T) if S == 1 else got == opt, (S, opt, got)
