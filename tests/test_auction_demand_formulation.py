"""Ask demands (pm_set_ask_demand) restated on the CPU, against the numpy checkers run on the twin instance, whose ask
table repeats row t demand[t] times (np.repeat of F's rows and of the caps):

* the demand remap of a stored state keeps feasible, unshared, eps-CS holds, and warm and repair passes from it end
  within D of scipy's optimum of the twin instance, and on it with cost_scale = D + 1;
* the per-ask certificate (one row term per ask, weighted by its demand; holds, costs and slacks per slot) equals the
  twin's certificate on random and adversarial states;
* the fold of a slot assignment to groups (counts per ask, their scan, members gathered and sorted) equals a direct fold.
"""
import numpy as np
import pytest

import auction_certificate as ac
from auction_demand import demand_certificate, fold_like_device, offsets, remap
import auction_repair_checker as rp
import auction_reverse_checker as rc
import auction_warm_checker as wc

NONE = wc.NONE


def random_instance(T, W, seed, density=0.3):
    rng = np.random.default_rng(seed)
    F = rng.random((T, W)) < density
    ap = rng.integers(1, 40, W).astype(np.uint32)
    cap = rng.integers(5, 50, T).astype(np.uint32)
    d = rng.integers(1, 5, T).astype(np.uint32)
    return F, ap, cap, d, rng


def new_demands(d, rng):
    d2 = d.copy()
    for t in rng.choice(len(d), max(1, len(d) // 4), replace=False):
        d2[t] = max(1, int(d2[t]) + int(rng.choice([-3, -2, -1, 1, 2, 3])))
    return d2


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("S_exact", [False, True])
def test_remapped_state_warm_and_repair(seed, S_exact):
    F, ap, cap, d, rng = random_instance(12, 40, seed)
    Fx, capx = np.repeat(F, d, axis=0), np.repeat(cap, d)
    S = int(d.sum()) + 1 if S_exact else 1
    a, p, _ = wc.cold(Fx, ap, capx, S)
    d2 = new_demands(d, rng)
    a2, added, _ = remap(a, d, d2)
    Fx2, capx2 = np.repeat(F, d2, axis=0), np.repeat(cap, d2)
    D2 = int(d2.sum())
    # kept holds: feasible, unshared, and eps-CS against every worker at the stored prices
    wc.check_feasible_injective(Fx2, a2)
    rp.check_held_eps_cs(Fx2, ap, capx2, S, p, a2)
    assert all(a2[s] == NONE for s in added)
    opt = rc.optimum(Fx2, ap, capx2, S)
    aw, pw, _, _ = wc.warm(Fx2, ap, capx2, S, p, a2, len(ap), [], added)
    out = rp.repair(Fx2, ap, capx2, S, p, a2, len(ap), [], added, check=True)
    for got in (aw, out["assigned"]):
        wc.check_feasible_injective(Fx2, got)
        cost = wc.total_cost(got, ap, capx2) * S
        assert opt <= cost <= opt + D2
        if S_exact:
            assert cost == opt


def assert_same_certificate(F, ap, cap, d, S, price, a_slots):
    got = demand_certificate(F, ap, cap, d, S, price, a_slots)
    want = ac.certificate(np.repeat(F, d, axis=0), ap, np.repeat(cap, d), S, price, a_slots)
    for f in ac.FIELDS:
        if f != "evals":   # T x W here, D x W for the twin: the sweep stays per ask
            assert got[f] == want[f], f
    assert np.array_equal(got["ask_bound"], want["ask_bound"][offsets(d)[:-1]])


@pytest.mark.parametrize("seed", range(8))
def test_weighted_certificate_equals_twin_random(seed):
    F, ap, cap, d, rng = random_instance(10, 30, 100 + seed)
    S = int(rng.integers(1, 5))
    D = int(d.sum())
    a, p, _ = wc.cold(np.repeat(F, d, axis=0), ap, np.repeat(cap, d), S)
    assert_same_certificate(F, ap, cap, d, S, p, a)
    # random states: any prices, any assignment (infeasible, shared and out-of-range holds included)
    for _ in range(5):
        price = rng.integers(0, 60 * S, len(ap)).astype(np.int64)
        a_r = rng.integers(0, len(ap) + 3, D).astype(np.uint32)
        a_r[rng.random(D) < 0.3] = NONE
        assert_same_certificate(F, ap, cap, d, S, price, a_r)


def test_weighted_certificate_equals_twin_adversarial():
    F, ap, cap, d, rng = random_instance(8, 20, 7, density=0.5)
    D = int(d.sum())
    zero = np.zeros(len(ap), dtype=np.int64)
    for a in (np.full(D, NONE, dtype=np.uint32),            # nothing held
              np.zeros(D, dtype=np.uint32),                 # every slot on worker 0
              np.arange(D, dtype=np.uint32) % len(ap)):     # every slot holding, feasible or not
        for price in (zero, np.full(len(ap), 1 << 40, dtype=np.int64)):
            assert_same_certificate(F, ap, cap, d, 3, price, a)
    F0 = np.zeros_like(F)                                   # no feasible pair: every row term is the outside option
    assert_same_certificate(F0, ap, cap, d, 2, zero, np.full(D, NONE, dtype=np.uint32))


@pytest.mark.parametrize("seed", range(5))
def test_fold_to_groups(seed):
    F, ap, cap, d, rng = random_instance(15, 50, 200 + seed)
    a, _, _ = wc.cold(np.repeat(F, d, axis=0), ap, np.repeat(cap, d), 1)
    group_ask, group_off, members, count, best = fold_like_device(a, d, ap)
    off = offsets(d)
    direct = {t: sorted(int(w) for w in a[off[t]:off[t + 1]] if w != NONE) for t in range(len(d))}
    direct = {t: m for t, m in direct.items() if m}
    assert list(group_ask) == sorted(direct)
    for g, t in enumerate(group_ask):
        assert members[group_off[g]:group_off[g + 1]].tolist() == direct[t]
    assert all(count[t] == len(direct.get(t, [])) for t in range(len(d)))
    assert all(best[t] == (min((int(ap[w]) << 32) | w for w in direct[t]) if t in direct else np.iinfo(np.int64).max)
               for t in range(len(d)))
    ones = np.ones(len(d), dtype=np.uint32)                 # demands of 1: one solo group per held ask, ask order
    a1, _, _ = wc.cold(F, ap, cap, 1)
    ga, go, mem, _, _ = fold_like_device(a1, ones, ap)
    held = np.flatnonzero(a1 != NONE)
    assert np.array_equal(ga, held) and np.array_equal(go, np.arange(len(held) + 1)) and np.array_equal(mem, a1[held])
