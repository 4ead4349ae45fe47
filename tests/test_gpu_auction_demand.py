"""Auction demands on the device (pm_set_ask_demand): demands of 1 change nothing; an engine with demands equals the
engine whose ask table repeats each row demand times (its twin) bit for bit through cold, eps-scaled, warm and repair
passes and table deltas; demand changes under a stored state equal the numpy checkers run from the remapped state; the
grouped result form; the reference modes ignore demands; every refusal changes nothing; scipy's optimum at 2 000 slots;
and the certificate at cfg3 workers with 25 000 asks of demands 1 / 2 / 4 / 8."""
import numpy as np
import pytest

import auction_certificate as ac
import auction_repair_checker as rp
import auction_reverse_checker as rc
import auction_warm_checker as wc
from auction_demand import offsets, remap
from protocol_b200 import abi
from protocol_b200._lib import PrimeMatchError
from test_gpu_auction_reverse import scipy_instance
from test_gpu_auction_warm import cfg3, engine, tables

pytestmark = pytest.mark.gpu

NONE = wc.NONE
AUC = abi.PM_MODE_AUCTION
REV = AUC | abi.PM_AUCTION_REVERSE
WARM = AUC | abi.PM_AUCTION_WARM
REPAIR = WARM | abi.PM_AUCTION_REPAIR
TUNES = [0, 1, 2, 8 | 32, 64 | 32, 128 | 32, 0x100 | 16]   # a spread of test_gpu_auction_warm's settings
CERT = [f for f in ac.FIELDS if f != "evals"]             # evals: T x W with demands, D x W for the twin


def fold_slots(a_slots, d):
    """{ask: sorted workers} from a slot assignment."""
    off = offsets(d)
    out = {}
    for t in range(len(d)):
        w = sorted(int(x) for x in a_slots[off[t]:off[t + 1]] if x != NONE)
        if w:
            out[t] = w
    return out


def fold_result(res):
    return {ask: list(m) for ask, m in res.groups()}


def twin_tables(t, cap, d, floors=None):
    t2 = dict(t)
    t2["asks"] = np.ascontiguousarray(np.repeat(t["asks"], d))
    return t2, np.repeat(cap, d), (None if floors is None else np.repeat(floors, d))


def snapshot(eng, with_cert=True):
    res = eng.fetch()
    price, warm, released = eng.auction_state()
    out = dict(price=price, warm=warm, released=released, rounds=res.stats["n_rounds"], rev=eng.auction_reverse_stats(),
               res=res)
    if with_cert:
        out["cert"] = eng.auction_certificate(ask_bound=True)
    return out


def assert_twin(a, b, d):
    """a: the demand engine's snapshot, b: the twin's."""
    ra, rb = a["res"], b["res"]
    twin_fold = {}
    slot_ask = np.repeat(np.arange(len(d)), d)
    for ask, m in rb.groups():
        twin_fold.setdefault(int(slot_ask[ask]), []).extend(m)
    assert fold_result(ra) == {t: sorted(m) for t, m in twin_fold.items()}
    assert np.array_equal(a["price"], b["price"])
    assert (a["warm"], a["released"], a["rounds"], a["rev"]) == (b["warm"], b["released"], b["rounds"], b["rev"])
    if "cert" in a:
        for f in CERT:
            assert a["cert"][f] == b["cert"][f], f
        assert np.array_equal(a["cert"]["ask_bound"], b["cert"]["ask_bound"][offsets(d)[:-1]])


def demands(rng, T, choices=(1, 2, 3, 4)):
    return rng.choice(choices, T).astype(np.uint32)


# ------------------------------------------------------------------ neutral
@pytest.mark.parametrize("mode", [AUC, REV])
def test_all_ones_is_no_call(mode):
    t, cap = tables(80, 900, 41)
    runs = []
    for set_ones in (False, True):
        eng = engine(t, cap)
        if set_ones:
            eng.set_ask_demand(np.ones(len(cap), dtype=np.uint32))
        eng.set_auction_params(cost_scale=1, eps_start=16 if mode == REV else 1, eps_div=4)
        snaps = []
        for m in (mode, WARM, REPAIR):
            eng.match(m)
            s = snapshot(eng)
            s["res"] = (s["res"].worker_group.copy(), s["res"].worker_ask.copy(), s["res"].group_ask.copy(),
                        s["res"].group_off.copy(), s["res"].group_members.copy(), s["res"].ask_best.copy(),
                        s["res"].ask_count.copy())
            snaps.append(s)
            cap2 = cap.copy()
            cap2[::7] += 3
            eng.set_price_caps(cap2)
        runs.append(snaps)
        eng.close()
    for a, b in zip(*runs):
        for x, y in zip(a["res"], b["res"]):
            assert np.array_equal(x, y)
        assert np.array_equal(a["price"], b["price"]) and a["cert"].keys() == b["cert"].keys()
        assert all(np.array_equal(a["cert"][k], b["cert"][k]) if k == "ask_bound" else a["cert"][k] == b["cert"][k]
                   for k in a["cert"])
        assert (a["warm"], a["released"], a["rounds"], a["rev"]) == (b["warm"], b["released"], b["rounds"], b["rev"])


# ------------------------------------------------------------------ twin
class Pair:
    """A demand engine and its twin, changed together."""

    def __init__(self, t, cap, d, tune=0, floors=None, reputation=None, S=1):
        self.t, self.cap, self.d, self.floors = t, cap.copy(), d.copy(), None if floors is None else floors.copy()
        self.a = engine(t, cap, tune=tune, floors=floors, reputation=reputation, S=S)
        self.a.set_ask_demand(d)
        t2, cap2, fl2 = twin_tables(t, cap, d, floors)
        self.b = engine(t2, cap2, tune=tune, floors=fl2, reputation=reputation, S=S)
        self.asks = t["asks"].copy()

    def set_caps(self, cap):
        self.cap = cap
        self.a.set_price_caps(cap)
        self.b.set_price_caps(np.repeat(cap, self.d))

    def set_floors(self, floors):
        self.floors = floors
        self.a.set_min_reputation(floors)
        self.b.set_min_reputation(np.repeat(floors, self.d))

    def update_asks(self, idx, rows):
        self.asks[idx] = rows
        self.a.update_asks(idx, rows, self.t["opts"])
        off = offsets(self.d)
        sidx = np.concatenate([np.arange(off[i], off[i + 1]) for i in idx]).astype(np.uint32)
        self.b.update_asks(sidx, np.repeat(rows, self.d[idx]), self.t["opts"])

    def resize_asks(self, n, added=None):
        T = len(self.d)
        if n > T:
            self.a.resize_asks(n, added, self.t["opts"])
            self.b.resize_asks(int(self.d.sum()) + n - T, added, self.t["opts"])
            self.d = np.concatenate([self.d, np.ones(n - T, dtype=np.uint32)])
            self.asks = np.concatenate([self.asks, added])
            self.cap = np.concatenate([self.cap, np.zeros(n - T, dtype=np.uint32)])
            if self.floors is not None:
                self.floors = np.concatenate([self.floors, np.zeros(n - T, dtype=np.uint32)])
        else:
            self.a.resize_asks(n)
            self.b.resize_asks(int(self.d[:n].sum()))
            self.d, self.asks, self.cap = self.d[:n], self.asks[:n], self.cap[:n]
            if self.floors is not None:
                self.floors = self.floors[:n]

    def update_workers(self, idx, a, b):
        self.a.update_workers(idx, a, b)
        self.b.update_workers(idx, a, b)

    def params(self, **kw):
        self.a.set_auction_params(**kw)
        self.b.set_auction_params(**kw)

    def check(self, mode):
        self.a.match(mode)
        self.b.match(mode)
        assert_twin(snapshot(self.a), snapshot(self.b), self.d)

    def close(self):
        self.a.close()
        self.b.close()


def random_change(p: Pair, rng):
    T, W = len(p.d), len(p.t["wa"])
    k = int(rng.integers(0, 5))
    if k == 0:
        idx = np.unique(rng.choice(W, 6, replace=False)).astype(np.uint32)
        wa, wb = p.t["wa"][idx].copy(), p.t["wb"][idx].copy()
        wb["ext_ask_price"] = rng.integers(10, 1000, len(idx)).astype(np.uint32)
        p.update_workers(idx, wa, wb)
    elif k == 1:
        cap = p.cap.copy()
        i = rng.choice(T, 3, replace=False)
        cap[i] = rng.integers(50, 1500, 3).astype(np.uint32)
        p.set_caps(cap)
    elif k == 2 and p.floors is not None:
        fl = p.floors.copy()
        fl[rng.choice(T, 2, replace=False)] = rng.integers(0, 3, 2).astype(np.uint32)
        p.set_floors(fl)
    elif k == 3:
        idx = np.unique(rng.choice(T, 2, replace=False)).astype(np.uint32)
        p.update_asks(idx, p.t["asks"][rng.choice(len(p.t["asks"]), len(idx))])
    else:
        if rng.integers(0, 2) and T > 10:
            p.resize_asks(T - 2)
        else:
            p.resize_asks(T + 2, p.t["asks"][rng.choice(len(p.t["asks"]), 2)])
            cap = p.cap.copy()
            cap[-2:] = rng.integers(50, 1500, 2).astype(np.uint32)
            p.set_caps(cap)


@pytest.mark.parametrize("tune", TUNES)
def test_twin_cold_warm_repair_chain(tune):
    t, cap = tables(60, 800, 43)
    rng = np.random.default_rng(43 + tune)
    rep = rng.integers(0, 4, 800).astype(np.uint32)
    floors = rng.integers(0, 3, 60).astype(np.uint32)
    p = Pair(t, cap, demands(rng, 60), tune=tune, floors=floors, reputation=rep)
    p.check(AUC)
    for i in range(8):
        random_change(p, rng)
        p.check(REPAIR if i % 2 else WARM)
    p.close()


@pytest.mark.parametrize("seed", [44, 45])
def test_twin_eps_scaled_reverse(seed):
    t, cap = tables(70, 900, seed)
    rng = np.random.default_rng(seed)
    p = Pair(t, cap, demands(rng, 70, (1, 2, 4, 8)), S=int(4 * 70 + 1))
    p.params(cost_scale=4 * 70 + 1, eps_start=256, eps_div=4)
    p.check(REV)
    random_change(p, rng)
    p.check(REPAIR)
    p.close()


def test_twin_duplicated_asks_ties():
    t, cap = tables(40, 600, 46, dup=(3, 50, 60))
    rng = np.random.default_rng(46)
    p = Pair(t, cap, demands(rng, len(cap)))
    p.check(AUC)
    for _ in range(4):
        random_change(p, rng)
        p.check(WARM)
    p.close()


# ------------------------------------------------------------------ demand changes
@pytest.mark.parametrize("mode", [WARM, REPAIR])
@pytest.mark.parametrize("seed", [47, 48])
def test_demand_changes_match_checkers(mode, seed):
    t, cap = tables(50, 700, seed)
    m = wc.Market(t, cap)
    F = m.F()
    ap = t["wb"]["ext_ask_price"]
    W = len(ap)
    rng = np.random.default_rng(seed)
    d = demands(rng, 50)
    eng = engine(t, cap)
    eng.set_ask_demand(d)
    a_slots, price, n = wc.cold(np.repeat(F, d, axis=0), ap, np.repeat(cap, d), 1)
    eng.match(AUC)
    assert fold_result(eng.fetch()) == fold_slots(a_slots, d)
    assert np.array_equal(eng.auction_state()[0], price)
    for step in range(5):
        d_new = d.copy()
        held = [t_ for t_, w in fold_slots(a_slots, d).items()]
        pick = rng.choice(held, 3, replace=False) if len(held) >= 3 else rng.choice(50, 3)
        for t_ in pick:                                   # grow or shrink held asks, and one unheld
            d_new[t_] = max(1, int(d_new[t_]) + int(rng.choice([-2, -1, 1, 2])))
        d_new[int(rng.integers(0, 50))] = int(rng.integers(1, 6))
        a_new, added, freed = remap(a_slots, d, d_new, n_kept=W)
        eng.set_ask_demand(d_new)
        Fx, capx = np.repeat(F, d_new, axis=0), np.repeat(cap, d_new)
        if mode == WARM:
            a_slots, price, n, rel = wc.warm(Fx, ap, capx, 1, price, a_new, W, [], added)
        else:
            out = rp.repair(Fx, ap, capx, 1, price, a_new, W, [], added)
            a_slots, price, rel = out["assigned"], out["price"], out["released"]
        eng.match(mode)
        res = eng.fetch()
        got_price, warm, released = eng.auction_state()
        assert warm and released == len(rel)
        assert fold_result(res) == fold_slots(a_slots, d_new)
        assert np.array_equal(got_price, price)
        cert = eng.auction_certificate()
        assert cert["gap"] <= int(d_new.sum()) and cert["n_bad_holds"] == 0 and cert["n_shared"] == 0
        d = d_new


def test_demand_change_then_certificate_before_pass():
    """The remapped state is certified as it stands: dropped slots' workers show as priced and unowned."""
    t, cap = tables(40, 500, 49)
    rng = np.random.default_rng(49)
    d = demands(rng, 40, (2, 3, 4))
    eng = engine(t, cap)
    eng.set_ask_demand(d)
    eng.match(AUC)
    before = eng.auction_certificate()
    eng.set_ask_demand(np.ones(40, dtype=np.uint32))
    after = eng.auction_certificate()
    assert after["n_held"] <= before["n_held"] and after["n_shared"] == 0 and after["n_bad_holds"] == 0
    eng.match(WARM)
    assert eng.auction_state()[1]
    assert eng.auction_certificate()["gap"] <= 40


# ------------------------------------------------------------------ result form
def test_result_form():
    t, cap = tables(60, 800, 50)
    rng = np.random.default_rng(50)
    d = demands(rng, 60, (1, 3, 6))
    eng = engine(t, cap)
    eng.set_ask_demand(d)
    eng.match(AUC)
    r = eng.fetch()
    ap = t["wb"]["ext_ask_price"].astype(np.int64)
    assert np.all(np.diff(r.group_ask[:r.n_groups].astype(np.int64)) > 0)   # one group per ask, ask order
    assert len(r.group_members) == int(r.group_off[r.n_groups]) == int(r.ask_count.sum())
    held = set()
    for g, (ask, m) in enumerate(r.groups()):
        assert m == sorted(m) and 1 <= len(m) <= d[ask] and r.ask_count[ask] == len(m)
        assert all(r.worker_ask[w] == ask and r.worker_group[w] == g for w in m)
        assert r.ask_best[ask] == min((int(ap[w]) << 32) | w for w in m)
        held.update(m)
    assert r.n_groups == int(np.count_nonzero(r.ask_count))
    free = np.setdiff1d(np.arange(800), list(held))
    assert np.all(r.worker_ask[free] == NONE) and np.all(r.worker_group[free] == NONE)
    assert np.all(r.ask_best[r.ask_count == 0] == abi.PM_COST_INF)


def test_reference_modes_ignore_demands():
    t, cap = tables(60, 800, 51)
    outs = []
    for dem in (False, True):
        eng = engine(t, cap)
        if dem:
            eng.set_ask_demand(np.full(60, 5, dtype=np.uint32))
        r = []
        for mode in (abi.PM_MODE_FIRST_FIT, abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED):
            eng.match(mode)
            res = eng.fetch()
            r.append((res.worker_group.copy(), res.group_ask.copy(), res.group_off.copy(), res.group_members.copy(),
                      res.ask_best.copy(), res.ask_count.copy()))
        outs.append(r)
        eng.close()
    for a, b in zip(*outs):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


# ------------------------------------------------------------------ refusals
def test_refusals_change_nothing():
    t, cap = tables(30, 400, 52)
    eng = engine(t, cap)
    d = np.full(30, 2, dtype=np.uint32)
    eng.set_ask_demand(d)
    eng.match(AUC)

    def state():
        price, warm, rel = eng.auction_state()
        return price, warm, rel, eng.table_version(), fold_result(eng.fetch()), eng.auction_certificate()

    def same(x, y):
        assert np.array_equal(x[0], y[0]) and x[1:5] == y[1:5]
        assert all(x[5][k] == y[5][k] for k in ac.FIELDS)

    s0 = state()
    bad = [np.full(29, 1, dtype=np.uint32), np.concatenate([np.zeros(1), np.ones(29)]).astype(np.uint32),
           np.full(30, (1 << 30) // 30 + 1, dtype=np.uint32)]
    for arr in bad:
        with pytest.raises(PrimeMatchError) as ei:
            eng.set_ask_demand(arr)
        assert ei.value.status == abi.PM_E_INVALID
        same(state(), s0)
    assert eng._lib.pm_set_ask_demand(eng._h, None, 30) == abi.PM_E_INVALID
    same(state(), s0)
    with pytest.raises(PrimeMatchError) as ei:
        eng.auction_assignment()
    assert ei.value.status == abi.PM_E_UNSUPPORTED
    with pytest.raises(PrimeMatchError) as ei:
        eng.auction_restore(s0[0], np.full(30, NONE, dtype=np.uint32))
    assert ei.value.status == abi.PM_E_UNSUPPORTED
    same(state(), s0)
    eng.close()
    # growth that would take D to 2^30 (an engine without a stored state: nothing of that size is allocated)
    fresh = engine(t, cap)
    fresh.set_ask_demand(np.concatenate([[(1 << 30) - 31], np.ones(29)]).astype(np.uint32))
    v = fresh.table_version()
    with pytest.raises(PrimeMatchError) as ei:
        fresh.resize_asks(32, t["asks"][:2], t["opts"])
    assert ei.value.status == abi.PM_E_INVALID and fresh.table_version() == v
    fresh._lib.pm_set_asks(fresh._h, None, 0, None, 0)
    assert fresh._lib.pm_set_ask_demand(fresh._h, None, 0) == abi.PM_OK
    fresh.close()


def test_no_ask_table_is_state():
    from protocol_b200.engine import Engine
    eng = Engine()
    with pytest.raises(PrimeMatchError) as ei:
        eng.set_ask_demand(np.ones(3, dtype=np.uint32))
    assert ei.value.status == abi.PM_E_STATE
    eng.close()


# ------------------------------------------------------------------ anchors
def test_scipy_optimum_at_2000_slots():
    T, W = 500, 2000
    t, cap = scipy_instance(T, W, 7)
    rng = np.random.default_rng(7)
    d = demands(rng, T, (2, 4, 6))
    D = int(d.sum())
    m = wc.Market(t, cap)
    Fx, capx = np.repeat(m.F(), d, axis=0), np.repeat(cap, d)
    ap = t["wb"]["ext_ask_price"]
    opt = rc.optimum(Fx, ap, capx)
    eng = engine(t, cap)
    eng.set_ask_demand(d)
    for S, exact in ((1, False), (D + 1, True)):
        eng.set_auction_params(cost_scale=S, eps_start=max(1, S // 8), eps_div=4)
        eng.match(REV)
        a = np.full(D, NONE, dtype=np.uint32)
        off = offsets(d)
        for ask, mem in eng.fetch().groups():
            a[off[ask]:off[ask] + len(mem)] = mem
        wc.check_feasible_injective(Fx, a)
        cost = wc.total_cost(a, ap, capx)
        assert cost == opt if exact else opt <= cost <= opt + D
        cert = eng.auction_certificate()
        assert cert["gap"] <= D * 1 and cert["cost"] == cost * S
    eng.close()


def test_certificate_at_cfg3_workers():
    t, cap = cfg3()
    T = 25_000
    t = dict(t)
    t["asks"] = np.ascontiguousarray(t["asks"][:T])
    cap = cap[:T]
    d = np.random.default_rng(53).choice([1, 2, 4, 8], T).astype(np.uint32)
    eng = engine(t, cap)
    eng.set_ask_demand(d)
    eng.match(AUC)
    cert = eng.auction_certificate()
    assert cert["n_bad_holds"] == 0 and cert["n_shared"] == 0
    assert cert["gap"] <= int(d.sum())
    r = eng.fetch()
    assert len(r.group_members) == cert["n_held"] and np.all(r.ask_count <= d)
    eng.close()
