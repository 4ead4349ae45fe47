"""pm_auction_restore / pm_auction_assignment on the device: a state exported from one engine and restored into a fresh
one with the same tables carries every later pass bit for bit (results, prices, pm_auction_state, reverse stats,
rounds) under every PM_TUNE_AUCTION setting the warm tests use; adversarial states are audited exactly as the numpy
restatement (auction_restore_checker.py) audits them, and the next warm and repair passes equal the checkers started
from the audited state; a state survives pm_set_asks with an inserted ask, pm_set_worker_count, pm_set_model_table and
a move to a sibling engine; a scipy solution seeds a warm pass; refusals change nothing; and one restore at the 100k x 1M
size of BASELINE configs[2]."""
import ctypes as C
import time

import numpy as np
import pytest

import auction_certificate as ac
import auction_repair_checker as rp
import auction_restore_checker as rs
import auction_warm_checker as wc
from helpers import load_engine
from protocol_b200 import abi
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine
from test_gpu_auction_reverse import scipy_instance
from test_gpu_auction_warm import cfg3, engine, tables

pytestmark = pytest.mark.gpu

NONE = wc.NONE
AUC, REV = abi.PM_MODE_AUCTION, abi.PM_MODE_AUCTION | abi.PM_AUCTION_REVERSE
WARM = AUC | abi.PM_AUCTION_WARM
REPAIR = WARM | abi.PM_AUCTION_REPAIR
DROPS = ("n_dropped_bad", "n_dropped_shared", "n_dropped_slack")


class Both:
    """Forwards every table call to several engines: the same changes reach each of them."""

    def __init__(self, *engines):
        self.engines = engines

    def __getattr__(self, name):
        def call(*args, **kw):
            for e in self.engines:
                getattr(e, name)(*args, **kw)
        return call


def current_tables(m: wc.Market, t):
    return dict(asks=m.asks, opts=m.opts, wa=m.wa, wb=m.wb, bits=t["bits"], n_patterns=t["n_patterns"],
                n_models=t["n_models"], words=t["words"])


def fresh(m: wc.Market, t, tune=0, S=1, eps_start=1):
    """A new engine holding the market's current tables, caps, floors and reputation column."""
    eng = engine(current_tables(m, t), m.cap, tune=tune, floors=m.floors, reputation=m.reputation)
    eng.set_auction_params(cost_scale=S, eps_start=eps_start, eps_div=4)
    return eng


def export(eng):
    """(prices, assignment) of the stored state: what a caller keeps across a restart."""
    return eng.auction_state()[0], eng.auction_assignment()


def outcome(eng):
    """Everything a pass reports, minus times and the table version (which counts each engine's own calls)."""
    res = eng.fetch()
    st = {k: v for k, v in res.stats.items() if not k.startswith("ms_")}
    price, warm, released = eng.auction_state()
    return (res.worker_group.copy(), res.worker_ask.copy(), res.group_ask.copy(), res.group_members.copy(),
            res.ask_best.copy(), res.ask_count.copy(), st, price, warm, released, eng.auction_reverse_stats(),
            eng.auction_assignment())


def same(x, y):
    for a, b in zip(x, y):
        if isinstance(a, np.ndarray):
            assert np.array_equal(a, b)
        else:
            assert a == b, (a, b)
    return True


def same_cert(x, y):
    return all(x[k] == y[k] for k in ac.FIELDS) and np.array_equal(x["ask_bound"], y["ask_bound"])


def lsa_assignment(F, ap, cap, S=1):
    """scipy's optimal assignment (linear_sum_assignment on auction_reverse_checker.optimum's matrix), as uint32[T]."""
    from scipy.optimize import linear_sum_assignment

    T, W = F.shape
    BIG = 1 << 50
    M = np.full((T, W + T), BIG, dtype=np.int64)
    M[:, :W] = np.where(F, np.asarray(ap, dtype=np.int64)[None, :] * S, BIG)
    M[np.arange(T), W + np.arange(T)] = (np.asarray(cap, dtype=np.int64) + 1) * S
    r, c = linear_sum_assignment(M)
    a = np.full(T, NONE, dtype=np.uint32)
    a[r[c < W]] = c[c < W]
    return a, int(M[r, c].sum())


# ---------------------------------------------------------------- round trip
def round_trip(t, cap, seed, modes, tune=0, S=1, eps_start=1, floors=None, reputation=None):
    m = wc.Market(t, cap, reputation, floors)
    a = engine(t, cap, tune=tune, floors=floors, reputation=reputation)
    a.set_auction_params(cost_scale=S, eps_start=eps_start, eps_div=4)
    rng = np.random.default_rng(seed)
    a.match(modes[0])
    for mode in modes[1:]:
        price, assigned = export(a)
        got = np.full(len(m.asks), NONE, dtype=np.uint32)
        res = a.fetch()
        got[res.group_ask] = res.group_members
        assert np.array_equal(assigned, got)
        b = fresh(m, t, tune, S, eps_start)
        rep = b.auction_restore(price, assigned)
        assert all(rep[k] == 0 for k in DROPS) and rep["n_held"] == int((assigned != NONE).sum())
        assert rep["evals"] == len(m.asks) * m.n_workers
        assert same_cert(a.auction_certificate(ask_bound=True), b.auction_certificate(ask_bound=True))
        assert b.auction_state()[1:] == (False, 0) and b.auction_reverse_stats() == (0, 0, 0)
        m.store(price, assigned)
        for _ in range(int(rng.integers(1, 3))):
            wc.random_step(m, rng, eng=Both(a, b))
        a.match(mode)
        b.match(mode)
        assert same(outcome(a), outcome(b))
        b.close()
    a.close()


@pytest.mark.parametrize("eps_start", [1, 64])
@pytest.mark.parametrize("n_asks,n_workers,seed", [(50, 700, 2), (300, 2500, 3)])
def test_round_trip_carries_every_pass(n_asks, n_workers, seed, eps_start):
    t, cap = tables(n_asks, n_workers, seed)
    round_trip(t, cap, seed, [REV, WARM, REPAIR, AUC, REPAIR, WARM, REV, WARM], eps_start=eps_start)


def test_round_trip_with_floors_and_scale():
    t, cap = tables(120, 1500, 31)
    rng = np.random.default_rng(31)
    rep = rng.integers(0, 4, 1500).astype(np.uint32)
    floors = rng.integers(0, 3, 120).astype(np.uint32)
    round_trip(t, cap, 31, [AUC, WARM, REPAIR, REV, WARM], floors=floors, reputation=rep)
    round_trip(t, cap, 32, [REV, REPAIR, WARM, REPAIR], S=121, eps_start=64)


@pytest.mark.parametrize("tune", [1, 2, 8, 16, 32, 64, 128, 8 | 32, 64 | 32, 1 | 64, 128 | 32, 0x200, 0x100 | 16])
def test_round_trip_under_every_shortcut_setting(tune):
    t, cap = tables(25, 6000, 7, dup=(20, 5, 120))
    round_trip(t, cap, 70 + tune, [AUC, WARM, REPAIR, WARM], tune=tune)


# ---------------------------------------------------------------- adversarial states against the checkers
@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("S,eps_start", [(1, 1), (7, 64), (None, 1)])
def test_adversarial_states_equal_the_checkers(seed, S, eps_start):
    t, cap = tables(60, 900, 40 + seed)
    rng = np.random.default_rng(40 + seed)
    floors = rng.integers(0, 3, 60).astype(np.uint32) if seed == 1 else None
    rep = rng.integers(0, 4, 900).astype(np.uint32) if seed == 1 else None
    m = wc.Market(t, cap, rep, floors)
    T = len(cap)
    S = S or T + 1
    F, ap = m.F(), m.wb["ext_ask_price"]
    eng = fresh(m, t, S=S, eps_start=eps_start)
    for _ in range(3):
        price, assigned = rs.adversarial_state(F, ap, m.cap, S, rng, eps_start)
        want = rs.audit(F, ap, m.cap, S, price, assigned)
        got = eng.auction_restore(price, assigned)
        assert all(got[k] == want[k] for k in ("n_held", "evals") + DROPS), (got, want)
        kept = want["assigned"]
        assert np.array_equal(eng.auction_assignment(), kept)
        c = eng.auction_certificate(ask_bound=True)
        w = ac.certificate(F, ap, m.cap, S, price, kept)
        assert all(c[k] == w[k] for k in ac.FIELDS) and np.array_equal(c["ask_bound"], w["ask_bound"])
        assert np.array_equal(eng.auction_state()[0], price)
        # the warm pass from it
        eng.match(WARM)
        a, p, n, rel = wc.warm(F, ap, m.cap, S, price, kept, m.n_workers, [], [])
        got_a = eng.auction_assignment()
        got_p, warm, released = eng.auction_state()
        assert warm and released == len(rel) and eng.stats()["n_rounds"] == n
        assert np.array_equal(got_a, a) and np.array_equal(got_p, p)
        # the repair from the same audited state
        eng.auction_restore(price, assigned)
        eng.match(REPAIR)
        out = rp.repair(F, ap, m.cap, S, price, kept, m.n_workers, [], [])
        got_p, warm, released = eng.auction_state()
        assert warm and released == len(out["released"]) == 0
        assert np.array_equal(eng.auction_assignment(), out["assigned"]) and np.array_equal(got_p, out["price"])
        assert eng.stats()["n_rounds"] == out["fwd"]
        assert eng.auction_reverse_stats() == (1, out["rev"], out["bids"])
        cert = eng.auction_certificate()
        assert cert["n_bad_holds"] == cert["n_shared"] == cert["n_priced_unowned"] == 0 and 0 <= cert["gap"] <= T
    eng.close()


# ---------------------------------------------------------------- across the calls that discard the state
def check_warm_from(eng, m, S, price, assigned):
    """Restore, one warm pass, and the checker from the audited state; the result certifies within T."""
    T = len(m.asks)
    F, ap = m.F(), m.wb["ext_ask_price"]
    want = rs.audit(F, ap, m.cap, S, price, assigned)
    got = eng.auction_restore(price, assigned)
    assert all(got[k] == want[k] for k in ("n_held",) + DROPS)
    eng.match(WARM)
    a, p, n, rel = wc.warm(F, ap, m.cap, S, price, want["assigned"], m.n_workers, [], [])
    got_p, warm, released = eng.auction_state()
    assert warm and released == len(rel) and eng.stats()["n_rounds"] == n
    assert np.array_equal(eng.auction_assignment(), a) and np.array_equal(got_p, p)
    c = eng.auction_certificate()
    assert c["n_bad_holds"] == c["n_shared"] == c["n_priced_unowned"] == 0 and 0 <= c["gap"] <= T
    return want


def test_state_survives_every_discarding_call():
    t, cap = tables(300, 2500, 3)
    m = wc.Market(t, cap)
    eng = fresh(m, t)
    eng.match(AUC)
    price, assigned = export(eng)
    # pm_set_asks with an ask inserted in the middle: the export's ask indices move up past it
    k = 137
    asks = np.concatenate([m.asks[:k], m.asks[k + 5:k + 6], m.asks[k:]])
    cap2 = np.concatenate([m.cap[:k], [m.cap[k + 5]], m.cap[k:]]).astype(np.uint32)
    eng.set_asks(asks, m.opts)
    eng.set_price_caps(cap2)
    m2 = wc.Market(dict(current_tables(m, t), asks=asks), cap2)
    a2 = np.concatenate([assigned[:k], [NONE], assigned[k:]]).astype(np.uint32)
    want = check_warm_from(eng, m2, 1, price, a2)
    assert want["n_held"] == int((assigned != NONE).sum())   # nothing else changed: every hold kept
    # pm_set_worker_count with the same rows
    price, assigned = export(eng)
    eng.set_workers(m2.wa, m2.wb)
    check_warm_from(eng, m2, 1, price, assigned)
    # pm_set_model_table
    price, assigned = export(eng)
    eng.set_model_table(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    check_warm_from(eng, m2, 1, price, assigned)
    # a sibling engine
    price, assigned = export(eng)
    h = C.c_void_p()
    assert eng._lib.pm_create_sibling(eng._h, C.byref(h)) == abi.PM_OK
    sib = Engine.__new__(Engine)
    sib._lib, sib._h, sib.n_workers, sib.n_asks, sib._auction_workers = eng._lib, h, 0, 0, 0
    load_engine(sib, dict(current_tables(m2, t), asks=asks))
    sib.set_price_caps(cap2)
    check_warm_from(sib, m2, 1, price, assigned)
    sib.close()
    eng.close()


def test_external_seed_from_scipy_at_2000_x_2000():
    t, cap = scipy_instance(2000, 2000, 4)
    T = len(cap)
    F = wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    ap = t["wb"]["ext_ask_price"]
    seed, opt = lsa_assignment(F, ap, cap)
    eng = engine(t, cap)
    rep = eng.auction_restore(np.zeros(len(t["wa"]), dtype=np.int64), seed)
    assert rep["n_dropped_bad"] == rep["n_dropped_shared"] == 0
    eng.match(WARM)
    assert eng.auction_state()[1]
    c = eng.auction_certificate()
    assert c["n_bad_holds"] == c["n_shared"] == c["n_priced_unowned"] == 0 and 0 <= c["gap"] <= T
    assert opt <= c["cost"] <= opt + T
    eng.close()


# ---------------------------------------------------------------- refusals
def test_refusals_change_nothing():
    t, cap = tables(50, 700, 2)
    T, W = len(cap), len(t["wa"])
    twins = [engine(t, cap), engine(t, cap)]
    for e in twins:
        e.match(AUC)
    eng, lib = twins[0], twins[0]._lib
    price, assigned = export(eng)
    rep = abi.PmAuctionRestoreReport()

    def light(e):
        try:
            cert = e.auction_certificate(ask_bound=True)
        except PrimeMatchError as exc:   # disabled asks, a missing pattern: the certificate refuses them too
            cert = exc.status
        return (cert, e.auction_state(), e.auction_reverse_stats(), e.table_version(),
                {k: v for k, v in e.stats().items() if not k.startswith("ms_")}, e.auction_assignment())

    def check(before, after):
        assert before[0] == after[0] if isinstance(before[0], int) else same_cert(before[0], after[0])
        assert np.array_equal(before[1][0], after[1][0]) and before[1][1:] == after[1][1:]
        assert before[2:5] == after[2:5] and np.array_equal(before[5], after[5])

    def refused(status, p=price, a=assigned, nw=None, na=None, null_p=False, null_a=False):
        before = light(eng)
        pp = np.ascontiguousarray(p, dtype=np.int64)
        aa = np.ascontiguousarray(a, dtype=np.uint32)
        rc_ = lib.pm_auction_restore(eng._h, None if null_p else pp.ctypes.data, len(pp) if nw is None else nw,
                                     None if null_a else aa.ctypes.data, len(aa) if na is None else na, C.byref(rep))
        assert rc_ == status
        check(before, light(eng))

    top = rs.price_bound(cap, 1)
    refused(abi.PM_E_INVALID, null_p=True)
    refused(abi.PM_E_INVALID, null_a=True)
    refused(abi.PM_E_INVALID, nw=W - 1)
    refused(abi.PM_E_INVALID, na=T - 1)
    refused(abi.PM_E_INVALID, p=np.zeros(W + 1, dtype=np.int64))
    bad = assigned.copy()
    bad[3] = W
    refused(abi.PM_E_INVALID, a=bad)
    for v in (-1, top + 1):
        p = price.copy()
        p[7] = v
        refused(abi.PM_E_INVALID, p=p)
    assert lib.pm_auction_restore(None, None, 0, None, 0, None) == abi.PM_E_INVALID
    # an ask pointing at a missing model pattern (pm_update_asks keeps the state on both twins)
    opt = np.zeros(1, dtype=abi.GPU_OPT)
    opt["present"], opt["pattern_id"] = abi.PM_O_MODEL, 0xFFFFFFF0
    row = t["asks"][5:6].copy()
    row["n_opts"], row["opt_off"] = 1, 0
    for e in twins:
        e.update_asks([5], row, opt)
    refused(abi.PM_E_STATE)
    for e in twins:
        e.update_asks([5], t["asks"][5:6], t["opts"])
    # disabled asks
    for e in twins:
        e.set_ask_enabled([3], False)
    refused(abi.PM_E_UNSUPPORTED)
    for e in twins:
        e.set_ask_enabled([3], True)
    # the next passes equal the twin's, which never saw a refused call
    for mode in (WARM, REPAIR):
        for e in twins:
            e.match(mode)
        assert same(outcome(twins[0]), outcome(twins[1]))
    for e in twins:
        e.close()
    # refusals on engines without a stored state leave none behind
    e = Engine()
    with pytest.raises(PrimeMatchError) as exc:                 # no tables
        e.auction_restore(np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.uint32))
    assert exc.value.status == abi.PM_E_STATE
    load_engine(e, t)
    with pytest.raises(PrimeMatchError) as exc:                 # no caps
        e.auction_restore(price, assigned)
    assert exc.value.status == abi.PM_E_STATE
    e.set_price_caps(cap)
    e.set_auction_params(eps_start=(1 << 61) - 1)               # outside the integer domain: found by the sweep
    with pytest.raises(PrimeMatchError) as exc:
        e.auction_restore(price, assigned)
    assert exc.value.status == abi.PM_E_INVALID
    e.set_auction_params()
    e.set_shard(0, 350)
    with pytest.raises(PrimeMatchError) as exc:
        e.auction_restore(price, assigned)
    assert exc.value.status == abi.PM_E_UNSUPPORTED
    with pytest.raises(PrimeMatchError) as exc:
        e.auction_state()
    assert exc.value.status == abi.PM_E_STATE
    with pytest.raises(PrimeMatchError) as exc:
        e.auction_assignment()
    assert exc.value.status == abi.PM_E_STATE
    e.close()


# ---------------------------------------------------------------- full size
def test_restore_at_cfg3_size():
    """100k asks x 1M workers: A's cold state restored into B; equal certificates; 1 000 rows rewritten on both (half
    of them held); the two warm passes are bit-identical.  The restore time is printed, not asserted."""
    t, cap = cfg3()
    T, W = len(cap), len(t["wa"])
    a = engine(t, cap)
    a.match(AUC)
    price, assigned = export(a)
    b = engine(t, cap)
    t0 = time.perf_counter()
    rep = b.auction_restore(price, assigned)
    ms = (time.perf_counter() - t0) * 1e3
    print(f"\nrestore at 100k x 1M: {ms:.1f} ms, held {rep['n_held']}")
    assert all(rep[k] == 0 for k in DROPS) and rep["n_held"] == int((assigned != NONE).sum()) > 0
    assert rep["evals"] == T * W
    assert same_cert(a.auction_certificate(ask_bound=True), b.auction_certificate(ask_bound=True))
    rng = np.random.default_rng(5)
    held = assigned[assigned != NONE]
    idx = np.unique(np.concatenate([rng.choice(held, 500, replace=False), rng.choice(W, 500, replace=False)])).astype(np.uint32)
    wa, wb = t["wa"][idx].copy(), t["wb"][idx].copy()
    wb["ext_ask_price"] = np.maximum(1, wb["ext_ask_price"] // 2)
    for e in (a, b):
        e.update_workers(idx, wa, wb)
        e.match(WARM)
    assert a.auction_state()[1] and same(outcome(a), outcome(b))
    a.close()
    b.close()
