"""pm_auction_slot_assignment / pm_auction_restore_slots on the device: the per-slot export equals the twin engine's
pm_auction_assignment (the twin repeats row t demand[t] times) and the fold of pm_fetch_result after every pass kind
and table delta; a state exported from an engine with demands and restored into a fresh one carries every later pass
bit for bit, a demand change included, under every PM_TUNE_AUCTION setting the restore tests use; adversarial slot
states restored into a demand engine and into its twin give the same report (apart from evals), export, certificate
and next passes, equal to the numpy audit and the warm and repair checkers; with every demand 1 the slot calls are the
plain calls; the state survives the calls that discard it; refusals change nothing; and one round trip at the bench
tool's 25 000 asks x 1M workers."""
import ctypes as C
import time

import numpy as np
import pytest

import auction_certificate as ac
import auction_repair_checker as rp
import auction_restore_checker as rs
import auction_warm_checker as wc
from auction_demand import offsets, remap
from helpers import load_engine
from protocol_b200 import abi
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine
from test_gpu_auction_demand import Pair, demands, fold_result, fold_slots, random_change, twin_tables
from test_gpu_auction_restore import Both, current_tables, fresh, same, same_cert
from test_gpu_auction_warm import cfg3, engine, tables

pytestmark = pytest.mark.gpu

NONE = wc.NONE
AUC, REV = abi.PM_MODE_AUCTION, abi.PM_MODE_AUCTION | abi.PM_AUCTION_REVERSE
WARM = AUC | abi.PM_AUCTION_WARM
REPAIR = WARM | abi.PM_AUCTION_REPAIR
DROPS = ("n_dropped_bad", "n_dropped_shared", "n_dropped_slack")
CERT = [f for f in ac.FIELDS if f != "evals"]   # evals: T x W with demands, D x W for the twin
TUNES = [0, 1, 2, 8, 16, 32, 64, 128, 8 | 32, 64 | 32, 1 | 64, 128 | 32, 0x200, 0x100 | 16]   # test_gpu_auction_restore's


def outcome(eng):
    """Everything a pass reports, minus times and the table version, with the slot export."""
    res = eng.fetch()
    st = {k: v for k, v in res.stats.items() if not k.startswith("ms_")}
    price, warm, released = eng.auction_state()
    return (res.worker_group.copy(), res.worker_ask.copy(), res.group_ask.copy(), res.group_members.copy(),
            res.ask_best.copy(), res.ask_count.copy(), st, price, warm, released, eng.auction_reverse_stats(),
            eng.auction_slot_assignment())


def change_demands(d, rng, n=3):
    d2 = d.copy()
    for t in rng.choice(len(d), min(n, len(d)), replace=False):
        d2[t] = max(1, int(d2[t]) + int(rng.choice([-2, -1, 1, 2])))
    return d2


def same_cert_twin(c, ct, d):
    """The demand engine's certificate against its twin's: every field but evals, ask_bound at each ask's first slot."""
    assert all(c[k] == ct[k] for k in CERT), [(k, c[k], ct[k]) for k in CERT if c[k] != ct[k]]
    assert np.array_equal(c["ask_bound"], ct["ask_bound"][offsets(d)[:-1]])


# ---------------------------------------------------------------- the export
@pytest.mark.parametrize("tune", [0, 8 | 32, 0x100 | 16])
def test_slot_export_equals_twin_and_result(tune):
    t, cap = tables(60, 800, 61)
    rng = np.random.default_rng(61 + tune)
    rep = rng.integers(0, 4, 800).astype(np.uint32)
    floors = rng.integers(0, 3, 60).astype(np.uint32)
    p = Pair(t, cap, demands(rng, 60), tune=tune, floors=floors, reputation=rep)

    def check(after_pass):
        slots = p.a.auction_slot_assignment()
        assert len(slots) == int(p.d.sum())
        assert np.array_equal(slots, p.b.auction_assignment())
        if after_pass:
            assert fold_slots(slots, p.d) == fold_result(p.a.fetch())
        return slots

    p.check(AUC)
    check(True)
    for i in range(8):   # worker, cap, floor and ask deltas (random_change), each checked before and after the pass
        random_change(p, rng)
        check(False)
        p.check(REPAIR if i % 2 else WARM)
        check(True)
    p.params(cost_scale=1, eps_start=64, eps_div=4)   # eps-scaled with reverse rounds
    p.check(REV)
    check(True)
    slots, d = check(True), p.d
    p.b.close()
    for mode in (WARM, REPAIR, WARM):   # demand deltas: the export is the remap of the last one, then the pass's fold
        d2 = change_demands(d, rng, 5)
        p.a.set_ask_demand(d2)
        want, _, _ = remap(slots, d, d2)
        assert np.array_equal(p.a.auction_slot_assignment(), want)
        p.a.match(mode)
        slots, d = p.a.auction_slot_assignment(), d2
        assert fold_slots(slots, d) == fold_result(p.a.fetch())
    p.a.close()


# ---------------------------------------------------------------- round trip
def slot_round_trip(t, cap, seed, modes, tune=0, S=1, eps_start=1, floors=None, reputation=None, choices=(1, 2, 3, 4)):
    rng = np.random.default_rng(seed)
    m = wc.Market(t, cap, reputation, floors)
    d = demands(rng, len(cap), choices)
    a = engine(t, cap, tune=tune, floors=floors, reputation=reputation)
    a.set_ask_demand(d)
    a.set_auction_params(cost_scale=S, eps_start=eps_start, eps_div=4)
    a.match(modes[0])
    for i, mode in enumerate(modes[1:]):
        price, slots = a.auction_state()[0], a.auction_slot_assignment()
        assert fold_slots(slots, d) == fold_result(a.fetch())
        b = fresh(m, t, tune, S, eps_start)
        b.set_ask_demand(d)
        rep = b.auction_restore_slots(price, slots)
        assert all(rep[k] == 0 for k in DROPS) and rep["n_held"] == int((slots != NONE).sum())
        assert rep["evals"] == len(m.asks) * m.n_workers
        assert same_cert(a.auction_certificate(ask_bound=True), b.auction_certificate(ask_bound=True))
        assert b.auction_state()[1:] == (False, 0) and b.auction_reverse_stats() == (0, 0, 0)
        assert np.array_equal(b.auction_slot_assignment(), slots)
        m.store(price, slots)
        for _ in range(int(rng.integers(1, 3))):
            wc.random_step(m, rng, eng=Both(a, b))
        if i % 2:   # a demand change after the restore
            d = change_demands(d, rng)
            Both(a, b).set_ask_demand(d)
        a.match(mode)
        b.match(mode)
        assert same(outcome(a), outcome(b))
        b.close()
    a.close()


@pytest.mark.parametrize("eps_start", [1, 64])
def test_round_trip_carries_every_pass(eps_start):
    t, cap = tables(50, 700, 62)
    slot_round_trip(t, cap, 62, [REV, WARM, REPAIR, AUC, REPAIR, WARM, REV, WARM], eps_start=eps_start)


def test_round_trip_with_floors_scale_and_large_demands():
    t, cap = tables(80, 1500, 63)
    rng = np.random.default_rng(63)
    rep = rng.integers(0, 4, 1500).astype(np.uint32)
    floors = rng.integers(0, 3, 80).astype(np.uint32)
    slot_round_trip(t, cap, 63, [AUC, WARM, REPAIR, REV, WARM], floors=floors, reputation=rep)
    slot_round_trip(t, cap, 64, [REV, REPAIR, WARM, REPAIR], S=4 * 80 + 1, eps_start=64, choices=(1, 2, 4, 8))


@pytest.mark.parametrize("tune", TUNES)
def test_round_trip_under_every_shortcut_setting(tune):
    t, cap = tables(25, 6000, 7, dup=(20, 5, 120))
    slot_round_trip(t, cap, 170 + tune, [AUC, WARM, REPAIR, WARM], tune=tune)


# ---------------------------------------------------------------- adversarial states: demand engine, twin, checkers
@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("S,eps_start", [(1, 1), (7, 64), (None, 1)])
def test_adversarial_states_equal_the_twin_and_the_checkers(seed, S, eps_start):
    T, W = (40, 900) if S else (20, 600)   # cost_scale = D + 1: the checkers' rounds grow with it
    t, cap = tables(T, W, 65 + seed)
    rng = np.random.default_rng(65 + seed)
    floors = rng.integers(0, 3, T).astype(np.uint32) if seed == 1 else None
    rep = rng.integers(0, 4, W).astype(np.uint32) if seed == 1 else None
    d = demands(rng, T)
    D = int(d.sum())
    S = S or D + 1
    m = wc.Market(t, cap, rep, floors)
    slot_ask = np.repeat(np.arange(T), d)
    Fx, ap, capx = m.F()[slot_ask], m.wb["ext_ask_price"], cap[slot_ask]
    eng = fresh(m, t, S=S, eps_start=eps_start)
    eng.set_ask_demand(d)
    t2, cap2, fl2 = twin_tables(t, cap, d, floors)
    tw = engine(t2, cap2, floors=fl2, reputation=rep)
    tw.set_auction_params(cost_scale=S, eps_start=eps_start, eps_div=4)
    for _ in range(3):
        price, assigned = rs.adversarial_state(Fx, ap, capx, S, rng, eps_start)
        want = rs.audit(Fx, ap, capx, S, price, assigned)
        kept = want["assigned"]
        for mode in (WARM, REPAIR):
            got = eng.auction_restore_slots(price, assigned)
            got_t = tw.auction_restore(price, assigned)
            assert all(got[k] == got_t[k] == want[k] for k in ("n_held",) + DROPS), (got, got_t, want)
            assert got["evals"] == T * W and got_t["evals"] == D * W
            assert np.array_equal(eng.auction_slot_assignment(), kept)
            assert np.array_equal(tw.auction_assignment(), kept)
            same_cert_twin(eng.auction_certificate(ask_bound=True), tw.auction_certificate(ask_bound=True), d)
            assert np.array_equal(eng.auction_state()[0], price)
            eng.match(mode)
            tw.match(mode)
            got_p, warm, released = eng.auction_state()
            assert (got_p.tobytes(), warm, released) == (tw.auction_state()[0].tobytes(),) + tw.auction_state()[1:]
            assert eng.auction_reverse_stats() == tw.auction_reverse_stats()
            assert eng.stats()["n_rounds"] == tw.stats()["n_rounds"]
            slots = eng.auction_slot_assignment()
            assert np.array_equal(slots, tw.auction_assignment())
            if mode == WARM:
                a, p, n, rel = wc.warm(Fx, ap, capx, S, price, kept, W, [], [])
                assert warm and released == len(rel) and eng.stats()["n_rounds"] == n
                assert np.array_equal(slots, a) and np.array_equal(got_p, p)
            else:
                out = rp.repair(Fx, ap, capx, S, price, kept, W, [], [])
                assert warm and released == len(out["released"]) == 0
                assert np.array_equal(slots, out["assigned"]) and np.array_equal(got_p, out["price"])
                assert eng.stats()["n_rounds"] == out["fwd"]
                assert eng.auction_reverse_stats() == (1, out["rev"], out["bids"])
            assert fold_slots(slots, d) == fold_result(eng.fetch())
            cert = eng.auction_certificate()
            assert cert["n_bad_holds"] == cert["n_shared"] == cert["n_priced_unowned"] == 0 and 0 <= cert["gap"] <= D
    eng.close()
    tw.close()


# ---------------------------------------------------------------- every demand 1
def test_all_ones_slot_calls_are_the_plain_calls():
    t, cap = tables(60, 900, 66)
    rng = np.random.default_rng(66)
    plain, ones = engine(t, cap), engine(t, cap)
    ones.set_ask_demand(np.ones(60, dtype=np.uint32))
    for e in (plain, ones):
        e.match(AUC)
    exp = ones.auction_slot_assignment()
    assert exp.tobytes() == ones.auction_assignment().tobytes() == plain.auction_assignment().tobytes()
    m = wc.Market(t, cap)
    F, ap = m.F(), m.wb["ext_ask_price"]
    for _ in range(3):
        price, assigned = rs.adversarial_state(F, ap, cap, 1, rng)
        r1, r2 = ones.auction_restore_slots(price, assigned), plain.auction_restore(price, assigned)
        assert r1 == r2
        assert ones.auction_slot_assignment().tobytes() == plain.auction_assignment().tobytes()
        for mode in (WARM, REPAIR):
            ones.auction_restore_slots(price, assigned)
            plain.auction_restore(price, assigned)
            ones.match(mode)
            plain.match(mode)
            assert same(outcome(ones), outcome(plain))
    # demands set back to 1 under a stored state: the slot export is the plain export of the remapped state
    d = demands(rng, 60, (2, 3))
    ones.set_ask_demand(d)
    ones.match(AUC)
    slots = ones.auction_slot_assignment()
    ones.set_ask_demand(np.ones(60, dtype=np.uint32))
    want, _, _ = remap(slots, d, np.ones(60, dtype=np.uint32))
    got = ones.auction_slot_assignment()
    assert got.tobytes() == ones.auction_assignment().tobytes() == want.tobytes()
    price = ones.auction_state()[0]
    assert ones.auction_restore_slots(price, got) == plain.auction_restore(price, got)
    plain.close()
    ones.close()


# ---------------------------------------------------------------- across the calls that discard the state
def check_warm_from(eng, m, d, S, price, slots):
    """Restore per slot, one warm pass, and the checker on the twin from the audited state."""
    slot_ask = np.repeat(np.arange(len(d)), d)
    Fx, ap, capx = m.F()[slot_ask], m.wb["ext_ask_price"], m.cap[slot_ask]
    want = rs.audit(Fx, ap, capx, S, price, slots)
    got = eng.auction_restore_slots(price, slots)
    assert all(got[k] == want[k] for k in ("n_held",) + DROPS)
    eng.match(WARM)
    a, p, n, rel = wc.warm(Fx, ap, capx, S, price, want["assigned"], m.n_workers, [], [])
    got_p, warm, released = eng.auction_state()
    assert warm and released == len(rel) and eng.stats()["n_rounds"] == n
    assert np.array_equal(eng.auction_slot_assignment(), a) and np.array_equal(got_p, p)
    c = eng.auction_certificate()
    assert c["n_bad_holds"] == c["n_shared"] == c["n_priced_unowned"] == 0 and 0 <= c["gap"] <= len(slots)
    return want


def test_state_survives_every_discarding_call():
    t, cap = tables(200, 2500, 67)
    rng = np.random.default_rng(67)
    d = demands(rng, 200)
    m = wc.Market(t, cap)
    eng = fresh(m, t)
    eng.set_ask_demand(d)
    eng.match(AUC)
    price, slots = eng.auction_state()[0], eng.auction_slot_assignment()
    # pm_set_asks with a demand-3 ask inserted at k: set the demands again, insert 3 unheld slots at its offset
    k, dk = 83, 3
    asks = np.concatenate([m.asks[:k], m.asks[k + 5:k + 6], m.asks[k:]])
    cap2 = np.concatenate([m.cap[:k], [m.cap[k + 5]], m.cap[k:]]).astype(np.uint32)
    d2 = np.concatenate([d[:k], [dk], d[k:]]).astype(np.uint32)
    eng.set_asks(asks, m.opts)
    eng.set_price_caps(cap2)
    eng.set_ask_demand(d2)
    m2 = wc.Market(dict(current_tables(m, t), asks=asks), cap2)
    at = int(offsets(d)[k])
    s2 = np.concatenate([slots[:at], np.full(dk, NONE), slots[at:]]).astype(np.uint32)
    want = check_warm_from(eng, m2, d2, 1, price, s2)
    assert want["n_held"] == int((slots != NONE).sum())   # nothing else changed: every hold kept
    # pm_set_worker_count with the same rows
    price, slots = eng.auction_state()[0], eng.auction_slot_assignment()
    eng.set_workers(m2.wa, m2.wb)
    check_warm_from(eng, m2, d2, 1, price, slots)
    # pm_set_model_table
    price, slots = eng.auction_state()[0], eng.auction_slot_assignment()
    eng.set_model_table(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    check_warm_from(eng, m2, d2, 1, price, slots)
    # a sibling engine
    price, slots = eng.auction_state()[0], eng.auction_slot_assignment()
    h = C.c_void_p()
    assert eng._lib.pm_create_sibling(eng._h, C.byref(h)) == abi.PM_OK
    sib = Engine.__new__(Engine)
    sib._lib, sib._h, sib.n_workers, sib.n_asks, sib._auction_workers = eng._lib, h, 0, 0, 0
    load_engine(sib, dict(current_tables(m2, t), asks=asks))
    sib.set_price_caps(cap2)
    sib.set_ask_demand(d2)
    check_warm_from(sib, m2, d2, 1, price, slots)
    sib.close()
    eng.close()


# ---------------------------------------------------------------- refusals
def test_refusals_change_nothing():
    t, cap = tables(40, 600, 68)
    T, W = len(cap), len(t["wa"])
    d = demands(np.random.default_rng(68), T)
    D = int(d.sum())
    twins = [engine(t, cap), engine(t, cap)]
    for e in twins:
        e.set_ask_demand(d)
        e.match(AUC)
    eng, lib = twins[0], twins[0]._lib
    price, slots = eng.auction_state()[0], eng.auction_slot_assignment()
    rep = abi.PmAuctionRestoreReport()

    def state(e):
        try:
            cert = e.auction_certificate(ask_bound=True)
        except PrimeMatchError as exc:   # disabled asks, a missing pattern: the certificate refuses them too
            cert = exc.status
        try:
            res = fold_result(e.fetch())
        except PrimeMatchError as exc:   # after a demand change: no result until the next pass
            res = exc.status
        p, warm, rel = e.auction_state()
        return (p, warm, rel, e.table_version(), res, cert, e.auction_reverse_stats(),
                {k: v for k, v in e.stats().items() if not k.startswith("ms_")}, e.auction_slot_assignment())

    def same_state(x, y):
        assert np.array_equal(x[0], y[0]) and x[1:5] == y[1:5]
        assert x[5] == y[5] if isinstance(x[5], int) else same_cert(x[5], y[5])
        assert x[6:8] == y[6:8] and np.array_equal(x[8], y[8])

    def refused(status, p=price, a=slots, nw=None, ns=None, null_p=False, null_a=False):
        before = state(eng)
        pp = np.ascontiguousarray(p, dtype=np.int64)
        aa = np.ascontiguousarray(a, dtype=np.uint32)
        rc_ = lib.pm_auction_restore_slots(eng._h, None if null_p else pp.ctypes.data, len(pp) if nw is None else nw,
                                           None if null_a else aa.ctypes.data, len(aa) if ns is None else ns, C.byref(rep))
        assert rc_ == status
        same_state(before, state(eng))

    # the export
    before = state(eng)
    n = C.c_uint32(D - 1)
    out = np.zeros(D, dtype=np.uint32)
    assert lib.pm_auction_slot_assignment(eng._h, out.ctypes.data, C.byref(n)) == abi.PM_E_INVALID and n.value == D
    n = C.c_uint32(D + 1)
    assert lib.pm_auction_slot_assignment(eng._h, out.ctypes.data, C.byref(n)) == abi.PM_E_INVALID and n.value == D
    assert lib.pm_auction_slot_assignment(eng._h, out.ctypes.data, None) == abi.PM_E_INVALID
    assert lib.pm_auction_slot_assignment(None, None, C.byref(n)) == abi.PM_E_INVALID
    same_state(before, state(eng))
    # the restore
    top = rs.price_bound(cap, 1)
    refused(abi.PM_E_INVALID, null_p=True)
    refused(abi.PM_E_INVALID, null_a=True)
    refused(abi.PM_E_INVALID, nw=W - 1)
    refused(abi.PM_E_INVALID, ns=D - 1)
    refused(abi.PM_E_INVALID, a=slots[:T])                       # one entry per ask is not per slot
    refused(abi.PM_E_INVALID, p=np.zeros(W + 1, dtype=np.int64))
    bad = slots.copy()
    bad[3] = W
    refused(abi.PM_E_INVALID, a=bad)
    for v in (-1, top + 1):
        p = price.copy()
        p[7] = v
        refused(abi.PM_E_INVALID, p=p)
    assert lib.pm_auction_restore_slots(None, None, 0, None, 0, None) == abi.PM_E_INVALID
    # an array exported before a demand change (the change applied to both engines)
    d2 = d.copy()
    d2[5] += 2
    for e in twins:
        e.set_ask_demand(d2)
    refused(abi.PM_E_INVALID)
    # an ask pointing at a missing model pattern (pm_update_asks keeps the state and the demands)
    opt = np.zeros(1, dtype=abi.GPU_OPT)
    opt["present"], opt["pattern_id"] = abi.PM_O_MODEL, 0xFFFFFFF0
    row = t["asks"][5:6].copy()
    row["n_opts"], row["opt_off"] = 1, 0
    s2 = eng.auction_slot_assignment()
    for e in twins:
        e.update_asks([5], row, opt)
    refused(abi.PM_E_STATE, a=s2)
    for e in twins:
        e.update_asks([5], t["asks"][5:6], t["opts"])
    for e in twins:   # disabled asks
        e.set_ask_enabled([3], False)
    refused(abi.PM_E_UNSUPPORTED, a=s2)
    for e in twins:
        e.set_ask_enabled([3], True)
    # the next passes equal the twin's, which never saw a refused call
    for mode in (WARM, REPAIR):
        for e in twins:
            e.match(mode)
        assert same(outcome(twins[0]), outcome(twins[1]))
    for e in twins:
        e.close()
    # engines without a stored state keep none
    e = Engine()
    with pytest.raises(PrimeMatchError) as exc:                 # no tables
        e.auction_restore_slots(np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.uint32))
    assert exc.value.status == abi.PM_E_STATE
    load_engine(e, t)
    e.set_ask_demand(d)
    with pytest.raises(PrimeMatchError) as exc:                 # no stored state: no export, not even its size
        e.auction_slot_assignment()
    assert exc.value.status == abi.PM_E_STATE
    with pytest.raises(PrimeMatchError) as exc:                 # no caps
        e.auction_restore_slots(price, slots)
    assert exc.value.status == abi.PM_E_STATE
    e.set_price_caps(cap)
    e.set_auction_params(eps_start=(1 << 61) - 1)               # outside the integer domain: found by the sweep
    with pytest.raises(PrimeMatchError) as exc:
        e.auction_restore_slots(price, slots)
    assert exc.value.status == abi.PM_E_INVALID
    e.set_auction_params()
    e.set_shard(0, 300)
    with pytest.raises(PrimeMatchError) as exc:
        e.auction_restore_slots(price, slots)
    assert exc.value.status == abi.PM_E_UNSUPPORTED
    for call in (e.auction_state, e.auction_slot_assignment):
        with pytest.raises(PrimeMatchError) as exc:
            call()
        assert exc.value.status == abi.PM_E_STATE
    e.close()


# ---------------------------------------------------------------- full size
def test_round_trip_at_bench_size():
    """tools/auction_demand_bench.py's instance: cfg3's first 25 000 asks with demands in {1, 2, 4, 8} x 1M workers.
    A's cold state restored per slot into B; nothing dropped; 1 000 rows rewritten on both (half of them held); the two
    warm passes are bit-identical.  The restore time is printed, not asserted."""
    t, cap = cfg3()
    T = 25_000
    t = dict(t)
    t["asks"] = np.ascontiguousarray(t["asks"][:T])
    cap = cap[:T]
    W = len(t["wa"])
    d = np.random.default_rng(11).choice([1, 2, 4, 8], T).astype(np.uint32)
    a = engine(t, cap)
    a.set_ask_demand(d)
    a.match(AUC)
    price, slots = a.auction_state()[0], a.auction_slot_assignment()
    b = engine(t, cap)
    b.set_ask_demand(d)
    t0 = time.perf_counter()
    rep = b.auction_restore_slots(price, slots)
    ms = (time.perf_counter() - t0) * 1e3
    print(f"\nslot restore at {T} asks ({int(d.sum())} slots) x {W} workers: {ms:.1f} ms, held {rep['n_held']}")
    assert all(rep[k] == 0 for k in DROPS) and rep["n_held"] == int((slots != NONE).sum()) > 0
    assert rep["evals"] == T * W
    assert same_cert(a.auction_certificate(ask_bound=True), b.auction_certificate(ask_bound=True))
    rng = np.random.default_rng(5)
    held = slots[slots != NONE]
    idx = np.unique(np.concatenate([rng.choice(held, 500, replace=False), rng.choice(W, 500, replace=False)])).astype(np.uint32)
    wa, wb = t["wa"][idx].copy(), t["wb"][idx].copy()
    wb["ext_ask_price"] = np.maximum(1, wb["ext_ask_price"] // 2)
    for e in (a, b):
        e.update_workers(idx, wa, wb)
        e.match(WARM)
    assert a.auction_state()[1] and same(outcome(a), outcome(b))
    a.close()
    b.close()
