"""PM_AUCTION_WARM on the device: chains of auction passes over random table histories equal the sequential
checker's chain bit for bit (assignment, prices, rounds, warm or cold, asks released), under every PM_TUNE_AUCTION
setting; the cutoff and every call that discards the stored state give a cold pass; refusals; and a warm pass at the
100k x 1M size of BASELINE configs[2]."""
import os

import numpy as np
import pytest

import auction_warm_checker as wc
from helpers import load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine

pytestmark = pytest.mark.gpu

NONE = wc.NONE
WARM = abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM


def tables(n_asks, n_workers, seed, dup=None):
    w = synth.make_workers(n_workers, seed=synth.SEED_WORKERS + seed)
    a = synth.make_asks(n_asks, "mixed", seed=synth.SEED_ASKS + seed)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words)
    rng = np.random.default_rng(seed)
    wb = t["wb"].copy()
    if dup is None:   # _auction_tables of test_gpu_parity.py
        wb["ext_ask_price"] = rng.integers(10, 1000, n_workers).astype(np.uint32)
        cap = rng.integers(50, 1500, n_asks).astype(np.uint32)
    else:             # duplicated asks over a narrow price range: every tie rule
        copies, plo, phi = dup
        idx = rng.permutation(np.repeat(np.arange(n_asks), copies))
        t["asks"] = np.ascontiguousarray(t["asks"][idx])
        wb["ext_ask_price"] = rng.integers(plo, phi + 1, n_workers).astype(np.uint32)
        cap = rng.integers(max(plo - 2, 0), phi + 3, len(idx)).astype(np.uint32)
    t["wb"] = wb
    return t, cap


def engine(t, cap, tune=0, incr=None, floors=None, reputation=None, S=1):
    env = {}
    if tune:
        env["PM_TUNE_AUCTION"] = str(tune)
    if incr is not None:
        env["PM_TUNE_INCR"] = str(incr)
    os.environ.update(env)
    try:
        eng = Engine()
    finally:
        for k in env:
            os.environ.pop(k, None)
    load_engine(eng, t)
    eng.set_price_caps(cap)
    if reputation is not None:
        eng.set_worker_reputation(reputation)
    if floors is not None:
        eng.set_min_reputation(floors)
    if S != 1:
        eng.set_auction_params(cost_scale=S)
    return eng


def run(eng, T, mode=WARM):
    eng.match(mode)
    res = eng.fetch()
    got = np.full(T, NONE, dtype=np.uint32)
    for ask, members in res.groups():
        assert len(members) == 1
        got[ask] = members[0]
    price, warm, released = eng.auction_state()
    return got, price, res.stats, warm, released


def check_pass(eng, m, S, want_warm):
    T = len(m.asks)
    got, price, st, warm, released = run(eng, T)
    if want_warm:
        a, p, n, rel = m.warm(S)
        assert warm and released == len(rel)
    else:
        a, p, n = m.cold(S)
        assert not warm and released == 0
    assert np.array_equal(got, a)
    assert np.array_equal(price, p)
    assert st["n_rounds"] == n
    m.store(p, a)
    return st


def chain(t, cap, seed, steps, tune=0, S=1, floors=None, reputation=None, kinds=None):
    m = wc.Market(t, cap, reputation, floors)
    eng = engine(t, cap, tune=tune, floors=floors, reputation=reputation, S=S)
    rng = np.random.default_rng(seed)
    check_pass(eng, m, S, want_warm=False)   # no stored state yet: cold
    n_released = 0
    for _ in range(steps):
        for _ in range(int(rng.integers(1, 3))):
            wc.random_step(m, rng, eng=eng, kinds=kinds)
        check_pass(eng, m, S, want_warm=True)
        n_released += eng.auction_state()[2]
    eng.close()
    return n_released


@pytest.mark.parametrize("n_asks,n_workers,seed", [(50, 700, 2), (300, 2500, 3), (64, 1025, 4)])
def test_warm_chain_matches_checker(n_asks, n_workers, seed):
    t, cap = tables(n_asks, n_workers, seed)
    assert chain(t, cap, seed, 8) > 0


def test_warm_chain_with_reputation_floors_and_scale():
    t, cap = tables(120, 1500, 31)
    rng = np.random.default_rng(31)
    rep = rng.integers(0, 4, 1500).astype(np.uint32)
    floors = rng.integers(0, 3, 120).astype(np.uint32)
    chain(t, cap, 31, 8, floors=floors, reputation=rep)
    chain(t, cap, 32, 6, S=121)


@pytest.mark.parametrize("n_base,copies,n_workers,plo,phi,seed", [(12, 40, 3000, 10, 14, 5), (3, 200, 2500, 7, 9, 8)])
def test_warm_chain_identical_bidders_and_ties(n_base, copies, n_workers, plo, phi, seed):
    t, cap = tables(n_base, n_workers, seed, dup=(copies, plo, phi))
    chain(t, cap, seed, 6)


@pytest.mark.parametrize("tune", [1, 2, 8, 16, 32, 64, 128, 8 | 32, 64 | 32, 1 | 64, 128 | 32, 0x200, 0x100 | 16])
def test_warm_chain_every_shortcut_can_be_switched_off(tune):
    t, cap = tables(25, 6000, 7, dup=(20, 5, 120))
    chain(t, cap, 70 + tune, 4, tune=tune)


def test_cold_pass_prices_equal_the_oracle():
    t, cap = tables(300, 2500, 9)
    eng = engine(t, cap)
    got, price, st, warm, released = run(eng, 300, abi.PM_MODE_AUCTION)
    want, wprice, rounds = orc.soa_auction(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    assert np.array_equal(got, want) and np.array_equal(price, wprice) and st["n_rounds"] == rounds
    assert not warm and released == 0
    eng.close()


def test_state_before_any_auction_pass():
    t, cap = tables(20, 200, 1)
    eng = engine(t, cap)
    with pytest.raises(PrimeMatchError) as ex:
        eng.auction_state()
    assert ex.value.status == abi.PM_E_STATE
    eng.match(abi.PM_MODE_FIRST_FIT)            # a reference-mode pass stores no auction state
    with pytest.raises(PrimeMatchError) as ex:
        eng.auction_state()
    assert ex.value.status == abi.PM_E_STATE
    eng.close()


def test_cutoff_exceeded_runs_cold():
    t, cap = tables(64, 1025, 4)
    m = wc.Market(t, cap)
    eng = engine(t, cap, incr=5)
    check_pass(eng, m, 1, want_warm=False)
    rng = np.random.default_rng(4)
    wc.random_step(m, rng, n_rows=3, eng=eng, kinds=("price",))
    check_pass(eng, m, 1, want_warm=True)      # 3 rows: within the cutoff
    wc.random_step(m, rng, n_rows=10, eng=eng, kinds=("price",))
    assert m.n_changes() > 5
    check_pass(eng, m, 1, want_warm=False)     # 10 rows: cold, and equal to the cold checker on the current tables
    eng.close()


def test_discarding_calls_give_a_cold_pass():
    t, cap = tables(50, 700, 2)
    T = 50
    calls = [
        lambda e: (e.set_asks(t["asks"], t["opts"]), e.set_price_caps(cap)),
        lambda e: e.set_model_table(t["bits"], t["n_patterns"], t["n_models"], t["words"]),
        lambda e: e.set_workers(t["wa"], t["wb"]),                 # pm_set_worker_count + upsert
        lambda e: e.set_auction_params(),
        lambda e: e.set_shard(0, 0),
        lambda e: e.attach_comm(None),
    ]
    m = wc.Market(t, cap)
    eng = engine(t, cap)
    check_pass(eng, m, 1, want_warm=False)
    for call in calls:
        check_pass(eng, m, 1, want_warm=True)  # nothing changed: warm, nothing released
        call(eng)
        check_pass(eng, m, 1, want_warm=False)
    eng.close()


def test_reference_pass_between_changes_nothing():
    t, cap = tables(300, 2500, 3)
    rng = np.random.default_rng(3)
    m = wc.Market(t, cap)
    eng = engine(t, cap)
    check_pass(eng, m, 1, want_warm=False)
    for step in range(4):
        wc.random_step(m, rng, eng=eng, kinds=("price", "flags", "spec"))
        eng.match(abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS | abi.PM_INCREMENTAL)
        check_pass(eng, m, 1, want_warm=True)
    eng.close()


def test_refusals():
    t, cap = tables(50, 700, 2)
    eng = engine(t, cap)
    for mode in (abi.PM_MODE_FIRST_FIT | abi.PM_AUCTION_WARM, abi.PM_MODE_PROXIMITY | abi.PM_AUCTION_WARM,
                 abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS | abi.PM_AUCTION_WARM,
                 WARM | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS | abi.PM_INCREMENTAL):
        with pytest.raises(PrimeMatchError) as ex:
            eng.match(mode)
        assert ex.value.status == abi.PM_E_INVALID, hex(mode)
    with pytest.raises(PrimeMatchError) as ex:
        eng.match_local(abi.PM_MODE_FIRST_FIT | abi.PM_AUCTION_WARM)
    assert ex.value.status == abi.PM_E_INVALID
    eng.set_ask_enabled([3], False)
    with pytest.raises(PrimeMatchError) as ex:
        eng.match(WARM)
    assert ex.value.status == abi.PM_E_UNSUPPORTED
    eng.set_ask_enabled([3], True)
    eng.set_shard(0, 350)
    with pytest.raises(PrimeMatchError) as ex:
        eng.match(WARM)
    assert ex.value.status == abi.PM_E_UNSUPPORTED
    eng.close()


def cfg3():
    T, W = 100_000, 1_000_000
    w = synth.make_workers(W, seed=synth.SEED_WORKERS)
    a = synth.make_asks(T, "mixed", seed=synth.SEED_ASKS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b.copy(), bits=bits, n_patterns=npat, n_models=nmod, words=words)
    t["wb"]["ext_ask_price"] = np.exp(np.log(10) + synth._unit(synth.SEED_EXT, W, 1) * np.log(200)).astype(np.uint32)
    cap = np.exp(np.log(20) + synth._unit(synth.SEED_EXT, T, 2) * np.log(150)).astype(np.uint32)
    return t, cap


def test_warm_pass_at_cfg3_size():
    """100k asks x 1M workers (tools/auction_scale.py's instance): one cold pass, 1 000 rows rewritten (half of them held),
    one warm pass.  Feasible, injective, unowned workers at price 0, and eps-complementary slackness on a sample of asks
    against every worker (values from the device's prices, feasibility from the oracle's predicate)."""
    t, cap = cfg3()
    T, W = len(cap), len(t["wa"])
    eng = engine(t, cap)
    got, price, st, warm, _ = run(eng, T)
    assert not warm
    rng = np.random.default_rng(5)
    held = got[got != NONE]
    idx = np.unique(np.concatenate([rng.choice(held, 500, replace=False), rng.choice(W, 500, replace=False)])).astype(np.uint32)
    a, b = t["wa"][idx].copy(), t["wb"][idx].copy()
    b["ext_ask_price"] = np.maximum(1, b["ext_ask_price"] // 2)
    t["wa"][idx], t["wb"][idx] = a, b
    eng.update_workers(idx, a, b)
    got, price, st, warm, released = run(eng, T)
    assert warm and released > 0 and st["n_rounds"] > 0
    ap = t["wb"]["ext_ask_price"].astype(np.int64)
    sold = np.flatnonzero(got != NONE)
    assert len(np.unique(got[sold])) == len(sold) and np.all(ap[got[sold]] <= cap[sold])
    owned = np.zeros(W, dtype=bool)
    owned[got[sold]] = True
    assert np.all(price[~owned] == 0)
    value = -ap - price
    for tk in rng.choice(T, 40, replace=False):
        F = wc.feasible(t["wa"], t["wb"], t["asks"][tk:tk + 1], t["opts"], t["bits"], t["words"], cap[tk:tk + 1])[0]
        best = value[F].max() if F.any() else wc.NEG
        outside = -(int(cap[tk]) + 1)
        if got[tk] != NONE:
            assert F[got[tk]] and value[got[tk]] >= max(best, outside) - 1
        else:
            assert best < outside
    eng.close()
