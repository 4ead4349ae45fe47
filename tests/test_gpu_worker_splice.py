"""Removing and inserting worker rows anywhere in the table on the device (pm_remove_workers / pm_insert_workers).

Twins: engine A takes random worker splices among pm_update_workers, pm_resize_workers, pm_set_flags,
pm_set_ask_enabled and ask splices; engine B is loaded fresh with the current rows.  Every pm_fetch_result array and
pm_build_cost_tile must be equal, in every reference mode, on every path, with and without PM_INCREMENTAL, sharded
and through pm_multi, and the incremental pass stays incremental.  A tail splice equals pm_resize_workers (+
pm_update_workers) field by field.  Warm and repair auction passes after splices equal the numpy checkers run from the
host-remapped state, under every PM_TUNE_AUCTION shortcut switch and with reputation floors; past the cutoff the pass
is a fresh cold one.  At cfg3, 1 000 removed held workers and 1 000 inserted rows leave the engine equal to a fresh
one.  Refusals change nothing."""
import ctypes as C

import numpy as np
import pytest

import auction_repair_checker as rp
from helpers import load_engine
from protocol_b200 import abi
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine, MultiEngine
from protocol_b200.sharded import shard_range, wrap_device_buffers
from test_gpu_ask_deltas import MODES, PATHS, REPAIR, TUNES, WARM, pool_tables, same, twins
from test_gpu_ask_splice import SpliceRows
from test_gpu_auction_warm import engine as auction_engine
from test_gpu_auction_warm import run as auction_run
from test_gpu_auction_warm import tables as auction_tables
from test_gpu_incremental import GROUPS, INCR, LEAN
from test_worker_splice_formulation import Splice, SpliceMarket, exported, remap_holds, remap_prices

pytestmark = pytest.mark.gpu

NONE = abi.PM_NONE


class Workers:
    """The caller's worker table (planes, location, address rank) and its changes, sent to the engines given."""

    def __init__(self, w, rank):
        self.pool_a, self.pool_b, self.pool_lat, self.pool_lon = w.a.copy(), w.b.copy(), w.lat.copy(), w.lon.copy()
        self.a, self.b, self.lat, self.lon = w.a.copy(), w.b.copy(), w.lat.copy(), w.lon.copy()
        self.rank = rank.copy()
        self.next_rank = int(rank.max()) + 1 if len(rank) else 0

    def fresh_ranks(self, engs, idx):
        """New rows come with address rank 0; give each a rank of its own, as distinct addresses have (rows with equal
        ranks have no defined member order)."""
        for i in np.asarray(idx, dtype=np.int64):
            r = np.array([self.next_rank], dtype=np.uint32)
            self.next_rank += 1
            for e in engs:
                fn = e._lib.pm_multi_set_worker_addr_rank if isinstance(e, MultiEngine) else e._lib.pm_set_worker_addr_rank
                assert fn(e._h, C.c_void_p(r.ctypes.data), int(i), 1) == 0
            self.rank[i] = r[0]

    def step(self, rng, engs, kinds=("remove", "insert", "remove", "insert", "update", "resize", "flags")):
        W = len(self.a)
        kind = kinds[rng.integers(len(kinds))]
        if kind == "remove" and W > 50:
            idx = rng.integers(0, W, int(rng.integers(1, 40))).astype(np.uint32)   # any order, repeats once
            for e in engs:
                e.remove_workers(idx)
            sp = Splice(W, idx)
            for f in ("a", "b", "lat", "lon", "rank"):
                setattr(self, f, sp.apply(getattr(self, f), None))
        elif kind == "insert" or kind == "remove":
            k = int(rng.integers(1, 40))
            before = np.sort(rng.integers(0, W + 1, k)).astype(np.uint32)
            if rng.random() < 0.2:
                before[:] = rng.integers(0, 2) * W            # all at the front or all at the end
            src = rng.integers(0, len(self.pool_a), k)
            a, b, la, lo = self.pool_a[src], self.pool_b[src], self.pool_lat[src], self.pool_lon[src]
            with_loc = rng.random() < 0.7
            for e in engs:
                e.insert_workers(before, a, b, la if with_loc else None, lo if with_loc else None)
            sp = Splice(W, (), before)
            self.a, self.b = sp.apply(self.a, a), sp.apply(self.b, b)
            self.lat = sp.apply(self.lat, la if with_loc else None)
            self.lon = sp.apply(self.lon, lo if with_loc else None)
            self.rank = sp.apply(self.rank, None)
            self.fresh_ranks(engs, sp.at())
            kind = "insert"
        elif kind == "update":
            idx = np.unique(rng.integers(0, W, int(rng.integers(1, 30)))).astype(np.uint32)
            src = rng.integers(0, len(self.pool_a), len(idx))
            for e in engs:
                e.update_workers(idx, self.pool_a[src], self.pool_b[src], self.pool_lat[src], self.pool_lon[src])
            self.a[idx], self.b[idx] = self.pool_a[src], self.pool_b[src]
            self.lat[idx], self.lon[idx] = self.pool_lat[src], self.pool_lon[src]
        elif kind == "resize":
            n = W + int(rng.integers(-20, 20))
            for e in engs:
                e.resize_workers(n)
            if n < W:
                for f in ("a", "b", "lat", "lon", "rank"):
                    setattr(self, f, getattr(self, f)[:n].copy())
            else:
                z = n - W
                self.a = np.concatenate([self.a, np.zeros(z, abi.WORKER_A)])
                self.b = np.concatenate([self.b, np.zeros(z, abi.WORKER_B)])
                self.lat, self.lon = np.concatenate([self.lat, np.zeros(z)]), np.concatenate([self.lon, np.zeros(z)])
                self.rank = np.concatenate([self.rank, np.zeros(z, np.uint32)])
                self.fresh_ranks(engs, np.arange(W, n))
        else:
            idx = np.unique(rng.integers(0, W, int(rng.integers(1, 30)))).astype(np.uint32)
            flags = self.a["flags"][idx] ^ abi.PM_W_HEALTHY
            for e in engs:
                e.set_flags(idx, flags)
            self.a["flags"][idx] = flags
        return kind

    def fresh(self, eng):
        eng.set_workers(self.a, self.b)
        eng.set_locations(self.lat, self.lon)
        eng.set_addr_rank(self.rank)


def fresh_twin(B, rows, workers):
    rows.fresh(B)
    workers.fresh(B)


# ------------------------------------------------------------------ 1. twins: every mode and path
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("mode", list(MODES))
def test_twins_every_mode_and_path(mode, path):
    base, sizes, edges = MODES[mode]
    fa, fb, env = PATHS[path]
    seed = 800 + len(mode) * 3 + len(path)
    rng = np.random.default_rng(seed)
    w, pool, t = pool_tables(150, 3000, sizes, seed, edges=edges)
    rank = rng.permutation(len(w)).astype(np.uint32)
    A, B = twins(t, env, rank)
    rows = SpliceRows(pool, t["opts"], 150)
    wk = Workers(w, rank)
    A.match(base | fa)
    kinds = {}
    for step in range(12):
        kind = wk.step(rng, [A], **({"kinds": (("remove",), ("insert",))[step]} if step < 2 else {}))
        kinds[kind] = kinds.get(kind, 0) + 1
        if step % 3 == 2:
            rows.step(rng, [A])
        fresh_twin(B, rows, wk)
        A.match(base | fa)
        B.match(base | fb)
        same(A.fetch(), B.fetch(), f"{mode}/{path} step {step} ({kind})")
        if path in ("materialized", "fused") and step % 4 == 0:
            T = len(rows.asks)
            assert np.array_equal(A.cost_tile(0, T), B.cost_tile(0, T)), f"cost tile, step {step}"
    assert kinds.get("remove") and kinds.get("insert")
    A.close()
    B.close()


def test_splices_stay_incremental():
    """After removals the next incremental pass walks nothing; after insertions it walks the inserted rows only; a
    refused call lists nothing."""
    w, pool, t = pool_tables(300, 20000, GROUPS, 805, edges=False)
    rank = np.arange(20000, dtype=np.uint32)
    A, B = twins(t, None, rank)
    rows = SpliceRows(pool, t["opts"], 300)
    wk = Workers(w, rank)
    A.match(abi.PM_MODE_FIRST_FIT | INCR)
    T = 300
    for kind, n_walk in (("remove", 0), ("insert", None)):
        W = len(wk.a)
        before = len(wk.a)
        rng = np.random.default_rng(len(kind))
        wk.step(rng, [A], kinds=(kind,))
        n_ins = len(wk.a) - before if kind == "insert" else 0
        fresh_twin(B, rows, wk)
        A.match(abi.PM_MODE_FIRST_FIT | INCR)
        B.match(abi.PM_MODE_FIRST_FIT | LEAN)
        same(A.fetch(), B.fetch(), f"after {kind}")
        st = A.stats()
        assert st["n_tiles"] == (n_ins if n_walk is None else n_walk), (kind, st)
        assert st["evals"] <= st["n_tiles"] * T < T * W, (kind, st)
    with pytest.raises(PrimeMatchError):
        A.remove_workers([len(wk.a)])
    A.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert A.stats()["evals"] == 0
    A.close()
    B.close()


# ------------------------------------------------------------------ 2. a tail splice is pm_resize_workers
def _stats(e):
    return {k: v for k, v in e.stats().items() if not k.startswith("ms_")}


@pytest.mark.parametrize("demand", [False, True], ids=["one_slot", "demands"])
def test_tail_splice_equals_resize(demand):
    t, cap = auction_tables(80, 1500, 861)
    rng = np.random.default_rng(861)
    A, B = auction_engine(t, cap), auction_engine(t, cap)
    d = rng.integers(1, 4, 80).astype(np.uint32)
    for e in (A, B):
        if demand:
            e.set_ask_demand(d)
        e.match(abi.PM_MODE_FIRST_FIT | INCR)
        e.match(WARM)
    wa, wb = t["wa"], t["wb"]
    for step, mode in enumerate((WARM, REPAIR, abi.PM_MODE_AUCTION | abi.PM_AUCTION_REVERSE, REPAIR, WARM)):
        W = A.n_workers
        va, vb = A.table_version(), B.table_version()
        n = int(rng.integers(5, 40))
        if step % 2 == 0:
            A.remove_workers(np.arange(W - n, W)[::-1])
            B.resize_workers(W - n)
        else:
            src = rng.integers(0, len(wa), n)
            A.insert_workers(np.full(n, W, np.uint32), wa[src], wb[src])
            B.resize_workers(W + n)
            B.update_workers(np.arange(W, W + n, dtype=np.uint32), wa[src], wb[src])
        assert A.table_version() > va and B.table_version() > vb
        for m in (abi.PM_MODE_FIRST_FIT | INCR, mode):
            A.match(m)
            B.match(m)
            same(A.fetch(), B.fetch(), f"step {step} {m:#x}")
            assert _stats(A) == _stats(B), f"step {step} {m:#x}"
        pa, pb = A.auction_state(), B.auction_state()
        assert np.array_equal(pa[0], pb[0]) and pa[1:] == pb[1:]
        assert A.auction_reverse_stats() == B.auction_reverse_stats()
        assert np.array_equal(A.auction_slot_assignment(), B.auction_slot_assignment())
    A.close()
    B.close()


# ------------------------------------------------------------------ 3. the auction from the remapped state
def market_of(t, cap, rep=None, floors=None):
    m = SpliceMarket.__new__(SpliceMarket)
    SpliceMarket.__init__(m, t, cap, reputation=rep, floors=floors)
    return m


def splice_step(m, rng, eng, held_only):
    W = m.n_workers
    if rng.random() < 0.5 and W > 50:
        held = m.assigned[(m.assigned != NONE) & (m.assigned < W)]
        pool = held if held_only and len(held) else np.arange(W)
        idx = rng.choice(pool, min(len(pool), int(rng.integers(1, 12))), replace=False)
        m.splice(idx.astype(np.uint32), eng=eng)
        return "remove"
    k = int(rng.integers(1, 12))
    src = rng.integers(0, W, k)
    m.splice((), np.sort(rng.integers(0, W + 1, k)), m.wa[src].copy(), m.wb[src].copy(), eng=eng)
    return "insert"


def splice_chain(seed, steps, tune=0, repair=False, n_asks=60, n_workers=900, floors=False):
    t, cap = auction_tables(n_asks, n_workers, seed)
    rng = np.random.default_rng(seed)
    rep = fl = None
    if floors:
        rep = rng.integers(0, 4, n_workers).astype(np.uint32)
        fl = rng.integers(0, 3, n_asks).astype(np.uint32)
    m = market_of(t, cap, rep, fl)
    eng = auction_engine(t, cap, tune=tune, floors=fl, reputation=rep)
    mode = REPAIR if repair else WARM
    got, price, st, warm, released = auction_run(eng, n_asks, mode)
    a, p, n = m.cold()
    assert not warm and np.array_equal(got, a) and np.array_equal(price, p) and st["n_rounds"] == n
    m.store(p, a)
    kinds = set()
    for step in range(steps):
        for _ in range(int(rng.integers(1, 3))):
            before = exported(m.assigned)
            kinds.add(splice_step(m, rng, eng, held_only=step % 2 == 0))
            assert np.array_equal(eng.auction_assignment(), exported(m.assigned)), f"export, step {step}"
            assert np.array_equal(eng.auction_state()[0], m.price), f"prices, step {step}"
            assert len(before) == n_asks
        if floors and step % 2:   # the inserted rows come with reputation 0
            r = rng.integers(0, 4, m.n_workers).astype(np.uint32)
            m.set_reputation(0, r, eng)
        with pytest.raises(PrimeMatchError) as ex:
            eng.auction_certificate()
        assert ex.value.status == abi.PM_E_STATE
        got, price, st, warm, released = auction_run(eng, n_asks, mode)
        assert warm, f"step {step}"
        if repair:
            out = rp.market_repair(m)
            a, p = out["assigned"], out["price"]
            assert released == len(out["released"]) and st["n_rounds"] == out["fwd"]
        else:
            a, p, n, rel = m.warm()
            assert released == len(rel) and st["n_rounds"] == n
        assert np.array_equal(got, a), f"step {step}"
        assert np.array_equal(price, p), f"step {step}"
        m.store(p, a)
        cert = eng.auction_certificate()
        assert cert["n_bad_holds"] == 0 and cert["gap"] <= n_asks
    eng.close()
    return kinds


@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
@pytest.mark.parametrize("seed", [2, 3])
def test_auction_chain_matches_checker(seed, repair):
    assert splice_chain(870 + seed, 8, repair=repair) == {"remove", "insert"}


@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
def test_auction_chain_under_reputation_floors(repair):
    splice_chain(880, 6, repair=repair, floors=True)


@pytest.mark.parametrize("tune", TUNES)
def test_auction_chain_every_shortcut_can_be_switched_off(tune):
    splice_chain(890 + tune, 4, tune=tune, repair=bool(tune & 1), n_asks=30, n_workers=3000)


def test_slot_assignment_after_splices_with_demands():
    """With demands the per-slot export after a splice is the earlier one renamed, a removed holder PM_NONE, and the
    prices are the earlier ones moved with their rows.  The warm pass that follows equals a twin loaded with the
    current rows and given the remapped export through pm_auction_restore_slots (the inserted rows written on the
    twin too, as changed rows): the same groups, prices and rounds; after a removal it also releases each removed
    holder once more than the twin, whose restored slots hold nothing there."""
    t, cap = auction_tables(60, 2000, 871)
    rng = np.random.default_rng(871)
    d = rng.integers(1, 4, 60).astype(np.uint32)
    eng = auction_engine(t, cap)
    eng.set_ask_demand(d)
    eng.match(WARM)
    wa, wb = t["wa"].copy(), t["wb"].copy()
    for step in range(4):
        W = len(wa)
        before_export = eng.auction_slot_assignment()
        price_before = eng.auction_state()[0]
        if step % 2 == 0:
            held = before_export[before_export != NONE]
            idx = rng.choice(held, 6, replace=False)
            eng.remove_workers(idx)
            sp = Splice(W, idx)
            ins = None
        else:
            bf = np.sort(rng.integers(0, W + 1, 9)).astype(np.uint32)
            src = rng.integers(0, len(t["wa"]), 9)
            eng.insert_workers(bf, t["wa"][src], t["wb"][src])
            sp = Splice(W, (), bf)
            ins = (t["wa"][src], t["wb"][src])
        wa = sp.apply(wa, None if ins is None else ins[0])
        wb = sp.apply(wb, None if ins is None else ins[1])
        want = exported(remap_holds(sp, before_export, sp.n_old))
        assert np.array_equal(eng.auction_slot_assignment(), want), f"step {step}"
        want_price = remap_prices(sp, price_before, sp.n_old)
        assert np.array_equal(eng.auction_state()[0], want_price), f"prices, step {step}"
        twin = auction_engine(dict(t, wa=wa, wb=wb), cap)
        twin.set_ask_demand(d)
        twin.auction_restore_slots(want_price, want)
        if ins is not None:
            twin.update_workers(sp.at().astype(np.uint32), *ins)
        for e in (eng, twin):
            e.match(WARM)
        r, q = eng.fetch(), twin.fetch()
        same(r, q, f"step {step}")
        assert r.stats["n_rounds"] == q.stats["n_rounds"], f"step {step}"
        price, warm, released = eng.auction_state()
        p2, w2, rel2 = twin.auction_state()
        assert warm and w2 and len(price) == sp.n_new and np.array_equal(price, p2), f"step {step}"
        if ins is None:
            assert released == rel2 + 6, (released, rel2)
        twin.close()
    eng.close()


def test_auction_past_the_cutoff_equals_a_fresh_cold_pass():
    t, cap = auction_tables(60, 1500, 873)
    eng = auction_engine(t, cap, incr=6)
    auction_run(eng, 60, WARM)
    src = np.arange(8)
    eng.insert_workers(np.full(8, 10, np.uint32), t["wa"][src], t["wb"][src])   # 8 changed rows: past the cutoff of 6
    got, price, st, warm, _ = auction_run(eng, 60, WARM)
    sp = Splice(1500, (), np.full(8, 10))
    fresh = auction_engine(dict(t, wa=sp.apply(t["wa"], t["wa"][src]), wb=sp.apply(t["wb"], t["wb"][src])), cap)
    g2, p2, st2, w2, _ = auction_run(fresh, 60, abi.PM_MODE_AUCTION)
    assert not warm and not w2
    assert np.array_equal(got, g2) and np.array_equal(price, p2) and st["n_rounds"] == st2["n_rounds"]
    eng.close()
    fresh.close()


# ------------------------------------------------------------------ 4. sharded engines and pm_multi
def test_sharded_twins():
    """Three shard engines: the first two on fixed pm_set_shard ranges, which stay where they are while rows shift
    through them, the last on an open-ended range, which moves with W."""
    import torch

    n_shards = 3
    rng = np.random.default_rng(875)
    w, pool, t = pool_tables(160, 10007, [(1, 1), (2, 4), (3, 3)], 875, edges=False)
    rank = np.arange(len(w), dtype=np.uint32)
    engs, bounds = [], []
    for r in range(n_shards):
        lo, hi = shard_range(len(w), n_shards, r)
        e = Engine(cost_tile_bytes=1 << 20)
        load_engine(e, t, addr_rank=rank, locations=True)
        e.set_shard(lo, hi - lo if r < n_shards - 1 else 0)
        bounds.append((lo, hi))
        engs.append(e)
    B = Engine()
    load_engine(B, t)
    rows = SpliceRows(pool, t["opts"], 160)
    wk = Workers(w, rank)
    for step in range(8):
        if step:
            wk.step(rng, engs, kinds=("remove", "insert"))
        W = len(wk.a)
        ranges = bounds[:-1] + [(bounds[-1][0], W)]
        fresh_twin(B, rows, wk)
        T = len(rows.asks)
        for flags, ref in ((INCR, LEAN), (abi.PM_PATH_MATERIALIZED, abi.PM_PATH_MATERIALIZED)):
            mode = abi.PM_MODE_FIRST_FIT | flags
            bufs = []
            for e in engs:
                e.match_local(mode)
                e.sync()
                bufs.append(wrap_device_buffers(e, W, T))
            first = torch.cat([bufs[r][0][lo:hi] for r, (lo, hi) in enumerate(ranges)])
            best = torch.stack([b[1] for b in bufs]).min(dim=0).values
            cnt = torch.stack([b[2] for b in bufs]).sum(dim=0).to(torch.int32)
            B.match(abi.PM_MODE_FIRST_FIT | ref)
            q = B.fetch()
            for r, e in enumerate(engs):
                bufs[r][0].copy_(first)
                bufs[r][1].copy_(best)
                bufs[r][2].copy_(cnt)
                torch.cuda.synchronize()
                e.match_finish(mode)
                same(e.fetch(), q, f"rank {r}, step {step}, {flags:#x}")
            if flags == INCR and step:
                assert all(e.stats()["n_tiles"] < hi - lo for e, (lo, hi) in zip(engs, ranges)), step
    for e in engs + [B]:
        e.close()


def test_multi_twins():
    rng = np.random.default_rng(877)
    w, pool, t = pool_tables(150, 8000, GROUPS, 877, edges=False)
    M = MultiEngine([0])
    M.set_asks(t["asks"], t["opts"])
    M.set_model_table(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    M.set_workers(t["wa"], t["wb"])
    M.set_locations(t["lat"], t["lon"])
    rank = np.arange(len(w), dtype=np.uint32)
    M.set_addr_rank(rank)
    B = Engine()
    load_engine(B, t)
    rows = SpliceRows(pool, t["opts"], 150)
    wk = Workers(w, rank)
    M.match(abi.PM_MODE_FIRST_FIT | INCR)
    for step in range(8):
        wk.step(rng, [M])
        fresh_twin(B, rows, wk)
        M.match(abi.PM_MODE_FIRST_FIT | INCR)
        B.match(abi.PM_MODE_FIRST_FIT | LEAN)
        same(M.fetch(), B.fetch(), f"pm_multi, step {step}")
    lib, h = M._lib, M._h
    idx = np.array([1, len(wk.a)], dtype=np.uint32)
    assert lib.pm_multi_remove_workers(h, C.c_void_p(idx.ctypes.data), 2) == abi.PM_E_INVALID
    M.match(abi.PM_MODE_FIRST_FIT | INCR)
    same(M.fetch(), B.fetch(), "after a refused pm_multi_remove_workers")
    B.close()
    M.close()


# ------------------------------------------------------------------ 5. refusals change nothing
def test_refusals_change_nothing():
    t, cap = auction_tables(60, 1200, 879)
    eng = auction_engine(t, cap)
    eng.set_ask_demand(np.full(60, 2, np.uint32))
    eng.match(abi.PM_MODE_FIRST_FIT | INCR)
    eng.match(WARM)
    lib, h = eng._lib, eng._h
    P = lambda a: C.c_void_p(a.ctypes.data)
    a, b = np.ascontiguousarray(t["wa"][:2]), np.ascontiguousarray(t["wb"][:2])
    la = np.zeros(2)
    idx = np.array([3, 4], dtype=np.uint32)
    far = np.array([3, 1200], dtype=np.uint32)
    dec = np.array([5, 4], dtype=np.uint32)
    past = np.array([4, 1201], dtype=np.uint32)
    calls = [
        lambda: lib.pm_remove_workers(h, None, 2),
        lambda: lib.pm_remove_workers(h, P(far), 2),
        lambda: lib.pm_insert_workers(h, None, P(a), P(b), None, None, 2),
        lambda: lib.pm_insert_workers(h, P(idx), None, P(b), None, None, 2),
        lambda: lib.pm_insert_workers(h, P(idx), P(a), None, None, None, 2),
        lambda: lib.pm_insert_workers(h, P(idx), P(a), P(b), P(la), None, 2),
        lambda: lib.pm_insert_workers(h, P(idx), P(a), P(b), None, P(la), 2),
        lambda: lib.pm_insert_workers(h, P(dec), P(a), P(b), None, None, 2),
        lambda: lib.pm_insert_workers(h, P(past), P(a), P(b), None, None, 2),
        lambda: lib.pm_insert_workers(h, P(idx), P(a), P(b), None, None, 0xFFFFFFFF - 1200),
    ]
    v = eng.table_version()
    slots = eng.auction_slot_assignment()
    state = eng.auction_state()
    for i, call in enumerate(calls):
        assert call() == abi.PM_E_INVALID, i
    assert eng.table_version() == v
    assert np.array_equal(eng.auction_slot_assignment(), slots)
    after = eng.auction_state()
    assert np.array_equal(state[0], after[0]) and state[1:] == after[1:]
    eng.auction_certificate()                       # still the stored pass's
    e = Engine()
    assert e._lib.pm_remove_workers(e._h, P(idx), 2) == abi.PM_E_STATE
    assert e._lib.pm_insert_workers(e._h, P(idx), P(a), P(b), None, None, 2) == abi.PM_E_STATE
    e.close()
    eng.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert eng.stats()["evals"] == 0
    eng.remove_workers([2, 30])
    with pytest.raises(PrimeMatchError) as ex:
        eng.auction_certificate()
    assert ex.value.status == abi.PM_E_STATE
    eng.close()


# ------------------------------------------------------------------ 6. full size: cfg3
def test_cfg3_splice():
    """bench.py's market at cfg3: 1 000 held workers removed at scattered positions and 1 000 rows inserted.  The lean
    incremental pass and a cold auction pass equal a fresh engine's; the warm pass that follows certifies within T."""
    from test_gpu_bench_workloads import FF, TILE, load, workload
    from protocol_b200 import synth

    w, a, tbl, _ = workload("cfg3")
    T, W = len(a.asks), len(w.a)
    caps = np.exp(np.log(20) + synth._unit(synth.SEED_EXT, T, 3) * np.log(100)).astype(np.uint32)
    rng = np.random.default_rng(881)
    e = Engine(cost_tile_bytes=TILE)
    load(e, w, a, tbl)
    e.set_price_caps(caps)
    e.match(FF | LEAN | abi.PM_INCREMENTAL)
    e.match(abi.PM_MODE_AUCTION)
    held = e.auction_assignment()
    held = held[held != NONE]
    rm = rng.choice(held, 1000, replace=False).astype(np.uint32)
    e.remove_workers(rm[::-1])
    sp1 = Splice(W, rm)
    src = rng.integers(0, W, 1000)
    bf = np.sort(rng.integers(0, sp1.n_new + 1, 1000)).astype(np.uint32)
    e.insert_workers(bf, w.a[src], w.b[src])
    sp2 = Splice(sp1.n_new, (), bf)
    wa, wb = sp2.apply(sp1.apply(w.a, None), w.a[src]), sp2.apply(sp1.apply(w.b, None), w.b[src])
    f = Engine(cost_tile_bytes=TILE)
    f.set_asks(a.asks, a.opts)
    f.set_model_table(*tbl)
    f.set_workers(wa, wb)
    f.set_price_caps(caps)
    e.match(FF | LEAN | abi.PM_INCREMENTAL)
    f.match(FF | LEAN)
    same(e.fetch(), f.fetch(), "cfg3 lean incremental")
    assert e.stats()["n_tiles"] <= 1000
    e.match(WARM)
    assert e.auction_state()[1]
    cert = e.auction_certificate()
    assert cert["n_bad_holds"] == 0 and cert["gap"] <= T
    e.match(abi.PM_MODE_AUCTION)
    f.match(abi.PM_MODE_AUCTION)
    same(e.fetch(), f.fetch(), "cfg3 cold auction")
    e.close()
    f.close()
