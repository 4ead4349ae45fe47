"""Removing and inserting asks anywhere in the table on the device (pm_remove_asks / pm_insert_asks).

Twins: engine A takes random splices among the other table calls; engine B gets pm_set_asks with the current rows and
mask.  Every pm_fetch_result array and pm_build_cost_tile must be equal, in every reference mode, on every path, with
and without PM_INCREMENTAL, sharded and through pm_multi, and the incremental pass stays incremental.  A tail splice
equals pm_resize_asks field by field.  Warm and repair auction passes after splices equal the numpy checkers run from
the remapped state, under every PM_TUNE_AUCTION shortcut switch, with demands and reputation floors.  At cfg3, 1 000
removed held asks and 1 000 inserted rows leave the engine equal to a fresh one.  Refusals change nothing."""
import ctypes as C

import numpy as np
import pytest

import auction_repair_checker as rp
from helpers import load_engine
from protocol_b200 import abi, synth
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine, MultiEngine
from protocol_b200.sharded import shard_range, wrap_device_buffers
from test_ask_deltas_formulation import own_options
from test_ask_splice_formulation import SpliceMarket, splice_step
from test_gpu_ask_deltas import MODES, PATHS, REPAIR, TUNES, WARM, Rows, pool_tables, same, twins, workers_step
from test_gpu_auction_warm import engine as auction_engine
from test_gpu_auction_warm import run as auction_run
from test_gpu_auction_warm import tables as auction_tables
from test_gpu_incremental import GROUPS, INCR, LEAN

pytestmark = pytest.mark.gpu

NONE = abi.PM_NONE


class SpliceRows(Rows):
    """Rows with remove / insert steps too."""

    def step(self, rng, engs, kinds=("remove", "insert", "remove", "insert", "replace", "append", "shrink", "toggle")):
        T = len(self.asks)
        kind = kinds[rng.integers(len(kinds))]
        if kind == "remove" and T > 8:
            idx = rng.integers(0, T, int(rng.integers(1, 7))).astype(np.uint32)   # any order, repeats once
            for e in engs:
                e.remove_asks(idx)
            keep = np.setdiff1d(np.arange(T), idx)
            self.asks, self.mask = self.asks[keep].copy(), self.mask[keep].copy()
            return kind
        if kind == "insert":
            k = int(rng.integers(1, 6))
            before = np.sort(rng.integers(0, T + 1, k)).astype(np.uint32)
            rows = self.pool[rng.integers(0, len(self.pool), k)]
            sent = self.payload(rng, rows)
            for e in engs:
                e.insert_asks(before, *sent)
            self.asks = np.insert(self.asks, before.astype(np.int64), rows)
            self.mask = np.insert(self.mask, before.astype(np.int64), True)
            return kind
        return super().step(rng, engs, kinds=(kind,) if kind in ("replace", "append", "shrink", "toggle") else ("toggle",))


# ------------------------------------------------------------------ 1. twins: every mode and path
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("mode", list(MODES))
def test_twins_every_mode_and_path(mode, path):
    base, sizes, edges = MODES[mode]
    fa, fb, env = PATHS[path]
    seed = 500 + len(mode) * 3 + len(path)
    rng = np.random.default_rng(seed)
    w, pool, t = pool_tables(150, 3000, sizes, seed, edges=edges)
    rank = rng.permutation(len(w)).astype(np.uint32)
    A, B = twins(t, env, rank)
    rows = SpliceRows(pool, t["opts"], 150)
    A.match(base | fa)
    kinds = {}
    for step in range(12):
        kind = rows.step(rng, [A], **({"kinds": (("remove",), ("insert",))[step]} if step < 2 else {}))
        kinds[kind] = kinds.get(kind, 0) + 1
        if step % 4 == 3:
            workers_step(rng, w, [A, B])
        rows.fresh(B)
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
    """Removing asks that own workers walks only their orphans; inserting rows walks only the E-pass; a refused call
    lists nothing."""
    w, pool, t = pool_tables(300, 20000, GROUPS, 505, edges=False)
    W = 20000
    A, B = twins(t)
    rows = SpliceRows(pool, t["opts"], 300)
    A.match(abi.PM_MODE_FIRST_FIT | INCR)
    owners = np.bincount(A.fetch().worker_ask[A.fetch().worker_ask != NONE], minlength=300)
    idx = np.flatnonzero(owners)[[0, 3, 7]].astype(np.uint32)
    for call in (lambda e: e.remove_asks(idx), lambda e: e.insert_asks([0, 150, 150], pool[[400, 401, 402]], t["opts"])):
        call(A)
        if len(rows.asks) == 300:
            keep = np.setdiff1d(np.arange(300), idx)
            rows.asks, rows.mask = rows.asks[keep].copy(), rows.mask[keep].copy()
        else:
            rows.asks = np.insert(rows.asks, [0, 150, 150], pool[[400, 401, 402]])
            rows.mask = np.ones(len(rows.asks), bool)
        rows.fresh(B)
        A.match(abi.PM_MODE_FIRST_FIT | INCR)
        B.match(abi.PM_MODE_FIRST_FIT | LEAN)
        same(A.fetch(), B.fetch(), "after the splice")
        st = A.stats()
        assert st["n_tiles"] < W and st["evals"] < len(rows.asks) * W, st
    with pytest.raises(PrimeMatchError):
        A.remove_asks([len(rows.asks)])
    A.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert A.stats()["evals"] == 0
    A.close()
    B.close()


# ------------------------------------------------------------------ 2. a tail splice is pm_resize_asks
def _stats(e):
    return {k: v for k, v in e.stats().items() if not k.startswith("ms_")}


@pytest.mark.parametrize("demand", [False, True], ids=["one_slot", "demands"])
def test_tail_splice_equals_resize(demand):
    t, cap = auction_tables(110, 1500, 61)
    pool = t["asks"].copy()
    t = dict(t, asks=pool[:80])
    rng = np.random.default_rng(61)
    A, B = auction_engine(t, cap[:80]), auction_engine(t, cap[:80])
    d = rng.integers(1, 4, 80).astype(np.uint32)
    for e in (A, B):
        if demand:
            e.set_ask_demand(d)
        e.match(abi.PM_MODE_FIRST_FIT | INCR)
        e.match(WARM)
    caps = cap[:80].copy()
    for step, mode in enumerate((WARM, REPAIR, abi.PM_MODE_AUCTION | abi.PM_AUCTION_REVERSE, REPAIR)):
        T = len(caps)
        va, vb = A.table_version(), B.table_version()
        if step % 2 == 0:
            A.remove_asks(np.arange(T - 4, T)[::-1])
            B.resize_asks(T - 4)
            caps = caps[:T - 4]
        else:
            new = pool[80 + 4 * step:84 + 4 * step]
            A.insert_asks(np.full(4, T, np.uint32), *own_options(new, t["opts"]))
            B.resize_asks(T + 4, *own_options(new, t["opts"]))
            caps = np.concatenate([caps, rng.integers(50, 1500, 4).astype(np.uint32)])
        assert A.table_version() - va == B.table_version() - vb
        assert np.array_equal(A.auction_slot_assignment(), B.auction_slot_assignment()), step
        for e in (A, B):
            e.set_price_caps(caps)
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
def splice_chain(seed, steps, tune=0, repair=False, n_asks=60, n_workers=900, floors=False):
    t, cap = auction_tables(n_asks + 60, n_workers, seed)
    pool = t["asks"].copy()
    t = dict(t, asks=pool[:n_asks])
    rng = np.random.default_rng(seed)
    rep = fl = None
    if floors:
        rep = rng.integers(0, 4, n_workers).astype(np.uint32)
        fl = rng.integers(0, 3, n_asks).astype(np.uint32)
    m = SpliceMarket(t, cap[:n_asks], reputation=rep, floors=fl)
    eng = auction_engine(t, cap[:n_asks], tune=tune, floors=fl, reputation=rep)
    mode = REPAIR if repair else WARM
    got, price, st, warm, released = auction_run(eng, n_asks, mode)
    a, p, n = m.cold()
    assert not warm and np.array_equal(got, a) and np.array_equal(price, p) and st["n_rounds"] == n
    m.store(p, a)
    kinds = set()
    for step in range(steps):
        for _ in range(int(rng.integers(1, 3))):
            kinds.add(splice_step(m, pool, rng, eng=eng, held_only=step % 2 == 0))
        if floors:   # inserted rows come with floor 0: give them (and the other floor-0 asks) a floor
            fl = m.floors.copy()
            z = fl == 0
            fl[z] = rng.integers(0, 3, int(z.sum()))
            m.set_floors(fl, eng)
        T = len(m.asks)
        got, price, st, warm, released = auction_run(eng, T, mode)
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
        assert eng.auction_certificate()["n_bad_holds"] == 0
    eng.close()
    return kinds


@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
@pytest.mark.parametrize("seed", [2, 3])
def test_auction_chain_matches_checker(seed, repair):
    assert splice_chain(600 + seed, 8, repair=repair) == {"remove", "insert"}


@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
def test_auction_chain_under_reputation_floors(repair):
    splice_chain(640, 6, repair=repair, floors=True)


@pytest.mark.parametrize("tune", TUNES)
def test_auction_chain_every_shortcut_can_be_switched_off(tune):
    splice_chain(670 + tune, 4, tune=tune, repair=bool(tune & 1), n_asks=30, n_workers=3000)


def test_slot_assignment_after_splices_with_demands():
    """The export after a splice is the earlier one with the removed asks' slots cut out and PM_NONE for the inserted
    ones; the warm pass that follows equals a twin built by pm_set_asks + pm_auction_restore_slots of that export."""
    t, cap = auction_tables(120, 2000, 71)
    pool = t["asks"].copy()
    t = dict(t, asks=pool[:80])
    rng = np.random.default_rng(71)
    d = rng.integers(1, 4, 80).astype(np.uint32)
    eng = auction_engine(t, cap[:80])
    eng.set_ask_demand(d)
    eng.match(WARM)
    asks, caps = pool[:80].copy(), cap[:80].copy()
    for step in range(4):
        before_export = eng.auction_slot_assignment()
        off = np.concatenate([[0], np.cumsum(d)]).astype(np.int64)
        T = len(d)
        if step % 2 == 0:
            idx = rng.choice(T, 5, replace=False)
            eng.remove_asks(idx.astype(np.uint32))
            keep = np.setdiff1d(np.arange(T), idx)
            want = np.concatenate([before_export[off[k]:off[k + 1]] for k in keep])
            asks, caps, d = asks[keep], caps[keep], d[keep]
        else:
            before = np.sort(rng.integers(0, T + 1, 3)).astype(np.uint32)
            new = pool[100 + 3 * step:103 + 3 * step]
            eng.insert_asks(before, *own_options(new, t["opts"]))
            parts, j = [], 0
            for k in range(T + 1):
                while j < 3 and before[j] == k:
                    parts.append(np.full(1, NONE, np.uint32))
                    j += 1
                if k < T:
                    parts.append(before_export[off[k]:off[k + 1]])
            want = np.concatenate(parts)
            b = before.astype(np.int64)
            asks = np.insert(asks, b, new)
            caps = np.insert(caps, b, rng.integers(50, 1500, 3).astype(np.uint32))
            d = np.insert(d, b, 1).astype(np.uint32)
        got = eng.auction_slot_assignment()
        assert np.array_equal(got, want), f"step {step}"
        eng.set_price_caps(caps)
        price, _, _ = eng.auction_state()
        twin = auction_engine(dict(t, asks=asks), caps)
        twin.set_ask_demand(d)
        twin.auction_restore_slots(price, got)
        for e in (eng, twin):
            e.match(WARM)
        r, q = eng.fetch(), twin.fetch()
        same(r, q, f"step {step}")
        assert r.stats["n_rounds"] == q.stats["n_rounds"]
        assert np.array_equal(eng.auction_state()[0], twin.auction_state()[0])
        twin.close()
    eng.close()


# ------------------------------------------------------------------ 4. sharded engines and pm_multi
@pytest.mark.parametrize("n_shards", [2, 3])
def test_sharded_twins(n_shards):
    import torch

    rng = np.random.default_rng(700 + n_shards)
    w, pool, t = pool_tables(160, 10007, [(1, 1), (2, 4), (3, 3)], 713, edges=False)
    W = len(w)
    engs, ranges = [], []
    for r in range(n_shards):
        lo, hi = shard_range(W, n_shards, r)
        e = Engine(cost_tile_bytes=1 << 20)
        load_engine(e, t)
        e.set_shard(lo, hi - lo)
        engs.append(e)
        ranges.append((lo, hi))
    B = Engine()
    load_engine(B, t)
    rows = SpliceRows(pool, t["opts"], 160)
    for step in range(8):
        if step:
            rows.step(rng, engs)
        rows.fresh(B)
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
                same(e.fetch(), q, f"{n_shards} shards, rank {r}, step {step}, {flags:#x}")
    for e in engs + [B]:
        e.close()


@pytest.mark.parametrize("every_gpu", [False, True], ids=["device0", "every_gpu"])
def test_multi_twins(every_gpu):
    import torch

    devices = list(range(max(1, torch.cuda.device_count()))) if every_gpu else [0]
    rng = np.random.default_rng(721 + every_gpu)
    w, pool, t = pool_tables(150, 8000, GROUPS, 721, edges=False)
    M = MultiEngine(devices)
    M.set_asks(t["asks"], t["opts"])
    M.set_model_table(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    M.set_workers(t["wa"], t["wb"])
    B = Engine()
    load_engine(B, t)
    rows = SpliceRows(pool, t["opts"], 150)
    M.match(abi.PM_MODE_FIRST_FIT | INCR)
    for step in range(8):
        rows.step(rng, [M])
        rows.fresh(B)
        M.match(abi.PM_MODE_FIRST_FIT | INCR)
        B.match(abi.PM_MODE_FIRST_FIT | LEAN)
        same(M.fetch(), B.fetch(), f"pm_multi over {devices}, step {step}")
    lib, h = M._lib, M._h
    idx = np.array([1, len(rows.asks)], dtype=np.uint32)
    assert lib.pm_multi_remove_asks(h, C.c_void_p(idx.ctypes.data), 2) == abi.PM_E_INVALID
    M.match(abi.PM_MODE_FIRST_FIT | INCR)
    same(M.fetch(), B.fetch(), "after a refused pm_multi_remove_asks")
    B.close()
    M.close()


# ------------------------------------------------------------------ 5. refusals change nothing
def test_refusals_change_nothing():
    t, cap = auction_tables(90, 1200, 81)
    pool = t["asks"].copy()
    t = dict(t, asks=pool[:60])
    eng = auction_engine(t, cap[:60])
    eng.set_ask_demand(np.full(60, 2, np.uint32))
    eng.match(abi.PM_MODE_FIRST_FIT | INCR)
    eng.match(WARM)
    lib, h = eng._lib, eng._h
    P = lambda a: C.c_void_p(a.ctypes.data)
    good = np.ascontiguousarray(pool[60:62])
    opts = np.ascontiguousarray(t["opts"])
    bad_sizes = good.copy()
    bad_sizes["min_group_size"][1], bad_sizes["max_group_size"][1] = 5, 2
    bad_range = good.copy()
    bad_range["opt_off"][0], bad_range["n_opts"][0] = len(opts), 1
    idx = np.array([3, 4], dtype=np.uint32)
    far = np.array([3, 60], dtype=np.uint32)
    dec = np.array([5, 4], dtype=np.uint32)
    past = np.array([4, 61], dtype=np.uint32)
    calls = [
        lambda: lib.pm_remove_asks(h, None, 2),
        lambda: lib.pm_remove_asks(h, P(far), 2),
        lambda: lib.pm_insert_asks(h, None, P(good), 2, P(opts), len(opts)),
        lambda: lib.pm_insert_asks(h, P(idx), None, 2, P(opts), len(opts)),
        lambda: lib.pm_insert_asks(h, P(idx), P(good), 2, None, len(opts)),
        lambda: lib.pm_insert_asks(h, P(dec), P(good), 2, P(opts), len(opts)),
        lambda: lib.pm_insert_asks(h, P(past), P(good), 2, P(opts), len(opts)),
        lambda: lib.pm_insert_asks(h, P(idx), P(bad_sizes), 2, P(opts), len(opts)),
        lambda: lib.pm_insert_asks(h, P(idx), P(bad_range), 2, P(opts), len(opts)),
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
    eng.auction_certificate()                       # still the stored pass's: not resized
    e = Engine()
    assert e._lib.pm_remove_asks(e._h, P(idx), 2) == abi.PM_E_STATE
    assert e._lib.pm_insert_asks(e._h, P(idx), P(good), 2, P(opts), len(opts)) == abi.PM_E_STATE
    e.close()
    eng.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert eng.stats()["evals"] == 0
    eng.remove_asks([2, 30])
    with pytest.raises(PrimeMatchError) as ex:
        eng.auction_certificate()
    assert ex.value.status == abi.PM_E_STATE
    eng.close()


# ------------------------------------------------------------------ 6. full size: cfg3
def test_cfg3_splice():
    """bench.py's auction market at cfg3: 1 000 held asks removed at scattered positions and 1 000 rows inserted.  The
    lean incremental pass and a cold auction pass equal a fresh engine's; the warm and repair passes equal a twin built
    by pm_set_asks + pm_auction_restore_slots of the remapped export."""
    from test_gpu_bench_workloads import FF, TILE, load, workload

    w, a, tbl, _ = workload("cfg3")
    T = len(a.asks)
    caps0 = np.exp(np.log(20) + synth._unit(synth.SEED_EXT, T, 3) * np.log(100)).astype(np.uint32)
    rng = np.random.default_rng(79)
    plan = {}

    def spliced():
        e = Engine(cost_tile_bytes=TILE)
        load(e, w, a, tbl)
        e.set_price_caps(caps0)
        e.match(FF | LEAN | abi.PM_INCREMENTAL)
        e.match(abi.PM_MODE_AUCTION)
        if not plan:
            held = np.flatnonzero(e.auction_assignment() != NONE)
            plan["rm"] = np.sort(rng.choice(held, 1000, replace=False))
            keep = np.setdiff1d(np.arange(T), plan["rm"])
            plan["src"] = rng.integers(0, T, 1000)
            plan["before"] = np.sort(rng.integers(0, len(keep) + 1, 1000)).astype(np.uint32)
            b = plan["before"].astype(np.int64)
            plan["asks"] = np.insert(a.asks[keep], b, a.asks[plan["src"]])
            plan["caps"] = np.insert(caps0[keep], b, rng.integers(20, 2000, 1000).astype(np.uint32))
        e.remove_asks(plan["rm"].astype(np.uint32)[::-1])
        e.insert_asks(plan["before"], *own_options(a.asks[plan["src"]], a.opts))
        e.set_price_caps(plan["caps"])
        return e

    def fresh():
        f = Engine(cost_tile_bytes=TILE)
        f.set_asks(plan["asks"], a.opts)
        f.set_model_table(*tbl)
        f.set_workers(w.a, w.b)
        f.set_price_caps(plan["caps"])
        return f

    eng = spliced()
    ref = fresh()
    eng.match(FF | LEAN | abi.PM_INCREMENTAL)
    ref.match(FF | LEAN)
    same(eng.fetch(), ref.fetch(), "cfg3 lean incremental")
    assert eng.stats()["n_tiles"] < len(w.a)
    for mode in (WARM, REPAIR):
        A = eng if mode == WARM else spliced()
        twin = fresh()
        twin.auction_restore_slots(A.auction_state()[0], A.auction_slot_assignment())
        A.match(mode)
        twin.match(mode)
        r, q = A.fetch(), twin.fetch()
        same(r, q, f"cfg3 {mode:#x}")
        assert A.auction_state()[1] and twin.auction_state()[1]
        assert r.stats["n_rounds"] == q.stats["n_rounds"]
        assert np.array_equal(A.auction_state()[0], twin.auction_state()[0])
        twin.close()
        if A is not eng:
            A.close()
    eng.match(abi.PM_MODE_AUCTION)
    ref.match(abi.PM_MODE_AUCTION)
    same(eng.fetch(), ref.fetch(), "cfg3 cold auction")
    ref.close()
    eng.close()
