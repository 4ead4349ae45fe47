"""Ask-table deltas on the device (pm_update_asks / pm_resize_asks).  Twins: engine A takes the deltas, engine B gets
pm_set_asks with the current rows and the same mask after every step; every pm_fetch_result array and
pm_build_cost_tile must be equal, in every reference mode, on every path, with and without PM_INCREMENTAL, sharded and
through pm_multi.  The incremental pass stays incremental.  Warm and repair auction passes equal the checkers run from
the remapped stored state bit for bit; the certificate follows.  Refusals change nothing."""
import ctypes as C
import os

import numpy as np
import pytest

import auction_certificate as ac
import auction_repair_checker as rp
from helpers import load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine, MultiEngine
from protocol_b200.sharded import shard_range, wrap_device_buffers
from test_ask_deltas_formulation import AskMarket, ask_step, own_options
from test_gpu_auction_warm import engine as auction_engine
from test_gpu_auction_warm import run as auction_run
from test_gpu_auction_warm import tables as auction_tables
from test_gpu_incremental import GROUPS, INCR, LEAN, new_engine
from test_gpu_variants import wide_tables

pytestmark = pytest.mark.gpu

NONE = abi.PM_NONE
FIELDS = ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count")
WARM = abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM
REPAIR = WARM | abi.PM_AUCTION_REPAIR
TUNES = [1, 2, 8, 16, 32, 64, 128, 8 | 32, 64 | 32, 1 | 64, 128 | 32, 0x200, 0x100 | 16]   # test_gpu_auction_warm's


def same(r, q, what):
    for f in FIELDS:
        assert np.array_equal(getattr(r, f), getattr(q, f)), f"{what}: {f} differs"
    assert r.stats["n_bumped"] == q.stats["n_bumped"], what


class Rows:
    """The caller's side: the current ask rows (opt_off into one option pool) and the enabled mask.  `send`: how the
    caller sends new rows — "own" (each row with only its own option rows, rebased), "pool" (the whole option pool,
    opt_off into it), or "mixed" (own three times in four)."""

    def __init__(self, pool, opts, n0, send="mixed"):
        self.pool, self.opts, self.send = pool, opts, send
        self.asks = pool[:n0].copy()
        self.mask = np.ones(n0, bool)

    def payload(self, rng, rows):
        if self.send == "pool" or (self.send == "mixed" and rng.random() < 0.25):
            return rows, self.opts
        return own_options(rows, self.opts)

    def step(self, rng, engs, kinds=("replace", "append", "shrink", "append_shrink", "toggle", "replace_disabled")):
        T = len(self.asks)
        kind = kinds[rng.integers(len(kinds))]
        if kind in ("replace", "replace_disabled"):
            k = int(rng.integers(1, 6))
            idx = rng.integers(0, T, k).astype(np.uint32)             # repeated indices: the last entry decides
            if kind == "replace_disabled" and (~self.mask).any():
                idx[0] = np.flatnonzero(~self.mask)[0]
            rows = self.pool[rng.integers(0, len(self.pool), k)]
            sent = self.payload(rng, rows)
            for e in engs:
                e.update_asks(idx, *sent)
            for t, r in zip(idx, rows):
                self.asks[t] = r
        if kind in ("shrink", "append_shrink") and T > 8:
            n = T - int(rng.integers(1, 6))
            for e in engs:
                e.resize_asks(n)
            self.asks, self.mask = self.asks[:n].copy(), self.mask[:n].copy()
        if kind in ("append", "append_shrink"):
            rows = self.pool[rng.integers(0, len(self.pool), int(rng.integers(1, 6)))]
            sent = self.payload(rng, rows)
            for e in engs:
                e.resize_asks(len(self.asks) + len(rows), *sent)
            self.asks = np.concatenate([self.asks, rows])
            self.mask = np.concatenate([self.mask, np.ones(len(rows), bool)])
        if kind == "toggle":
            idx = rng.integers(0, T, int(rng.integers(1, 5)))
            en = rng.random(len(idx)) < 0.5
            for e in engs:
                e.set_ask_enabled(idx, en)
            for t, v in zip(idx, en):
                self.mask[t] = v
        return kind

    def fresh(self, eng):
        """What pm_set_asks gives for the current rows with the same mask."""
        eng.set_asks(self.asks, self.opts)
        if (~self.mask).any():
            eng.set_ask_enabled(np.flatnonzero(~self.mask), False)


def pool_tables(T, W, sizes, seed, edges=True):
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed, with_addresses=False)
    a = synth.make_asks(3 * T, "mixed", seed=synth.SEED_ASKS + seed, group_sizes=sizes)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    pool = a.asks.copy()
    if edges:   # min 0 asks (the empty group), max 0 asks (take nobody in the reference modes)
        pool["min_group_size"][::17] = 0
        pool["min_group_size"][5::29] = 0
        pool["max_group_size"][5::29] = 0
    t = dict(asks=pool[:T], opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words,
             lat=w.lat, lon=w.lon)
    return w, pool, t


def twins(t, env=None, rank=None):
    a, b = new_engine(**(env or {})), new_engine(**(env or {}))
    for e in (a, b):
        load_engine(e, t, addr_rank=rank, locations=True)
    return a, b


def workers_step(rng, w, engs):
    idx = np.unique(rng.integers(0, len(w), int(rng.integers(1, 40)))).astype(np.uint32)
    wa, wb = w.a[idx].copy(), w.b[idx].copy()
    wa["flags"] ^= np.where(rng.random(len(idx)) < 0.3, abi.PM_W_HEALTHY, 0).astype(np.uint32)
    for e in engs:
        e.update_workers(idx, wa, wb)
    w.a[idx], w.b[idx] = wa, wb


# ------------------------------------------------------------------ 1. twins: every mode and path
PATHS = {"materialized": (abi.PM_PATH_MATERIALIZED, abi.PM_PATH_MATERIALIZED, None),
         "int64_tile": (abi.PM_PATH_MATERIALIZED, abi.PM_PATH_MATERIALIZED, {"PM_TUNE_BUILD": 8}),
         "fused": (abi.PM_PATH_FUSED, abi.PM_PATH_FUSED, None), "fused_lean": (LEAN, LEAN, None),
         "incremental": (INCR, LEAN, None)}
MODES = {"first_fit": (abi.PM_MODE_FIRST_FIT, GROUPS, True), "proximity": (abi.PM_MODE_PROXIMITY, GROUPS, False),
         "proximity_solo": (abi.PM_MODE_PROXIMITY, [(1, 1)], False),
         "proximity_merge": (abi.PM_MODE_PROXIMITY_MERGE, [(1, 3), (2, 4)], False)}


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("mode", list(MODES))
def test_twins_every_mode_and_path(mode, path):
    base, sizes, edges = MODES[mode]
    fa, fb, env = PATHS[path]
    seed = len(mode) * 3 + len(path)
    rng = np.random.default_rng(seed)
    w, pool, t = pool_tables(150, 3000, sizes, seed, edges=edges)
    rank = rng.permutation(len(w)).astype(np.uint32)
    A, B = twins(t, env, rank)
    rows = Rows(pool, t["opts"], 150)
    A.match(base | fa)
    kinds = {}
    for step in range(12):
        kind = rows.step(rng, [A])
        kinds[kind] = kinds.get(kind, 0) + 1
        if step % 3 == 2:
            workers_step(rng, w, [A, B])
        rows.fresh(B)
        A.match(base | fa)
        B.match(base | fb)
        r, q = A.fetch(), B.fetch()
        same(r, q, f"{mode}/{path} step {step} ({kind})")
        if path in ("materialized", "fused") and step % 4 == 0:
            T = len(rows.asks)
            assert np.array_equal(A.cost_tile(0, T), B.cost_tile(0, T)), f"cost tile, step {step}"
    assert len(kinds) >= 3
    A.close()
    B.close()


def test_tail_hand_downs_and_changed_option_counts():
    """Updates that create under-filled tails (their workers handed down) and rows whose option count changes."""
    rng = np.random.default_rng(77)
    w, pool, t = pool_tables(120, 2500, [(3, 3), (4, 6), (2, 2), (1, 1)], 77)
    A, B = twins(t)
    rows = Rows(pool, t["opts"], 120)
    n_opts = set()
    for step in range(10):
        rows.step(rng, [A], kinds=("replace",))
        n_opts |= set(rows.asks["n_opts"].tolist())
        rows.fresh(B)
        for f in (abi.PM_PATH_MATERIALIZED, INCR):
            A.match(abi.PM_MODE_FIRST_FIT | f)
            B.match(abi.PM_MODE_FIRST_FIT | (LEAN if f == INCR else f))
            r = A.fetch()
            same(r, B.fetch(), f"step {step} {f:#x}")
    assert r.stats["n_bumped"] > 0 and len(n_opts) > 1
    A.close()
    B.close()


def test_generic_predicate_operand_past_2_31():
    """A replaced row with a cpu_cores threshold >= 2^31 sends every pass to the generic predicate; replacing it back
    returns to the fast one; the twins agree throughout."""
    w, pool, t = pool_tables(100, 3000, GROUPS, 12, edges=False)
    A, B = twins(t)
    rows = Rows(pool, t["opts"], 100)
    big = pool[:1].copy()
    big["flags"] = abi.PM_A_HAS_REQ | abi.PM_A_REQ_CPU | abi.PM_A_REQ_CPU_CORES
    big["cpu_cores"] = (1 << 31) + 5
    big["n_opts"] = 0
    for row in (big, pool[7:8].copy()):
        A.update_asks([9], row, rows.opts)
        rows.asks[9] = row[0]
        rows.fresh(B)
        for f in (abi.PM_PATH_MATERIALIZED, abi.PM_PATH_FUSED, INCR):
            A.match(abi.PM_MODE_FIRST_FIT | f)
            B.match(abi.PM_MODE_FIRST_FIT | (LEAN if f == INCR else f))
            same(A.fetch(), B.fetch(), f"cpu_cores {int(row['cpu_cores'][0])} {f:#x}")
        assert np.array_equal(A.cost_tile(0, 100), B.cost_tile(0, 100))
    A.close()
    B.close()


def test_wide_catalogue_worker_major():
    w, a, obits, pbits, npat, nmod, words = wide_tables(300, 5000, 3000, 30, 41, last_rows=True)
    t = dict(asks=a.asks[:150], opts=a.opts, wa=w.a, wb=w.b, bits=pbits, n_patterns=npat, n_models=nmod, words=words,
             lat=w.lat, lon=w.lon)
    rng = np.random.default_rng(41)
    A, B = twins(t)
    rows = Rows(a.asks.copy(), a.opts, 150)
    for step in range(8):
        rows.step(rng, [A])
        rows.fresh(B)
        for f in (abi.PM_PATH_MATERIALIZED, INCR):
            A.match(abi.PM_MODE_FIRST_FIT | f)
            B.match(abi.PM_MODE_FIRST_FIT | (LEAN if f == INCR else f))
            same(A.fetch(), B.fetch(), f"step {step} {f:#x}")
    A.close()
    B.close()


class RawOptions:
    """The engine's option-row bookkeeping as prime_match.h states it: each delta appends the option ranges its rows
    reference; raw_opts is compacted (to exactly the live rows) when its dead rows outnumber the live ones."""

    def __init__(self, n_raw, asks):
        self.raw, self.compactions = n_raw, 0
        self.live = int(asks["n_opts"].sum())

    def delta(self, asks_after, new_rows):
        self.raw += int(new_rows["n_opts"].sum()) if new_rows is not None else 0
        self.live = int(asks_after["n_opts"].sum())
        if self.raw - self.live > self.live:
            self.raw = self.live
            self.compactions += 1
            return True
        return False


def test_appended_options_then_compaction():
    """A caller that sends each changed row with its own option rows: many deltas append to raw_opts and scatter the
    rows (pm_scatter_asks) before the dead rows outnumber the live ones and one compaction packs them; the twins agree
    after every step on both sides of it."""
    rng = np.random.default_rng(90)
    w, pool, t = pool_tables(150, 4000, GROUPS, 90)
    packed, own = own_options(pool[:150], t["opts"])      # the first table holds only the rows' own options
    A, B = twins(dict(t, asks=packed, opts=own))
    rows = Rows(pool, t["opts"], 150, send="own")
    model = RawOptions(len(own), packed)
    appended_before = None
    for step in range(60):
        T = len(rows.asks)
        if step % 7 == 6:
            new = pool[rng.integers(0, len(pool), 3)]
            A.resize_asks(T + 3, *own_options(new, rows.opts))
            rows.asks = np.concatenate([rows.asks, new])
            rows.mask = np.concatenate([rows.mask, np.ones(3, bool)])
        else:
            idx = rng.choice(T, 4, replace=False).astype(np.uint32)
            new = pool[rng.integers(0, len(pool), 4)]
            A.update_asks(idx, *own_options(new, rows.opts))
            rows.asks[idx] = new
        if model.delta(rows.asks, new) and appended_before is None:
            appended_before = step
        rows.fresh(B)
        fa, fb = (INCR, LEAN) if step % 5 else (abi.PM_PATH_MATERIALIZED, abi.PM_PATH_MATERIALIZED)
        A.match(abi.PM_MODE_FIRST_FIT | fa)
        B.match(abi.PM_MODE_FIRST_FIT | fb)
        same(A.fetch(), B.fetch(), f"step {step} (compactions so far {model.compactions})")
        if step % 10 == 0:
            assert np.array_equal(A.cost_tile(0, len(rows.asks)), B.cost_tile(0, len(rows.asks))), f"step {step}"
    assert appended_before is not None and appended_before >= 10, appended_before   # many appends, then a compaction
    assert model.compactions >= 1
    A.close()
    B.close()


def test_repeated_indices_the_last_entry_decides():
    w, pool, t = pool_tables(100, 3000, GROUPS, 31, edges=False)
    A, B = twins(t)
    rows = Rows(pool, t["opts"], 100)
    idx = np.array([5, 9, 5, 40, 5, 9], dtype=np.uint32)
    new = pool[[200, 201, 202, 203, 204, 205]]
    A.match(abi.PM_MODE_FIRST_FIT | INCR)
    A.update_asks(idx, *own_options(new, rows.opts))
    rows.asks[5], rows.asks[9], rows.asks[40] = new[4], new[5], new[3]
    rows.fresh(B)
    for fa, fb in ((INCR, LEAN), (abi.PM_PATH_MATERIALIZED, abi.PM_PATH_MATERIALIZED)):
        A.match(abi.PM_MODE_FIRST_FIT | fa)
        B.match(abi.PM_MODE_FIRST_FIT | fb)
        same(A.fetch(), B.fetch(), f"{fa:#x}")
    assert np.array_equal(A.cost_tile(0, 100), B.cost_tile(0, 100))
    A.close()
    B.close()


# ------------------------------------------------------------------ 2. it stays incremental
def test_replacing_a_few_asks_stays_incremental():
    w, pool, t = pool_tables(300, 20000, GROUPS, 5, edges=False)
    T, W = 300, 20000
    A, B = twins(t)
    rows = Rows(pool, t["opts"], T)
    A.match(abi.PM_MODE_FIRST_FIT | INCR)
    ff = orc.soa_first_feasible(w.a, w.b, rows.asks, rows.opts, t["bits"], t["words"])
    idx = np.array([3, 40, 41, 200], dtype=np.uint32)
    new = pool[[400, 500, 3, 650]]
    A.update_asks(idx, *own_options(new, rows.opts))
    rows.asks[idx] = new
    rows.fresh(B)
    A.match(abi.PM_MODE_FIRST_FIT | INCR)
    B.match(abi.PM_MODE_FIRST_FIT | LEAN)
    same(A.fetch(), B.fetch(), "after 4 replaced asks")
    st = A.stats()
    orphans = int(np.isin(ff, idx).sum())
    assert orphans > 0
    assert st["evals"] < T * W and st["n_tiles"] == orphans, (st["evals"], st["n_tiles"], orphans)
    A.close()
    B.close()


# ------------------------------------------------------------------ 3. sharded engines and pm_multi
@pytest.mark.parametrize("n_shards", [2, 3])
def test_sharded_twins(n_shards):
    import torch

    rng = np.random.default_rng(n_shards)
    w, pool, t = pool_tables(160, 10007, [(1, 1), (2, 4), (3, 3)], 13, edges=False)
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
    rows = Rows(pool, t["opts"], 160)
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


def test_multi_twins():
    import torch

    devices = list(range(max(1, torch.cuda.device_count())))
    rng = np.random.default_rng(21)
    w, pool, t = pool_tables(150, 8000, GROUPS, 21, edges=False)
    M = MultiEngine(devices)
    M.set_asks(t["asks"], t["opts"])
    M.set_model_table(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    M.set_workers(t["wa"], t["wb"])
    B = Engine()
    load_engine(B, t)
    rows = Rows(pool, t["opts"], 150)
    M.match(abi.PM_MODE_FIRST_FIT | INCR)
    for step in range(8):
        rows.step(rng, [M])
        rows.fresh(B)
        M.match(abi.PM_MODE_FIRST_FIT | INCR)
        B.match(abi.PM_MODE_FIRST_FIT | LEAN)
        same(M.fetch(), B.fetch(), f"pm_multi over {devices}, step {step}")
    B.close()
    M.close()


# ------------------------------------------------------------------ 4. the auction from the remapped state
def auction_chain(seed, steps, tune=0, repair=False, n_asks=60, n_workers=900):
    t, cap = auction_tables(n_asks + 60, n_workers, seed)
    pool = t["asks"].copy()
    t = dict(t, asks=pool[:n_asks])
    m = AskMarket(t, cap[:n_asks])
    eng = auction_engine(t, cap[:n_asks], tune=tune)
    rng = np.random.default_rng(seed)
    mode = REPAIR if repair else WARM
    got, price, st, warm, released = auction_run(eng, n_asks, mode)
    a, p, n = m.cold()
    assert not warm and np.array_equal(got, a) and np.array_equal(price, p) and st["n_rounds"] == n
    m.store(p, a)
    kinds = set()
    for step in range(steps):
        for _ in range(int(rng.integers(1, 3))):
            kinds.add(ask_step(m, pool, rng, eng=eng))
        T = len(m.asks)
        got, price, st, warm, released = auction_run(eng, T, mode)
        assert warm, f"step {step}"
        if repair:
            out = rp.market_repair(m)
            a, p = out["assigned"], out["price"]
            assert released == len(out["released"]) and st["n_rounds"] == out["fwd"]
            assert eng.auction_reverse_stats() == (1, out["rev"], out["bids"])
        else:
            a, p, n, rel = m.warm()
            assert released == len(rel) and st["n_rounds"] == n
        assert np.array_equal(got, a), f"step {step}"
        assert np.array_equal(price, p), f"step {step}"
        m.store(p, a)
        cert = eng.auction_certificate()
        assert cert["gap"] <= T and cert["n_bad_holds"] == 0
    eng.close()
    return kinds


@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
@pytest.mark.parametrize("seed", [2, 3, 4])
def test_auction_chain_matches_checker(seed, repair):
    kinds = auction_chain(seed, 8, repair=repair)
    assert {"replace", "append", "shrink"} <= kinds


@pytest.mark.parametrize("tune", TUNES)
def test_auction_chain_every_shortcut_can_be_switched_off(tune):
    auction_chain(70 + tune, 4, tune=tune, repair=bool(tune & 1), n_asks=30, n_workers=3000)


@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
def test_appended_asks_under_reputation_floors(repair):
    """Appended asks get floor 0 (and cap 0) until the floors and caps are set again; the warm and repair passes after
    the append, and after the new floors, equal the checkers; the certificate audits the floors as they stand."""
    t, cap = auction_tables(90, 1200, 44)
    pool = t["asks"].copy()
    t = dict(t, asks=pool[:60])
    rng = np.random.default_rng(44)
    rep = rng.integers(0, 4, 1200).astype(np.uint32)
    floors = rng.integers(0, 3, 60).astype(np.uint32)
    m = AskMarket(t, cap[:60], reputation=rep, floors=floors)
    eng = auction_engine(t, cap[:60], floors=floors, reputation=rep)
    mode = REPAIR if repair else WARM

    def check(T, what):
        got, price, st, warm, released = auction_run(eng, T, mode)
        if repair:
            out = rp.market_repair(m)
            a, p = out["assigned"], out["price"]
            assert released == len(out["released"]) and st["n_rounds"] == out["fwd"], what
        else:
            a, p, n, rel = m.warm()
            assert released == len(rel) and st["n_rounds"] == n, what
        assert warm and np.array_equal(got, a) and np.array_equal(price, p), what
        m.store(p, a)
        cert = eng.auction_certificate()
        want = ac.market_certificate(m, 1, p, a)
        assert all(cert[f] == want[f] for f in ac.FIELDS), what
        return a

    got, price, *_ = auction_run(eng, 60, abi.PM_MODE_AUCTION)
    m.store(price, got)
    m.append(pool[70:75], eng)                        # cap 0, floor 0: only a worker asking 0 could take them
    assert (m.floors[60:] == 0).all() and (m.cap[60:] == 0).all()
    check(65, "after the append")
    caps = m.cap.copy()
    caps[60:] = rng.integers(300, 1500, 5)
    m.set_caps(caps, eng)
    fl = m.floors.copy()
    fl[60:] = [3, 0, 2, 3, 1]
    m.set_floors(fl, eng)
    a = check(65, "after the new caps and floors")
    held = a[60:][a[60:] != NONE]
    assert len(held) and (rep[held] >= fl[60:][a[60:] != NONE]).all()
    eng.close()


def test_auction_certificate_after_update_and_resize():
    t, cap = auction_tables(100, 1200, 9)
    pool = t["asks"].copy()
    t = dict(t, asks=pool[:60])
    m = AskMarket(t, cap[:60])
    eng = auction_engine(t, cap[:60])
    got, price, *_ = auction_run(eng, 60, WARM)
    m.store(price, got)
    # an update: the certificate audits the stored state against the new rows
    m.replace([1, 2, 30], pool[[70, 71, 72]], eng)
    want = ac.market_certificate(m, 1, price, got)
    cert = eng.auction_certificate(ask_bound=True)
    for f in ac.FIELDS:
        assert cert[f] == want[f], f
    assert np.array_equal(cert["ask_bound"], want["ask_bound"])
    # a resize: PM_E_STATE until the next pass, and nothing changes
    v = eng.table_version()
    m.append(pool[80:82], eng)
    before = eng.auction_state()
    with pytest.raises(PrimeMatchError) as ex:
        eng.auction_certificate()
    assert ex.value.status == abi.PM_E_STATE
    after = eng.auction_state()
    assert np.array_equal(before[0], after[0]) and before[1:] == after[1:] and eng.table_version() > v
    got, price, st, warm, released = auction_run(eng, 62, WARM)
    a, p, n, rel = m.warm()
    assert warm and np.array_equal(got, a) and np.array_equal(price, p)
    assert eng.auction_certificate()["gap"] <= 62
    eng.close()


def test_auction_above_the_cutoff_equals_a_fresh_cold_pass():
    t, cap = auction_tables(120, 1500, 17)
    pool = t["asks"].copy()
    t = dict(t, asks=pool[:80])
    eng = auction_engine(t, cap[:80], incr=6)
    auction_run(eng, 80, WARM)
    eng.resize_asks(72)                     # frees the workers of 8 asks ...
    eng.resize_asks(76, pool[90:94], t["opts"])   # ... and 4 appended asks: past the cutoff of 6
    caps = np.concatenate([cap[:72], cap[90:94]])
    eng.set_price_caps(caps)
    got, price, st, warm, _ = auction_run(eng, 76, WARM)
    fresh = auction_engine(dict(t, asks=np.concatenate([pool[:72], pool[90:94]])), caps)
    g2, p2, st2, w2, _ = auction_run(fresh, 76, abi.PM_MODE_AUCTION)
    assert not warm and not w2
    assert np.array_equal(got, g2) and np.array_equal(price, p2) and st["n_rounds"] == st2["n_rounds"]
    eng.close()
    fresh.close()


# ------------------------------------------------------------------ 5. refusals change nothing
def test_refusals_change_nothing():
    rng = np.random.default_rng(8)
    w, pool, t = pool_tables(100, 3000, GROUPS, 8, edges=False)
    A, B = twins(t)
    rows = Rows(pool, t["opts"], 100)
    A.match(abi.PM_MODE_FIRST_FIT | INCR)
    lib, h = A._lib, A._h
    good = np.ascontiguousarray(pool[:2])
    opts = np.ascontiguousarray(t["opts"])
    bad_sizes = good.copy()
    bad_sizes["min_group_size"][1], bad_sizes["max_group_size"][1] = 5, 2
    bad_range = good.copy()
    bad_range["opt_off"][0] = len(opts)
    bad_range["n_opts"][0] = 1
    idx = np.array([3, 4], dtype=np.uint32)
    far = np.array([3, 100], dtype=np.uint32)
    P = lambda a: C.c_void_p(a.ctypes.data)
    calls = [
        lambda: lib.pm_update_asks(h, None, P(good), 2, P(opts), len(opts)),
        lambda: lib.pm_update_asks(h, P(idx), None, 2, P(opts), len(opts)),
        lambda: lib.pm_update_asks(h, P(idx), P(good), 2, None, len(opts)),
        lambda: lib.pm_update_asks(h, P(far), P(good), 2, P(opts), len(opts)),
        lambda: lib.pm_update_asks(h, P(idx), P(bad_sizes), 2, P(opts), len(opts)),
        lambda: lib.pm_update_asks(h, P(idx), P(bad_range), 2, P(opts), len(opts)),
        lambda: lib.pm_resize_asks(h, 102, None, P(opts), len(opts)),
        lambda: lib.pm_resize_asks(h, 102, P(bad_sizes), P(opts), len(opts)),
        lambda: lib.pm_resize_asks(h, 102, P(bad_range), P(opts), len(opts)),
        lambda: lib.pm_resize_asks(h, 1 << 30, P(good), P(opts), len(opts)),
    ]
    v = A.table_version()
    for i, call in enumerate(calls):
        assert call() == abi.PM_E_INVALID, i
    assert A.table_version() == v
    e = Engine()
    assert e._lib.pm_update_asks(e._h, P(idx), P(good), 2, P(opts), len(opts)) == abi.PM_E_STATE
    assert e._lib.pm_resize_asks(e._h, 2, P(good), P(opts), len(opts)) == abi.PM_E_STATE
    e.close()
    A.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert A.stats()["evals"] == 0                   # nothing was listed
    for step in range(4):
        rows.step(rng, [A])
        rows.fresh(B)
        A.match(abi.PM_MODE_FIRST_FIT | INCR)
        B.match(abi.PM_MODE_FIRST_FIT | LEAN)
        same(A.fetch(), B.fetch(), f"after refusals, step {step}")
    A.close()
    B.close()


def test_auction_refusals_keep_the_warm_state():
    t, cap = auction_tables(70, 900, 6)
    pool = t["asks"].copy()
    t = dict(t, asks=pool[:50])
    m = AskMarket(t, cap[:50])
    eng = auction_engine(t, cap[:50])
    got, price, *_ = auction_run(eng, 50, WARM)
    m.store(price, got)
    with pytest.raises(PrimeMatchError):
        eng.update_asks([50], pool[:1], t["opts"])
    with pytest.raises(PrimeMatchError):
        eng.resize_asks(52)                              # growth without rows
    m.replace([4], pool[60:61], eng)
    got, price, st, warm, released = auction_run(eng, 50, WARM)
    a, p, n, rel = m.warm()
    assert warm and np.array_equal(got, a) and np.array_equal(price, p) and st["n_rounds"] == n
    eng.close()
