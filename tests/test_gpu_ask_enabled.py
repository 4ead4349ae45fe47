"""Enabled configurations (pm_set_ask_enabled).  A disabled ask behaves as if it were absent from the table: every array
pm_fetch_result returns equals what pm_set_asks with only the enabled asks returns, indices mapped back, and what the CPU
oracle forms on that subset — on every evaluation path, predicate variant and acceptance-table form, for the edge asks
(min 0, max 0, tail hand-down), sharded, and through the plugin.  PM_INCREMENTAL keeps its stored evaluation across
toggles: asks enabled since are walked against every worker, the orphans of asks disabled since are walked again, and
every array still equals a flagless twin's."""
import numpy as np
import pytest

from helpers import TableBuilder, groups_equal, load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine
from protocol_b200.plugin import NodeGroupConfiguration, NodeGroupsPlugin, NodeStatus, Task
from test_gpu_incremental import CAND, GROUPS, INCR, LEAN, Twin, addr, all_groups, assert_same, full_stats, new_engine, node
from protocol_b200.sharded import shard_range, wrap_device_buffers
from test_gpu_variants import wide_tables

pytestmark = pytest.mark.gpu

NONE = abi.PM_NONE
INF = abi.PM_COST_INF
FIELDS = ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count")


def subset(asks, mask):
    """The enabled rows alone: what pm_set_asks gets from a caller that compacts (option rows stay shared)."""
    return asks[mask]


def mapped(sub, mask):
    """A result of the compacted table, its ask indices mapped back to the full table's."""
    full = np.nonzero(mask)[0].astype(np.uint32)
    up = lambda x: np.where(x == NONE, NONE, full[np.minimum(x, max(len(full) - 1, 0))] if len(full) else NONE).astype(np.uint32)
    best = np.full(len(mask), INF, dtype=np.int64)
    cnt = np.zeros(len(mask), dtype=np.uint32)
    best[mask], cnt[mask] = sub.ask_best, sub.ask_count
    return dict(worker_group=sub.worker_group, worker_ask=up(sub.worker_ask), group_ask=up(sub.group_ask),
                group_off=sub.group_off, group_members=sub.group_members, ask_best=best, ask_count=cnt)


def assert_as_if_absent(r, sub, mask, what=""):
    m = mapped(sub, mask)
    for f in FIELDS:
        assert np.array_equal(getattr(r, f), m[f]), f"{what}: {f} differs from the compacted table's"
    assert r.stats["n_bumped"] == sub.stats["n_bumped"], what
    assert not np.isin(r.worker_ask, np.nonzero(~mask)[0]).any() and not np.isin(r.group_ask, np.nonzero(~mask)[0]).any()


def masked_pair(t, mask, env=None, locations=False, rank=None):
    """(engine with the full table and `mask` applied, engine given the enabled rows only)."""
    m, s = new_engine(**(env or {})), new_engine(**(env or {}))
    load_engine(m, t, addr_rank=rank, locations=locations)
    load_engine(s, dict(t, asks=subset(t["asks"], mask)), addr_rank=rank, locations=locations)
    m.set_ask_enabled(np.nonzero(~mask)[0], False)
    return m, s


def tables(T, W, group_sizes=None, seed_shift=0, kind="mixed"):
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed_shift, with_addresses=False)
    a = synth.make_asks(T, kind, seed=synth.SEED_ASKS + seed_shift, group_sizes=group_sizes)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    return w, a, dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words,
                      lat=w.lat, lon=w.lon)


def random_mask(T, rng, p=0.65):
    mask = rng.random(T) < p
    mask[rng.integers(0, T, 3)] = False
    return mask


# ------------------------------------------------------------------ 1. every mode and path = compacted table = oracle
PATHS = {"materialized": (abi.PM_PATH_MATERIALIZED, None), "materialized_int64": (abi.PM_PATH_MATERIALIZED, {"PM_TUNE_BUILD": 8}),
         "fused": (abi.PM_PATH_FUSED, None), "fused_lean": (LEAN, None)}
MODES = {"first_fit": (abi.PM_MODE_FIRST_FIT, GROUPS), "proximity": (abi.PM_MODE_PROXIMITY, GROUPS),
         "proximity_solo": (abi.PM_MODE_PROXIMITY, None), "proximity_merge": (abi.PM_MODE_PROXIMITY_MERGE, [(1, 3), (2, 4)])}


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("mode", list(MODES))
def test_masked_equals_compacted_and_oracle(mode, path):
    base, sizes = MODES[mode]
    flags, env = PATHS[path]
    rng = np.random.default_rng(len(mode) * 7 + len(path))
    w, a, t = tables(260, 4000, group_sizes=sizes, seed_shift=len(mode))
    mask = random_mask(len(a), rng)
    rank = rng.permutation(len(w)).astype(np.uint32)
    m, s = masked_pair(t, mask, env, locations=True, rank=rank)
    m.match(base | flags)
    s.match(base | flags)
    r, q = m.fetch(), s.fetch()
    assert_as_if_absent(r, q, mask, f"{mode}/{path}")
    if base != abi.PM_MODE_PROXIMITY_MERGE:
        og = orc.soa_form_groups(w.a, w.b, subset(a.asks, mask), a.opts, t["bits"], t["words"], addr_rank=rank, lat=w.lat,
                                 lon=w.lon, proximity=base == abi.PM_MODE_PROXIMITY)
        assert groups_equal(q, og), f"{mode}/{path}: compacted table differs from the oracle"
    assert len(r.group_ask) > 10
    m.close()
    s.close()


# ------------------------------------------------------------------ 2. predicate variants and acceptance tables
VARIANTS = {"generic": None, "shared_word": (200, 112, 1), "global_table": (3000, 112, 2), "worker_major": (3000, 30, 41)}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_predicate_variants_and_wide_catalogues(variant):
    rng = np.random.default_rng(len(variant))
    if variant == "generic":
        env = {"PM_TUNE_GENERIC": 1}
        w, a, t = tables(300, 5000, group_sizes=GROUPS, seed_shift=9)
        pbits, words = t["bits"], t["words"]
    else:
        env = None
        n_models, n_patterns, shift = VARIANTS[variant]
        w, a, obits, pbits, npat, nmod, words = wide_tables(400, 5000, n_models, n_patterns, seed_shift=shift, last_rows=True)
        t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=pbits, n_patterns=npat, n_models=nmod, words=words,
                 lat=w.lat, lon=w.lon)
    mask = random_mask(len(a), rng)
    m, s = masked_pair(t, mask, env)
    for flags in (abi.PM_PATH_MATERIALIZED, abi.PM_PATH_FUSED, LEAN):
        m.match(abi.PM_MODE_FIRST_FIT | flags)
        s.match(abi.PM_MODE_FIRST_FIT | flags)
        assert_as_if_absent(m.fetch(), s.fetch(), mask, f"{variant} {flags:#x}")
    ff = orc.soa_first_feasible(w.a, w.b, subset(a.asks, mask), a.opts, pbits, words)
    assert (mapped(s.fetch(), mask)["worker_ask"] != NONE).sum() <= (ff != NONE).sum()
    # the cost tile: a disabled ask's rows are infeasible, an enabled ask's rows are the compacted table's
    T = len(a)
    tile, sub_tile = m.cost_tile(0, T), s.cost_tile(0, int(mask.sum()))
    assert (tile[~mask] == INF).all()
    assert np.array_equal(tile[mask], sub_tile)
    m.close()
    s.close()


# ------------------------------------------------------------------ 3. edge asks
def _edge_tables():
    tb = TableBuilder()
    loc = (45.5, -73.5)
    for i in range(7):
        tb.add_node({"gpu_count": 8, "gpu_model": "NVIDIA H100", "gpu_mem": 80000}, location=loc)
    for i in range(3):
        tb.add_node({"gpu_count": 1, "gpu_model": "RTX 4090", "gpu_mem": 24000}, location=loc)
    tb.add_config(None, 0, 2)                         # 0: min 0 -> the trailing empty group
    tb.add_config("gpu:count=8", 3, 3)                # 1: 7 workers -> 2 groups + a tail of 1 handed down
    tb.add_config("gpu:model=H100", 0, 0)             # 2: max 0 -> proximity refuses while it is enabled
    tb.add_config("gpu:count=8", 2, 2)                # 3: the tail's next feasible ask (disabled below)
    tb.add_config(None, 1, 1)                         # 4: ... so the tail comes here
    return tb.tables()


@pytest.mark.parametrize("mode", [abi.PM_MODE_FIRST_FIT, abi.PM_MODE_PROXIMITY], ids=["first_fit", "proximity"])
def test_edge_asks(mode):
    t = _edge_tables()
    T = len(t["asks"])
    e = Engine()
    load_engine(e, t, locations=True)
    if mode == abi.PM_MODE_PROXIMITY:
        with pytest.raises(PrimeMatchError) as ex:
            e.match(mode)
        assert ex.value.status == abi.PM_E_UNSUPPORTED
    e.set_ask_enabled([0, 2, 3], False)
    for flags in (abi.PM_PATH_MATERIALIZED, LEAN):
        e.match(mode | flags)                          # a disabled max == 0 ask: no refusal
        r = e.fetch()
        mask = np.ones(T, bool)
        mask[[0, 2, 3]] = False
        og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"][mask], t["opts"], t["bits"], t["words"], lat=t["lat"],
                                 lon=t["lon"], proximity=mode == abi.PM_MODE_PROXIMITY)
        up = np.nonzero(mask)[0]
        assert np.array_equal(r.group_ask, up[og.cfg]) and np.array_equal(r.group_members, og.members)
        assert 0 not in r.group_ask.tolist()                    # no empty group of the disabled min == 0 ask
        assert (r.group_off[1:] > r.group_off[:-1]).all()       # no empty group at all
        tail = [wk for c, ws in r.groups() if c == 4 for wk in ws if wk < 7]
        assert len(tail) == 1                                   # the 7th H100 worker skips ask 3 and lands on ask 4
        assert not r.ask_count[[0, 2, 3]].any() and (r.ask_best[[0, 2, 3]] == INF).all()
    e.set_ask_enabled(np.arange(T), False)
    e.match(mode)
    r = e.fetch()
    assert r.n_groups == 0 and (r.worker_ask == NONE).all() and (r.ask_best == INF).all() and not r.ask_count.any()
    e.close()


# ------------------------------------------------------------------ 4. refusals and resets
def test_refusals_and_resets():
    w, a, t = tables(200, 3000, group_sizes=GROUPS, seed_shift=4)
    T, W = len(a), len(w)
    e = Engine()
    load_engine(e, t)
    e.match(abi.PM_MODE_FIRST_FIT | INCR)
    full = e.fetch()
    for idx in ([T], [3, T + 7], [1 << 31]):
        with pytest.raises(PrimeMatchError) as ex:
            e.set_ask_enabled(idx, False)
        assert ex.value.status == abi.PM_E_INVALID
    e.match(abi.PM_MODE_FIRST_FIT | INCR)          # nothing changed: not ask 3 either
    assert e.stats()["evals"] == 0
    assert_same(e.fetch(), full, "after refused calls")
    e.set_price_caps(np.full(T, 1 << 20, dtype=np.uint32))
    e.set_ask_enabled([5], False)
    with pytest.raises(PrimeMatchError) as ex:
        e.match(abi.PM_MODE_AUCTION)
    assert ex.value.status == abi.PM_E_UNSUPPORTED
    e.set_ask_enabled([5], True)
    e.match(abi.PM_MODE_AUCTION)
    # pm_set_asks enables everything again and discards the stored evaluation
    e.set_ask_enabled(np.arange(0, T, 2), False)
    e.set_asks(a.asks, a.opts)
    e.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert full_stats(e.stats(), T, W)
    assert_same(e.fetch(), full, "after pm_set_asks")
    e.close()


# ------------------------------------------------------------------ 5. PM_INCREMENTAL across toggles
def _orphans(ff_prev, dis, written):
    o = np.isin(ff_prev, list(dis))
    o[list(written)] = False
    return int(o.sum())


def _first_feasible(w_a, w_b, a, bits, words, mask):
    ff = orc.soa_first_feasible(w_a, w_b, a.asks[mask], a.opts, bits, words)
    up = np.nonzero(mask)[0].astype(np.uint32)
    return np.where(ff == NONE, NONE, up[np.minimum(ff, max(len(up) - 1, 0))]).astype(np.uint32)


@pytest.mark.parametrize("mode", [abi.PM_MODE_FIRST_FIT, abi.PM_MODE_PROXIMITY], ids=["first_fit", "proximity"])
def test_random_toggle_history(mode):
    rng = np.random.default_rng(40 + mode)
    T, W = 240, 4000
    w = synth.make_workers(W, with_addresses=False)
    pool = synth.make_workers(3000, seed=synth.SEED_WORKERS + 91)
    a = synth.make_asks(T, "mixed", group_sizes=GROUPS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    wa, wb = w.a.copy(), w.b.copy()
    tw = Twin(mode)
    tw.load(wa, wb, a, bits, npat, nmod, words, w.lat, w.lon, rng.permutation(W).astype(np.uint32))
    mask = np.ones(T, bool)
    tw.run("first pass")
    ff = _first_feasible(wa, wb, a, bits, words, mask)
    seen = {}
    for step in range(36):
        op = ["toggle", "off_on", "disable_top", "enable0", "rows_and_toggle", "none"][step % 6] if step < 12 else \
            rng.choice(["toggle", "off_on", "disable_top", "enable0", "rows_and_toggle", "none"])
        before = mask.copy()
        written = set()
        if op in ("toggle", "rows_and_toggle"):
            idx = rng.choice(T, int(rng.integers(1, 12)), replace=False)
            on = rng.random(len(idx)) < 0.5
            tw.set_ask_enabled(idx, on)
            mask[idx] = on
        elif op == "off_on":            # the same ask off and on again: neither enabled nor disabled since
            j = int(rng.choice(np.nonzero(mask)[0]))
            tw.set_ask_enabled([j], False)
            tw.set_ask_enabled([j, j], [False, True])
        elif op == "disable_top":       # the first ask of many workers
            owners = np.bincount(ff[ff != NONE], minlength=T)
            j = int(np.argmax(owners))
            tw.set_ask_enabled([j], False)
            mask[j] = False
        elif op == "enable0":
            tw.set_ask_enabled([0], False)
            tw.run(f"step {step} disable 0")
            ff = _first_feasible(wa, wb, a, bits, words, mask & (np.arange(T) != 0))
            before = mask & (np.arange(T) != 0)
            tw.set_ask_enabled([0], True)
            mask[0] = True
        if op == "rows_and_toggle":
            u = np.unique(rng.integers(0, W, int(rng.integers(1, 50)))).astype(np.uint32)
            sel = rng.integers(0, len(pool), len(u))
            ra, rb = pool.a[sel].copy(), pool.b[sel].copy()
            ra["flags"][rng.random(len(u)) < 0.3] ^= abi.PM_W_ASSIGNED
            tw.update_workers(u, ra, rb, pool.lat[sel], pool.lon[sel])
            wa[u], wb[u] = ra, rb
            written = set(u.tolist())
        tw.set_addr_rank(rng.permutation(W).astype(np.uint32))
        r = tw.run(f"step {step} ({op})")
        st = r.stats
        en, dis = set(np.nonzero(mask & ~before)[0]), set(np.nonzero(~mask & before)[0])
        assert st["n_tiles"] == len(written) + _orphans(ff, dis, written), (step, op, st)
        if not en and not dis and not written:
            assert st["evals"] == 0, (step, op, st)
        else:
            assert st["evals"] <= T * st["n_tiles"] + len(en) * W, (step, op, st)
        ff = _first_feasible(wa, wb, a, bits, words, mask)
        assert not np.isin(r.worker_ask, np.nonzero(~mask)[0]).any()
        seen[op] = seen.get(op, 0) + 1
    assert len(seen) == 6, seen
    tw.close()


def test_orphans_beyond_one_cta_and_enabling_ask0():
    """Ask 1 accepts every candidate and owns most of 20 000 workers: disabling it orphans more than 5 000 of them,
    walked from ask 2 on.  Enabling ask 0 (also a catch-all) ahead of every owner takes them all back."""
    W, T = 20_000, 400
    w = synth.make_workers(W, with_addresses=False)
    a = synth.make_asks(T, "mixed", group_sizes=GROUPS)
    asks = a.asks.copy()
    for j in (0, 1):
        asks[j] = 0
        asks[j]["opt_off"] = 0
        asks[j]["min_group_size"] = asks[j]["max_group_size"] = 1
    a = synth.Asks(asks=asks, opts=a.opts, pattern_strings=a.pattern_strings)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    tw = Twin(abi.PM_MODE_FIRST_FIT)
    tw.load(w.a, w.b, a, bits, npat, nmod, words)
    tw.set_ask_enabled([0], False)
    r = tw.run("ask 0 off: a full pass")
    owners = int((r.worker_ask == 1).sum())
    assert owners > 5000
    tw.set_ask_enabled([1], False)
    r = tw.run("orphans")
    assert r.stats["n_tiles"] == owners and r.stats["evals"] > 0
    assert not (r.worker_ask == 1).any()
    tw.set_ask_enabled([0], True)
    r = tw.run("enable ask 0")
    assert r.stats["n_tiles"] == 0 and 0 < r.stats["evals"] <= W
    assert (r.worker_ask == 0).sum() >= owners
    tw.close()


@pytest.mark.parametrize("cutoff", [200, 100_000_000])
def test_fallback_threshold(cutoff):
    """The E-pass counts |E| W / T written rows against PM_TUNE_INCR: 10 asks (134 rows) run incrementally under a
    cutoff of 200, 20 asks (267 rows) evaluate everything."""
    T, W = 300, 4000
    w, a, t = tables(T, W, group_sizes=GROUPS, seed_shift=6)
    tw = Twin(abi.PM_MODE_FIRST_FIT, PM_TUNE_INCR=cutoff)
    tw.load(w.a, w.b, a, t["bits"], t["n_patterns"], t["n_models"], t["words"])
    for n_en in (10, 20):
        tw.set_ask_enabled(np.arange(100, 100 + n_en), False)
        tw.run(f"{n_en} off")
        tw.set_ask_enabled(np.arange(100, 100 + n_en), True)
        st = tw.run(f"{n_en} on").stats
        if -(-n_en * W // T) <= cutoff:
            assert st["n_tiles"] == 0 and 0 < st["evals"] <= n_en * W, (n_en, st)
        else:
            assert full_stats(st, T, W), (n_en, st)
    tw.close()


# ------------------------------------------------------------------ 6. sharded engines honour the mask
@pytest.mark.parametrize("path", [abi.PM_PATH_MATERIALIZED, abi.PM_PATH_FUSED], ids=["materialized", "fused"])
@pytest.mark.parametrize("n_shards", [2, 3])
def test_sharded_masked(n_shards, path):
    """Shard engines on one GPU (pm_set_shard), each with the full table and the mask, merged as the collective merges
    them (test_gpu_sharded.py): the result is the compacted table's."""
    import torch

    w, a, t = tables(300, 10007, group_sizes=[(1, 1), (2, 4), (3, 3)], seed_shift=13)
    mask = random_mask(len(a), np.random.default_rng(n_shards))
    mode = abi.PM_MODE_FIRST_FIT | path
    W, T = len(w), len(a)
    engs, bufs, ranges = [], [], []
    for r in range(n_shards):
        lo, hi = shard_range(W, n_shards, r)
        e = Engine(cost_tile_bytes=1 << 20)
        load_engine(e, t)
        e.set_ask_enabled(np.nonzero(~mask)[0], False)
        e.set_shard(lo, hi - lo)
        e.match_local(mode)
        e.sync()
        engs.append(e)
        bufs.append(wrap_device_buffers(e, W, T))
        ranges.append((lo, hi))
    first = torch.cat([bufs[r][0][lo:hi] for r, (lo, hi) in enumerate(ranges)])
    best = torch.stack([b[1] for b in bufs]).min(dim=0).values
    cnt = torch.stack([b[2] for b in bufs]).sum(dim=0).to(torch.int32)
    s = Engine()
    load_engine(s, dict(t, asks=subset(a.asks, mask)))
    s.match(mode)
    q = s.fetch()
    for r, e in enumerate(engs):
        bufs[r][0].copy_(first)
        bufs[r][1].copy_(best)
        bufs[r][2].copy_(cnt)
        torch.cuda.synchronize()
        e.match_finish(mode)
        assert_as_if_absent(e.fetch(), q, mask, f"{n_shards} shards, rank {r}")
    for e in engs + [s]:
        e.close()


# ------------------------------------------------------------------ 7. the plugin: task events toggle configurations
@pytest.mark.parametrize("proximity", [False, True], ids=["first_fit", "proximity"])
def test_plugin_task_events_keep_the_incremental_pass(proximity):
    rng = np.random.default_rng(70 + proximity)
    cfgs = [NodeGroupConfiguration(f"cfg-{c}", mn, mn + int(rng.integers(0, 3)),
                                   f"gpu:count={[1, 2, 4, 8][c % 4]}" if c % 5 else None)
            for c, mn in enumerate(rng.integers(1, 4, 24).tolist())]
    e1, e2 = Engine(), Engine()
    a = NodeGroupsPlugin(cfgs, engine=e1, proximity_enabled=proximity)
    b = NodeGroupsPlugin(cfgs, engine=e2, proximity_enabled=proximity)
    n = 0
    for _ in range(3000):
        nd = node(n, np.random.default_rng(n))
        for p in (a, b):
            p.add_node(nd)
        n += 1
    tasks = {}
    toggle_only = 0
    for step in range(30):
        ops = []
        if rng.random() < 0.7 or not tasks:
            topo = [c.name for c in cfgs if rng.random() < 0.15]
            ops.append(("add", Task(allowed_topologies=topo)))
        if tasks and rng.random() < 0.5:
            ops.append(("del", list(tasks)[int(rng.integers(0, len(tasks)))]))
        nodes_changed = step % 3 == 0
        if nodes_changed:
            ops += [("status", int(rng.integers(0, n)), int(rng.choice([NodeStatus.Healthy, NodeStatus.Dead])))
                    for _ in range(int(rng.integers(1, 20)))]
        for op in ops:
            for p in (a, b):
                if op[0] == "add":
                    p.add_task(op[1])
                elif op[0] == "del":
                    p.delete_task(op[1])
                else:
                    p.update_node_status(addr(op[1]), op[2])
            if op[0] == "add":
                tasks[op[1].id] = op[1]
            elif op[0] == "del":
                tasks.pop(op[1])
        e2.resize_workers(0)   # b's plugin uploads everything: a full evaluation
        fa, fb = a.try_form_new_groups(), b.try_form_new_groups()
        assert fa == fb, f"step {step}: {fa} vs {fb}"
        assert all_groups(a) == all_groups(b), f"step {step}: published groups differ"
        st = e1.stats()
        if step and not nodes_changed:   # configurations toggled, no node changed: not a full evaluation
            assert st["n_tiles"] < n, (step, st)
            toggle_only += 1
    assert toggle_only >= 10, toggle_only
    assert len(all_groups(a)) > 10
    for p in (a, b):
        p.close()
    e1.close()
    e2.close()


# ------------------------------------------------------------------ 8. full size
def test_full_size_toggles_incremental_equals_full_pass():
    W, T = 1_000_000, 100_000
    w = synth.make_workers(W)
    a = synth.make_asks(T, "mixed")
    bits, npat, nmod, words = synth.intern_tables(w, a)
    rng = np.random.default_rng(2)
    e, f = Engine(), Engine()
    for x in (e, f):
        x.set_asks(a.asks, a.opts)
        x.set_model_table(bits, npat, nmod, words)
        x.set_workers(w.a, w.b)
    e.match(abi.PM_MODE_FIRST_FIT | INCR)
    ff = e.fetch().worker_ask
    owners = np.bincount(ff[ff != NONE], minlength=T)
    for rnd, j in enumerate((1, 10, 100)):
        off = np.concatenate([np.argsort(owners)[::-1][:j // 2 + 1], rng.choice(np.nonzero(owners == 0)[0], j // 2)])
        on = rng.choice(T, j, replace=False)
        for x in (e, f):
            x.set_ask_enabled(on, True)
            x.set_ask_enabled(off, False)
        e.match(abi.PM_MODE_FIRST_FIT | INCR)
        r = e.fetch()
        # the top owners' workers are orphans, walked again; nothing else is
        assert r.stats["n_tiles"] < W and r.stats["evals"] < T * W // 4, (rnd, r.stats)
        f.match(abi.PM_MODE_FIRST_FIT | LEAN)
        assert_same(r, f.fetch(), f"round {rnd}")
        ff = r.worker_ask
        owners = np.bincount(ff[ff != NONE], minlength=T)
    e.close()
    f.close()
