"""PM_INCREMENTAL: a pass that re-evaluates only the worker rows written since the engine's stored evaluation must
return exactly what the same pass without the flag returns — every array pm_fetch_result hands back — whatever the
history of table calls, whichever predicate variant the kernels select, on either side of the cutoff.  The stats say
which path ran: `evals` = pair evaluations executed, `n_tiles` = worker rows re-evaluated."""
import os

import numpy as np
import pytest

from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine
from protocol_b200.plugin import (ComputeSpecs, GpuSpecs, NodeGroupConfiguration, NodeGroupsPlugin, NodeStatus,
                                  OrchestratorNode, Task)
from test_gpu_variants import many_option_tables, wide_tables

pytestmark = pytest.mark.gpu

LEAN = abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS
INCR = LEAN | abi.PM_INCREMENTAL
CAND = abi.PM_W_HEALTHY | abi.PM_W_P2P
GROUPS = [(1, 1), (2, 3), (3, 5), (4, 4), (2, 8)]   # under-filled tails and hand-downs


def new_engine(**env):
    """An engine created with PM_TUNE_* knobs set (they are read at pm_create)."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return Engine(timing=True)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def assert_same(r, q, what=""):
    for f in ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count"):
        assert np.array_equal(getattr(r, f), getattr(q, f)), f"{what}: {f} differs"
    assert r.stats["n_bumped"] == q.stats["n_bumped"], what
    assert not r.ask_count.any() and (r.ask_best == abi.PM_COST_INF).all(), what


class Twin:
    """The same table calls on two engines: `inc` passes with PM_INCREMENTAL, `ref` without."""

    def __init__(self, mode, **env):
        self.mode = mode
        self.inc, self.ref = new_engine(**env), new_engine(**env)
        self.engines = (self.inc, self.ref)

    def __getattr__(self, name):
        def call(*args, **kw):
            for e in self.engines:
                getattr(e, name)(*args, **kw)
        return call

    def load(self, wa, wb, a, bits, npat, nmod, words, lat=None, lon=None, rank=None):
        self.set_asks(a.asks, a.opts)
        self.set_model_table(bits, npat, nmod, words)
        self.set_workers(wa, wb)
        if lat is not None:
            self.set_locations(lat, lon)
        if rank is not None:
            self.set_addr_rank(rank)

    def run(self, what=""):
        self.inc.match(self.mode | INCR)
        r = self.inc.fetch()
        self.ref.match(self.mode | LEAN)
        q = self.ref.fetch()
        assert_same(r, q, what)
        return r

    def close(self):
        for e in self.engines:
            e.close()


def full_stats(st, T, W):
    return st["evals"] == T * W and st["n_tiles"] == W


# ------------------------------------------------------------------ 1. random delta history
@pytest.mark.parametrize("mode", [abi.PM_MODE_FIRST_FIT, abi.PM_MODE_PROXIMITY], ids=["first_fit", "proximity"])
def test_random_delta_history(mode):
    rng = np.random.default_rng(5 + mode)
    W0, T = 3000, 240
    w = synth.make_workers(W0, with_addresses=False)
    pool = synth.make_workers(4000, seed=synth.SEED_WORKERS + 77)   # rows that get written in
    a = synth.make_asks(T, "mixed", group_sizes=GROUPS)
    a2 = synth.make_asks(T, "mixed", seed=synth.SEED_ASKS + 5, group_sizes=GROUPS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    tw = Twin(mode)
    W = W0
    tw.load(w.a, w.b, a, bits, npat, nmod, words, w.lat, w.lon, rng.permutation(W).astype(np.uint32))
    tw.run("first pass")
    assert full_stats(tw.inc.stats(), T, W)
    asks = a
    counts = {}

    def rows(n):
        sel = rng.integers(0, len(pool), n)
        ra, rb = pool.a[sel].copy(), pool.b[sel].copy()
        flip = rng.random(n)
        ra["flags"][flip < 0.2] ^= abi.PM_W_ASSIGNED
        ra["flags"][(flip >= 0.2) & (flip < 0.3)] ^= abi.PM_W_HEALTHY
        return ra, rb, pool.lat[sel], pool.lon[sel]

    for step in range(42):
        op = ["update", "update_dup", "flags", "upsert", "grow", "shrink", "none", "none", "asks", "bits"][step % 10] \
            if step < 10 else rng.choice(["update", "update_dup", "flags", "upsert", "grow", "shrink", "none", "asks", "bits"],
                                         p=[0.2, 0.1, 0.15, 0.1, 0.1, 0.1, 0.15, 0.05, 0.05])
        dirty, full = set(), False
        if op in ("update", "update_dup"):
            u = np.unique(rng.integers(0, W, int(rng.integers(1, 60))))
            ra, rb, la, lo = rows(len(u))
            pick = np.arange(len(u))
            if op == "update_dup":   # duplicate indices carry the same row and count once
                pick = np.concatenate([pick, rng.integers(0, len(u), len(u))])
            tw.update_workers(u[pick], ra[pick], rb[pick], la[pick], lo[pick])
            dirty = set(u.tolist())
        elif op == "flags":
            u = np.unique(rng.integers(0, W, int(rng.integers(1, 40))))
            f = np.where(rng.random(len(u)) < 0.5, CAND, CAND | abi.PM_W_ASSIGNED)
            f = (f | abi.PM_W_HAS_SPECS | abi.PM_W_HAS_GPU | abi.PM_W_HAS_GPU_COUNT | abi.PM_W_HAS_LOC).astype(np.uint32)
            idx = np.concatenate([u, u[:3], [W + 5]]).astype(np.uint32)   # repeats and an index past the table
            tw.set_flags(idx, np.concatenate([f, f[:3], [CAND]]).astype(np.uint32))
            dirty = set(u.tolist())
        elif op == "upsert":
            first = int(rng.integers(0, W - 50))
            n = int(rng.integers(1, 50))
            ra, rb, _, _ = rows(n)
            for e in tw.engines:
                e.upsert_workers(ra, rb, first)
            dirty = set(range(first, first + n))
        elif op == "grow":
            n = W + int(rng.integers(1, 300))
            tw.resize_workers(n)
            dirty = set(range(W, n))
            W = n
            new = np.arange(W - len(dirty), W, dtype=np.uint32)
            ra, rb, la, lo = rows(len(new))
            tw.update_workers(new, ra, rb, la, lo)   # the grown rows get contents (still the same dirty rows)
        elif op == "shrink":
            W = W - int(rng.integers(1, 300))
            tw.resize_workers(W)
        elif op == "asks":
            asks = a2 if asks is a else a
            tw.set_asks(asks.asks, asks.opts)
            full = True
        elif op == "bits":
            tw.set_model_table(bits, npat, nmod, words)
            full = True
        # ranks and locations write nothing the predicate reads; a rank per row keeps member order total
        tw.set_addr_rank(rng.permutation(W).astype(np.uint32))
        r = tw.run(f"step {step} ({op})")
        st = r.stats
        counts[op] = counts.get(op, 0) + 1
        if full:
            assert full_stats(st, T, W), (step, op, st)
        elif op == "shrink" or op == "none":
            assert st["n_tiles"] == 0 and st["evals"] == 0, (step, op, st)
        else:
            assert st["n_tiles"] == len(dirty), (step, op, st["n_tiles"], len(dirty))
            assert st["evals"] <= T * len(dirty), (step, op, st)
    assert r.stats["n_bumped"] >= 0 and len(r.group_ask) > 20
    assert all(counts.get(k, 0) >= 1 for k in ("update", "update_dup", "flags", "upsert", "grow", "shrink", "none", "asks",
                                                "bits")), counts
    tw.close()


def test_history_hands_down_and_bumps():
    """Group sizes that leave under-filled tails on every pass: the hand-down sweep runs on the working copy and
    bumps workers, and the stored evaluation stays the evaluation's."""
    rng = np.random.default_rng(11)
    w = synth.make_workers(2000)
    a = synth.make_asks(60, "mixed", group_sizes=[(3, 5), (4, 7), (2, 9)])
    bits, npat, nmod, words = synth.intern_tables(w, a)
    tw = Twin(abi.PM_MODE_FIRST_FIT)
    tw.load(w.a, w.b, a, bits, npat, nmod, words)
    bumped = 0
    for step in range(12):
        r = tw.run(f"step {step}")
        bumped += r.stats["n_bumped"]
        u = np.unique(rng.integers(0, len(w), 30)).astype(np.uint32)
        f = w.a["flags"][u] ^ np.uint32(abi.PM_W_ASSIGNED)
        w.a["flags"][u] = f
        tw.set_flags(u, f)
    assert bumped > 0
    tw.close()


# ------------------------------------------------------------------ 2. every predicate variant
def _variant_run(w, a, pbits, npat, nmod, words, rng, env=None, big=False):
    """Full pass, then three rounds of ~300 written rows: rows whose first feasible ask is 0, the last row, none,
    ordinary rows and non-candidates; worker_ask (all groups solo) is each worker's first feasible ask."""
    T = len(a)
    tw = Twin(abi.PM_MODE_FIRST_FIT, **(env or {}))
    wa, wb = w.a.copy(), w.b.copy()
    tw.load(wa, wb, a, pbits, npat, nmod, words)
    tw.run("full")
    ff = orc.soa_first_feasible(wa, wb, a.asks, a.opts, pbits, words)
    kinds = {}
    for rnd in range(3):
        src = rng.permutation(len(w))[:2000]
        src_ff = ff[src]
        pick = []
        for name, sel in (("row0", src_ff == 0), ("last", src_ff == src_ff[src_ff != abi.PM_NONE].max()),
                          ("none", src_ff == abi.PM_NONE), ("any", np.ones(len(src), bool))):
            got = src[sel][:80]
            kinds[name] = kinds.get(name, 0) + len(got)
            pick.append(got)
        pick = np.concatenate(pick)
        dst = np.unique(rng.integers(0, len(w), len(pick)))
        pick = pick[:len(dst)]
        na, nb = w.a[pick].copy(), w.b[pick].copy()
        if big and rnd == 1:   # operands >= 2^31 on written rows: the partial range check picks the generic predicate
            nb["ram_mb"][:5] = 0x80000000
            na["gpu_mem_mb"][5:8] = 0xF0000000
        wa[dst], wb[dst] = na, nb
        tw.update_workers(dst, na, nb)
        r = tw.run(f"round {rnd}")
        assert r.stats["n_tiles"] == len(dst)
        ff = orc.soa_first_feasible(wa, wb, a.asks, a.opts, pbits, words)
        if (a.asks["min_group_size"] == 1).all() and (a.asks["max_group_size"] == 1).all():
            assert np.array_equal(r.worker_ask, ff), f"round {rnd}: first feasible ask differs from the oracle"
    assert kinds["row0"] and kinds["none"] and kinds["last"], kinds
    tw.close()


@pytest.mark.parametrize("generic", ["0", "1"])
def test_fast_and_generic_predicates(generic):
    rng = np.random.default_rng(21)
    w = synth.make_workers(6000)
    a = synth.make_asks(700, "mixed")
    bits, npat, nmod, words = synth.intern_tables(w, a)
    _variant_run(w, a, bits, npat, nmod, words, rng, env={"PM_TUNE_GENERIC": generic}, big=True)


@pytest.mark.parametrize("n_models,n_patterns,shift", [(200, 112, 1), (3000, 112, 2), (100_000, 40, 3), (3000, 30, 41),
                                                       (100_000, 24, 35)],
                         ids=["200_shared", "3000_global", "100k_global", "3000_worker_major", "100k_worker_major"])
def test_wide_catalogues(n_models, n_patterns, shift):
    w, a, obits, pbits, npat, nmod, words = wide_tables(500, 6000, n_models, n_patterns, seed_shift=shift, last_rows=True)
    _variant_run(w, a, pbits, npat, nmod, words, np.random.default_rng(shift))


@pytest.mark.parametrize("n_models", [16, 200])
def test_asks_with_more_options_than_the_stage_holds(n_models):
    w, a, obits, pbits, npat, nmod, words = many_option_tables(n_models)
    _variant_run(w, a, pbits, npat, nmod, words, np.random.default_rng(n_models))


def test_many_row_chunks_catch_all_last_row():
    """T = 40 000 asks: a few hundred written workers split the asks into many chunks.  The last ask accepts every
    candidate, so workers without specs find it at the very last row, past every other chunk."""
    rng = np.random.default_rng(3)
    w = synth.make_workers(5000)
    a = synth.make_asks(40_000, "mixed")
    tail = np.zeros(1, dtype=abi.ASK)
    tail["opt_off"] = len(a.opts)
    tail["min_group_size"] = tail["max_group_size"] = 1
    a = synth.Asks(asks=np.concatenate([a.asks, tail]), opts=a.opts, pattern_strings=a.pattern_strings)
    T = len(a)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    tw = Twin(abi.PM_MODE_FIRST_FIT)
    tw.load(w.a, w.b, a, bits, npat, nmod, words)
    tw.run("full")
    dst = np.unique(rng.integers(0, len(w), 400)).astype(np.uint32)
    na, nb = w.a[dst].copy(), w.b[dst].copy()
    na["flags"][: len(dst) // 3] = CAND                  # candidates without specs: only the catch-all takes them
    na["flags"][len(dst) // 3: len(dst) // 2] = 0          # not candidates
    tw.update_workers(dst, na, nb)
    r = tw.run("chunks")
    assert (r.worker_ask[dst[: len(dst) // 3]] == T - 1).all()
    assert (r.worker_ask[dst[len(dst) // 3: len(dst) // 2]] == abi.PM_NONE).all()
    assert r.stats["n_tiles"] == len(dst) and 0 < r.stats["evals"] <= T * len(dst)
    tw.close()


# ------------------------------------------------------------------ 3. both sides of the cutoff
@pytest.mark.parametrize("cutoff", ["0", "50", "100000000"])
def test_cutoff(cutoff):
    rng = np.random.default_rng(7)
    w = synth.make_workers(4000)
    a = synth.make_asks(300, "mixed", group_sizes=GROUPS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    T, W = len(a), len(w)
    tw = Twin(abi.PM_MODE_FIRST_FIT, PM_TUNE_INCR=cutoff)
    tw.load(w.a, w.b, a, bits, npat, nmod, words)
    tw.run("full")
    for k in (10, 100, 3000):
        dst = rng.permutation(W)[:k].astype(np.uint32)
        f = w.a["flags"][dst] ^ np.uint32(abi.PM_W_ASSIGNED)
        tw.set_flags(dst, f)
        st = tw.run(f"k={k}").stats
        if int(cutoff) >= k:
            assert st["n_tiles"] == k and st["evals"] <= T * k, (k, st)
        else:
            assert full_stats(st, T, W), (k, st)
    tw.close()


# ------------------------------------------------------------------ 4. refusals and what invalidates
def _small_engine(**env):
    w = synth.make_workers(3000)
    a = synth.make_asks(200, "mixed", group_sizes=GROUPS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    e = new_engine(**env)
    e.set_asks(a.asks, a.opts)
    e.set_model_table(bits, npat, nmod, words)
    e.set_workers(w.a, w.b)
    e.set_locations(w.lat, w.lon)
    return e, w, a


def test_refusals():
    e, w, a = _small_engine()
    for mode in (abi.PM_MODE_FIRST_FIT | abi.PM_INCREMENTAL,
                 abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED | abi.PM_INCREMENTAL,
                 abi.PM_MODE_FIRST_FIT | abi.PM_NO_ASK_STATS | abi.PM_INCREMENTAL,
                 abi.PM_MODE_AUCTION | INCR):
        with pytest.raises(PrimeMatchError) as ex:
            e.match(mode)
        assert ex.value.status == abi.PM_E_INVALID, hex(mode)
    e.set_shard(0, 1500)
    with pytest.raises(PrimeMatchError) as ex:
        e.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert ex.value.status == abi.PM_E_UNSUPPORTED
    e.close()


def test_set_shard_invalidates():
    e, w, a = _small_engine()
    T, W = len(a), len(w)
    e.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert full_stats(e.stats(), T, W)
    e.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert e.stats()["evals"] == 0 and e.stats()["n_tiles"] == 0
    e.set_shard(0, 0)   # the whole table again, but the stored evaluation is gone
    e.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert full_stats(e.stats(), T, W)
    e.close()


def test_side_columns_re_evaluate_nothing():
    e, w, a = _small_engine()
    e.match(abi.PM_MODE_PROXIMITY | INCR)
    before = e.fetch()
    e.set_locations(w.lat[::-1].copy(), w.lon[::-1].copy())
    e.set_addr_rank(np.arange(len(w), dtype=np.uint32)[::-1].copy())
    e.set_worker_reputation(np.arange(len(w), dtype=np.uint32))
    e.match(abi.PM_MODE_PROXIMITY | INCR)
    st = e.stats()
    assert st["evals"] == 0 and st["n_tiles"] == 0
    # a flagless pass on the same tables gives the same groups (locations and ranks did change them)
    after = e.fetch()
    e.match(abi.PM_MODE_PROXIMITY | LEAN)
    assert_same(after, e.fetch(), "side columns")
    assert not np.array_equal(before.group_members, after.group_members)
    e.close()


# ------------------------------------------------------------------ 5. the plugin at scale
MODELS = ["NVIDIA H100", "NVIDIA A100 80GB", "RTX 4090", "NVIDIA L40S"]
CITIES = [(45.5186, -73.5545), (32.7942, -96.7475), (48.85, 2.35), (35.68, 139.69), None]


def addr(i):
    return "0x" + f"{(i * 2654435761) & 0xFFFFFFFF:08x}".upper() + f"{i:032x}"


def node(i, rng):
    spec = ComputeSpecs(gpu=GpuSpecs(count=int(rng.choice([1, 2, 4, 8])), model=MODELS[int(rng.integers(0, 4))],
                                     memory_mb=80000), ram_mb=64000, storage_gb=1000) if rng.random() > 0.05 else None
    return OrchestratorNode(addr(i), status=NodeStatus.Healthy if rng.random() > 0.1 else NodeStatus.Discovered,
                            p2p_id=f"p2p-{i}", compute_specs=spec, location=CITIES[int(rng.integers(0, 5))])


def all_groups(p):
    return p._json(p._lib.pm_plugin_get_all_groups, cap=1 << 26)   # thousands of groups: more than the default buffer


def test_plugin_at_scale():
    rng = np.random.default_rng(31)
    cfgs = []
    for c in range(50):
        mn = int(rng.integers(1, 5))
        req = f"gpu:count={[1, 2, 4, 8][c % 4]}" + (f";gpu:model={MODELS[c % 4].split()[-1]}" if c % 3 else "")
        cfgs.append(NodeGroupConfiguration(f"cfg-{c}", mn, mn + int(rng.integers(0, 4)), req if c % 7 else None))
    e1, e2 = Engine(), Engine()
    a = NodeGroupsPlugin(cfgs, engine=e1, proximity_enabled=False)
    b = NodeGroupsPlugin(cfgs, engine=e2, proximity_enabled=False)
    task = Task(allowed_topologies=[c.name for c in cfgs])
    for p in (a, b):
        p.add_task(task)
    n = 0
    for _ in range(20_000):
        nd = node(n, np.random.default_rng(n))
        for p in (a, b):
            p.add_node(nd)
        n += 1
    incremental = 0
    for step in range(30):
        ops = [("add", n + i) for i in range(int(rng.integers(0, 30)))]
        n += len(ops)
        ops += [("status", int(rng.integers(0, n)), int(rng.choice([NodeStatus.Healthy, NodeStatus.Dead])))
                for _ in range(int(rng.integers(0, 40)))]
        for p in (a, b):
            for op in ops:
                if op[0] == "add":
                    p.add_node(node(op[1], np.random.default_rng(op[1])))
                else:
                    p.update_node_status(addr(op[1]), op[2])
        e2.resize_workers(0)   # b's plugin has to upload everything: a full evaluation
        fa, fb = a.try_form_new_groups(), b.try_form_new_groups()
        assert fa == fb, f"step {step}: {fa} vs {fb} groups formed"
        assert all_groups(a) == all_groups(b), f"step {step}: published groups differ"
        st = e1.stats()
        if step and st["n_tiles"] < n:
            incremental += 1
            assert st["evals"] <= st["n_tiles"] * len(cfgs), st
    assert incremental >= 10, incremental
    assert len(all_groups(a)) > 100
    for p in (a, b):
        p.close()
    e1.close()
    e2.close()


# ------------------------------------------------------------------ 6. full size, once
def test_full_size_incremental_equals_full_pass():
    W, T = 1_000_000, 100_000
    w = synth.make_workers(W)
    a = synth.make_asks(T, "mixed")
    bits, npat, nmod, words = synth.intern_tables(w, a)
    rng = np.random.default_rng(1)
    e = Engine()
    e.set_asks(a.asks, a.opts)
    e.set_model_table(bits, npat, nmod, words)
    e.set_workers(w.a, w.b)
    e.match(abi.PM_MODE_FIRST_FIT | INCR)
    assert full_stats(e.stats(), T, W)
    dst = np.unique(rng.integers(0, W, 400)).astype(np.uint32)
    src = rng.integers(0, W, len(dst))
    na, nb = w.a[src].copy(), w.b[src].copy()
    na["flags"][::5] ^= abi.PM_W_ASSIGNED
    e.update_workers(dst, na, nb)
    e.match(abi.PM_MODE_FIRST_FIT | INCR)
    r = e.fetch()
    assert r.stats["n_tiles"] == len(dst) and r.stats["evals"] <= T * len(dst)
    w.a[dst], w.b[dst] = na, nb
    f = Engine()
    f.set_asks(a.asks, a.opts)
    f.set_model_table(bits, npat, nmod, words)
    f.set_workers(w.a, w.b)
    f.match(abi.PM_MODE_FIRST_FIT | LEAN)
    assert_same(r, f.fetch(), "full size")
    e.close()
    f.close()
