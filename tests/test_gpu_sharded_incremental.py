"""PM_INCREMENTAL on sharded engines: shard engines on one GPU through pm_match_local (the host merges the three
arrays, as the collective does), and pm_multi through pm_multi_match.  Every rank keeps the stored evaluation of its
own range and re-walks only that range's written rows, its orphans and, after asks were enabled, its workers against
them.  Through a random history of table calls every array pm_fetch_result returns must equal an unsharded engine's
full lean pass, and the stats must say that each rank walked exactly its share of the change."""
import os

import numpy as np
import pytest

from protocol_b200 import abi, synth
from protocol_b200.engine import Engine, MultiEngine
from protocol_b200.sharded import shard_range, wrap_device_buffers
from test_gpu_incremental import CAND, GROUPS, INCR, LEAN, assert_same, new_engine

pytestmark = pytest.mark.gpu


def _n_devices():
    import torch
    return torch.cuda.device_count()


def reference_pass(ref, mode):
    """The unsharded full lean pass: (its first feasible ask per worker, its result)."""
    W, T = ref.n_workers, ref.n_asks
    ref.match_local(mode | LEAN)
    ref.sync()
    first = wrap_device_buffers(ref, W, T)[0].cpu().numpy().view(np.uint32).copy()
    ref.match_finish(mode | LEAN)
    return first, ref.fetch()


class History:
    """Random table calls, applied by `apply(name, *args)` to every engine the test drives; remembers which rows were
    written and which asks were disabled / enabled since the last pass."""

    def __init__(self, rng, W, T, locations):
        self.rng, self.W, self.T, self.locations = rng, W, T, locations
        self.pool = synth.make_workers(4000, seed=synth.SEED_WORKERS + 77)
        self.on = np.ones(T, bool)
        self.reset()

    def reset(self):
        self.written = set()
        self.on_before = self.on.copy()

    def rows(self, n):
        sel = self.rng.integers(0, len(self.pool), n)
        ra, rb = self.pool.a[sel].copy(), self.pool.b[sel].copy()
        flip = self.rng.random(n)
        ra["flags"][flip < 0.2] ^= abi.PM_W_ASSIGNED
        ra["flags"][(flip >= 0.2) & (flip < 0.3)] ^= abi.PM_W_HEALTHY
        return ra, rb, self.pool.lat[sel], self.pool.lon[sel]

    def step(self, op, apply, first, lo=0, hi=None):
        """One table call of kind `op`; rows are drawn from [lo, hi) (default: the whole table)."""
        rng, W = self.rng, self.W
        hi = W if hi is None else hi
        if op == "update":
            u = np.unique(rng.integers(lo, hi, int(rng.integers(1, 60))))
            ra, rb, la, lo_ = self.rows(len(u))
            apply("update_workers", u, ra, rb, *((la, lo_) if self.locations else ()))
            self.written |= set(u.tolist())
        elif op == "flags":
            u = np.unique(rng.integers(lo, hi, int(rng.integers(1, 40))))
            f = np.where(rng.random(len(u)) < 0.5, CAND, CAND | abi.PM_W_ASSIGNED)
            f = (f | abi.PM_W_HAS_SPECS | abi.PM_W_HAS_GPU | abi.PM_W_HAS_GPU_COUNT | abi.PM_W_HAS_LOC).astype(np.uint32)
            apply("set_flags", u.astype(np.uint32), f)
            self.written |= set(u.tolist())
        elif op == "upsert":
            n = int(rng.integers(1, 40))
            first_row = int(rng.integers(0, W - n))
            ra, rb, _, _ = self.rows(n)
            apply("upsert_workers", ra, rb, first_row)
            self.written |= set(range(first_row, first_row + n))
        elif op in ("grow", "shrink"):
            n = W + int(rng.integers(1, 40)) if op == "grow" else W - int(rng.integers(1, 40))
            apply("resize_workers", n)
            if n > W:
                new = np.arange(W, n, dtype=np.uint32)
                ra, rb, la, lo_ = self.rows(len(new))
                apply("update_workers", new, ra, rb, *((la, lo_) if self.locations else ()))
                self.written |= set(range(W, n))
            self.written = {i for i in self.written if i < n}
            self.W = n
        elif op == "toggle":
            idx = rng.choice(self.T, int(rng.integers(1, 12)), replace=False)
            en = rng.random(len(idx)) < 0.5
            apply("set_ask_enabled", idx, en)
            self.on[idx] = en
        elif op == "disable_top":   # the asks that own the most workers
            owners = np.bincount(first[first != abi.PM_NONE], minlength=self.T)
            top = np.argsort(owners)[::-1][:3]
            apply("set_ask_enabled", top, False)
            self.on[top] = False
        elif op == "enable_all":
            apply("set_ask_enabled", np.arange(self.T), True)
            self.on[:] = True
        if self.locations or op in ("grow", "shrink"):   # a rank per row keeps member order total
            apply("set_addr_rank", rng.permutation(self.W).astype(np.uint32))

    def expected_tiles(self, lo, hi, stored, entered=()):
        """Rows a rank walks in full: its range's written rows (and those that entered it) plus its orphans."""
        rows = {i for i in self.written | set(entered) if lo <= i < hi}
        dis = set(np.nonzero(self.on_before & ~self.on)[0].tolist())
        orphans = [w for w in range(lo, hi) if w not in rows and int(stored[w]) in dis]
        return len(rows) + len(orphans)


# ------------------------------------------------------------------ 1. shard engines on one GPU
class Shards:
    """Shard engines on device 0 over equal shares of the table; the last one is open-ended (pm_set_shard(lo, 0)), so
    the rows a resize adds or cuts off are its own."""

    def __init__(self, n_shards, W, **env):
        self.engines = [new_engine(**env) for _ in range(n_shards)]
        self.ref = Engine()
        self.bounds = [shard_range(W, n_shards, r) for r in range(n_shards)]

    def apply(self, name, *args):
        for e in self.engines + [self.ref]:
            getattr(e, name)(*args)

    def set_ranges(self):
        last = len(self.engines) - 1
        for r, (e, (lo, hi)) in enumerate(zip(self.engines, self.bounds)):
            e.set_shard(lo, 0 if r == last else hi - lo)

    def ranges(self):
        W = self.ref.n_workers
        return [(lo, W if r == len(self.engines) - 1 else hi) for r, (lo, hi) in enumerate(self.bounds)]

    def run(self, mode, what):
        """match_local on every shard, the merge, match_finish; returns (reference first ask, reference result,
        per-shard stats)."""
        import torch

        W, T = self.ref.n_workers, self.ref.n_asks
        for e in self.engines:
            e.match_local(mode | INCR)
        bufs = []
        for e in self.engines:
            e.sync()
            bufs.append(wrap_device_buffers(e, W, T))
        ranges = self.ranges()
        for r, (lo, hi) in enumerate(ranges):
            fa = bufs[r][0]
            assert bool((fa[:lo] == -1).all()) and bool((fa[hi:] == -1).all()), f"{what}: shard {r} outside its range"
        first = torch.cat([bufs[r][0][lo:hi] for r, (lo, hi) in enumerate(ranges)])
        best = torch.stack([b[1] for b in bufs]).min(dim=0).values
        cnt = torch.stack([b[2] for b in bufs]).sum(dim=0).to(torch.int32)
        ref_first, q = reference_pass(self.ref, mode)
        assert np.array_equal(first.cpu().numpy().view(np.uint32), ref_first), f"{what}: first feasible ask differs"
        stats = []
        for r, e in enumerate(self.engines):
            bufs[r][0].copy_(first)
            bufs[r][1].copy_(best)
            bufs[r][2].copy_(cnt)
            torch.cuda.synchronize()
            e.match_finish(mode | INCR)
            res = e.fetch()
            assert_same(res, q, f"{what}, shard {r}")
            stats.append(res.stats)
        return ref_first, q, stats

    def close(self):
        for e in self.engines + [self.ref]:
            e.close()


def load(apply, w, a, bits, npat, nmod, words, locations):
    apply("set_asks", a.asks, a.opts)
    apply("set_model_table", bits, npat, nmod, words)
    apply("set_workers", w.a, w.b)
    if locations:
        apply("set_locations", w.lat, w.lon)
    apply("set_addr_rank", np.random.default_rng(0).permutation(len(w)).astype(np.uint32))


OPS = ["update", "flags", "upsert", "grow", "shrink", "toggle", "disable_top", "none", "enable_all"]


@pytest.mark.parametrize("n_shards,W,resize", [(2, 3001, True), (3, 3001, True), (7, 5, False)],
                         ids=["2_shards", "3_shards", "7_shards_5_workers"])
@pytest.mark.parametrize("mode", [abi.PM_MODE_FIRST_FIT, abi.PM_MODE_PROXIMITY], ids=["first_fit", "proximity"])
def test_shard_engines_random_history(n_shards, W, resize, mode):
    rng = np.random.default_rng(n_shards * 10 + mode)
    T = 240
    prox = mode == abi.PM_MODE_PROXIMITY
    w = synth.make_workers(W, with_addresses=False)
    a = synth.make_asks(T, "mixed", group_sizes=GROUPS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    sh = Shards(n_shards, W)
    load(sh.apply, w, a, bits, npat, nmod, words, prox)
    sh.set_ranges()
    h = History(rng, W, T, prox)
    first, _, stats = sh.run(mode, "first pass")
    for (lo, hi), st in zip(sh.ranges(), stats):
        assert st["n_tiles"] == hi - lo and st["evals"] == T * (hi - lo), st
    ops = OPS if resize else [op for op in OPS if op not in ("grow", "shrink", "upsert")]
    seen = set()
    for step in range(40):
        op = ops[step % len(ops)] if step < len(ops) else str(rng.choice(ops))
        if op == "shrink" and h.W - 40 <= sh.bounds[-1][0]:
            op = "grow"   # the last shard's start stays inside the table
        h.reset()
        h.step(op, sh.apply, first)
        stored = first
        first, q, stats = sh.run(mode, f"step {step} ({op})")
        for r, ((lo, hi), st) in enumerate(zip(sh.ranges(), stats)):
            want = h.expected_tiles(lo, hi, stored)
            assert st["n_tiles"] == want, (step, op, r, st["n_tiles"], want)
            if op == "none":
                assert st["evals"] == 0, (step, r, st)
        seen.add(op)
    assert seen == set(ops), seen
    assert len(q.group_ask) > 0
    sh.close()


def test_per_shard_cutoff():
    """A small PM_TUNE_INCR and rows written into one shard only: that shard evaluates its range in full, the others
    stay incremental, and the merged result is unchanged."""
    rng = np.random.default_rng(3)
    W, T = 6000, 200
    w = synth.make_workers(W, with_addresses=False)
    a = synth.make_asks(T, "mixed", group_sizes=GROUPS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    sh = Shards(3, W, PM_TUNE_INCR=50)
    load(sh.apply, w, a, bits, npat, nmod, words, False)
    sh.set_ranges()
    first, _, _ = sh.run(abi.PM_MODE_FIRST_FIT, "first pass")
    h = History(rng, W, T, False)
    ranges = sh.ranges()
    for r_hot in range(3):
        lo, hi = ranges[r_hot]
        h.reset()
        dst = rng.choice(np.arange(lo, hi), 120, replace=False).astype(np.uint32)
        ra, rb, _, _ = h.rows(len(dst))
        sh.apply("update_workers", dst, ra, rb)
        first, _, stats = sh.run(abi.PM_MODE_FIRST_FIT, f"hot shard {r_hot}")
        for r, ((lo, hi), st) in enumerate(zip(ranges, stats)):
            if r == r_hot:
                assert st["n_tiles"] == hi - lo and st["evals"] == T * (hi - lo), (r, st)
            else:
                assert st["n_tiles"] == 0 and st["evals"] == 0, (r, st)
    sh.close()


@pytest.mark.parametrize("call", ["set_shard", "set_asks", "set_model_table", "set_worker_count"])
def test_invalidation_on_a_shard_engine(call):
    W, T = 3000, 200
    w = synth.make_workers(W, with_addresses=False)
    a = synth.make_asks(T, "mixed", group_sizes=GROUPS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    lo, hi = 1000, 2200
    e = new_engine()
    load(lambda name, *args: getattr(e, name)(*args), w, a, bits, npat, nmod, words, False)
    e.set_shard(lo, hi - lo)
    mode = abi.PM_MODE_FIRST_FIT | INCR
    e.match_local(mode)
    e.sync()
    e.match_local(mode)
    e.match_finish(mode)
    st = e.stats()
    assert st["evals"] == 0 and st["n_tiles"] == 0, st
    if call == "set_shard":
        e.set_shard(lo, hi - lo)
    elif call == "set_asks":
        e.set_asks(a.asks, a.opts)
    elif call == "set_model_table":
        e.set_model_table(bits, npat, nmod, words)
    else:
        e.set_workers(w.a, w.b)   # pm_set_worker_count + pm_upsert_workers
    e.match_local(mode)
    e.match_finish(mode)
    st = e.stats()
    assert st["n_tiles"] == hi - lo and st["evals"] == T * (hi - lo), st
    e.close()


# ------------------------------------------------------------------ 2. pm_multi
def multi_history(devices, steps, seed):
    n = len(devices)
    rng = np.random.default_rng(seed)
    W, T = 4000 * n + n // 2 + 1, 300   # not a multiple of n
    w = synth.make_workers(W, with_addresses=False)
    a = synth.make_asks(T, "mixed", group_sizes=GROUPS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    m = MultiEngine(devices, timing=True)
    ref = Engine()

    def apply(name, *args):
        getattr(m, name)(*args)
        getattr(ref, name)(*args)

    load(apply, w, a, bits, npat, nmod, words, False)
    h = History(rng, W, T, False)
    mode = abi.PM_MODE_FIRST_FIT

    def run(what):
        m.match(mode | INCR)
        r = m.fetch()
        first, q = reference_pass(ref, mode)
        assert_same(r, q, what)
        return first, [m.stats(i) for i in range(n)]

    first, st = run("first pass")
    assert sum(s["evals"] for s in st) == T * W and sum(s["n_tiles"] for s in st) == W, st
    ops = ["update", "flags", "upsert", "grow", "shrink", "toggle", "disable_top", "none", "enable_all"]
    for step in range(steps):
        op = ops[step % len(ops)] if step < len(ops) else str(rng.choice(ops))
        h.reset()
        W_old = h.W
        if op == "grow":   # 1 ... n + 1 rows: every boundary moves by a row or so
            W_new = W_old + int(rng.integers(1, n + 2))
            apply("resize_workers", W_new)
            new = np.arange(W_old, W_new, dtype=np.uint32)
            ra, rb, _, _ = h.rows(len(new))
            apply("update_workers", new, ra, rb)
            h.written |= set(new.tolist())
            h.W = W_new
            apply("set_addr_rank", rng.permutation(h.W).astype(np.uint32))
        else:
            h.step(op, apply, first)
        stored = first
        first, st = run(f"step {step} ({op})")
        tiles = []
        for r, s in enumerate(st):
            a0, a1 = shard_range(W_old, n, r)
            lo, hi = shard_range(h.W, n, r)
            entered = [i for i in range(lo, hi) if not a0 <= i < a1]
            tiles.append(h.expected_tiles(lo, hi, stored, entered))
            assert s["n_tiles"] == tiles[-1], (step, op, r, s["n_tiles"], tiles[-1])
        n_en = int((h.on & ~h.on_before).sum())
        total = sum(s["evals"] for s in st)
        assert total <= T * sum(tiles) + n_en * h.W, (step, op, total)
        if op == "none":
            assert total == 0
    m.close()
    ref.close()


def test_multi_on_one_device():
    """pm_multi over device 0 alone: pm_multi_resize_workers and pm_multi_update_workers reach the engine, and its
    incremental passes equal full ones."""
    multi_history([0], 24, 5)


def test_multi_over_every_gpu():
    n = _n_devices()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    multi_history(list(range(n)), 30, 7)
