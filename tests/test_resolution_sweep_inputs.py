"""Inputs of tests/test_gpu_resolution_sweeps.py and the evidence that each one reaches the path it targets.

The resolution kernels (pm_sweep: first-fit under-filled tails; pm_merge_sweep: try_merge_solo_groups under the
proximity policy) are single CTAs of 1024 threads whose loops stride by 1024 threads or 32 warps.  Every input here is
built to push one of those loops past its first stride, and every input has a guard that proves it from the oracle
alone, so this file runs without a GPU: if a change to `synth` shrinks an input, the guard fails here instead of the
GPU case silently testing less.

First-fit evidence (`sweep_trace`) restates nothing of the sweep: from the oracle's groups (orc.soa_form_groups, the
per-configuration loop of mod.rs:478-628) and the oracle's predicate (orc.soa_eval_matrix), a worker reaches every
compatible configuration up to the one whose group takes it.  A configuration that some worker reaches without being
taken there had an under-filled tail; the worker was handed from it to the next configuration it reaches.
"""
from __future__ import annotations

import functools
import os

import numpy as np
import pytest

from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200.engine import Interner

NONE = abi.PM_NONE
STRIDE = 1024                      # threads of pm_sweep / pm_merge_sweep
THREADS = max(1, len(os.sched_getaffinity(0)))
SIZES = [(1, 1), (2, 2), (2, 4), (3, 3), (4, 8), (1, 3), (5, 16), (3, 5), (6, 6), (7, 9)]
FULL = (abi.PM_W_HEALTHY | abi.PM_W_P2P | abi.PM_W_HAS_SPECS | abi.PM_W_HAS_GPU | abi.PM_W_HAS_GPU_COUNT
        | abi.PM_W_HAS_GPU_MEM | abi.PM_W_HAS_GPU_MODEL | abi.PM_W_HAS_CPU | abi.PM_W_HAS_CPU_CORES | abi.PM_W_HAS_RAM
        | abi.PM_W_HAS_STORAGE)


# ------------------------------------------------------------------------------------------------ table assembly
def crafted_workers(n, count, mem=40000, model_id=0, cores=16, ram=64000, storage=1000):
    """n fully specified, healthy candidate workers; per-worker columns may be arrays."""
    a = np.zeros(n, dtype=abi.WORKER_A)
    b = np.zeros(n, dtype=abi.WORKER_B)
    a["gpu_count"], a["gpu_mem_mb"], a["model_id"], a["flags"] = count, mem, model_id, FULL
    b["cpu_cores"], b["ram_mb"], b["storage_gb"] = cores, ram, storage
    return a, b


class Asks:
    """Ask rows in priority order, from synth blocks and requirement strings parsed by the product's parser against
    an interner that holds the workers' model strings (ids = catalogue positions)."""

    def __init__(self, model_strings, pattern_strings=synth.PATTERN_CATALOGUE):
        self.it = Interner()
        for i, m in enumerate(model_strings):
            assert self.it.model(m) == i
        for i, p in enumerate(pattern_strings):
            assert self.it.pattern(p) == i
        self.blocks = []           # (ask rows, option rows with block-local offsets)
        self._parsed = {}

    def synth_block(self, asks: synth.Asks, lo=0, hi=None):
        hi = len(asks) if hi is None else hi
        rows = asks.asks[lo:hi].copy()
        o0 = int(rows["opt_off"][0]) if len(rows) else 0
        o1 = int(rows["opt_off"][-1] + rows["n_opts"][-1]) if len(rows) else 0
        rows["opt_off"] -= o0
        self.blocks.append((rows, asks.opts[o0:o1].copy()))

    def add(self, req, mn, mx):
        if req not in self._parsed:
            self._parsed[req] = self.it.parse(req)
        row, o = self._parsed[req]
        row = row.copy()
        row["opt_off"], row["min_group_size"], row["max_group_size"] = 0, mn, mx
        self.blocks.append((np.array([row], dtype=abi.ASK), o.copy()))

    def __len__(self):
        return sum(len(r) for r, _ in self.blocks)

    def tables(self, wa, wb, lat=None, lon=None):
        rows, opts, off = [], [], 0
        for r, o in self.blocks:
            r = r.copy()
            r["opt_off"] += off
            rows.append(r)
            opts.append(o)
            off += len(o)
        bits, npat, nmod, words = self.it.table()
        n = len(wa)
        return dict(asks=np.concatenate(rows), opts=np.concatenate(opts).astype(abi.GPU_OPT), wa=wa, wb=wb, bits=bits,
                    n_patterns=npat, n_models=nmod, words=words,
                    lat=np.zeros(n) if lat is None else lat, lon=np.zeros(n) if lon is None else lon)


def _workers(*parts):
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


# ------------------------------------------------------------------------------------------------ first-fit inputs
PLANTED = {1023: (5, 5), 1024: (3, 3), 2047: (4, 4), 2048: (3, 3)}   # index -> (min, max) of the gpu:count=3 asks


@functools.lru_cache(maxsize=None)
def many_configs():
    """Case 1: 5000 mixed asks with group sizes that leave frequent tails over 60 000 synth workers, plus gpu:count=3
    asks at 1023, 1024, 2047 and 2048 that seven count-3 workers reach in turn: each is an under-filled tail that
    hands the same two workers across a chunk boundary of 1024, and the last one hands them to nobody."""
    w = synth.make_workers(60_000, seed=synth.SEED_WORKERS + 101, with_addresses=True)
    a = synth.make_asks(4996, "mixed", seed=synth.SEED_ASKS + 101, group_sizes=SIZES)
    k = Asks(w.model_strings)
    prev = 0
    for i, idx in enumerate(sorted(PLANTED)):
        k.synth_block(a, prev, idx - i)
        k.add("gpu:count=3", *PLANTED[idx])
        prev = idx - i
    k.synth_block(a, prev)
    wa, wb = _workers((w.a, w.b), crafted_workers(7, 3))
    rank = np.concatenate([w.addr_rank, np.arange(len(w), len(w) + 7, dtype=np.uint32)])
    return k.tables(wa, wb), rank


@functools.lru_cache(maxsize=None)
def cascade():
    """Cases 2 and 5: a chain of 2200 gpu:count=5 asks at every other index from 1 to 4399, between mixed asks.  The
    first link holds 40 count-5 workers as (16, 16): 8 are handed on; every later link is (9, 9), reached only by those
    8 (its base segment is empty), so all 8 move on again, across four chunk boundaries.  The last link is (1, 8).
    Interleaved: count-5 asks with max_group_size 0 (feasible for nobody, the chain skips them) and asks with
    min_group_size 0 that nobody reaches (a trailing empty group each)."""
    w = synth.make_workers(20_000, seed=synth.SEED_WORKERS + 102)
    a = synth.make_asks(2200, "mixed", seed=synth.SEED_ASKS + 102, group_sizes=SIZES)
    k = Asks(w.model_strings)
    for i in range(2200):
        k.synth_block(a, i, i + 1)
        k.add("gpu:count=5", *((16, 16) if i == 0 else (1, 8) if i == 2199 else (9, 9)))
        if i % 97 == 5:
            k.add("gpu:count=5", 0, 0)
        if i % 101 == 7:
            k.add("gpu:count=6", 0, 3)
    fives = crafted_workers(40, 5)
    wa, wb = _workers((w.a[:9000], w.b[:9000]), fives, (w.a[9000:], w.b[9000:]))
    return k.tables(wa, wb), None


@functools.lru_cache(maxsize=None)
def big_pops():
    """Cases 3, 4 and 7 over 20 000 synth workers.
    * 4100 count-7 workers: (2999, 3000) forms one group of 3000 (more than 1024 members to order by address rank)
      and hands 1100 on; only the half with 80 GB reaches a later ask, the rest are left unassigned.
    * 150 count-9 workers: (99, 100) hands 50 on (more than 32, fewer than 1024).
    * 200 count-6 workers, even positions 60 GB, odd 30 GB: A = (60, 60) over the 100 even ones hands the 40 largest on
      to B = (100, 100), whose own segment is the 100 odd ones; B's 40 largest alternate between the two sources."""
    w = synth.make_workers(20_000, seed=synth.SEED_WORKERS + 103, with_addresses=True)
    a = synth.make_asks(600, "mixed", seed=synth.SEED_ASKS + 103, group_sizes=SIZES)
    k = Asks(w.model_strings)
    k.synth_block(a, 0, 100)
    k.add("gpu:count=7", 2999, 3000)
    k.add("gpu:count=6;gpu:memory_mb_min=50000", 60, 60)
    k.synth_block(a, 100, 300)
    k.add("gpu:count=9", 99, 100)
    k.add("gpu:count=6", 100, 100)
    k.synth_block(a, 300, 500)
    k.add("gpu:count=7;gpu:memory_mb_min=50000", 1, 1)
    k.add("gpu:count=6", 1, 1)
    k.add("gpu:count=9", 1, 2)
    k.synth_block(a, 500)
    sevens = crafted_workers(4100, 7, mem=np.where(np.arange(4100) % 2 == 0, 80000, 24000))
    nines = crafted_workers(150, 9)
    sixes = crafted_workers(200, 6, mem=np.where(np.arange(200) % 2 == 0, 60000, 30000))
    parts = [(w.a[:5000], w.b[:5000]), sevens, (w.a[5000:12000], w.b[5000:12000]), nines, sixes,
             (w.a[12000:], w.b[12000:])]
    wa, wb = _workers(*parts)
    rng = np.random.default_rng(103)
    rank = rng.permutation(len(wa)).astype(np.uint32)
    return k.tables(wa, wb), rank


def _with_group_sizes(a, seed):
    """Cycle SIZES over the asks of a wide-catalogue table (its own ask order stays the priority order)."""
    pick = synth.splitmix64(seed, len(a.asks), 30) % np.uint64(len(SIZES))
    gs = np.asarray(SIZES, dtype=np.uint32)[pick.astype(np.int64)]
    a.asks["min_group_size"], a.asks["max_group_size"] = gs[:, 0], gs[:, 1]


@functools.lru_cache(maxsize=None)
def wide(n_models, n_patterns):
    """Case 6: test_gpu_variants' wide catalogues with group sizes: the sweep decides hand-downs with ask_meets on the
    31-models-per-word table while the evaluation ran the BITS = 1 / 0 or worker-major kernels."""
    from test_gpu_variants import wide_tables

    w, a, obits, pbits, npat, nmod, words = wide_tables(700, 8000, n_models=n_models, n_patterns=n_patterns,
                                                        seed_shift=200 + n_patterns, last_rows=True)
    _with_group_sizes(a, 200 + n_models)
    # every option names models: compatible sets stay small, so tails are frequent and targets depend on the clause
    no_model = (a.opts["present"] & abi.PM_O_MODEL) == 0
    pid = synth.splitmix64(300 + n_models, len(a.opts), 31) % np.uint64(n_patterns)
    a.opts["pattern_id"][no_model] = pid.astype(np.uint32)[no_model]
    a.opts["present"] |= abi.PM_O_MODEL
    t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=obits, n_patterns=npat, n_models=nmod, words=words,
             lat=w.lat, lon=w.lon)
    return t, pbits


@functools.lru_cache(maxsize=None)
def large_operands():
    """Case 6, generic predicate: u32 operands >= 2^31 and a wrapping count x memory product decide where a handed-down
    worker goes.  Three (3, 3) asks over five such workers each hand two on; of each pair the next ask's wide clause
    (ram >= 3e9, memory_mb_min >= 2.5e9, total_memory_max 10 through a product that wraps to 0) accepts one, and the
    other falls through to a plain ask further down."""
    w = synth.make_workers(3000, seed=synth.SEED_WORKERS + 104)
    a = synth.make_asks(300, "mixed", seed=synth.SEED_ASKS + 104, group_sizes=SIZES)
    k = Asks(w.model_strings)
    k.synth_block(a, 0, 100)
    k.add("gpu:count=65536", 3, 3)
    k.add("gpu:count=11", 3, 3)
    k.add("gpu:count=12", 3, 3)
    k.synth_block(a, 100, 200)
    k.add("gpu:count=65536;gpu:total_memory_max=10", 1, 1)
    k.add("gpu:count=11;ram_mb=3000000000", 1, 1)
    k.add("gpu:count=12;gpu:memory_mb_min=2500000000", 1, 1)
    k.add("gpu:count=65536", 1, 1)
    k.add("gpu:count=11", 1, 1)
    k.add("gpu:count=12", 1, 1)
    k.synth_block(a, 200)
    # five each: (3, 3) keeps three and hands on the last two, one accepted by the wide clause and one not
    wrap = crafted_workers(5, 65536, mem=np.array([65536, 65537, 65536, 65536, 65537]))   # 2^32 wraps to 0; 2^16 stays
    ram = crafted_workers(5, 11, ram=np.array([3_500_000_000, 1000, 3_000_000_000, 3_000_000_000, 2_999_999_999]))
    mem = crafted_workers(5, 12, mem=np.array([3_000_000_000, 40000, 2_500_000_000, 2_500_000_000, 2_499_999_999]))
    wa, wb = _workers((w.a[:1000], w.b[:1000]), wrap, ram, mem, (w.a[1000:], w.b[1000:]))
    return k.tables(wa, wb), None


@functools.lru_cache(maxsize=None)
def late_tails():
    """Case 1, the other way round: whole chunks of 1024 without an under-filled tail before and between the ones that
    have one.  3000 solo asks, and seven count-3 workers: (5, 5) at 1500 hands two on to (3, 3) at 2700, which hands
    them on to (1, 1) at 2990."""
    w = synth.make_workers(20_000, seed=synth.SEED_WORKERS + 105)
    a = synth.make_asks(2997, "mixed", seed=synth.SEED_ASKS + 105)
    k = Asks(w.model_strings)
    k.synth_block(a, 0, 1500)
    k.add("gpu:count=3", 5, 5)
    k.synth_block(a, 1500, 2699)
    k.add("gpu:count=3", 3, 3)
    k.synth_block(a, 2699, 2988)
    k.add("gpu:count=3", 1, 1)
    k.synth_block(a, 2988)
    wa, wb = _workers((w.a[:7000], w.b[:7000]), crafted_workers(7, 3), (w.a[7000:], w.b[7000:]))
    return k.tables(wa, wb), None


FIRST_FIT_CASES = {"many_configs": many_configs, "late_tails": late_tails, "cascade": cascade, "big_pops": big_pops,
                   "large_operands": large_operands}


# ------------------------------------------------------------------------------------------------ first-fit evidence
def oracle_groups(t, addr_rank=None):
    return orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], addr_rank=addr_rank)


def sweep_trace(t, og, band=128):
    """Per configuration: K (workers that reach it), base (of those, the ones it is the first feasible configuration
    of), pop (reached but not taken); hand-downs as (from, to, worker) with to = NONE for workers left over."""
    T, W = len(t["asks"]), len(t["wa"])
    taken_at = np.full(W, T, dtype=np.int64)
    for g in range(len(og.cfg)):
        taken_at[og.members[og.off[g]:og.off[g + 1]]] = og.cfg[g]
    K = np.zeros(T, dtype=np.int64)
    base = np.zeros(T, dtype=np.int64)
    pop = np.zeros(T, dtype=np.int64)
    last = np.full(W, -1, dtype=np.int64)
    src, dst, who = [], [], []
    for t0 in range(0, T, band):
        t1 = min(T, t0 + band)
        cost = orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], t0, t1, 0, W,
                                   threads=THREADS, want_cost=True, want_rows=False, want_cols=False)["cost"]
        reach = (cost != abi.PM_COST_INF) & (taken_at[None, :] >= np.arange(t0, t1)[:, None])
        for i in range(t1 - t0):
            c = t0 + i
            ws = np.flatnonzero(reach[i])
            prev = last[ws]
            K[c], base[c], pop[c] = len(ws), int((prev < 0).sum()), int((taken_at[ws] > c).sum())
            h = prev >= 0
            src.append(prev[h])
            dst.append(np.full(int(h.sum()), c, dtype=np.int64))
            who.append(ws[h])
            last[ws] = c
    left = np.flatnonzero((taken_at == T) & (last >= 0))
    src.append(last[left])
    dst.append(np.full(len(left), NONE, dtype=np.int64))
    who.append(left)
    mn = t["asks"]["min_group_size"].astype(np.int64)
    mx = t["asks"]["max_group_size"].astype(np.int64)
    r = np.where(mx > 0, K % np.maximum(mx, 1), 0)
    bad = (r > 0) & (r < mn)
    # the oracle's groups and its predicate tell one story: exactly the under-filled tails were handed on, whole
    assert np.array_equal(pop, np.where(bad, r, 0))
    return dict(K=K, base=base, pop=pop, bad=bad, src=np.concatenate(src), dst=np.concatenate(dst),
                who=np.concatenate(who))


@functools.lru_cache(maxsize=None)
def first_fit_case(name):
    t, rank = FIRST_FIT_CASES[name]()
    og = oracle_groups(t, rank)
    return t, rank, og, sweep_trace(t, og)


def _chunk_crossings(tr):
    moved = tr["dst"] != NONE
    return int(((tr["src"][moved] // STRIDE) != (tr["dst"][moved] // STRIDE)).sum())


def guard_first_fit(name, t, og, tr):
    """The evidence each input exists for; returns the number of hand-downs the engine must report as n_bumped."""
    bad = np.flatnonzero(tr["bad"])
    assert len(bad), "no under-filled tail at all"
    n_none = int((tr["dst"] == NONE).sum())
    if name == "many_configs":
        assert len(t["asks"]) == 5000 and len(t["wa"]) > 60_000
        assert set(PLANTED) <= set(bad.tolist()) and bad.max() >= 2 * STRIDE
        assert len(bad) > 800 and (bad >= 2 * STRIDE).sum() > 150 and bad.max() >= 3 * STRIDE            # frequent tails in every chunk
        for frm, to in ((1023, 1024), (1024, 2047), (2047, 2048)):
            assert ((tr["src"] == frm) & (tr["dst"] == to)).sum() == 2            # across a chunk boundary
        assert ((tr["src"] == 2048) & (tr["dst"] == NONE)).sum() == 2
        assert _chunk_crossings(tr) >= 5
    elif name == "late_tails":
        assert bad.tolist() == [1500, 2700] and len(t["asks"]) == 3000
        assert ((tr["src"] == 1500) & (tr["dst"] == 2700)).sum() == 2 and ((tr["src"] == 2700) & (tr["dst"] == 2990)).sum() == 2
    elif name == "cascade":
        links = np.flatnonzero(tr["bad"] & (tr["base"] == 0) & (tr["pop"] == 8) & (tr["K"] == 8))
        chain = links[np.isin(links, np.flatnonzero(t["asks"]["max_group_size"] == 9))]
        assert len(chain) >= 2100 and chain.min() < STRIDE and chain.max() >= 4 * STRIDE
        gaps = np.diff(chain)
        assert (gaps <= 4).all()                                               # one unbroken chain
        zero_max = np.flatnonzero(t["asks"]["max_group_size"] == 0)
        zero_min = np.flatnonzero((t["asks"]["min_group_size"] == 0) & (t["asks"]["max_group_size"] > 0))
        assert len(zero_max) > 20 and len(zero_min) > 20
        assert (zero_max > chain.min()).sum() > 20 and (zero_min < chain.max()).sum() > 20   # among the links
        assert tr["K"][zero_max].sum() == 0                                    # skipped by every hand-down
        assert (np.isin(og.cfg, zero_min)).sum() == len(zero_min)              # one empty group each
        assert _chunk_crossings(tr) >= 4
    elif name == "big_pops":
        assert tr["pop"].max() > STRIDE and ((tr["pop"] > 32) & (tr["pop"] < STRIDE)).any()
        big = int(np.argmax(tr["pop"]))
        assert n_none > 500 and ((tr["src"] == big) & (tr["dst"] == NONE)).sum() > 500
        sizes = np.diff(og.off)
        assert sizes.max() > STRIDE                                            # pm_order_members over > 1024 members
        # B pops from both sources, alternating: sort its popped workers by index, count source switches
        b = [c for c in np.flatnonzero(tr["bad"]) if tr["base"][c] and tr["base"][c] < tr["K"][c]]
        switches = 0
        for c in b:
            out = np.sort(tr["who"][tr["src"] == c])
            came_in = np.isin(out, tr["who"][tr["dst"] == c])
            switches = max(switches, int((came_in[1:] != came_in[:-1]).sum()))
        assert switches >= 30
    elif name == "large_operands":
        big = (t["wb"]["ram_mb"] >= 1 << 31) | (t["wa"]["gpu_mem_mb"] >= 1 << 31) | \
              ((t["wa"]["gpu_count"].astype(np.uint64) * t["wa"]["gpu_mem_mb"]) >= 1 << 32)
        moved = np.isin(tr["who"], np.flatnonzero(big)) & (tr["dst"] != NONE)
        assert moved.sum() == 6 and len(set(tr["dst"][moved].tolist())) == 6   # both fates of every wide clause
    return int(tr["pop"].sum())


def guard_wide(t, og, tr):
    """Hand-downs whose target accepted the worker through a model clause past the first acceptance word."""
    moved = tr["dst"] != NONE
    mid = t["wa"]["model_id"][tr["who"][moved]]
    tgt = tr["dst"][moved]
    has_model = np.zeros(len(t["asks"]), dtype=bool)
    pm = np.flatnonzero((t["opts"]["present"] & abi.PM_O_MODEL) != 0)
    owner = np.searchsorted(t["asks"]["opt_off"].astype(np.int64), pm, side="right") - 1
    has_model[owner] = True
    n = int(((mid >= 62) & has_model[tgt]).sum())
    assert n >= 20, f"{n} hand-downs decided past the first acceptance word"
    return int(tr["pop"].sum())


# ------------------------------------------------------------------------------------------------ merge inputs
def merge_nodes(n, seed, located="cities", points=None, counts=None):
    """Synth workers as the plugin's nodes: (workers, located mask).  located: 'cities' (synth), 'none', or 'points'
    (`counts[i]` nodes on points[i], in interleaved order)."""
    w = synth.make_workers(n, seed=seed, with_addresses=True, healthy_frac=1.0)
    w.a["flags"] |= abi.PM_W_P2P
    if located == "none":
        w.a["flags"] &= ~np.uint32(abi.PM_W_HAS_LOC)
    elif located == "points":
        which = np.repeat(np.arange(len(counts)), counts)
        which = which[np.random.default_rng(seed).permutation(len(which))]
        w.lat, w.lon = np.asarray(points)[which, 0].copy(), np.asarray(points)[which, 1].copy()
        w.a["flags"] |= abi.PM_W_HAS_LOC
    return w


# configurations: (name, min, max, requirement) in template order
MERGE_CASES = {
    # 1 + 2: the first configuration's min exceeds its ~1600 compatible nodes: none merge, all are handed to the next,
    # whose list (4000) and hand-down list (> 1024) both pass the first stride
    "handdown": dict(n=4000, seed=901, located="cities",
                     cfgs=[("cfg-big", 2000, 4000, "gpu:count=1"), ("cfg-any", 2, 5, None), ("solo", 1, 1, None)]),
    # 3: nobody located, batches of 1500 filled in list order
    "list_order": dict(n=4000, seed=902, located="none",
                       cfgs=[("cfg-1500", 1500, 1500, None), ("cfg-pair", 2, 2, "gpu:count=2"), ("solo", 1, 1, None)]),
    # 4: two points, every distance tied at 0 within a point: position breaks ties across strides
    "ties": dict(n=3000, seed=903, located="points", points=[(45.5186, -73.5545), (32.7942, -96.7475)],
                 counts=[1700, 1300], cfgs=[("cfg-1200", 2, 1200, None), ("solo", 1, 1, None)]),
    # 5: 1100 configurations nobody fits before the ones that merge
    "many_configs": dict(n=300, seed=904, located="cities",
                         cfgs=[(f"cfg-none-{i}", 2, 3, f"gpu:count={9 + i}") for i in range(1090)]
                         + [("cfg-c1", 2, 3, "gpu:count=1"), ("cfg-c2", 2, 4, "gpu:count=2"),
                            ("cfg-c4", 2, 2, "gpu:count=4"), ("cfg-any", 2, 3, None), ("solo", 1, 1, None)]),
}


def merge_oracle_setup(case):
    """(workers, oracle nodes, available configurations in priority order, oracle configs) for a merge case."""
    spec = MERGE_CASES[case]
    w = merge_nodes(spec["n"], spec["seed"], spec["located"], spec.get("points"), spec.get("counts"))
    onodes = []
    for i in range(len(w)):
        f = int(w.a["flags"][i])
        has = lambda b: bool(f & b)
        kw = {}
        if has(abi.PM_W_HAS_SPECS):
            kw = dict(gpu_count=int(w.a["gpu_count"][i]), gpu_model=w.model_strings[int(w.a["model_id"][i])],
                      gpu_mem=int(w.a["gpu_mem_mb"][i]) if has(abi.PM_W_HAS_GPU_MEM) else None,
                      cpu_cores=int(w.b["cpu_cores"][i]), ram=int(w.b["ram_mb"][i]), storage=int(w.b["storage_gb"][i]))
        loc = (float(w.lat[i]), float(w.lon[i])) if has(abi.PM_W_HAS_LOC) else None
        onodes.append(orc.make_node(address=w.addresses[i], specs=has(abi.PM_W_HAS_SPECS), location=loc, **kw))
    reqs = [orc.Req(r) if r else None for _, _, _, r in spec["cfgs"]]
    ocfgs = [(name, mn, mx, r) for (name, mn, mx, _), r in zip(spec["cfgs"], reqs)]
    sorted_cfgs = [ocfgs[i] for i in orc.sort_configs(ocfgs)]
    avail = [sorted_cfgs[i] for i in orc.available_configs(sorted_cfgs, [1] * len(sorted_cfgs))]
    return w, onodes, avail, reqs


def merge_list_lengths(onodes, avail, want):
    """Per merge configuration (max >= 2), how many solo nodes reach it and how many of those were handed down:
    the list pm_merge_sweep builds for it.  A node reaches every compatible configuration until a batch takes it."""
    taken_at = np.full(len(onodes), len(avail))
    for c, ms in want.as_list():
        taken_at[ms] = c
    reach, handed = np.zeros(len(avail), dtype=np.int64), np.zeros(len(avail), dtype=np.int64)
    seen = np.zeros(len(onodes), dtype=bool)
    for c, (_, mn, mx, req) in enumerate(avail):
        if mx < 2:
            continue
        ok = np.array([orc.node_compatible(nd, req) for nd in onodes]) & (taken_at >= c)
        reach[c], handed[c] = ok.sum(), (ok & seen).sum()
        seen |= ok
    return reach, handed


def guard_merge(case, w, onodes, avail, want):
    spec = MERGE_CASES[case]
    reach, handed = merge_list_lengths(onodes, avail, want)
    groups = want.as_list()
    sizes = np.array([len(m) for _, m in groups])
    located = (w.a["flags"] & abi.PM_W_HAS_LOC) != 0
    if case == "handdown":
        big = [n for n, *_ in avail].index("cfg-big")
        assert STRIDE < reach[big] < avail[big][1] and not any(c == big for c, _ in groups)
        nxt = [n for n, *_ in avail].index("cfg-any")
        assert handed[nxt] > STRIDE and reach[nxt] > 2 * STRIDE
        assert sizes[[c == nxt for c, _ in groups]].sum() > 2 * STRIDE         # seeds and members past the first stride
    elif case == "list_order":
        assert not located.any() and (sizes == 1500).sum() == 2
    elif case == "ties":
        pts = np.unique(np.stack([w.lat, w.lon], 1), axis=0)
        assert len(pts) == 2 and max(spec["counts"]) > STRIDE and (sizes == 1200).sum() >= 2
    elif case == "many_configs":
        assert len(avail) > STRIDE and min(c for c, _ in groups) >= STRIDE and len(groups) > 10
    return reach, handed


# ------------------------------------------------------------------------------------------------ the CPU guards
@pytest.mark.parametrize("name", sorted(FIRST_FIT_CASES))
def test_first_fit_inputs_reach_their_paths(name):
    t, rank, og, tr = first_fit_case(name)
    assert guard_first_fit(name, t, og, tr) > 0


@pytest.mark.parametrize("n_models,n_patterns", [(200, 112), (3000, 112), (3000, 30)])
def test_wide_catalogue_inputs_hand_down_past_word_zero(n_models, n_patterns):
    t, _ = wide(n_models, n_patterns)
    og = oracle_groups(t)
    guard_wide(t, og, sweep_trace(t, og))


@pytest.mark.parametrize("case", sorted(MERGE_CASES))
def test_merge_inputs_reach_their_paths(case):
    w, onodes, avail, _ = merge_oracle_setup(case)
    want = orc.merge_solo_groups(onodes, [(f"g{i:05d}", i, False) for i in range(len(onodes))], avail, proximity=True)
    guard_merge(case, w, onodes, avail, want)


def test_trace_matches_a_hand_worked_chain():
    """sweep_trace on a table small enough to follow by hand: 5 workers, (3, 3) then (2, 2) then (1, 1)."""
    k = Asks([m for m, _ in synth.MODEL_CATALOGUE])
    k.add("gpu:count=1", 3, 3)
    k.add("gpu:count=1", 2, 2)
    k.add("gpu:count=1", 1, 1)
    wa, wb = crafted_workers(5, 1)
    t = k.tables(wa, wb)
    og = oracle_groups(t)
    tr = sweep_trace(t, og)
    # 5 reach the first: one group of 3, workers 3 and 4 handed on; the second takes both
    assert tr["K"].tolist() == [5, 2, 0] and tr["pop"].tolist() == [2, 0, 0] and tr["base"].tolist() == [5, 0, 0]
    assert sorted(zip(tr["src"].tolist(), tr["dst"].tolist(), tr["who"].tolist())) == [(0, 1, 3), (0, 1, 4)]
    assert og.as_list() == [(0, [0, 1, 2]), (1, [3, 4])]
