"""Inputs of tests/test_gpu_proximity_sweeps.py and the evidence that each one reaches the path it targets.

Proximity formation (PM_MODE_PROXIMITY, the reference's default policy) runs on pm_proximity_grid, a cooperative launch
of ceil(W / 512) CTAs of 512 threads (at most the co-resident count, never fewer than the SMs when it runs at all), and
falls back to pm_proximity_sweep, one CTA of 1024 threads.  Their loops have boundaries no small table reaches: the
configuration scan in chunks of 512 / 1024 that skips a chunk nobody reaches, hand-down lists of up to 128 sorted in
shared memory and longer ones rebuilt by an ordered compaction, seed-parallel batches for groups of 2..4 with at least
two CTAs, per-group selection in chunks of 16 where CTA j owns list positions [512 j, 512 j + 512), ordered partitions
of unlocated groups across those chunks.  Every input here is built to cross one of them, and every input has a guard
that proves it from the checker alone, so this file runs without a GPU: if a change to `synth` shrinks an input, the
guard fails here instead of the GPU case silently testing less.

Every located worker stands on a certified place (the 64 synth cities, and 1 km traps written beyond ±90 where a case
needs them): a difference on the GPU is then a kernel bug, not two libm's rounding a near-tie.  The evidence is
`sweep_trace` applied to the proximity checker's groups (orc.soa_form_groups, latitude-banded: test_oracle_groups.py
proves it equal to the literal loop).  Its assertion holds unchanged under proximity: a configuration hands on exactly
its under-filled tail, r = K mod max when 0 < r < min — only WHICH workers go depends on the policy.

Disabled asks (pm_set_ask_enabled) behave as if absent: the checker runs on the enabled rows alone and its indices
are mapped back; the guards speak of the full table.
"""
from __future__ import annotations

import functools
import math

import numpy as np
import pytest

from helpers import assert_distance_certificate
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from test_resolution_sweep_inputs import NONE, SIZES, Asks, crafted_workers, sweep_trace

GRID = 512                      # threads of a pm_proximity_grid CTA: the scan chunk and the list positions a CTA owns
SINGLE = 1024                   # threads of pm_proximity_sweep
XS_SMEM = 128                   # hand-downs up to this long are walked and sorted in shared memory
TOPK = 16                       # neighbours selected per grid barrier
MAX_GRID_W = 132 * GRID         # up to here the grid is ceil(W / 512) CTAs on an H100
LOC = abi.PM_W_HAS_LOC
KM_PER_DEG = 6371.0 * np.pi / 180.0
CATALOGUE = [m for m, _ in synth.MODEL_CATALOGUE]


def n_ctas(W):
    assert W <= MAX_GRID_W, "the grid width is only known up to 132 x 512 workers"
    return max(1, -(-W // GRID))


def beyond_90(lat, lon):
    """The same place with its latitude written beyond ±90."""
    return math.copysign(180.0, lat) - lat, lon + 180.0


# ------------------------------------------------------------------------------------------------ table assembly
class Pop:
    """Workers in index order and where they stand: synth blocks (on the synth cities) and crafted families placed
    on `points` by index (-1: no location)."""

    def __init__(self, points=synth.CITIES):
        self.points = np.asarray(points, dtype=np.float64)
        self.parts = []
        self.n = 0

    def _add(self, a, b, lat, lon):
        self.parts.append((a, b, lat, lon))
        self.n += len(a)
        return np.arange(self.n - len(a), self.n)

    def synth(self, w, lo=0, hi=None):
        hi = len(w) if hi is None else hi
        return self._add(w.a[lo:hi], w.b[lo:hi], w.lat[lo:hi], w.lon[lo:hi])

    def crafted(self, where, count, **kw):
        where = np.asarray(where, dtype=np.int64)
        a, b = crafted_workers(len(where), count, **kw)
        loc = where >= 0
        a["flags"][loc] |= LOC
        p = self.points[np.maximum(where, 0)]
        return self._add(a, b, np.where(loc, p[:, 0], 0.0), np.where(loc, p[:, 1], 0.0))

    def tables(self, k: Asks):
        cat = lambda i: np.concatenate([p[i] for p in self.parts])
        return k.tables(cat(0), cat(1), cat(2), cat(3))


def spread(n, seed, located=1.0, cities=64):
    """n places drawn from the first `cities` synth cities, a fraction `located` of them located."""
    rng = np.random.default_rng(seed)
    where = rng.integers(0, cities, n)
    where[rng.random(n) >= located] = -1
    return where


def mixed_mem(n80, n24):
    """gpu memory of a family whose 80 GB and 24 GB members alternate by index while both last."""
    m = np.full(n80 + n24, 80000)
    k = min(n80, n24)
    m[1:2 * k:2] = 24000
    m[2 * k:] = 80000 if n80 > n24 else 24000
    return m


def add(k: Asks, req, mn, mx):
    """Asks.add, and None: an ask without requirements (every candidate fits)."""
    if req is not None:
        return k.add(req, mn, mx)
    row = np.zeros(1, dtype=abi.ASK)
    row["min_group_size"], row["max_group_size"] = mn, mx
    k.blocks.append((row, np.zeros(0, dtype=abi.GPU_OPT)))


class Case:
    """One input: full tables, the enabled mask, an address rank, and named ask / worker indices for its guard."""

    def __init__(self, t, on=None, rank=None, **named):
        self.t = t
        T = len(t["asks"])
        self.on = np.ones(T, bool) if on is None else on
        self.rank = np.random.default_rng(T).permutation(len(t["wa"])).astype(np.uint32) if rank is None else rank
        self.named = named

    def __getattr__(self, k):
        try:
            return self.__dict__["named"][k]
        except KeyError:
            raise AttributeError(k) from None


# ------------------------------------------------------------------------------------------------ 1. many_configs
PLANTED = {511: (5, 5), 512: (3, 3), 1023: (4, 4), 1024: (3, 3), 2047: (3, 3), 2048: (3, 3)}


@functools.lru_cache(maxsize=None)
def many_configs():
    """5000 mixed asks over 60 000 synth workers (118 CTAs), plus gpu:count=3 asks at 511/512, 1023/1024 and
    2047/2048 that seven located count-3 workers reach in turn.  At 511, (5, 5): the seed (Montreal) takes the four
    other Montreal workers, so the two far ones — not the last two by index — are handed on, across every chunk
    boundary of 512 and 1024, and the last ask hands them to nobody."""
    w = synth.make_workers(60_000, seed=synth.SEED_WORKERS + 201)
    a = synth.make_asks(5000 - len(PLANTED), "mixed", seed=synth.SEED_ASKS + 201, group_sizes=SIZES)
    k = Asks(w.model_strings)
    prev = 0
    for i, idx in enumerate(sorted(PLANTED)):
        k.synth_block(a, prev, idx - i)
        k.add("gpu:count=3", *PLANTED[idx])
        prev = idx - i
    k.synth_block(a, prev)
    pop = Pop()
    pop.synth(w)
    threes = pop.crafted([0, 1, 0, 0, 5, 0, 0], 3)
    return Case(pop.tables(k), threes=threes)


# ------------------------------------------------------------------------------------------------ 2. empty_runs
NOBODY = "gpu:count=1000"


@functools.lru_cache(maxsize=None)
def empty_runs():
    """Runs of configurations nobody reaches between the ones that have members, over 3000 synth workers (6 CTAs):
    [0, 1024) ends exactly on a chunk boundary of both kernels; [1025, 1725) is longer than one grid chunk and shorter
    than two; [1726, 3226) longer than one single-CTA chunk.  Disabled (0, 0) asks stand inside the runs (enabled they
    would make proximity refuse); an unreached (0, 2) ask inside the last run still emits its empty group.  The
    reached asks hand tails across the runs; a solo ask takes the synth workers at the end."""
    k = Asks(CATALOGUE)
    off, named = [], {}

    def run(n, disabled=(), min0=()):
        for i in range(n):
            if i in disabled:
                off.append(len(k))
                k.add("gpu:count=3", 0, 0)
            elif i in min0:
                named.setdefault("min0", []).append(len(k))
                k.add(NOBODY, 0, 2)
            else:
                k.add(NOBODY, 1 + i % 3, 1 + i % 3 + i % 5)

    def reached(name, req, mn, mx):
        named[name] = len(k)
        add(k, req, mn, mx)

    run(1024, disabled=(300, 700))
    reached("r1", "gpu:count=3", 3, 3)                 # 10 count-3 workers: three groups, one handed on
    run(700, disabled=(200,))
    reached("r2", "gpu:count=3;gpu:count=5", 2, 2)     # 9 count-5 workers and the handed-on one: five pairs
    run(1500, disabled=(100, 1300))
    reached("r3", "gpu:count=6", 2, 3)
    run(600, disabled=(50, 450), min0=(300,))
    reached("r4", "gpu:count=7", 4, 4)                 # 9: two groups, one handed to the solo ask
    reached("solo", None, 1, 1)
    pop = Pop()
    pop.synth(synth.make_workers(3000, seed=synth.SEED_WORKERS + 202))
    pop.crafted(spread(10, 1), 3)
    pop.crafted(spread(9, 2, located=0.7), 5)
    pop.crafted([7] * 5 + [9] * 3, 6)
    pop.crafted(spread(9, 4), 7)
    t = pop.tables(k)
    on = np.ones(len(k), bool)
    on[off] = False
    return Case(t, on, disabled=np.array(off), **named)


# ------------------------------------------------------------------------------------------------ 3. handdown_sizes
HANDDOWNS = {127: (5, 100, (2, 4)), 128: (6, 101, (3, 3)), 129: (7, 100, (17, 17)), 2000: (9, 300, (33, 33))}


@functools.lru_cache(maxsize=None)
def handdown_sizes():
    """For h in 127, 128, 129, 2000: ask A_h = (h + 3, h + 3) over 2h + 3 located 80 GB workers of one gpu count forms
    one proximity group (its seed and the h + 2 nearest) and hands exactly h on to B_h, whose own base segment is the
    24 GB workers of that count, interleaved with A_h's by index.  B_h: groups of 4 and 3 (seed-parallel batches on a
    merged list), 17 and 33 (several selection passes).  A_2000's group has 2003 members (more than 512 neighbours) and
    B_2000 receives 2000: an ordered compaction on the grid, a bitonic sort with P = 2048 on the single CTA."""
    k = Asks(CATALOGUE)
    pop = Pop()
    named = {}
    for h, (count, n24, size) in HANDDOWNS.items():
        m = h + 3
        named[f"a{h}"] = len(k)
        k.add(f"gpu:count={count};gpu:memory_mb_min=50000", m, m)
        named[f"b{h}"] = len(k)
        k.add(f"gpu:count={count}", *size)
        mem = mixed_mem(m + h, n24)
        where = spread(len(mem), count, located=0.95 if h == 2000 else 1.0)
        where[(mem == 24000) & (np.arange(len(mem)) % 10 == 3)] = -1            # some of B's own without location
        named[f"w{h}"] = pop.crafted(where, count, mem=mem)
    named["tail"] = len(k)
    add(k, None, 1, 1)
    return Case(pop.tables(k), **named)


# ------------------------------------------------------------------------------------------------ 4. cascade
@functools.lru_cache(maxsize=None)
def cascade():
    """A chain of 2200 gpu:count=5 asks at every other index from 1 to about 4400, between mixed asks, over 20 000
    synth workers (40 CTAs) and 124 located count-5 workers.  The first link (64, 64) forms one proximity group and
    hands 60 on; link 300, (50, 50), forms one from the handed-down list and hands 10 on; link 700, (3, 3), forms three
    (a batch) and hands one on; the last link is (1, 8).  Every other link is (61, 61): its base segment is empty and
    all it receives moves on, across four chunk boundaries of 512 and two of 1024.  Among the links: disabled (0, 0)
    count-5 asks (the chain skips them) and (0, 3) asks nobody reaches (an empty group each)."""
    w = synth.make_workers(20_000, seed=synth.SEED_WORKERS + 204)
    a = synth.make_asks(2200, "mixed", seed=synth.SEED_ASKS + 204, group_sizes=SIZES)
    k = Asks(w.model_strings)
    off, links = [], []
    for i in range(2200):
        k.synth_block(a, i, i + 1)
        links.append(len(k))
        k.add("gpu:count=5", *{0: (64, 64), 300: (50, 50), 700: (3, 3), 2199: (1, 8)}.get(i, (61, 61)))
        if i % 97 == 5:
            off.append(len(k))
            k.add("gpu:count=5", 0, 0)
        if i % 101 == 7:
            k.add("gpu:count=6", 0, 3)
    pop = Pop()
    pop.synth(w, 0, 9000)
    fives = pop.crafted(spread(124, 204), 5)
    pop.synth(w, 9000)
    on = np.ones(len(k), bool)
    on[off] = False
    return Case(pop.tables(k), on, links=np.array(links), disabled=np.array(off), fives=fives)


# ------------------------------------------------------------------------------------------------ 5. batches
def _trap_points():
    """The synth cities, then for six of them a place 1 km north written beyond ±90 (R·|Δlatitude| > 4000 km)."""
    hubs = [c for c in range(64) if abs(synth.CITIES[c, 0]) < 70][:6]
    traps = [beyond_90(synth.CITIES[c, 0] + 1.0 / KM_PER_DEG, synth.CITIES[c, 1]) for c in hubs]
    return np.concatenate([synth.CITIES, np.array(traps)]), hubs


BATCH_SCALES = {"one_cta": 380, "two_ctas": 900, "wide": 60_000}


@functools.lru_cache(maxsize=None)
def batches(scale):
    """Groups of 2, 3 and 4 with synth workers around them up to W (1, 2 or 118 CTAs):
    * pairs over co-located clusters of 6 and 5 (a batch's later seed is an earlier seed's neighbour; lists of four
      distances of 0 run out of spares);
    * trios with three located candidates and five without (no pruning: f64::MAX neighbours);
    * quads with one located candidate and 30 without (the batch has fewer located seeds than its width);
    * a (2, 3) ask over five (remaining / max < 2: no batch at all);
    * six consecutive pair asks, the odd ones holding a seed's 1 km neighbour written beyond ±90 (the "latitude beyond
      90" flag slots alternate);
    * on the wide scale, 8-GPU synth workers in pairs (hundreds of batches) before a solo ask for the rest."""
    pts, hubs = _trap_points()
    W = BATCH_SCALES[scale]
    k = Asks(CATALOGUE)
    pop = Pop(pts)
    named = {}

    def ask(name, req, mn, mx):
        named[name] = len(k)
        add(k, req, mn, mx)

    ask("pairs", "gpu:count=3", 2, 2)
    named["w_pairs"] = pop.crafted([11] * 6 + [3, 40] + [12] * 5 + spread(9, 51).tolist(), 3)
    ask("trios", "gpu:count=5", 3, 3)
    named["w_trios"] = pop.crafted([-1, 4, -1, -1, 20, -1, 33, -1], 5)
    ask("quads", "gpu:count=6", 4, 4)
    named["w_quads"] = pop.crafted([-1] * 7 + [17] + [-1] * 23, 6)
    ask("short", "gpu:count=7", 2, 3)
    named["w_short"] = pop.crafted([2, 8, 2, 30, -1], 7)
    named["alt"] = []
    for j in range(6):
        named["alt"].append(len(k))
        k.add(f"gpu:count={9 + j}", 2, 2)
        hub = hubs[j]
        where = [hub, 64 + j if j % 2 else 21, 21, 45, 50, 21, -1, 45]     # odd: the hub's neighbour is the trap
        pop.crafted(where, 9 + j)
    if scale == "wide":
        ask("eights", "gpu:count=8", 2, 2)
    ask("solo", None, 1, 1)
    w = synth.make_workers(W - pop.n, seed=synth.SEED_WORKERS + 205)
    pop.synth(w)
    return Case(pop.tables(k), **named)


# ------------------------------------------------------------------------------------------------ 6. big_groups
@functools.lru_cache(maxsize=None)
def big_groups():
    """Selection in chunks of 16 past one CTA (17 CTAs):
    * (17, 17), (18, 18), (32, 32), (33, 33) over 512 m + r candidates, r < 16 (the last CTA runs out of live
      candidates inside a chunk), 60 % located: later groups have a located seed and are filled with f64::MAX
      candidates by list position across CTAs;
    * (550, 600) over 2360 with 100 located: a located group of 600, two full unlocated groups by the ordered
      partition (they straddle CTA chunks) and an unlocated group of 560 taken in list order (past one chunk of 512);
    * (1, 1) and (0, 1) asks receiving 200 and 150 hand-downs (compaction) in lists of 1100 and 650 that mix located
      and unlocated workers over several CTA chunks."""
    k = Asks(CATALOGUE)
    pop = Pop()
    named = {}
    for count, (mn, mx), K in ((3, (17, 17), 1024 + 5), (5, (18, 18), 512 + 7), (6, (32, 32), 1536 + 3),
                               (7, (33, 33), 1024 + 15)):
        named[f"g{mx}"] = len(k)
        k.add(f"gpu:count={count}", mn, mx)
        pop.crafted(spread(K, 300 + count, located=0.6), count)
    named["g600"] = len(k)
    k.add("gpu:count=9", 550, 600)
    where = np.full(2360, -1)
    where[np.random.default_rng(309).choice(2360, 100, replace=False)] = spread(100, 310)
    pop.crafted(where, 9)
    for count, n80, n24, (mn, mx) in ((11, 200, 900, (1, 1)), (12, 150, 500, (0, 1))):
        named[f"x{count}"] = len(k)
        k.add(f"gpu:count={count};gpu:memory_mb_min=50000", 300, 300)
        named[f"y{count}"] = len(k)
        k.add(f"gpu:count={count}", mn, mx)
        pop.crafted(spread(n80 + n24, 320 + count, located=0.5), count, mem=mixed_mem(n80, n24))
    return Case(pop.tables(k), **named)


CASES = {"many_configs": many_configs, "empty_runs": empty_runs, "handdown_sizes": handdown_sizes, "cascade": cascade,
         "batches_one_cta": functools.partial(batches, "one_cta"), "batches_two_ctas": functools.partial(batches, "two_ctas"),
         "batches_wide": functools.partial(batches, "wide"), "big_groups": big_groups}


# ------------------------------------------------------------------------------------------------ evidence
def enabled_tables(case):
    return dict(case.t, asks=case.t["asks"][case.on])


class Evidence:
    """The checker's groups for a case (on the enabled asks, indices mapped back to the full table) and what they
    imply: per configuration K (list length), xc (hand-downs received), located (located members of the list)."""

    def __init__(self, case):
        t, sub = case.t, enabled_tables(case)
        self.case, self.T, self.W = case, len(t["asks"]), len(t["wa"])
        assert_distance_certificate(t["lat"], t["lon"], (t["wa"]["flags"] & LOC) != 0)
        self.og = orc.soa_form_groups(sub["wa"], sub["wb"], sub["asks"], sub["opts"], sub["bits"], sub["words"],
                                      addr_rank=case.rank, lat=sub["lat"], lon=sub["lon"], proximity="banded")
        tr = sweep_trace(sub, self.og)
        up = np.flatnonzero(case.on)
        self.up = up
        full = lambda x: np.bincount(up, weights=x, minlength=self.T).astype(np.int64)
        self.K, self.base, self.pop = full(tr["K"]), full(tr["base"]), full(tr["pop"])
        self.src = up[tr["src"]]
        self.dst = np.where(tr["dst"] == NONE, NONE, up[np.minimum(tr["dst"], len(up) - 1)])
        self.who = tr["who"]
        self.xc = np.bincount(self.dst[self.dst != NONE], minlength=self.T)
        ff = orc.soa_first_feasible(sub["wa"], sub["wb"], sub["asks"], sub["opts"], sub["bits"], sub["words"])
        self.first = np.where(ff == NONE, NONE, up[np.minimum(ff, len(up) - 1)]).astype(np.int64)
        self.loc = (t["wa"]["flags"] & LOC) != 0
        self.located = np.bincount(self.first[(self.first != NONE) & self.loc], minlength=self.T)[:self.T] + \
            np.bincount(self.dst[(self.dst != NONE) & self.loc[self.who]], minlength=self.T)[:self.T]
        self.cfg = up[self.og.cfg]
        self.sizes = np.diff(self.og.off)
        self.n_bumped = int(self.pop.sum())

    def members(self, g):
        return self.og.members[self.og.off[g]:self.og.off[g + 1]]

    def groups_of(self, c):
        return np.flatnonzero(self.cfg == c)

    def handed(self, frm, to):
        return np.sort(self.who[(self.src == frm) & (self.dst == to)])

    def received(self, c):
        return np.sort(self.who[self.dst == c])

    def candidates(self, c):
        """The list the kernels build for c: its base segment merged with what it receives, in index order."""
        return np.union1d(np.flatnonzero(self.first == c), self.received(c))

    def grouped_non_solo(self):
        """Non-empty groups of configurations with max >= 2: the groups the grid kernel forms in batches or one at a
        time (pm_stats n_rounds + n_build_launches)."""
        mx = self.case.t["asks"]["max_group_size"][self.cfg]
        return int(((self.sizes > 0) & (mx >= 2)).sum())

    def batches_must_run(self):
        """Configurations where the grid must open a seed-parallel batch: groups of 2..4, at least two CTAs, room for
        two full groups and a located candidate to seed them."""
        mx = self.case.t["asks"]["max_group_size"].astype(np.int64)
        return np.flatnonzero((mx >= 2) & (mx <= 4) & (self.K // np.maximum(mx, 1) >= 2) & (self.located >= 1)) \
            if n_ctas(self.W) >= 2 else np.zeros(0, np.int64)


@functools.lru_cache(maxsize=None)
def evidence(name):
    return Evidence(CASES[name]())


def _crossings(ev, stride):
    moved = ev.dst != NONE
    return int(((ev.src[moved] // stride) != (ev.dst[moved] // stride)).sum())


def _amin(ev):
    return ev.case.t["asks"]["min_group_size"].astype(np.int64)


def _amax(ev):
    return ev.case.t["asks"]["max_group_size"].astype(np.int64)


def _straddles(ev, g):
    """A group whose members' list positions lie in more than one CTA chunk of 512."""
    pos = np.searchsorted(ev.candidates(ev.cfg[g]), ev.members(g))
    return (pos // GRID).min() != (pos // GRID).max()


# ------------------------------------------------------------------------------------------------ guards
def guard(name):
    """The evidence each input exists for, with numbers; returns the Evidence."""
    ev = evidence(name)
    c = ev.case
    mn, mx = _amin(ev), _amax(ev)
    if name == "many_configs":
        assert ev.T == 5000 and 100 * GRID < ev.W <= MAX_GRID_W and n_ctas(ev.W) == 118
        chain = sorted(PLANTED)
        for frm, to in zip(chain, chain[1:]):
            assert ev.handed(frm, to).tolist() == [c.threes[1], c.threes[4]], f"{frm} -> {to}"
        assert len(ev.handed(2048, NONE)) == 2
        assert ev.handed(511, 512).tolist() != c.threes[-2:].tolist()      # proximity chose, not list order
        assert _crossings(ev, GRID) >= 5 and _crossings(ev, SINGLE) >= 3
        bad = np.flatnonzero(ev.pop)
        assert len(bad) > 500 and all(((bad // GRID) == j).any() for j in range(8))   # tails in every chunk up to 4096
    elif name == "empty_runs":
        reached = np.flatnonzero((ev.K > 0) | ((mn == 0) & c.on))
        assert reached.tolist() == sorted([c.r1, c.r2, c.r3, c.r4, c.solo] + c.min0)
        runs = np.diff(np.concatenate([[-1], reached])) - 1
        # runs of unreached asks before each reached one: [0, 1024) ends on a boundary of 512 and of 1024
        assert c.r1 == 2 * GRID == SINGLE and runs[0] == SINGLE
        assert GRID < runs[1] < 2 * GRID and runs[2] > SINGLE
        assert all(((c.disabled > lo) & (c.disabled < hi)).any()
                   for lo, hi in ((-1, c.r1), (c.r1, c.r2), (c.r2, c.r3), (c.r3, c.r4)))
        assert (mx[c.disabled] == 0).all() and (mn[c.disabled] == 0).all()
        assert ev.K[c.min0].sum() == 0 and all((ev.cfg == m).sum() == 1 and ev.sizes[ev.cfg == m][0] == 0 for m in c.min0)
        assert len(ev.handed(c.r1, c.r2)) == 1 and len(ev.handed(c.r4, c.solo)) == 1
    elif name == "handdown_sizes":
        assert n_ctas(ev.W) >= 2
        for h in HANDDOWNS:
            a, b = getattr(c, f"a{h}"), getattr(c, f"b{h}")
            assert ev.K[a] == 2 * h + 3 and ev.pop[a] == h and ev.xc[b] == h, f"A_{h} hands {ev.pop[a]}, B_{h} gets {ev.xc[b]}"
            assert ev.base[b] == HANDDOWNS[h][1] and len(ev.handed(a, b)) == h
            # the received and the base segment interleave in index order
            lst = ev.candidates(b)
            came = np.isin(lst, ev.received(b))
            assert int((came[1:] != came[:-1]).sum()) >= 40, f"B_{h}"
        assert ev.sizes[ev.groups_of(c.a2000)].tolist() == [2003] and ev.xc[c.b2000] > SINGLE
        assert (ev.sizes[ev.groups_of(c.b129)] == 17).sum() == 13 and (ev.sizes[ev.groups_of(c.b2000)] == 33).sum() >= 60
        assert {c.b127, c.b128} <= set(ev.batches_must_run().tolist())
        assert ev.xc[c.b127] < XS_SMEM <= ev.xc[c.b128] < ev.xc[c.b129]     # 127 / 128 sorted in shared memory, 129 compacted
    elif name == "cascade":
        links = c.links
        chain = links[(ev.K[links] > 0) & (ev.base[links] == 0) & (ev.pop[links] == ev.K[links])]
        assert len(chain) >= 2100 and chain.min() < GRID and chain.max() >= 4 * SINGLE
        assert (np.diff(links[ev.K[links] > 0]) <= 4).all()                   # every link is reached: one unbroken chain
        formed = links[(ev.K[links] > 0) & (ev.pop[links] < ev.K[links])]
        assert len(formed) == 4 and ev.K[formed].tolist() == [124, 60, 10, 1]
        assert (ev.base[formed[1:]] == 0).all()                                # proximity groups from handed-down lists
        assert (ev.xc[links[1:]] > 0).all()
        zero_min = np.flatnonzero((mn == 0) & (mx > 0))
        assert len(c.disabled) > 20 and len(zero_min) > 20
        assert (c.disabled > chain.min()).sum() > 20 and (zero_min < chain.max()).sum() > 20
        assert ev.K[c.disabled].sum() == 0 and (np.isin(ev.cfg, zero_min)).sum() == len(zero_min)
        assert _crossings(ev, GRID) >= 8 and _crossings(ev, SINGLE) >= 4
        assert ev.xc[links].max() == 60
    elif name.startswith("batches"):
        W = ev.W
        ncta = n_ctas(W)
        assert {"batches_one_cta": ncta == 1, "batches_two_ctas": ncta == 2, "batches_wide": ncta == 118}[name]
        must = set(ev.batches_must_run().tolist())
        # co-located clusters of 5 and more among the pairs' candidates
        lst = ev.candidates(c.pairs)
        pts = np.stack([c.t["lat"][lst], c.t["lon"][lst]], 1)[ev.loc[lst]]
        _, counts = np.unique(pts, axis=0, return_counts=True)
        assert counts.max() >= 6 and (counts >= 5).sum() >= 2
        assert ev.located[c.trios] == 3 < 4 <= ev.K[c.trios] and ev.located[c.quads] == 1 and ev.K[c.quads] // 4 >= 2
        assert ev.K[c.short] // 3 < 2
        alt = np.array(c.alt)
        processed = np.flatnonzero((ev.K > 0) | (mn == 0))
        assert np.array_equal(processed[np.searchsorted(processed, alt[0]):][:6], alt)   # consecutive for the kernel
        beyond = [bool((np.abs(c.t["lat"][ev.candidates(a)]) > 90).any()) for a in alt]
        assert beyond == [False, True] * 3
        if ncta >= 2:
            assert {c.pairs, c.quads, *c.alt} <= must and c.short not in must
        else:
            assert not must
        if name == "batches_wide":
            assert ev.K[c.eights] > 5000
    elif name == "big_groups":
        assert n_ctas(ev.W) == 17
        for m in (17, 18, 32, 33):
            g = getattr(c, f"g{m}")
            K, L = ev.K[g], ev.located[g]
            assert K % GRID < TOPK and K > GRID and 0 < L < K and mx[g] == m
            mixed = [gi for gi in ev.groups_of(g) if 0 < ev.loc[ev.members(gi)].sum() < ev.sizes[gi]]
            assert mixed, f"no group of {m} with a located seed filled by f64::MAX candidates"
        g600 = ev.groups_of(c.g600)
        locs = [int(ev.loc[ev.members(gi)].sum()) for gi in g600]
        assert ev.sizes[g600].tolist() == [600, 600, 600, 560] and locs == [100, 0, 0, 0]
        assert _straddles(ev, g600[1]) and _straddles(ev, g600[2]) and ev.sizes[g600[3]] - 1 > GRID
        for x, y in ((c.x11, c.y11), (c.x12, c.y12)):
            assert ev.pop[x] == ev.K[x] and ev.xc[y] > XS_SMEM and ev.K[y] > 2 * GRID / 2
            lst = ev.candidates(y)
            assert 0 < ev.loc[lst].sum() < len(lst) and len(lst) > GRID
        assert ev.K[c.y11] > 2 * GRID and mx[c.y11] == 1 and mn[c.y12] == 0 and mx[c.y12] == 1
        assert (ev.cfg == c.y12).sum() == ev.K[c.y12] + 1                   # every member its own group, then the empty one
    return ev


@pytest.mark.parametrize("name", sorted(CASES))
def test_proximity_inputs_reach_their_paths(name):
    ev = guard(name)
    assert ev.n_bumped >= 0 and len(ev.og) > 0


def test_trace_counts_tails_under_proximity():
    """sweep_trace on proximity groups small enough to follow by hand: six located workers, (4, 4) then (2, 2).  The
    tail handed on is the two farthest from the seed, not the last two by index."""
    k = Asks(CATALOGUE)
    k.add("gpu:count=1", 4, 4)
    k.add("gpu:count=1", 2, 2)
    pop = Pop()
    pop.crafted([0, 1, 0, 0, 1, 0], 1)
    t = pop.tables(k)
    og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], lat=t["lat"], lon=t["lon"],
                             proximity=True)
    tr = sweep_trace(t, og)
    assert tr["K"].tolist() == [6, 2] and tr["pop"].tolist() == [2, 0]
    assert sorted(tr["who"].tolist()) == [1, 4]
    assert og.as_list() == [(0, [0, 2, 3, 5]), (1, [1, 4])]
