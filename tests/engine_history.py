"""Long random histories of one engine: every table call, every pass kind and the auction certificate, and a host
mirror that says what each call must do.

`History` extends the warm checker's `Market` (worker rows, caps, floors, reputation, resizes and the auction's change
set) with what the reference modes read (locations, address ranks, the ask table with its group sizes, the model table,
the enabled mask) and with the two change trackers of prime_match.h, restated from the header and DESIGN §4-§6b:

  reference tracker (PM_INCREMENTAL): a stored evaluation exists after every successful reference-mode pass; rows
      written since through pm_update_workers / pm_set_flags / pm_upsert_workers (each once) and rows a grow adds are
      dirty; a shrink drops the dirty rows it cuts off; asks enabled / disabled since count against the stored mask
      (off and on again counts as neither); the next incremental pass walks the dirty rows and the orphans of the asks
      disabled since, or everything when there is no stored evaluation or the count passes the PM_TUNE_INCR cutoff.
      pm_set_asks, pm_set_model_table, pm_set_worker_count and a reference-mode pass that fails discard it; a call
      refused on its mode bits and every auction-mode pass, refused or not, leave it as it is.
  auction tracker (PM_AUCTION_WARM): a stored state exists after every successful auction pass; Market tracks R0 and
      A0; pm_set_asks, pm_set_model_table, pm_set_worker_count and pm_set_auction_params discard it; a refused auction
      pass keeps it; reference-mode passes and certificates leave it alone.

`generate` draws the seeded histories the GPU suite runs (tests/test_gpu_engine_history.py) and the CPU suite audits
(tests/test_engine_history_inputs.py).  Events are plain data, so a failing history can be replayed and shortened
(`shrink`).
"""
from __future__ import annotations

import functools
import os

import numpy as np

import auction_warm_checker as wc
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth

NONE = abi.PM_NONE
INF = abi.PM_COST_INF
FF, PROX, AUC = abi.PM_MODE_FIRST_FIT, abi.PM_MODE_PROXIMITY, abi.PM_MODE_AUCTION
LEAN = abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS
INCR = LEAN | abi.PM_INCREMENTAL
WARM = AUC | abi.PM_AUCTION_WARM
MODES = {
    "materialized": FF | abi.PM_PATH_MATERIALIZED, "fused": FF | abi.PM_PATH_FUSED, "lean": FF | LEAN,
    "lean_incr": FF | INCR, "proximity": PROX | LEAN, "proximity_incr": PROX | INCR,
    "auction": AUC, "reverse": AUC | abi.PM_AUCTION_REVERSE, "warm": WARM, "repair": WARM | abi.PM_AUCTION_REPAIR,
    "auction_incr": AUC | INCR,   # always refused (PM_E_INVALID): the incremental flag is for the reference modes
}
REFERENCE = ("materialized", "fused", "lean", "lean_incr", "proximity", "proximity_incr")
INCREMENTAL = ("lean_incr", "proximity_incr")
AUCTION = ("auction", "reverse", "warm", "repair")
PASSES = REFERENCE + AUCTION + ("certificate",)
CALLS = ("update", "set_flags", "upsert", "grow", "shrink", "reputation", "caps", "floors", "ask_off", "ask_on",
         "locations", "addr_rank", "set_asks", "model_table", "auction_params", "set_workers")
RARE = ("set_asks", "model_table", "auction_params", "set_workers")
REFUSALS = ("auction_disabled", "auction_domain", "auction_incremental", "proximity_max0", "certificate_no_state",
            "certificate_resized", "certificate_disabled")
GROUPS = [(1, 1), (2, 3), (3, 5), (4, 4), (2, 8)]
PARAMS = [(1, 1, 4), (1, 64, 4), (3, 1, 4)]
# (P + K + 2) * 2 + E < 2^61 holds for every ordinary price and for 0x7FFFFFFF / 0x80000000, not for 0xFFFFFFFE up
DOMAIN_EDGE = (2, (1 << 61) - (1 << 32) - (1 << 21), 1024)
EDGE_PRICES = [0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF]
NARROW_LIMIT = 0x7FFFFFFF        # the 32-bit cost tile holds prices below it
SIGN = 1 << 31
SETTINGS = {"default": {}, "generic": {"PM_TUNE_GENERIC": 1}, "unpiped": {"PM_TUNE_PIPE": 0},
            "incr40": {"PM_TUNE_INCR": 40}, "auction128": {"PM_TUNE_AUCTION": 128}}
TILE_BYTES = {"unpiped": 1 << 20}     # several cost tiles
DEFAULT_CUTOFF = 1 << 18              # PM_TUNE_INCR's default
SHAPES = ("mixed", "wide")
BIG = os.environ.get("PM_TEST_BIG") == "1"
N_CALLS = 360 if BIG else 120


def cutoff_of(setting):
    return int(SETTINGS[setting].get("PM_TUNE_INCR", DEFAULT_CUTOFF))


N_SLOTS = len(SHAPES) * len(SETTINGS)


def slot_of(shape, setting):
    return SHAPES.index(shape) * len(SETTINGS) + list(SETTINGS).index(setting)


def seed_of(shape, setting, k=0):
    return 1000 * (SHAPES.index(shape) + 1) + 10 * list(SETTINGS).index(setting) + k


def workers_small(wa, wb):
    """The fast predicate's operand limits over every row (values < 2^31, gpu count < 2^16, count * memory < 2^31)."""
    f = wa["flags"]
    small = (wb["cpu_cores"] | wb["ram_mb"] | wb["storage_gb"]) < SIGN
    hc, hm = (f & abi.PM_W_HAS_GPU_COUNT) != 0, (f & abi.PM_W_HAS_GPU_MEM) != 0
    small &= ~hc | (wa["gpu_count"] < 65536)
    small &= ~hm | (wa["gpu_mem_mb"] < SIGN)
    small &= ~(hc & hm) | (wa["gpu_count"].astype(np.uint64) * wa["gpu_mem_mb"].astype(np.uint64) < SIGN)
    return bool(small.all())


def prices_narrow(wb):
    return bool((wb["ext_ask_price"] < NARROW_LIMIT).all())


def in_domain(wb, cap, params):
    S, E, _ = params
    P = int(wb["ext_ask_price"].max()) if len(wb) else 0
    K = int(np.asarray(cap).max()) if len(cap) else 0
    return (P + K + 2) * max(S, 1) + max(E, 1) < (1 << 61)


# ------------------------------------------------------------------------------------------------ the fixed tables
@functools.lru_cache(maxsize=4)
def setup(shape):
    """Two ask tables of one shape (the second a permutation of the first with other group sizes, the max 0 ask `z` at
    the same index), two model tables of one shape that differ in some acceptance bits, the first worker table with
    prices, reputation and locations from synth.CITIES, the caps and floors."""
    T, W = 240, 3000
    rng = np.random.default_rng(77 + SHAPES.index(shape))
    if shape == "mixed":
        w = synth.make_workers(W, with_addresses=False)
        a = synth.make_asks(T, "mixed", group_sizes=GROUPS)
        bits, npat, nmod, words = synth.intern_tables(w, a)
    else:
        from test_gpu_variants import wide_tables
        w, a, obits, bits, npat, nmod, words = wide_tables(T, W, 3000, 30, seed_shift=41)
        gs = np.asarray(GROUPS, dtype=np.uint32)[rng.integers(0, len(GROUPS), T)]
        a.asks["min_group_size"], a.asks["max_group_size"] = gs[:, 0], gs[:, 1]
    asks, opts = a.asks.copy(), a.opts
    # ask z has max_group_size 0: proximity mode refuses while it is enabled, the reference modes never fill it, and the
    # auction, which has no group sizes, fills it like any other; it keeps a requirement many workers meet
    F = wc.feasible(w.a, w.b, asks, opts, bits, words, np.full(T, 0xFFFFFFFF, dtype=np.uint32))
    z = T // 3 + int(np.argmax(F[T // 3:].sum(axis=1) > 50))
    asks[z]["min_group_size"] = asks[z]["max_group_size"] = 0
    perm = rng.permutation(T)
    perm[perm == z] = perm[z]
    perm[z] = z
    asks2 = asks[perm].copy()
    gs = np.asarray(GROUPS, dtype=np.uint32)[rng.integers(0, len(GROUPS), T)]
    asks2["min_group_size"], asks2["max_group_size"] = gs[:, 0], gs[:, 1]
    asks2[z]["min_group_size"] = asks2[z]["max_group_size"] = 0
    bits2 = np.array(bits, dtype=np.uint32).copy()
    for p in rng.choice(npat, min(npat, 4), replace=False):
        for m in rng.choice(nmod, max(1, nmod // 3), replace=False):
            bits2[p * words + (m >> 5)] ^= np.uint32(1 << (m & 31))
    wb = w.b.copy()
    wb["ext_ask_price"] = rng.integers(10, 1000, W).astype(np.uint32)
    lat, lon = synth.CITIES[rng.integers(0, len(synth.CITIES), W)].T.copy()
    return dict(T=T, W=W, z=z, asks=[asks, asks2], opts=opts, bits=[np.asarray(bits, dtype=np.uint32), bits2],
                npat=npat, nmod=nmod, words=words, wa=w.a.copy(), wb=wb, lat=lat, lon=lon,
                rank=rng.permutation(W).astype(np.uint32), cap=rng.integers(50, 1500, T).astype(np.uint32),
                rep=rng.integers(0, 4, W).astype(np.uint32), floors=rng.integers(0, 3, T).astype(np.uint32))


# ------------------------------------------------------------------------------------------------ the mirror
class History(wc.Market):
    def __init__(self, shape, cutoff=DEFAULT_CUTOFF):
        s = setup(shape)
        self.s, self.cutoff, self.z = s, cutoff, s["z"]
        t = dict(wa=s["wa"], wb=s["wb"], asks=s["asks"][0], opts=s["opts"], bits=s["bits"][0], words=s["words"])
        super().__init__(t, s["cap"], s["rep"], s["floors"])
        self.lat, self.lon, self.rank = s["lat"].copy(), s["lon"].copy(), s["rank"].copy()
        self.ask_table = self.bits_table = 0
        self.mask = np.ones(len(self.asks), dtype=bool)
        self.params = PARAMS[0]
        # reference tracker
        self.eval = False
        self.dirty, self.over = set(), False
        self.eval_mask, self.eval_ff = self.mask.copy(), None
        self.eval_facts = None              # (workers_small, prices_narrow) at the stored evaluation
        self.flipped = set()                # which of the two facts changed since the stored evaluation
        # auction tracker
        self.auc_state, self.auc_w, self.auc_over = False, 0, False
        self.auc_toggled = set()

    # ---- facts
    def facts(self):
        return workers_small(self.wa, self.wb), prices_narrow(self.wb)

    def _note_facts(self):
        if self.eval_facts is not None:
            now = self.facts()
            for name, a, b in zip(("fast", "narrow"), self.eval_facts, now):
                if a != b:
                    self.flipped.add(name)

    def first_feasible(self):
        up = np.flatnonzero(self.mask).astype(np.uint32)
        ff = orc.soa_first_feasible(self.wa, self.wb, self.asks[self.mask], self.opts, self.bits, self.words)
        return np.where(ff == NONE, NONE, up[np.minimum(ff, max(len(up) - 1, 0))] if len(up) else NONE).astype(np.uint32)

    # ---- the two trackers
    def _mark(self, rows):
        rows = {int(i) for i in rows if i < self.n_workers}
        if self.eval and not self.over:
            self.dirty |= rows
            self.over = len(self.dirty) > self.cutoff
        if self.auc_state:
            self.auc_over |= len(self.rows) > self.cutoff
        self._note_facts()

    def discard_eval(self):
        self.eval, self.dirty, self.over = False, set(), False
        self.eval_facts, self.flipped = None, set()

    def discard_auction(self):
        self.auc_state, self.auc_over, self.auc_toggled = False, False, set()
        self.store(None, None)

    def incremental_plan(self):
        """(full, n_tiles, enabled since, disabled since, count certain) of the next incremental pass."""
        W, T = self.n_workers, len(self.asks)
        if not self.eval or self.cutoff == 0 or T == 0 or W == 0:
            return True, W, set(), set(), True
        en = set(np.flatnonzero(self.mask & ~self.eval_mask).tolist())
        dis = set(np.flatnonzero(~self.mask & self.eval_mask).tolist())
        e_rows = -(-len(en) * W // T)
        full_now = len(self.dirty) + e_rows > self.cutoff
        full = self.over or full_now
        sure = self.over == (len(self.dirty) > self.cutoff)   # a shrink since the count passed the cutoff: unspecified
        if full:
            return True, W, en, dis, sure
        ff = self.eval_ff
        orphans = np.isin(ff, list(dis)) if dis else np.zeros(W, dtype=bool)
        orphans[list(self.dirty)] = False
        return False, len(self.dirty) + int(orphans.sum()), en, dis, sure

    def warm_plan(self):
        """(warm, certain) of the next PM_AUCTION_WARM pass."""
        if not self.auc_state:
            return False, True
        fits = self.n_changes() <= self.cutoff
        return (fits and not self.auc_over), self.auc_over == (len(self.rows) > self.cutoff)

    def changed_asks(self):
        d = (self.cap != self.cap0) | (self.floors_or_zero() != self.floors0)
        return sorted(set(np.flatnonzero(d).tolist()) | self.auc_toggled)

    # ---- predictions of refusals (the set of statuses the header allows)
    def refusal(self, kind):
        """(refusal name, statuses) or (None, None) for a pass or certificate that must run."""
        if kind == "auction_incr":
            return "auction_incremental", {abi.PM_E_INVALID}
        if kind == "proximity" or kind == "proximity_incr":
            if self.mask[self.z] and self.asks[self.z]["max_group_size"] == 0:
                return "proximity_max0", {abi.PM_E_UNSUPPORTED}
            return None, None
        if kind in AUCTION:
            st, why = set(), None
            if not self.mask.all():
                st.add(abi.PM_E_UNSUPPORTED)
                why = "auction_disabled"
            if not in_domain(self.wb, self.cap, self.params):
                st.add(abi.PM_E_INVALID)
                why = why or "auction_domain"
            return (why, st) if st else (None, None)
        if kind == "certificate":
            st, why = set(), None
            if not self.auc_state:
                st.add(abi.PM_E_STATE)
                why = "certificate_no_state"
            elif self.n_workers != self.auc_w:
                st.add(abi.PM_E_STATE)
                why = "certificate_resized"
            if not self.mask.all():
                st.add(abi.PM_E_UNSUPPORTED)
                why = why or "certificate_disabled"
            if not in_domain(self.wb, self.cap, self.params):
                st.add(abi.PM_E_INVALID)
                why = why or "certificate_domain"
            return (why, st) if st else (None, None)
        return None, None

    # ---- outcomes of passes
    def reference_done(self, ok):
        if not ok:
            self.discard_eval()
            return
        self.eval, self.dirty, self.over = True, set(), False
        self.eval_mask = self.mask.copy()
        self.eval_ff = self.first_feasible()
        self.eval_facts, self.flipped = self.facts(), set()

    def auction_done(self, price, assigned):
        self.store(price, assigned)
        self.auc_state, self.auc_w, self.auc_over, self.auc_toggled = True, self.n_workers, False, set()

    # ---- table calls (the mirror's side)
    def apply(self, ev):
        name, x = ev[0], ev[1]
        W = self.n_workers
        if name == "update":
            idx = x["idx"]
            self.wa[idx], self.wb[idx] = x["a"], x["b"]
            if x["lat"] is not None:
                self.lat[idx], self.lon[idx] = x["lat"], x["lon"]
            self.rows |= {int(i) for i in idx if i < self.n_kept}
            self._mark(idx)
        elif name == "set_flags":
            idx = x["idx"]
            ok = idx < W
            self.wa["flags"][idx[ok]] = x["flags"][ok]
            self.rows |= {int(i) for i in idx[ok] if i < self.n_kept}
            self._mark(idx[ok])
        elif name == "upsert":
            f, n = x["first"], len(x["a"])
            self.wa[f:f + n], self.wb[f:f + n] = x["a"], x["b"]
            self.rows |= {i for i in range(f, f + n) if i < self.n_kept}
            self._mark(range(f, f + n))
        elif name == "grow":
            n = W + len(x["a"])
            self.resize(n, x["a"], x["b"])
            self.lat, self.lon, self.rank = x["lat"].copy(), x["lon"].copy(), x["rank"].copy()
            if self.eval_ff is not None:     # rows past the old end hold no stored first ask
                self.eval_ff = np.concatenate([self.eval_ff, np.full(n - W, NONE, dtype=np.uint32)])
            self._mark(range(W, n))
        elif name == "shrink":
            self.resize(x["n"])
            self.lat, self.lon, self.rank = self.lat[:x["n"]].copy(), self.lon[:x["n"]].copy(), x["rank"].copy()
            self.dirty = {r for r in self.dirty if r < x["n"]}
            if self.eval_ff is not None:
                self.eval_ff = self.eval_ff[:x["n"]].copy()
            self._note_facts()
        elif name == "reputation":
            self.set_reputation(x["first"], x["values"])
            if self.auc_state:
                self.auc_over |= len(self.rows) > self.cutoff
        elif name == "caps":
            self.set_caps(x["cap"])
        elif name == "floors":
            self.set_floors(x["floors"])
        elif name in ("ask_off", "ask_on"):
            on = name == "ask_on"
            changed = [int(t) for t in x["idx"] if self.mask[t] != on]
            self.mask[x["idx"]] = on
            if self.auc_state:
                self.auc_toggled |= set(changed)
        elif name == "locations":
            self.lat, self.lon = x["lat"].copy(), x["lon"].copy()
        elif name == "addr_rank":
            self.rank = x["rank"].copy()
        elif name == "set_asks":
            self.ask_table = x["table"]
            self.asks = self.s["asks"][x["table"]]
            self.mask = np.ones(len(self.asks), dtype=bool)
            self.discard_eval()
            self.discard_auction()
        elif name == "model_table":
            self.bits_table = x["table"]
            self.bits = self.s["bits"][x["table"]]
            self.discard_eval()
            self.discard_auction()
        elif name == "auction_params":
            self.params = x["params"]
            self.discard_auction()
        elif name == "set_workers":
            self.wa, self.wb = x["a"].copy(), x["b"].copy()
            self.lat, self.lon, self.rank = x["lat"].copy(), x["lon"].copy(), x["rank"].copy()
            self.reputation = x["rep"].copy()
            self.discard_eval()
            self.discard_auction()
        else:
            raise ValueError(name)


# ------------------------------------------------------------------------------------------------ the engine's side
def drive(eng, ev):
    """Apply one table call to an engine."""
    name, x = ev[0], ev[1]
    if name == "update":
        eng.update_workers(x["idx"], x["a"], x["b"], x["lat"], x["lon"])
    elif name == "set_flags":
        eng.set_flags(x["idx"], x["flags"])
    elif name == "upsert":
        eng.upsert_workers(np.ascontiguousarray(x["a"]), np.ascontiguousarray(x["b"]), x["first"])
    elif name == "grow":
        W = eng.n_workers
        eng.resize_workers(W + len(x["a"]))
        eng.upsert_workers(np.ascontiguousarray(x["a"]), np.ascontiguousarray(x["b"]), W)
        eng.set_locations(x["lat"], x["lon"])
        eng.set_addr_rank(x["rank"])
    elif name == "shrink":
        eng.resize_workers(x["n"])
        eng.set_addr_rank(x["rank"])
    elif name == "reputation":
        eng.set_worker_reputation(x["values"], x["first"])
    elif name == "caps":
        eng.set_price_caps(x["cap"])
    elif name == "floors":
        eng.set_min_reputation(x["floors"])
    elif name in ("ask_off", "ask_on"):
        eng.set_ask_enabled(x["idx"], name == "ask_on")
    elif name == "locations":
        eng.set_locations(x["lat"], x["lon"])
    elif name == "addr_rank":
        eng.set_addr_rank(x["rank"])
    elif name == "set_asks":
        s = x["setup"]
        eng.set_asks(s["asks"][x["table"]], s["opts"])
        eng.set_price_caps(x["cap"])
        eng.set_min_reputation(x["floors"])
    elif name == "model_table":
        s = x["setup"]
        eng.set_model_table(s["bits"][x["table"]], s["npat"], s["nmod"], s["words"])
    elif name == "auction_params":
        S, E, d = x["params"]
        eng.set_auction_params(cost_scale=S, eps_start=E, eps_div=d)
    elif name == "set_workers":
        eng.set_workers(x["a"], x["b"])
        eng.set_locations(x["lat"], x["lon"])
        eng.set_addr_rank(x["rank"])
        eng.set_worker_reputation(x["rep"])
    else:
        raise ValueError(name)


def load(eng, h: History):
    """Load an engine with the mirror's current tables (a fresh engine's start, or the start of a history)."""
    s = h.s
    eng.set_asks(s["asks"][h.ask_table], s["opts"])
    eng.set_model_table(s["bits"][h.bits_table], s["npat"], s["nmod"], s["words"])
    eng.set_workers(h.wa, h.wb)
    eng.set_locations(h.lat, h.lon)
    eng.set_addr_rank(h.rank)
    eng.set_price_caps(h.cap)
    eng.set_worker_reputation(h.reputation)
    eng.set_min_reputation(h.floors_or_zero())
    S, E, d = h.params
    eng.set_auction_params(cost_scale=S, eps_start=E, eps_div=d)
    if not h.mask.all():
        eng.set_ask_enabled(np.flatnonzero(~h.mask), False)


# ------------------------------------------------------------------------------------------------ the generator
class Gen:
    """Draws table calls against a mirror (so that indices, held rows and edge rows follow the history)."""

    def __init__(self, h: History, rng):
        self.h, self.rng = h, rng
        s = h.s
        self.pool_a, self.pool_b = s["wa"], s["wb"]

    def rows(self, n):
        """n rows: copies of the first table's rows with flags flipped, other counts, models and prices, and sometimes
        an edge operand or an edge price."""
        rng, h = self.rng, self.h
        src = rng.integers(0, len(self.pool_a), n)
        a, b = self.pool_a[src].copy(), self.pool_b[src].copy()
        flip = rng.random(n)
        a["flags"][flip < 0.15] ^= abi.PM_W_ASSIGNED
        a["flags"][(flip >= 0.15) & (flip < 0.25)] ^= abi.PM_W_HEALTHY
        b["ext_ask_price"] = rng.integers(10, 1000, n)
        for i in np.flatnonzero(rng.random(n) < 0.12):
            k = int(rng.integers(0, 7))
            if k == 0:
                b["ram_mb"][i] = 0x80000000
            elif k == 1:
                b["cpu_cores"][i] = 0xFFFFFFFF
            elif k == 2:
                b["storage_gb"][i] = 0x90000000
            elif k == 3:
                a["gpu_mem_mb"][i] = 0xF0000000
                a["flags"][i] |= abi.PM_W_HAS_GPU_MEM
            elif k == 4:
                a["gpu_count"][i] = [0x10000, 0xFFFFFFFF][int(rng.integers(0, 2))]
                a["flags"][i] |= abi.PM_W_HAS_GPU_COUNT
            else:
                b["ext_ask_price"][i] = EDGE_PRICES[int(rng.integers(0, 2 if h.params == DOMAIN_EDGE else 4))]
        return a, b

    def edge_rows(self):
        h = self.h
        wa, wb = h.wa, h.wb
        f = wa["flags"]
        hc, hm = (f & abi.PM_W_HAS_GPU_COUNT) != 0, (f & abi.PM_W_HAS_GPU_MEM) != 0
        bad = ((wb["cpu_cores"] | wb["ram_mb"] | wb["storage_gb"]) >= SIGN) | (hc & (wa["gpu_count"] >= 65536)) \
            | (hm & (wa["gpu_mem_mb"] >= SIGN)) | (wb["ext_ask_price"] >= NARROW_LIMIT)
        return np.flatnonzero(bad)

    def pick(self, k):
        """k distinct rows: held rows, edge rows (to write them back) or any."""
        rng, h = self.rng, self.h
        W = h.n_workers
        r = rng.random()
        pool = np.arange(W)
        if r < 0.3 and h.assigned is not None:
            held = h.assigned[h.assigned != NONE]
            held = held[held < W]
            if len(held):
                pool = held
        elif r < 0.55:
            e = self.edge_rows()
            if len(e):
                pool = e
        return np.unique(rng.choice(pool, size=min(k, len(pool)), replace=False)).astype(np.uint32)

    def points(self, n):
        return synth.CITIES[self.rng.integers(0, len(synth.CITIES), n)].T.copy()

    def call(self, name):
        rng, h = self.rng, self.h
        W, T = h.n_workers, len(h.asks)
        s = h.s
        if name == "update":
            big = 0.35 if h.cutoff < 1000 else 0.1
            u = self.pick(int(rng.integers(40, 90) if rng.random() < big else rng.integers(1, 30)))
            a, b = self.rows(len(u))
            sel = np.arange(len(u))
            if rng.random() < 0.4:                       # duplicate indices carry the same row
                sel = np.concatenate([sel, rng.integers(0, len(u), max(1, len(u) // 2))])
            lat = lon = None
            if rng.random() < 0.5:
                lat, lon = self.points(len(u))
                lat, lon = lat[sel], lon[sel]
            return ("update", dict(idx=u[sel], a=a[sel], b=b[sel], lat=lat, lon=lon))
        if name == "set_flags":
            u = self.pick(int(rng.integers(1, 25)))
            f = h.wa["flags"][u] ^ np.where(rng.random(len(u)) < 0.5, abi.PM_W_ASSIGNED, abi.PM_W_HEALTHY).astype(np.uint32)
            rep = rng.integers(0, len(u), min(3, len(u)))  # repeats carry the same flags; one index past the table
            idx = np.concatenate([u, u[rep], [W + 3]]).astype(np.uint32)
            return ("set_flags", dict(idx=idx, flags=np.concatenate([f, f[rep], [abi.PM_W_HEALTHY]]).astype(np.uint32)))
        if name == "upsert":
            n = int(rng.integers(1, 30))
            a, b = self.rows(n)
            return ("upsert", dict(first=int(rng.integers(0, W - n)), a=a, b=b))
        if name == "grow":
            n = int(rng.integers(1, 60))
            a, b = self.rows(n)
            la, lo = self.points(n)
            return ("grow", dict(a=a, b=b, lat=np.concatenate([h.lat, la]), lon=np.concatenate([h.lon, lo]),
                                 rank=rng.permutation(W + n).astype(np.uint32)))
        if name == "shrink":
            n = W - int(rng.integers(1, 60))
            return ("shrink", dict(n=n, rank=rng.permutation(n).astype(np.uint32)))
        if name == "reputation":
            first = int(rng.integers(0, W - 1))
            return ("reputation", dict(first=first, values=rng.integers(0, 4, min(int(rng.integers(1, 25)), W - first))
                                       .astype(np.uint32)))
        if name == "caps":
            cap = h.cap.copy()
            i = rng.choice(T, int(rng.integers(1, 12)), replace=False)
            cap[i] = np.clip(cap[i].astype(np.int64) + rng.integers(-100, 100, len(i)), 0, 2000)
            return ("caps", dict(cap=cap))
        if name == "floors":
            fl = h.floors_or_zero().copy()
            i = rng.choice(T, int(rng.integers(1, 12)), replace=False)
            fl[i] = rng.integers(0, 3, len(i))
            return ("floors", dict(floors=fl.astype(np.uint32)))
        if name == "ask_off":
            on = np.flatnonzero(h.mask)
            i = rng.choice(on, min(len(on), int(rng.integers(1, 8))), replace=False)
            if rng.random() < 0.3 and h.mask[h.z]:
                i = np.union1d(i, [h.z])
            return ("ask_off", dict(idx=np.unique(i).astype(np.uint32)))
        if name == "ask_on":
            off = np.flatnonzero(~h.mask)
            if rng.random() < 0.6 or len(off) < 2:
                i = off
            else:
                i = rng.choice(off, int(rng.integers(1, len(off))), replace=False)
            return ("ask_on", dict(idx=np.unique(i).astype(np.uint32)))
        if name == "locations":
            lat, lon = h.lat.copy(), h.lon.copy()
            i = rng.choice(W, W // 10, replace=False)
            lat[i], lon[i] = self.points(len(i))
            return ("locations", dict(lat=lat, lon=lon))
        if name == "addr_rank":
            return ("addr_rank", dict(rank=rng.permutation(W).astype(np.uint32)))
        if name == "set_asks":
            return ("set_asks", dict(table=1 - h.ask_table, setup=s, cap=h.cap.copy(), floors=h.floors_or_zero().copy()))
        if name == "model_table":
            return ("model_table", dict(table=1 - h.bits_table, setup=s))
        if name == "auction_params":
            choices = [p for p in PARAMS if p != h.params]
            return ("auction_params", dict(params=choices[int(rng.integers(0, len(choices)))]))
        if name == "set_workers":
            n = int(rng.integers(W - 40, W + 40))
            a, b = self.rows(n)
            la, lo = self.points(n)
            return ("set_workers", dict(a=a, b=b, lat=la, lon=lo, rank=rng.permutation(n).astype(np.uint32),
                                        rep=rng.integers(0, 4, n).astype(np.uint32)))
        raise ValueError(name)


ALL_PAIRS = [(c, k) for c in CALLS for k in PASSES]


def generate(shape, seed, n_calls=N_CALLS, cutoff=DEFAULT_CUTOFF, slot=0, n_slots=1):
    """A seeded history: a list of events, ("call", (name, payload)) or ("pass", kind).  The mirror it returns has
    lived through the history with the trackers only (no auction state values).  History `slot` of `n_slots` also
    makes every n_slots-th (table call -> pass kind) pair from the slot on, so that the histories together make all."""
    rng = np.random.default_rng(seed)
    must = ALL_PAIRS[slot::n_slots]
    h = History(shape, cutoff)
    g = Gen(h, rng)
    events = []
    seen_call, seen_pass = set(), set()
    last_pass, calls_since = "start", []
    domain_at = n_calls // 2

    def emit_call(ev):
        events.append(("call", ev))
        h.apply(ev)
        calls_since.append(ev[0])

    def emit_pass(kind):
        nonlocal last_pass, calls_since
        events.append(("pass", kind))
        why, _ = h.refusal(kind)
        if kind in REFERENCE:
            h.reference_done(why is None)
        elif kind in AUCTION and why is None:   # the checkers' state: later writes can aim at the held rows
            a, p, _, _, _ = expect_auction(h, kind, h.warm_plan()[0] if kind in ("warm", "repair") else False)
            h.auction_done(p, a)
        if why is not None and not follow:   # what the refusal kept: the next incremental and warm passes show it
            follow.extend(["lean_incr", "warm"])
        if kind != "auction_incr":          # the refused flag combination is no pass of any kind
            for c in calls_since:
                seen_call.add((c, kind))
            seen_pass.add((last_pass, kind))
            last_pass = kind
            calls_since = []

    def mine(a, b):
        """An unseen (pass -> pass) pair this slot is to make."""
        return a in PASSES and (a, b) not in seen_pass and (PASSES.index(a) * len(PASSES) + PASSES.index(b)) % n_slots == slot

    follow = []
    emit_pass("lean_incr")
    while len(events) < n_calls:
        if len([e for e in events if e[0] == "pass"]) == domain_at // 2 and h.params != DOMAIN_EDGE:
            # a refusal outside the integer domain, reached through a written row, between passes on a stored state
            high = np.flatnonzero(h.wb["ext_ask_price"] >= 0xFFFFFFFE).astype(np.uint32)
            if len(high):                           # only the row written below leaves the domain
                a, b = h.wa[high].copy(), h.wb[high].copy()
                b["ext_ask_price"] = 500
                emit_call(("update", dict(idx=high, a=a, b=b, lat=None, lon=None)))
            emit_call(("auction_params", dict(params=DOMAIN_EDGE)))
            if not h.mask.all():
                emit_call(("ask_on", dict(idx=np.flatnonzero(~h.mask).astype(np.uint32))))
            emit_pass("auction")
            row = np.array([int(rng.integers(0, h.n_workers))], dtype=np.uint32)
            a, b = h.wa[row].copy(), h.wb[row].copy()
            old = (a.copy(), b.copy())
            b["ext_ask_price"] = 0xFFFFFFFF
            emit_call(("update", dict(idx=row, a=a, b=b, lat=None, lon=None)))
            emit_pass("warm")                       # refused: the stored state stays
            emit_pass("lean_incr")
            emit_pass("certificate")                # refused too
            emit_call(("update", dict(idx=row, a=old[0], b=old[1], lat=None, lon=None)))
            emit_pass("repair" if rng.random() < 0.5 else "warm")
            emit_call(("auction_params", dict(params=PARAMS[int(rng.integers(0, len(PARAMS)))])))
            continue
        n_passes = len([e for e in events if e[0] == "pass"])
        if n_passes == 12 and h.mask.all():
            # warm or repair after reference passes of both modes, with asks left disabled across them
            emit_pass("auction")
            emit_call(("ask_off", dict(idx=np.union1d(rng.choice(len(h.asks), 5, replace=False), [h.z]).astype(np.uint32))))
            emit_pass("lean")
            emit_pass("certificate")                # refused: disabled asks
            emit_call(g.call("update"))
            emit_pass("proximity_incr")
            emit_call(("ask_on", dict(idx=np.flatnonzero(~h.mask).astype(np.uint32))))
            emit_pass("repair" if slot % 2 else "warm")
            continue
        # aim at a (call -> pass) pair not seen yet in this history, preferring a pass that also makes a new
        # (pass -> pass) pair; otherwise a few random calls and any pass
        targets = [(c, k) for c in CALLS for k in PASSES if (c, k) not in seen_call]
        fresh = [t for t in targets if mine(last_pass, t[1])] or [t for t in targets if (last_pass, t[1]) not in seen_pass]
        targets = fresh or targets
        names = [c for c in CALLS if not (c == "shrink" and h.n_workers < 2000)]
        p = np.array([0.15 if c in RARE else 1.0 for c in names])
        for _ in range(int(rng.integers(0, 3))):
            emit_call(g.call(names[int(rng.choice(len(names), p=p / p.sum()))]))
        if n_passes == 20:
            # past the cutoff between two reference passes (a full pass under a small PM_TUNE_INCR), and a side column
            emit_pass("lean")
            u = np.unique(rng.choice(h.n_workers, min(h.cutoff + 20, 120), replace=False)).astype(np.uint32)
            a, b = g.rows(len(u))
            emit_call(("update", dict(idx=u, a=a, b=b, lat=None, lon=None)))
            emit_call(g.call("addr_rank"))
            emit_pass("lean_incr")
            continue
        if n_passes == 26:
            # past the cutoff between two auction passes (a cold PM_AUCTION_WARM pass under a small PM_TUNE_INCR)
            if not h.mask.all():
                emit_call(("ask_on", dict(idx=np.flatnonzero(~h.mask).astype(np.uint32))))
            emit_pass("auction")
            u = np.unique(rng.choice(h.n_workers, min(h.cutoff + 20, 120), replace=False)).astype(np.uint32)
            a, b = g.rows(len(u))
            emit_call(("update", dict(idx=u, a=a, b=b, lat=None, lon=None)))
            emit_pass("warm")
            continue
        if n_passes == 34:
            # an incremental pass with written rows after an auction pass and a certificate since its evaluation
            emit_pass("lean")
            emit_call(g.call("update"))
            if not h.mask.all():
                emit_call(("ask_on", dict(idx=np.flatnonzero(~h.mask).astype(np.uint32))))
            emit_pass("auction")
            emit_pass("certificate")
            emit_call(g.call("set_flags"))
            emit_pass("lean_incr")
            continue
        forced = bool(follow)
        if follow:
            kind = follow.pop(0)
        elif must and n_passes >= 2 and n_passes % 4:
            j = next((i for i, (_, k) in enumerate(must) if mine(last_pass, k)),
                     next((i for i, (_, k) in enumerate(must) if (last_pass, k) not in seen_pass), 0))
            c, kind = must.pop(j)
            emit_call(g.call(c))
        elif targets and rng.random() < 0.85:
            tw = np.array([0.5 if c in RARE else 1.0 for c, _ in targets])
            c, kind = targets[int(rng.choice(len(targets), p=tw / tw.sum()))]
            if c == "ask_on" and h.mask.all():
                emit_call(g.call("ask_off"))
            if c != "shrink" or h.n_workers >= 2000:
                emit_call(g.call(c))
        else:
            if not h.mask.all() and rng.random() < 0.5:
                emit_call(g.call("ask_on"))
            kinds = [k for k in PASSES if mine(last_pass, k)] or [k for k in PASSES if (last_pass, k) not in seen_pass] \
                or list(PASSES)
            kind = kinds[int(rng.integers(0, len(kinds)))]
        if rng.random() < 0.04:
            emit_pass("auction_incr")
        if kind in AUCTION or kind == "certificate":
            if not h.mask.all() and (forced or rng.random() < 0.75):
                emit_call(("ask_on", dict(idx=np.flatnonzero(~h.mask).astype(np.uint32))))
        elif kind.startswith("proximity"):
            if h.mask[h.z] and rng.random() < 0.75:
                emit_call(("ask_off", dict(idx=np.array([h.z], dtype=np.uint32))))
        emit_pass(kind)
    for c, kind in must:                    # the slot's pairs the loop had no room for
        emit_call(g.call(c))
        emit_pass(kind)
    for i in range(slot, len(PASSES) ** 2, n_slots):
        a, b = PASSES[i // len(PASSES)], PASSES[i % len(PASSES)]
        if (a, b) not in seen_pass:
            if last_pass != a:
                emit_pass(a)
            emit_pass(b)
    return events, h


# ------------------------------------------------------------------------------------------------ shortening
def shrink(events, fails, max_rounds=4):
    """Drop events while `fails(events)` stays true (delta debugging over chunks, then single events).  Calls that a
    later event's payload depends on (sizes) may make a shortened history invalid: `fails` should treat an exception
    other than the assertion it looks for as "does not fail"."""
    cur = list(events)
    for _ in range(max_rounds):
        changed = False
        n = max(1, len(cur) // 2)
        while n >= 1:
            i = 0
            while i < len(cur):
                trial = cur[:i] + cur[i + n:]
                if trial and fails(trial):
                    cur, changed = trial, True
                else:
                    i += n
            n //= 2
        if not changed:
            break
    return cur


# ------------------------------------------------------------------------------------------------ what a pass returns
def expect_reference(h: History, kind):
    """Every array pm_fetch_result returns for a reference pass on the mirror's tables: the oracle's groups on the
    enabled asks (indices mapped back to the full table) and, on paths with ask statistics, the oracle's row minima
    and counts (INF / 0 for disabled asks and on the lean paths); for first fit also n_bumped, the hand-downs the
    oracle's groups imply (test_resolution_sweep_inputs.sweep_trace)."""
    T, W = len(h.asks), h.n_workers
    prox = kind.startswith("proximity")
    og = orc.soa_form_groups(h.wa, h.wb, h.asks[h.mask], h.opts, h.bits, h.words, addr_rank=h.rank, lat=h.lat, lon=h.lon,
                             proximity="banded" if prox else False)
    up = np.flatnonzero(h.mask).astype(np.uint32)
    cfg = up[og.cfg].astype(np.uint32) if len(og.cfg) else np.zeros(0, dtype=np.uint32)
    wg = np.full(W, NONE, dtype=np.uint32)
    wk = np.full(W, NONE, dtype=np.uint32)
    for g in range(len(cfg)):
        m = og.members[og.off[g]:og.off[g + 1]]
        wg[m], wk[m] = g, cfg[g]
    out = dict(worker_group=wg, worker_ask=wk, group_ask=cfg, group_off=og.off, group_members=og.members,
               ask_best=np.full(T, INF, dtype=np.int64), ask_count=np.zeros(T, dtype=np.uint32))
    if not prox:   # first fit: every worker handed on from an under-filled tail is one n_bumped
        from test_resolution_sweep_inputs import sweep_trace

        t = dict(asks=h.asks[h.mask], opts=h.opts, wa=h.wa, wb=h.wb, bits=h.bits, words=h.words)
        out["n_bumped"] = int(sweep_trace(t, og)["pop"].sum())
    if kind in ("materialized", "fused"):
        ev = orc.soa_eval_matrix(h.wa, h.wb, h.asks, h.opts, h.bits, h.words, 0, T, 0, W, threads=8)
        out["ask_best"] = np.where(h.mask, ev["row_best"], INF).astype(np.int64)
        out["ask_count"] = np.where(h.mask, ev["row_count"], 0).astype(np.uint32)
    return out


def expect_auction(h: History, kind, warm):
    """(assignment, prices, forward rounds, released, (phases, reverse rounds, reverse bids)) of an auction pass: the
    oracle's cold pass, the reverse checker, the warm checker or the repair checker."""
    import auction_repair_checker as rp
    import auction_reverse_checker as rc

    S, E, d = h.params
    ap = h.wb["ext_ask_price"]
    if warm and kind == "warm":
        a, p, n, rel = h.warm(S)
        return a, p, n, len(rel), (0, 0, 0)
    if warm and kind == "repair":
        out = rp.market_repair(h, S)
        return out["assigned"], out["price"], out["fwd"], len(out["released"]), (1, out["rev"], out["bids"])
    if kind == "reverse":
        a, p, fwd, rev, bids, phases = rc.scaled(h.F(), ap, h.cap, S, E, d, reverse_rounds=True)
        return a, p, fwd, 0, (phases, rev, bids)
    a, p, n = orc.soa_auction(h.wa, h.wb, h.asks, h.opts, h.bits, h.words, h.cap, S, E, d, reputation=h.reputation,
                              min_reputation=h.floors_or_zero())
    return a, p, n, 0, (0, 0, 0)


def expect_certificate(h: History):
    import auction_certificate as ac

    return ac.market_certificate(h, h.params[0], h.price, h.assigned)
