"""Long random histories of one engine: every table call, every pass kind and the auction certificate, and a host
mirror that says what each call must do.

`History` extends the delta tests' `AskMarket` (worker rows, caps, floors, reputation, resizes, the ask rows as
pm_update_asks / pm_resize_asks change them and the auction's change set) with what the reference modes read
(locations, address ranks, the model table, the enabled mask) and with the two change trackers of prime_match.h,
restated from the header and DESIGN §4-§6b:

  reference tracker (PM_INCREMENTAL): a stored evaluation exists after every successful reference-mode pass; rows
      written since through pm_update_workers / pm_set_flags / pm_upsert_workers (each once) and rows a grow adds are
      dirty; a shrink drops the dirty rows it cuts off; asks enabled / disabled since count against the stored mask
      (off and on again counts as neither); a replaced ask is in E when enabled now and in D when enabled at the stored
      evaluation; appended asks were not enabled at it; an ask shrink cuts the mask and sets every stored first ask past
      the new end to NONE (those workers are no orphans).  pm_remove_asks / pm_insert_asks move every stored first ask
      with its row; a removed one lands on the next kept row, its heir, which is in D with the replaced bit whatever
      its own state (NONE with no kept row after it, as a shrink); inserted asks are appended ones.  The next
      incremental pass walks the dirty rows and the
      orphans of D, or everything when there is no stored evaluation or the dirty rows plus ceil(|E| W / T) pass the
      PM_TUNE_INCR cutoff.  pm_set_asks, pm_set_model_table, pm_set_worker_count and a reference-mode pass that fails
      discard it; a call refused on its mode bits and every auction-mode pass, refused or not, leave it as it is.
  auction tracker (PM_AUCTION_WARM): a stored state exists after every successful auction pass; AskMarket tracks R0,
      A0 (toggled, replaced and appended asks) and the removed asks that held a worker; any ask resize since marks it
      resized (the certificate waits for the next pass); pm_set_asks, pm_set_model_table, pm_set_worker_count and
      pm_set_auction_params discard it; a refused auction pass keeps it; reference-mode passes and certificates leave
      it alone.
  ask demands (pm_set_ask_demand, "Auction demands"): ask t with demand d[t] is d[t] slots, the rows of the twin table
      that repeats row t d[t] times; the stored assignment, A0 and the warm and repair checkers are over slots.
      pm_set_asks resets every demand to 1, pm_update_asks keeps a replaced row's demand (all its slots join A0), an
      append adds asks of demand 1 (empty slots in A0), a shrink drops the removed asks' demands and counts the held
      workers of their slots below n_kept in removed_held; pm_remove_asks does the same for the removed asks and moves
      the kept asks' slots with them, pm_insert_asks adds asks of demand 1 like an append.  A demand change under a stored state keeps each ask's first
      min(old, new) slots; over several changes before one pass the slots kept are the minimum over the chain
      (`dem_kept`); a removed slot's worker is unowned at its stored price and counts in removed_held when it lies below
      n_kept; the other slots are in A0.  The warm decision counts |R0| + (W - n_kept) + |A0 in slots| + removed_held.
      A demand change touches neither the reference tracker nor the fast / narrow facts; a refused one changes nothing.
  restore (pm_auction_assignment / pm_auction_restore, "Auction state restore"): the export is the stored assignment
      over the current asks and the stored pass's prices; a restore is refused while a demand exceeds 1 or an ask is
      disabled (PM_E_UNSUPPORTED), for a missing pattern (PM_E_STATE), for lengths other than W and T, a worker >= W, a
      price outside [0, (K + 1) S + max(E, 1)] or tables outside the integer domain (PM_E_INVALID), and changes nothing
      then; else the stored state is auction_restore_checker.audit of the given one, with no change since it (R0, A0,
      removed_held and the resize flag cleared, auc_w = W), warm 0, released 0 and reverse stats 0.  The reference
      tracker, pm_fetch_result and pm_table_version stay.

Ask rows referencing a model pattern the model table lacks make every pass, auction pass, certificate and cost tile
return PM_E_STATE while they are in the table, enabled or not.

`generate` draws the seeded histories the GPU suite runs (tests/test_gpu_engine_history.py) and the CPU suite audits
(tests/test_engine_history_inputs.py).  Events are plain data, so a failing history can be replayed and shortened
(`shrink`).
"""
from __future__ import annotations

import functools
import os

import numpy as np

import auction_demand as ad
import auction_restore_checker as rs
import auction_warm_checker as wc
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from test_ask_deltas_formulation import AskMarket, own_options

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
         "locations", "addr_rank", "set_asks", "model_table", "auction_params", "set_workers", "update_asks",
         "append_asks", "shrink_asks", "remove_asks", "insert_asks", "ask_delta_refused", "demand", "demand_refused",
         "restore", "restore_refused", "move")
RARE = ("set_asks", "model_table", "auction_params", "set_workers", "ask_delta_refused", "demand_refused",
        "restore_refused", "move")
ASK_DELTAS = ("update_asks", "append_asks", "shrink_asks", "remove_asks", "insert_asks")
# auction-only calls: no pm_multi_ form, and nothing a reference pass reads
AUCTION_CALLS = ("demand", "demand_refused", "restore", "restore_refused", "move")
REFUSALS = ("auction_disabled", "auction_domain", "auction_incremental", "proximity_max0", "certificate_no_state",
            "certificate_resized", "certificate_disabled", "certificate_asks_resized", "pattern_missing",
            "ask_delta_refused", "demand_refused", "restore_refused")
# the PM_E_INVALID cases of pm_update_asks / pm_resize_asks / pm_remove_asks / pm_insert_asks (each changes nothing,
# pm_table_version and n_asks included)
DELTA_REFUSALS = ("index", "sizes", "range", "grow_without_rows", "grow_bad_range", "too_many")
SPLICE_REFUSALS = ("remove_index", "remove_null", "insert_decreasing", "insert_past_end", "insert_sizes", "insert_range")
# the PM_E_INVALID cases of pm_set_ask_demand (each changes nothing, pm_table_version included)
DEMAND_REFUSALS = ("length", "zero", "total", "null")
# refused exports and restores: (case, statuses of the restore); "demand", "no_state" also try the export
RESTORE_REFUSALS = ("length_w", "length_t", "worker", "price_neg", "price_high", "demand", "disabled", "missing",
                    "domain", "export_demand", "export_no_state")
RESTORE_VARIANTS = ("own", "stale", "adversarial", "resized")
EDGE_ASKS = ("max0", "min0", "no_opts", "big_cpu", "none", "missing")
GROUPS = [(1, 1), (2, 3), (3, 5), (4, 4), (2, 8)]
PARAMS = [(1, 1, 4), (1, 64, 4), (3, 1, 4)]
# (P + K + 2) * 2 + E < 2^61 holds for every ordinary price and for 0x7FFFFFFF / 0x80000000, not for 0xFFFFFFFE up
DOMAIN_EDGE = (2, (1 << 61) - (1 << 32) - (1 << 21), 1024)
EDGE_PRICES = [0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF]
NARROW_LIMIT = 0x7FFFFFFF        # the 32-bit cost tile holds prices below it
SIGN = 1 << 31
SETTINGS = {"default": {}, "generic": {"PM_TUNE_GENERIC": 1}, "int64": {"PM_TUNE_BUILD": 8},
            "incr40": {"PM_TUNE_INCR": 40}, "auction128": {"PM_TUNE_AUCTION": 128}}
TILE_BYTES = {"int64": 1 << 20}       # several cost tiles
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


def option_rows(asks):
    """Per ask the option rows pm_ask_convert reads ([opt_off, opt_off + n_opts) when the ask has requirements)."""
    has = (asks["flags"] & abi.PM_A_HAS_REQ) != 0
    return [range(int(o), int(o) + int(k)) if h else range(0) for o, k, h in zip(asks["opt_off"], asks["n_opts"], has)]


def asks_small(asks, opts):
    """The fast predicate's operand limits over every ask row, enabled or not (pm_ask_convert's kAskNotSmall)."""
    f = asks["flags"]
    has = (f & abi.PM_A_HAS_REQ) != 0
    cpu = np.where(has & ((f & abi.PM_A_REQ_CPU) != 0) & ((f & abi.PM_A_REQ_CPU_CORES) != 0), asks["cpu_cores"], 0)
    ram = np.where(has & ((f & abi.PM_A_REQ_RAM) != 0), asks["ram_mb"], 0)
    sto = np.where(has & ((f & abi.PM_A_REQ_STORAGE) != 0), asks["storage_gb"], 0)
    if ((cpu | ram | sto) >= SIGN).any():
        return False
    rows = np.array(sorted({o for r in option_rows(asks) for o in r}), dtype=np.int64)
    if len(rows) == 0:
        return True
    q = opts[rows]
    p = q["present"]
    count = ((p & abi.PM_O_COUNT) != 0) & (q["count"] >= 65536)
    mem_lo = np.maximum(np.where((p & abi.PM_O_MEM) != 0, q["memory_mb"], 0),
                        np.where((p & abi.PM_O_MEM_MIN) != 0, q["memory_mb_min"], 0))
    mem_hi = np.where((p & abi.PM_O_MEM_MAX) != 0, q["memory_mb_max"], 0xFFFFFFFF)
    mem_lo = np.where(mem_lo > mem_hi, 0, mem_lo)
    tot_lo = np.where((p & abi.PM_O_TOT_MIN) != 0, q["total_memory_min"], 0)
    tot_hi = np.where((p & abi.PM_O_TOT_MAX) != 0, q["total_memory_max"], 0xFFFFFFFF)
    tot_lo = np.where(tot_lo > tot_hi, 0, tot_lo)
    return not (count | (mem_lo >= SIGN) | (tot_lo >= SIGN)).any()


def missing_pattern(asks, opts, n_patterns):
    """bool[T]: the ask has an option row whose model pattern the model table lacks.  pm_ask_convert stores
    pattern_id + 1 as a 32-bit pattern row and the engine refuses when the largest row exceeds n_patterns, so a
    pattern_id >= n_patterns is missing (0xFFFFFFFF included: its row would wrap to 0, "no model clause")."""
    q = opts["pattern_id"].astype(np.int64)
    miss = ((opts["present"] & abi.PM_O_MODEL) != 0) & (q >= n_patterns)
    return np.array([bool(miss[list(r)].any()) if len(r) else False for r in option_rows(asks)], dtype=bool)


def split_toggles(mask, eval_mask, replaced, heirs=()):
    """E and D of the next incremental pass: E = enabled now and (replaced or not enabled at the stored evaluation),
    D = enabled at the stored evaluation and (replaced or disabled now), and every heir (the next kept row of a removed
    ask, which holds its workers now) whatever its own state; the orphans of a replaced ask or a heir are walked from
    the ask itself."""
    rep = np.zeros(len(mask), dtype=bool)
    rep[sorted(replaced)] = True
    en = mask & (rep | ~eval_mask)
    dis = eval_mask & (rep | ~mask)
    return set(np.flatnonzero(en).tolist()), set(np.flatnonzero(dis).tolist()) | set(heirs)


def renamed(s, new):
    """A set of ask indices through an index map (new[t] < 0: removed)."""
    return {int(new[t]) for t in s if new[t] >= 0}


def walked_rows(stored, dirty, dis):
    """n_tiles of an incremental pass: the written rows and the orphans (workers whose stored first ask is in D) that
    are not among them."""
    orphans = np.isin(stored, sorted(dis)) if dis else np.zeros(len(stored), dtype=bool)
    orphans[sorted(dirty)] = False
    return len(dirty) + int(orphans.sum())


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
    # the option table both ask tables index, with two option rows past it whose model patterns the model tables lack:
    # the first pattern past the table, and 0xFFFFFFFF (whose 32-bit pattern row pattern_id + 1 wraps to 0)
    miss = np.zeros(2, dtype=abi.GPU_OPT)
    miss["present"] = abi.PM_O_MODEL
    miss["pattern_id"] = [npat, 0xFFFFFFFF]
    opts = np.concatenate([np.ascontiguousarray(opts), miss])
    # rows a delta sends besides the two tables' rows: a max_group_size 0 ask and a min_group_size 0 ask (copies of z,
    # which many workers meet), a row without option rows, a cpu_cores threshold >= 2^31 (the generic predicate), a
    # row no worker meets, and the two rows with a missing pattern
    edge = np.repeat(asks[z:z + 1], len(EDGE_ASKS) + 1).copy()
    edge[0]["min_group_size"], edge[0]["max_group_size"] = 0, 0
    edge[1]["min_group_size"], edge[1]["max_group_size"] = 0, 3
    edge[2]["n_opts"], edge[2]["min_group_size"], edge[2]["max_group_size"] = 0, 1, 2
    edge[3] = (abi.PM_A_HAS_REQ | abi.PM_A_REQ_CPU | abi.PM_A_REQ_CPU_CORES, 0, 0, (1 << 31) + 5, 0, 0, 1, 1)
    edge[4] = (abi.PM_A_HAS_REQ | abi.PM_A_REQ_RAM, 0, 0, 0, 0xFFFFFFFF, 0, 1, 1)
    edge[5] = (abi.PM_A_HAS_REQ, 1, len(opts) - 2, 0, 0, 0, 1, 1)
    edge[6] = (abi.PM_A_HAS_REQ, 1, len(opts) - 1, 0, 0, 0, 1, 1)
    # a row inside the fast predicate's domain with a core-count threshold neither table has: one feature more (the
    # wide tables hold exactly 64, the feature kernel's budget)
    feature = asks[z:z + 1].copy()
    feature["flags"] |= abi.PM_A_HAS_REQ | abi.PM_A_REQ_CPU | abi.PM_A_REQ_CPU_CORES
    feature["cpu_cores"], feature["min_group_size"], feature["max_group_size"] = 3, 1, 2
    return dict(T=T, W=W, z=z, asks=[asks, asks2], opts=opts, bits=[np.asarray(bits, dtype=np.uint32), bits2],
                npat=npat, nmod=nmod, words=words, wa=w.a.copy(), wb=wb, lat=lat, lon=lon,
                rank=rng.permutation(W).astype(np.uint32), cap=rng.integers(50, 1500, T).astype(np.uint32),
                rep=rng.integers(0, 4, W).astype(np.uint32), floors=rng.integers(0, 3, T).astype(np.uint32),
                pool=np.concatenate([asks, asks2]), edge=edge, feature=feature)


# ------------------------------------------------------------------------------------------------ the mirror
class History(AskMarket):
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
        self.replaced = set()               # asks replaced since the stored evaluation
        self.appended = set()               # asks appended or inserted since it
        self.heirs = set()                  # kept rows that took a removed ask's stored first asks since it
        self.dropped = 0                   # stored first asks an ask shrink set to NONE since it
        self.eval_facts = None              # (workers_small, prices_narrow, asks_small) at the stored evaluation
        self.flipped = set()                # which of the facts changed since the stored evaluation
        # auction tracker (A0 is AskMarket's `toggled`, over asks; changed_slots() spreads it over slots)
        self.auc_state, self.auc_w, self.auc_over = False, 0, False
        self.resized = False                # an ask resize since the stored state
        self.d = np.ones(len(self.asks), dtype=np.uint32)
        self.d_pass = self.d.copy()
        self.last_report = None             # the report of the last successful restore
        self.outcomes = {}                  # generate(): event index -> an auction pass's prediction or restore report

    # ---- facts
    def facts(self):
        return workers_small(self.wa, self.wb), prices_narrow(self.wb), asks_small(self.asks, self.opts)

    def _note_facts(self):
        if self.eval_facts is not None:
            now = self.facts()
            for name, a, b in zip(("fast", "narrow", "ask_fast"), self.eval_facts, now):
                if a != b:
                    self.flipped.add(name)

    def max0_on(self):
        """The enabled asks with max_group_size == 0 (PM_MODE_PROXIMITY refuses while there is one)."""
        return np.flatnonzero(self.mask & (self.asks["max_group_size"] == 0))

    def pattern_missing(self):
        return bool(missing_pattern(self.asks, self.opts, self.s["npat"]).any())

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
        self.replaced, self.appended, self.heirs, self.dropped = set(), set(), set(), 0
        self.eval_facts, self.flipped = None, set()

    def discard_auction(self):
        self.auc_state, self.auc_over, self.resized = False, False, False
        self.store(None, None)

    # ---- slots (the twin table: row t repeated d[t] times)
    def store(self, price, assigned):
        super().store(price, assigned)
        self.dem_kept = None                # the leading slots of each ask a demand change kept (None: all)
        if hasattr(self, "d"):
            self.d_pass = self.d.copy()     # the demands at the stored state (cut and extended with the asks)

    def slot_F(self, F=None):
        return np.repeat(self.F() if F is None else F, self.d, axis=0)

    def slot_cap(self):
        return np.repeat(self.cap, self.d)

    def slot_floors(self):
        return np.repeat(self.floors_or_zero(), self.d)

    def held_asks(self):
        """The asks holding at least one worker in the stored state."""
        if not self.auc_state or self.assigned is None:
            return np.zeros(0, dtype=np.int64)
        if len(self.d) == 0:
            return np.zeros(0, dtype=np.int64)
        return np.flatnonzero(np.add.reduceat((self.assigned != NONE).astype(np.int64), ad.offsets(self.d)[:-1]))

    def kept_slots(self):
        """Per ask the leading slots that keep their stored hold at the next warm pass: 0 for an ask of A0."""
        kept = self.d.astype(np.int64) if self.dem_kept is None else np.minimum(self.dem_kept, self.d).astype(np.int64)
        kept[self.changed_asks()] = 0
        return kept

    def changed_slots(self):
        """A0 over slots: every slot of an ask of A0, and the slots past each ask's kept ones."""
        off = ad.offsets(self.d)
        k = np.arange(off[-1]) - np.repeat(off[:-1], self.d)
        return np.flatnonzero(k >= np.repeat(self.kept_slots(), self.d)).tolist()

    def n_changes(self):
        return len(self.rows) + (self.n_workers - self.n_kept) + len(self.changed_slots()) + self.removed_held

    def _freed(self, gone):
        """The workers of removed slots that count against the cutoff: those below n_kept."""
        gone = np.asarray(gone)
        return int(((gone != NONE) & (gone < self.n_kept)).sum())

    def _slot_freed(self, gone):
        """The workers of the slots a demand change removed that count against the cutoff."""
        return self._freed(gone)

    def _kept_after(self, new):
        """The slots kept over the chain of demand changes since the stored state."""
        return np.minimum(self.d if self.dem_kept is None else self.dem_kept, new)

    def _free_price(self, workers):
        """A removed slot's worker is unowned at its stored price: nothing to do."""

    def set_demand(self, new):
        new = np.asarray(new, dtype=np.uint32)
        if np.array_equal(new, self.d):     # the same demands: nothing changes
            return
        if self.auc_state:
            o_old, o_new = ad.offsets(self.d), ad.offsets(new)
            a, _, _ = ad.remap(self.assigned, self.d, new)
            gone = np.concatenate([self.assigned[o_old[t] + min(int(self.d[t]), int(new[t])):o_old[t + 1]]
                                   for t in range(len(new))] or [np.zeros(0, np.uint32)])
            gone = gone[gone != NONE]
            self.removed_held += self._slot_freed(gone)
            self._free_price(gone)
            self.dem_kept = self._kept_after(new)
            self.assigned = a
            assert len(a) == int(o_new[-1])
        self.d = new.copy()

    # ---- restore
    def export_refusal(self):
        st = set()
        if not self.auc_state:
            st.add(abi.PM_E_STATE)
        if (self.d > 1).any():
            st.add(abi.PM_E_UNSUPPORTED)
        return st

    def export(self):
        """(prices of the stored pass's rows, the stored assignment over the current asks)."""
        return self.price.copy(), self.assigned.copy()

    def restore_refusal(self, price, assigned):
        """The statuses a restore of (price, assigned) may return, or an empty set when it must succeed."""
        st = set()
        W, T = self.n_workers, len(self.asks)
        price, assigned = np.asarray(price, dtype=np.int64), np.asarray(assigned, dtype=np.uint32)
        if self.pattern_missing():
            st.add(abi.PM_E_STATE)
        if not self.mask.all() or (self.d > 1).any():
            st.add(abi.PM_E_UNSUPPORTED)
        S, E, _ = self.params
        top = rs.price_bound(self.cap, S, E)
        if len(price) != W or len(assigned) != T or ((assigned != NONE) & (assigned >= W)).any() \
                or (price < 0).any() or (price > top).any() or not in_domain(self.wb, self.cap, self.params):
            st.add(abi.PM_E_INVALID)
        return st

    def _restore_clear(self, price, kept):
        self.store(price, kept)

    def restore(self, price, assigned):
        """A successful restore: the audited state is the stored one, nothing changed since it.  Returns the report."""
        price = np.array(price, dtype=np.int64)
        out = rs.audit(self.F(), self.wb["ext_ask_price"], self.cap, self.params[0], price, assigned)
        self._restore_clear(price, out["assigned"])
        self.auc_state, self.auc_w, self.auc_over, self.resized = True, self.n_workers, False, False
        self.last_report = {k: out[k] for k in ("n_held", "n_dropped_bad", "n_dropped_shared", "n_dropped_slack", "evals")}
        return {k: out[k] for k in ("n_held", "n_dropped_bad", "n_dropped_shared", "n_dropped_slack", "evals")}

    def fit(self, price, assigned):
        """A state trimmed to the current tables: prices cut or zero-padded to W, holds >= W dropped, the assignment
        cut or padded with PM_NONE to T."""
        W, T = self.n_workers, len(self.asks)
        p = np.zeros(W, dtype=np.int64)
        p[:min(W, len(price))] = np.asarray(price, dtype=np.int64)[:W]
        a = np.full(T, NONE, dtype=np.uint32)
        a[:min(T, len(assigned))] = np.asarray(assigned, dtype=np.uint32)[:T]
        a[(a != NONE) & (a >= W)] = NONE
        return p, a

    def e_rows(self, en):
        """|E| x W / T rounded up: what the E-pass counts against the cutoff (the current T)."""
        T = len(self.asks)
        return -(-len(en) * self.n_workers // T) if T else 0

    def incremental_plan(self):
        """(full, n_tiles, enabled since, disabled since, count certain) of the next incremental pass."""
        W, T = self.n_workers, len(self.asks)
        if not self.eval or self.cutoff == 0 or T == 0 or W == 0:
            return True, W, set(), set(), True
        en, dis = self.split()
        full_now = len(self.dirty) + self.e_rows(en) > self.cutoff
        full = self.over or full_now
        sure = self.over == (len(self.dirty) > self.cutoff)   # a shrink since the count passed the cutoff: unspecified
        if full:
            return True, W, en, dis, sure
        return False, walked_rows(self.eval_ff, self.dirty, dis), en, dis, sure

    def warm_plan(self):
        """(warm, certain) of the next PM_AUCTION_WARM pass."""
        if not self.auc_state:
            return False, True
        fits = self.n_changes() <= self.cutoff
        return (fits and not self.auc_over), self.auc_over == (len(self.rows) > self.cutoff)

    # ---- the ask table in place (AskMarket keeps the rows, caps, floors and A0; these keep the rest)
    def update_asks(self, idx, rows):
        self.replace(idx, rows)
        if self.eval:
            self.replaced |= {int(t) for t in idx}
        self._note_facts()

    def append_asks(self, rows):
        k, T = len(rows), len(self.asks)
        if self.eval:
            self.appended |= set(range(T, T + k))
        self.append(rows)                   # the new asks have demand 1: one empty slot each, in A0
        self.d = np.concatenate([self.d, np.ones(k, dtype=np.uint32)])
        self.d_pass = np.concatenate([self.d_pass, np.ones(k, dtype=np.uint32)])
        if self.dem_kept is not None:
            self.dem_kept = np.concatenate([self.dem_kept, np.ones(k, dtype=self.dem_kept.dtype)])
        self.mask = np.concatenate([self.mask, np.ones(k, dtype=bool)])
        self.eval_mask = np.concatenate([self.eval_mask, np.zeros(k, dtype=bool)])
        self.resized |= self.auc_state
        self._note_facts()

    def shrink_asks(self, n):
        n_slots = int(ad.offsets(self.d)[n])
        a = self.assigned
        if a is not None:                   # the removed asks' slots: their held workers below n_kept count
            self.removed_held += self._freed(a[n_slots:])
            self.assigned = None
        self.shrink(n)
        if a is not None:
            self.assigned = a[:n_slots].copy()
        self.d, self.d_pass = self.d[:n].copy(), self.d_pass[:n].copy()
        if self.dem_kept is not None:
            self.dem_kept = self.dem_kept[:n].copy()
        self.mask, self.eval_mask = self.mask[:n].copy(), self.eval_mask[:n].copy()
        self.replaced = {t for t in self.replaced if t < n}
        self.appended = {t for t in self.appended if t < n}
        self.heirs = {t for t in self.heirs if t < n}
        if self.eval_ff is not None:   # a worker whose stored first ask was removed had no feasible ask before it
            cut = (self.eval_ff != NONE) & (self.eval_ff >= n)
            self.dropped += int(cut.sum()) if self.eval else 0
            self.eval_ff = np.where(cut, NONE, self.eval_ff).astype(np.uint32)
        self.resized |= self.auc_state
        self._note_facts()

    def split(self):
        """(E, D) of the next incremental pass."""
        return split_toggles(self.mask, self.eval_mask, self.replaced, self.heirs)

    def _new_heirs(self, rm, keep):
        """The kept rows that take the stored first asks of removed rows: the next kept row after a row enabled at the
        stored evaluation or itself a heir (no kept row after it: none)."""
        succ = np.searchsorted(keep, rm)
        return {int(s) for t, s in zip(rm, succ) if s < len(keep) and (self.eval_mask[t] or int(t) in self.heirs)}

    def _removed_freed(self, gone):
        """The workers of a removed ask's slots that count against the cutoff."""
        return self._freed(gone)

    def _per_ask(self, f):
        """Apply f to every per-ask column (asks, caps, floors, demands, masks)."""
        self.asks, self.cap, self.cap0, self.floors0 = f(self.asks), f(self.cap), f(self.cap0), f(self.floors0)
        if self.floors is not None:
            self.floors = f(self.floors)
        self.d, self.d_pass = f(self.d), f(self.d_pass)
        if self.dem_kept is not None:
            self.dem_kept = f(self.dem_kept)
        self.mask, self.eval_mask = f(self.mask), f(self.eval_mask)

    def remove_asks(self, idx):
        """pm_remove_asks: the rows after the removed ones move up.  Each stored first ask moves with its row; a removed
        one lands on the next kept row, its heir (D with the replaced bit), or is NONE with no kept row after it.  Kept
        asks keep their slots; a removed ask's held slots below n_kept count in removed_held."""
        T = len(self.asks)
        rm = np.unique(np.asarray(idx, dtype=np.int64))
        keep = np.setdiff1d(np.arange(T), rm)
        new = np.full(T, -1, np.int64)
        new[keep] = np.arange(len(keep))
        heirs = self._new_heirs(rm, keep) if self.eval else set()
        self.replaced, self.appended = renamed(self.replaced, new), renamed(self.appended, new)
        self.heirs = renamed(self.heirs, new) | heirs
        if self.eval_ff is not None:
            f = self.eval_ff.astype(np.int64)
            g = f - np.searchsorted(rm, f, side="left")
            cut = (f != NONE) & (g >= len(keep))
            self.dropped += int(cut.sum()) if self.eval else 0
            self.eval_ff = np.where((f == NONE) | cut, NONE, g).astype(np.uint32)
        if self.assigned is not None:
            off = ad.offsets(self.d)
            gone = np.zeros(int(off[-1]), dtype=bool)
            for t in rm:
                gone[off[t]:off[t + 1]] = True
            self.removed_held += self._removed_freed(self.assigned[gone])
            self.assigned = self.assigned[~gone].copy()
        self._per_ask(lambda v: v[keep].copy())
        self.toggled = renamed(self.toggled, new)
        self.resized |= self.auc_state
        self._note_facts()

    def insert_asks(self, before, rows):
        """pm_insert_asks: rows[i] goes before the current row before[i].  Stored first asks move with their rows; the
        inserted rows are in E (appended), with demand 1, cap 0, floor 0 and one empty slot in A0."""
        T, k = len(self.asks), len(before)
        before = np.asarray(before, dtype=np.int64)
        new = np.arange(T) + np.searchsorted(before, np.arange(T), side="right")
        at = before + np.arange(k)
        self.replaced, self.heirs = renamed(self.replaced, new), renamed(self.heirs, new)
        self.appended = renamed(self.appended, new) | ({int(a) for a in at} if self.eval else set())
        if self.eval_ff is not None:
            f = self.eval_ff.astype(np.int64)
            self.eval_ff = np.where(f == NONE, NONE, f + np.searchsorted(before, f, side="right")).astype(np.uint32)
        if self.assigned is not None:
            self.assigned = np.insert(self.assigned, ad.offsets(self.d)[before], NONE).astype(np.uint32)
        z = np.zeros(k, dtype=np.uint32)
        self.asks, self.cap, self.cap0 = np.insert(self.asks, before, rows), np.insert(self.cap, before, z), \
            np.insert(self.cap0, before, z)
        self.floors0 = np.insert(self.floors0, before, z)
        if self.floors is not None:
            self.floors = np.insert(self.floors, before, z)
        self.d, self.d_pass = np.insert(self.d, before, z + 1), np.insert(self.d_pass, before, z + 1)
        if self.dem_kept is not None:
            self.dem_kept = np.insert(self.dem_kept, before, np.ones(k, dtype=self.dem_kept.dtype))
        self.mask, self.eval_mask = np.insert(self.mask, before, True), np.insert(self.eval_mask, before, False)
        self.toggled = renamed(self.toggled, new) | self._inserted_a0(at)
        self.resized |= self.auc_state
        self._note_facts()
        return at

    def _inserted_a0(self, at):
        """The inserted asks A0 gains: all of them (their one slot holds nothing)."""
        return {int(a) for a in at}

    # ---- predictions of refusals (the set of statuses the header allows)
    def refusal(self, kind):
        """(refusal name, statuses) or (None, None) for a pass or certificate that must run."""
        if kind == "auction_incr":
            return "auction_incremental", {abi.PM_E_INVALID}
        if kind in REFERENCE and self.pattern_missing():
            return "pattern_missing", {abi.PM_E_STATE}
        if kind == "proximity" or kind == "proximity_incr":
            if len(self.max0_on()):
                return "proximity_max0", {abi.PM_E_UNSUPPORTED}
            return None, None
        if kind in AUCTION:
            if self.pattern_missing():   # refused before the pass: the stored state stays
                return "pattern_missing", {abi.PM_E_STATE}
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
            elif self.resized:
                st.add(abi.PM_E_STATE)
                why = "certificate_asks_resized"
            elif self.pattern_missing():
                st.add(abi.PM_E_STATE)
                why = "pattern_missing"
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
        self.replaced, self.appended, self.heirs, self.dropped = set(), set(), set(), 0
        self.eval_mask = self.mask.copy()
        self.eval_ff = self.first_feasible()
        self.eval_facts, self.flipped = self.facts(), set()

    def auction_done(self, price, assigned):
        self.store(price, assigned)
        self.auc_state, self.auc_w, self.auc_over, self.resized = True, self.n_workers, False, False

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
                self.toggled |= set(changed)
        elif name == "locations":
            self.lat, self.lon = x["lat"].copy(), x["lon"].copy()
        elif name == "addr_rank":
            self.rank = x["rank"].copy()
        elif name == "update_asks":
            self.update_asks(x["idx"], x["rows"])
        elif name == "append_asks":
            self.append_asks(x["rows"])
            if x["cap"] is not None:
                self.set_caps(x["cap"])
        elif name == "shrink_asks":
            if x["n"] != len(self.asks):    # pm_resize_asks to the current size changes nothing
                self.shrink_asks(x["n"])
        elif name == "remove_asks":
            self.remove_asks(x["idx"])
        elif name == "insert_asks":
            self.insert_asks(x["before"], x["rows"])
            if x["cap"] is not None:
                self.set_caps(x["cap"])
        elif name in ("ask_delta_refused", "demand_refused", "restore_refused"):   # refused: nothing changes
            pass
        elif name == "demand":
            self.set_demand(x["d"])
        elif name == "restore":
            self.last_report = None
            for price, assigned in x["attempts"]:   # the first one the engine takes
                if not self.restore_refusal(price, assigned):
                    self.restore(price, assigned)
                    break
        elif name == "move":                # a fresh engine with no stored evaluation takes the state
            price, assigned = x["fit"]
            self.restore(price, assigned)
            self.discard_eval()
        elif name == "set_asks":
            self.ask_table = x["table"]
            self.asks = self.s["asks"][x["table"]].copy()
            self.mask = np.ones(len(self.asks), dtype=bool)
            self.d = np.ones(len(self.asks), dtype=np.uint32)
            self.cap, self.floors = x["cap"].copy(), x["floors"].copy()
            self.eval_mask = self.mask.copy()
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
    elif name == "update_asks":
        eng.update_asks(x["idx"], *delta_rows(x))
    elif name == "append_asks":
        eng.resize_asks(x["n"], *delta_rows(x))
        if x["cap"] is not None:
            eng.set_price_caps(x["cap"])
    elif name == "shrink_asks":
        eng.resize_asks(x["n"])
    elif name == "remove_asks":
        eng.remove_asks(x["idx"])
    elif name == "insert_asks":
        eng.insert_asks(x["before"], *delta_rows(x))
        if x["cap"] is not None:
            eng.set_price_caps(x["cap"])
    elif name == "ask_delta_refused":
        refuse_delta(eng, x)
    elif name == "demand":
        eng.set_ask_demand(x["d"])
    elif name == "demand_refused":
        refuse_demand(eng, x)
    elif name in ("restore", "restore_refused", "move"):
        raise ValueError(f"{name}: the runner sends it (it checks the export and the report)")
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


def delta_rows(x):
    """(rows, opts) as a delta sends them: each row with only its own option rows, or with the whole option table."""
    return own_options(x["rows"], x["opts"]) if x["own"] else (x["rows"], x["opts"])


def refuse_delta(eng, x):
    """One PM_E_INVALID case of pm_update_asks / pm_resize_asks / pm_remove_asks / pm_insert_asks: the call is refused
    and pm_table_version stays.  That the tables themselves stay is shown by the incremental and warm passes that
    follow every refusal (the history's `follow`), which compare the engine with the mirror."""
    from protocol_b200._lib import PrimeMatchError

    T, rows, opts = x["T"], x["rows"], x["opts"]
    assert getattr(eng, "n_asks", T) == T
    bad_sizes = rows.copy()
    bad_sizes["min_group_size"][-1], bad_sizes["max_group_size"][-1] = 5, 2
    bad_range = rows.copy()
    bad_range["opt_off"][0], bad_range["n_opts"][0] = len(opts), 1
    bad_range["flags"][0] |= abi.PM_A_HAS_REQ
    def remove_null():   # a NULL idx with n > 0 (pm_multi keeps no ask count on the host)
        import ctypes

        fn = eng._lib.pm_remove_asks if hasattr(eng, "n_asks") else eng._lib.pm_multi_remove_asks
        rc = fn(eng._h, ctypes.c_void_p(None), 2)
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, "pm_remove_asks: null")

    calls = {"index": lambda: eng.update_asks(np.array([1, T], dtype=np.uint32), rows, opts),
             "sizes": lambda: eng.update_asks(np.array([1, 2], dtype=np.uint32), bad_sizes, opts),
             "range": lambda: eng.update_asks(np.array([1, 2], dtype=np.uint32), bad_range, opts),
             "grow_without_rows": lambda: eng.resize_asks(T + 2),
             "grow_bad_range": lambda: eng.resize_asks(T + 2, bad_range, opts),
             "too_many": lambda: eng.resize_asks(1 << 30, rows, opts),
             "remove_index": lambda: eng.remove_asks(np.array([3, T, 1], dtype=np.uint32)),
             "remove_null": remove_null,
             "insert_decreasing": lambda: eng.insert_asks(np.array([2, 1], dtype=np.uint32), rows, opts),
             "insert_past_end": lambda: eng.insert_asks(np.array([1, T + 1], dtype=np.uint32), rows, opts),
             "insert_sizes": lambda: eng.insert_asks(np.array([0, T], dtype=np.uint32), bad_sizes, opts),
             "insert_range": lambda: eng.insert_asks(np.array([1, 1], dtype=np.uint32), bad_range, opts)}
    v = eng.table_version()
    try:
        calls[x["case"]]()
    except PrimeMatchError as ex:
        assert ex.status == abi.PM_E_INVALID, (x["case"], ex.status)
    else:
        raise AssertionError(f"ask delta {x['case']}: accepted")
    assert eng.table_version() == v, (x["case"], "pm_table_version changed")
    # the wrapper's own count (it moves only after the library returns PM_OK), not a read of the engine
    assert getattr(eng, "n_asks", T) == T, (x["case"], "the wrapper's n_asks changed")


def refuse_demand(eng, x):
    """One PM_E_INVALID case of pm_set_ask_demand: the call is refused and pm_table_version stays."""
    import ctypes

    from protocol_b200._lib import PrimeMatchError

    T = x["T"]
    d = np.ones(T, dtype=np.uint32)
    v = eng.table_version()
    if x["case"] == "null":     # a NULL pointer with n_asks > 0
        rc = eng._lib.pm_set_ask_demand(eng._h, ctypes.c_void_p(None), T)
        assert rc == abi.PM_E_INVALID, ("null", rc)
    else:
        if x["case"] == "length":
            d = np.ones(T + (1 if T % 2 else -1), dtype=np.uint32)
        elif x["case"] == "zero":
            d[T // 2] = 0
        elif x["case"] == "total":   # D >= 2^30
            d[-1] = (1 << 30) - (T - 1)
        try:
            eng.set_ask_demand(d)
        except PrimeMatchError as ex:
            assert ex.status == abi.PM_E_INVALID, (x["case"], ex.status)
        else:
            raise AssertionError(f"demand {x['case']}: accepted")
    assert eng.table_version() == v, (x["case"], "pm_table_version changed")


def load(eng, h: History, twin=False):
    """Load an engine with the mirror's current tables (a fresh engine's start, or the start of a history), demands
    included; twin: the twin tables instead (every ask row, cap and floor repeated d[t] times, every demand 1)."""
    s = h.s
    eng.set_asks(np.repeat(h.asks, h.d) if twin else h.asks, h.opts)
    if (h.d != 1).any() and not twin:
        eng.set_ask_demand(h.d)
    eng.set_model_table(s["bits"][h.bits_table], s["npat"], s["nmod"], s["words"])
    eng.set_workers(h.wa, h.wb)
    eng.set_locations(h.lat, h.lon)
    eng.set_addr_rank(h.rank)
    eng.set_price_caps(h.slot_cap() if twin else h.cap)
    eng.set_worker_reputation(h.reputation)
    eng.set_min_reputation(h.slot_floors() if twin else h.floors_or_zero())
    S, E, d = h.params
    eng.set_auction_params(cost_scale=S, eps_start=E, eps_div=d)
    if not h.mask.all():
        assert not twin
        eng.set_ask_enabled(np.flatnonzero(~h.mask), False)


# ------------------------------------------------------------------------------------------------ the generator
class Gen:
    """Draws table calls against a mirror (so that indices, held rows and edge rows follow the history)."""

    def __init__(self, h: History, rng):
        self.h, self.rng = h, rng
        s = h.s
        self.pool_a, self.pool_b = s["wa"], s["wb"]
        self.saved = None                   # a state exported earlier (the stale restore's)

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

    def ask_rows(self, k, edge=0.15, missing=True):
        """k ask rows from both tables, sometimes an edge row (EDGE_ASKS; the missing-pattern rows only if `missing`)."""
        rng, s = self.rng, self.h.s
        rows = s["pool"][rng.integers(0, len(s["pool"]), k)].copy()
        n_edge = len(s["edge"]) if missing else len(s["edge"]) - 2
        for i in np.flatnonzero(rng.random(k) < edge):
            j = int(rng.integers(0, n_edge))
            if j >= len(s["edge"]) - 2 and rng.random() < 0.7:   # rarer than the other edge rows
                j = int(rng.integers(0, len(s["edge"]) - 2))
            rows[i] = s["edge"][j]
        return rows

    def delta(self, name, rows, **x):
        return (name, dict(x, rows=rows, opts=self.h.opts, own=bool(self.rng.random() < 0.7)))

    def update_asks(self, idx, rows=None):
        """Replace asks idx; the rows of asks with a missing pattern are replaced too (by ordinary rows)."""
        h = self.h
        miss = np.flatnonzero(missing_pattern(h.asks, h.opts, h.s["npat"]))
        rows = self.ask_rows(len(idx)) if rows is None else rows
        if len(miss):
            idx = np.concatenate([np.asarray(idx, dtype=np.uint32), miss.astype(np.uint32)])
            rows = np.concatenate([rows, self.ask_rows(len(miss), edge=0)])
        return self.delta("update_asks", rows, idx=np.asarray(idx, dtype=np.uint32))

    def held_asks(self):
        """Asks holding a worker in the stored auction state, and asks that are many workers' stored first ask."""
        h = self.h
        held = h.held_asks()
        first = np.zeros(0, dtype=np.int64)
        if h.eval and h.eval_ff is not None:
            ff = h.eval_ff[h.eval_ff != NONE].astype(np.int64)
            if len(ff):
                c = np.bincount(ff, minlength=len(h.asks))
                first = np.argsort(-c, kind="stable")[:8]
                first = first[c[first] > 0]
        return held, first

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
            if rng.random() < 0.3:
                i = np.union1d(i, h.max0_on())
            return ("ask_off", dict(idx=np.unique(i).astype(np.uint32)))
        if name == "update_asks":
            held, first = self.held_asks()
            k = int(rng.integers(1, 4))
            r = rng.random()
            if r < 0.3 and len(held):
                idx = rng.choice(held, min(k, len(held)), replace=False)
            elif r < 0.55 and len(first):
                idx = rng.choice(first, min(k, len(first)), replace=False)
            elif r < 0.7 and not h.mask.all():
                idx = rng.choice(np.flatnonzero(~h.mask), 1)
            else:
                idx = rng.integers(0, T, k)
            idx = np.asarray(idx, dtype=np.uint32)
            if rng.random() < 0.2:                      # a repeated index: the last entry decides
                idx = np.concatenate([idx, idx[:1]])
            return self.update_asks(idx)
        if name == "append_asks":
            k = int(rng.integers(1, 4 if T < 280 else 2))
            cap = None
            if rng.random() < 0.6:
                cap = np.concatenate([h.cap, rng.integers(50, 1500, k)]).astype(np.uint32)
            return self.delta("append_asks", self.ask_rows(k), n=T + k, cap=cap)
        if name == "shrink_asks":
            n = T - int(rng.integers(1, 6 if T > 210 else 2)) if rng.random() < 0.95 else T   # T: changes nothing
            return ("shrink_asks", dict(n=n))
        if name == "remove_asks":   # unsorted, sometimes a repeated index; held asks, first asks, max_group_size 0 rows
            held, first = self.held_asks()
            k = int(rng.integers(1, 5 if T > 210 else 2))
            r = rng.random()
            z = np.flatnonzero(h.asks["max_group_size"] == 0)
            pool = held if r < 0.3 and len(held) else first if r < 0.55 and len(first) else \
                z if r < 0.7 and len(z) else np.arange(T)
            idx = rng.permutation(rng.choice(pool, min(k, len(pool)), replace=False))
            if rng.random() < 0.3:
                idx = np.concatenate([idx, idx[:1]])
            return ("remove_asks", dict(idx=idx.astype(np.uint32)))
        if name == "insert_asks":   # equal positions, the front and the end (= an append); sometimes caps for them
            k = int(rng.integers(1, 4 if T < 280 else 2))
            r = rng.random()
            before = np.zeros(k) if r < 0.2 else np.full(k, T) if r < 0.35 else np.sort(rng.integers(0, T + 1, k))
            if rng.random() < 0.3:
                before[:] = before[0]
            before = before.astype(np.uint32)
            cap = None
            if rng.random() < 0.6:
                cap = np.insert(h.cap, before.astype(np.int64), rng.integers(50, 1500, k)).astype(np.uint32)
            return self.delta("insert_asks", self.ask_rows(k), before=before, cap=cap)
        if name == "ask_delta_refused":
            cases = DELTA_REFUSALS + SPLICE_REFUSALS
            return self.delta("ask_delta_refused", self.ask_rows(2, edge=0), T=T, case=cases[int(rng.integers(0, len(cases)))])
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
        if name == "set_asks":   # caps and floors of the new table's length, the current ones where they reach
            cap, fl = s["cap"].copy(), s["floors"].copy()
            n = min(T, len(cap))
            cap[:n], fl[:n] = h.cap[:n], h.floors_or_zero()[:n]
            return ("set_asks", dict(table=1 - h.ask_table, setup=s, cap=cap, floors=fl))
        if name == "model_table":
            return ("model_table", dict(table=1 - h.bits_table, setup=s))
        if name == "auction_params":
            choices = [p for p in PARAMS if p != h.params]
            return ("auction_params", dict(params=choices[int(rng.integers(0, len(choices)))]))
        if name == "demand":
            d = h.d.copy()
            r = rng.random()
            if r < 0.12:
                d[:] = 1
            elif r < 0.2:
                d[int(rng.integers(0, T))] = int(rng.integers(20, 120))      # one large demand
            else:                                                            # held asks and unheld ones, 1..4
                held = h.held_asks()
                free = np.setdiff1d(np.arange(T), held)
                idx = [rng.choice(p, min(len(p), int(rng.integers(1, 5))), replace=False) for p in (held, free) if len(p)]
                idx = np.concatenate(idx).astype(np.int64)
                d[idx] = rng.integers(1, 5, len(idx))
            return ("demand", dict(d=d.astype(np.uint32)))
        if name == "demand_refused":
            return ("demand_refused", dict(T=T, case=DEMAND_REFUSALS[int(rng.integers(0, len(DEMAND_REFUSALS)))]))
        if name == "restore":
            own = h.auc_state and not h.export_refusal()
            variants = ["adversarial"] + (["own", "own"] if own else []) + (["stale"] if self.saved is not None else [])
            return self.restore(variants[int(rng.integers(0, len(variants)))])
        if name == "restore_refused":
            cases = ["length_w", "length_t", "worker", "price_neg", "price_high"]
            cases += ["demand"] if (h.d > 1).any() else []
            cases += ["disabled"] if not h.mask.all() else []
            cases += ["export_no_state"] if not h.auc_state else ["export_demand"] if (h.d > 1).any() else []
            return self.restore_refused(cases[int(rng.integers(0, len(cases)))])
        if name == "move":
            raw = h.export()
            return ("move", dict(export=raw, fit=h.fit(*raw)))
        if name == "set_workers":
            n = int(rng.integers(W - 40, W + 40))
            a, b = self.rows(n)
            la, lo = self.points(n)
            return ("set_workers", dict(a=a, b=b, lat=la, lon=lo, rank=rng.permutation(n).astype(np.uint32),
                                        rep=rng.integers(0, 4, n).astype(np.uint32)))
        raise ValueError(name)


    def restore(self, variant):
        """A restore into the same engine: the own state as exported (after a worker resize: refused, then trimmed),
        a state exported earlier, or adversarial_state on the current tables."""
        h, rng = self.h, self.rng
        if variant in ("own", "resized") and (not h.auc_state or h.export_refusal()) \
                or variant == "stale" and self.saved is None:
            variant = "adversarial"             # nothing to export
        x = dict(variant=variant, export=None)
        if variant in ("own", "resized"):
            x["variant"] = "own" if h.n_workers == h.auc_w else "resized"
            x["export"] = raw = h.export()
            self.saved = raw
            x["attempts"] = [raw] if h.n_workers == h.auc_w else [raw, h.fit(*raw)]
        elif variant == "stale":
            p, a = h.fit(*self.saved)
            x["attempts"] = [(p, a), (np.minimum(p, rs.price_bound(h.cap, h.params[0], h.params[1])), a)]
        else:
            x["attempts"] = [rs.adversarial_state(h.F(), h.wb["ext_ask_price"], h.cap, h.params[0], rng, h.params[1])]
        return ("restore", x)

    def restore_refused(self, case):
        """One refused export or restore: a corrupted state, or a valid one while the tables refuse it."""
        h = self.h
        W, T = h.n_workers, len(h.asks)
        if h.auc_state:
            p, a = h.fit(*h.export()) if not (h.d > 1).any() else (np.zeros(W, np.int64), np.full(T, NONE, np.uint32))
        else:
            p, a = np.zeros(W, dtype=np.int64), np.full(T, NONE, dtype=np.uint32)
        p, a = p.copy(), a.copy()
        if case == "length_w":
            p = np.zeros(W + 1 if self.rng.random() < 0.5 else W - 1, dtype=np.int64)
        elif case == "length_t":
            a = np.full(T + 1, NONE, dtype=np.uint32)
        elif case == "worker":
            a[int(self.rng.integers(0, T))] = W
        elif case == "price_neg":
            p[int(self.rng.integers(0, W))] = -1
        elif case == "price_high":
            p[int(self.rng.integers(0, W))] = rs.price_bound(h.cap, h.params[0], h.params[1]) + 1
        return ("restore_refused", dict(case=case, price=p, assigned=a, export=case.startswith("export")))


ALL_PAIRS = [(c, k) for c in CALLS for k in PASSES]


def generate(shape, seed, n_calls=N_CALLS, cutoff=DEFAULT_CUTOFF, slot=0, n_slots=1, observe=None):
    """A seeded history: a list of events, ("call", (name, payload)), ("pass", kind) or ("probe", (t0, nt)) (a
    pm_build_cost_tile of asks [t0, t0 + nt), which changes nothing).  The mirror it returns has lived through the
    history, auction states included.  History `slot` of `n_slots` also makes every n_slots-th (table call -> pass
    kind) pair from the slot on, so that the histories together make all.  observe(h, event, before): called after
    each call with the mirror and before each pass, probe or refused call with it."""
    rng = np.random.default_rng(seed)
    must = ALL_PAIRS[slot::n_slots]
    h = History(shape, cutoff)
    g = Gen(h, rng)
    events = []
    seen_call, seen_pass = set(), set()
    last_pass, calls_since = "start", []
    domain_at = n_calls // 2
    done = set()                             # the scripted steps made so far

    def emit_call(ev):
        events.append(("call", ev))
        if observe is not None:
            observe(h, events[-1], True)
        if ev[0] == "restore_refused":
            assert h.restore_refusal(ev[1]["price"], ev[1]["assigned"]) or ev[1]["export"], ev[1]["case"]
            assert not ev[1]["export"] or h.export_refusal(), ev[1]["case"]
        h.apply(ev)
        if ev[0] in ("restore", "move"):
            h.outcomes[len(events) - 1] = h.last_report
        calls_since.append(ev[0])
        if observe is not None:
            observe(h, events[-1], False)
        if ev[0] in ("ask_delta_refused", "demand_refused", "restore_refused") and not follow:
            follow.extend(["lean_incr", "warm"])     # what it left: the next incremental and warm passes show it
        if ev[0] in ASK_DELTAS and len(h.asks) and rng.random() < 0.25:
            probe()

    def emit_named(c):
        """g.call(c), after the calls a restore or a move needs to be taken (all asks on, every demand 1, a stored
        state within the price bound); a move that still cannot be taken is a restore."""
        if c in ("restore", "move") and rng.random() < 0.85:
            all_on()
            if (h.d > 1).any():
                emit_call(("demand", dict(d=np.ones(len(h.asks), dtype=np.uint32))))
        if c == "move":
            if not h.auc_state and not h.refusal("auction")[0]:
                emit_pass("auction")
            if not h.auc_state or h.export_refusal() or h.restore_refusal(*h.fit(*h.export())):
                c = "restore"
        emit_call(g.call(c))

    def probe():
        T = len(h.asks)
        t0 = int(rng.integers(0, T))
        events.append(("probe", (t0, int(rng.integers(1, min(T - t0, 40) + 1)))))
        if observe is not None:
            observe(h, events[-1], True)

    def emit_pass(kind):
        nonlocal last_pass, calls_since
        events.append(("pass", kind))
        if observe is not None:
            observe(h, events[-1], True)
        why, _ = h.refusal(kind)
        if kind in REFERENCE:
            h.reference_done(why is None)
        elif kind in AUCTION and why is None:   # the checkers' state: later writes can aim at the held rows
            warm = h.warm_plan()[0] if kind in ("warm", "repair") else False
            out = expect_auction(h, kind, warm)
            h.outcomes[len(events) - 1] = (warm,) + out
            h.auction_done(out[1], out[0])
        if why is not None and not follow:   # what the refusal kept: the next incremental and warm passes show it
            follow.extend(["lean_incr", "warm"])
        if kind != "auction_incr":          # the refused flag combination is no pass of any kind
            for c in calls_since:
                seen_call.add((c, kind))
            seen_pass.add((last_pass, kind))
            last_pass = kind
            calls_since = []
        if why == "pattern_missing":        # the next update replaces the rows again
            emit_call(g.update_asks(np.zeros(0, dtype=np.uint32), h.s["pool"][:0]))
        elif kind in AUCTION and why is None and rng.random() < 0.25:
            probe()                         # with the max_group_size 0 rows in the auction's form

    def all_on():
        if not h.mask.all():
            emit_call(("ask_on", dict(idx=np.flatnonzero(~h.mask).astype(np.uint32))))

    def scripted(n_passes):
        """The ask-delta steps every history makes once (each from its pass count on)."""
        s, T = h.s, len(h.asks)
        if n_passes >= 4 and "held" not in done:
            # replace the asks that are many workers' stored first ask: one by a row that still accepts them (other
            # group sizes), one by a row that accepts none; then the same for asks holding auction workers
            done.add("held")
            emit_pass("lean")
            _, first = g.held_asks()
            keep = h.asks[first[:1]].copy()
            keep["min_group_size"], keep["max_group_size"] = 1, 2
            emit_call(g.update_asks(first[:2], np.concatenate([keep, s["edge"][4:5]])[:len(first[:2])]))
            emit_pass("lean_incr")
            all_on()
            emit_pass("auction")
            held, _ = g.held_asks()
            if len(held):
                t = held[int(rng.integers(0, len(held)))]
                keep = h.asks[[t]].copy()
                emit_call(g.update_asks(np.array([t, held[0]], dtype=np.uint32), np.concatenate([keep, s["edge"][4:5]])))
            emit_pass("repair" if slot % 2 else "warm")
            return True
        if n_passes >= 9 and "disabled" not in done:
            # replace a disabled row, then enable it; replace the max_group_size 0 asks with ordinary rows and append
            # a new one
            done.add("disabled")
            emit_pass("lean")
            t = np.array([int(rng.integers(0, T))], dtype=np.uint32)
            emit_call(("ask_off", dict(idx=t)))
            emit_call(g.update_asks(t, s["pool"][[int(rng.integers(0, len(s["pool"])))]]))
            emit_pass("lean_incr")
            emit_call(("ask_on", dict(idx=t)))
            z = np.flatnonzero(h.asks["max_group_size"] == 0).astype(np.uint32)
            if len(z):
                emit_call(g.update_asks(z, g.ask_rows(len(z), edge=0)))
            emit_call(g.delta("append_asks", s["edge"][:1].copy(), n=len(h.asks) + 1, cap=None))
            emit_pass("lean_incr")
            emit_pass("proximity_incr")     # refused: the appended max_group_size 0 ask
            return True
        if n_passes >= 16 and "missing" not in done:
            done.add("missing")
            t = np.array([int(rng.integers(0, T))], dtype=np.uint32)
            emit_call(g.delta("update_asks", s["edge"][5 + slot % 2:6 + slot % 2].copy(), idx=t))
            emit_call(g.restore_refused("missing"))
            emit_pass(["lean_incr", "auction", "certificate", "warm"][slot % 4])
            return True
        if n_passes >= 28 and h.cutoff < 1000 and "removed_held" not in done:
            # the removed asks that held a worker decide the cutoff: shrink past held asks, then write (unchanged) kept
            # rows until the changes without them reach the cutoff and with them pass it; a warm pass, then a repair
            # pass, must both run cold
            done.add("removed_held")
            for kind in ("warm", "repair"):
                all_on()
                emit_pass("auction")
                cut_held(3)
                if h.auc_state and h.removed_held:
                    base = h.n_changes() - h.removed_held
                    free = np.setdiff1d(np.arange(h.n_kept), sorted(h.rows))
                    u = rng.choice(free, max(0, h.cutoff - base), replace=False).astype(np.uint32)
                    if len(u):
                        u.sort()
                        emit_call(("update", dict(idx=u, a=h.wa[u].copy(), b=h.wb[u].copy(), lat=None, lon=None)))
                emit_pass(kind)
            return True
        if n_passes >= 36 and "shrink_held" not in done:
            # shrink past asks that hold auction workers, then warm and repair passes; shrink and grow back to the
            # same size before a certificate, which is refused
            done.add("shrink_held")
            all_on()
            emit_pass("auction")
            cut_held(4)
            emit_pass("warm")
            cut_held(2)
            emit_pass("repair")
            emit_call(("shrink_asks", dict(n=len(h.asks) - 2)))
            emit_call(g.delta("append_asks", g.ask_rows(2, missing=False), n=len(h.asks) + 2, cap=None))
            emit_pass("certificate")        # refused: the ask table was resized since the last auction pass
            return True
        n0 = len(events)
        if scripted_demand(n_passes) or scripted_splice(n_passes):   # on top of the history's length
            extra[0] += len([e for e in events[n0:] if e[0] != "probe"])
            return True
        if n_passes >= 24 and h.cutoff < 1000 and "e_rows" not in done:
            # appended asks alone past the cutoff: e_rows = ceil(|E| W / T) > PM_TUNE_INCR
            done.add("e_rows")
            emit_pass("lean")
            k = -(-(h.cutoff + 1) * len(h.asks) // h.n_workers) + 1
            emit_call(g.delta("append_asks", g.ask_rows(k, missing=False), n=len(h.asks) + k, cap=None))
            emit_pass("lean_incr")
            emit_call(("shrink_asks", dict(n=len(h.asks) - k)))
            emit_pass("lean_incr")          # the workers whose stored first ask was appended have none now
            return True
        return False

    def cut_held(j):                     # past the last j asks that hold a worker (at most 20 asks)
        held = h.held_asks()
        k = len(h.asks) - int(held[-j]) if len(held) >= j else 3
        emit_call(("shrink_asks", dict(n=len(h.asks) - min(max(k, 1), 20))))

    def demand_held(k, value):
        """Demand `value` on up to k asks that hold a worker (others when fewer hold one)."""
        d = h.d.copy()
        held = h.held_asks()
        pool = held if len(held) else np.arange(len(h.asks))
        idx = rng.choice(pool, min(k, len(pool)), replace=False)
        d[idx] = value
        emit_call(("demand", dict(d=d)))
        return idx

    def write_unchanged(n):
        """n unchanged kept rows no change lists yet (R0 grows by n, nothing else changes)."""
        free = np.setdiff1d(np.arange(h.n_kept), sorted(h.rows))
        u = np.sort(rng.choice(free, max(0, n), replace=False)).astype(np.uint32)
        if len(u):
            emit_call(("update", dict(idx=u, a=h.wa[u].copy(), b=h.wb[u].copy(), lat=None, lon=None)))

    def ones():
        if (h.d > 1).any():
            emit_call(("demand", dict(d=np.ones(len(h.asks), dtype=np.uint32))))

    def slot_state(k=8, value=3):
        """A stored state with demand `value` on asks that held a worker: a cold pass, the demands, a warm pass."""
        all_on()
        emit_pass("auction")
        demand_held(k, value)
        emit_pass("auction")

    def scripted_demand(n_passes):
        """The demand and restore steps every history makes once (each from its pass count on)."""
        if n_passes >= 6 and "restore_refusals" not in done:
            # refused exports and restores: without a state, with a demand above 1, with disabled asks
            done.add("restore_refusals")
            choices = [p for p in PARAMS if p != h.params]
            emit_call(("auction_params", dict(params=choices[int(rng.integers(0, len(choices)))])))
            emit_call(g.restore_refused("export_no_state"))
            all_on()
            emit_pass("auction")
            for case in ("length_w", "length_t", "worker", "price_neg", "price_high"):
                emit_call(g.restore_refused(case))
            demand_held(4, 2)
            emit_call(g.restore_refused("export_demand"))
            emit_call(g.restore_refused("demand"))
            ones()
            emit_call(("ask_off", dict(idx=np.array([int(rng.integers(0, len(h.asks)))], dtype=np.uint32))))
            emit_call(g.restore_refused("disabled"))
            return True
        if n_passes >= 14 and "mixed_window" not in done:
            # one window of mixed changes before a warm pass, then again before a repair pass
            done.add("mixed_window")
            slot_state()
            for kind in ("warm", "repair"):
                emit_call(g.call("demand"))
                big = np.flatnonzero(h.d > 1)
                held = np.intersect1d(h.held_asks(), big)
                t = held if len(held) else big if len(big) else h.held_asks()
                emit_call(g.update_asks(np.array([t[int(rng.integers(0, len(t)))]], dtype=np.uint32)))
                emit_call(g.delta("append_asks", g.ask_rows(2, missing=False), n=len(h.asks) + 2, cap=None))
                cut_held(2)
                i = np.array([int(rng.integers(0, len(h.asks)))], dtype=np.uint32)
                emit_call(("ask_off", dict(idx=i)))
                emit_call(("ask_on", dict(idx=i)))
                emit_call(g.call("update"))
                all_on()
                emit_pass(kind)
            return True
        if n_passes >= 18 and "chain" not in done:
            # 3 -> 1 -> 3 on held asks before one warm pass (past the cutoff by the chain's added slots under a small
            # PM_TUNE_INCR); then a worker shrink before a demand cut whose freed workers lie past n_kept
            done.add("chain")
            slot_state(6, 3)
            d3 = h.d.copy()
            idx = np.flatnonzero(h.d == 3)
            emit_call(("demand", dict(d=np.where(h.d == 3, 1, h.d).astype(np.uint32))))
            emit_call(("demand", dict(d=d3)))
            if h.cutoff < 1000 and h.auc_state:
                write_unchanged(h.cutoff + 1 - h.n_changes())
            emit_pass("warm")
            all_on()
            demand_held(6, 3)
            emit_pass("warm")
            if h.auc_state:   # the held slot workers past their ask's first slot, highest first
                off = ad.offsets(h.d)
                cand = [(int(h.assigned[s_]), t) for t in np.flatnonzero(h.d > 1)
                        for s_ in range(off[t] + 1, off[t + 1]) if h.assigned[s_] != NONE]
                cand = [c for c in cand if c[0] >= h.n_workers - 200]
                if cand:
                    w, t = max(cand)
                    emit_call(("shrink", dict(n=w, rank=rng.permutation(w).astype(np.uint32))))
                    d = h.d.copy()
                    d[t] = 1
                    emit_call(("demand", dict(d=d)))
                    if h.cutoff < 1000:
                        write_unchanged(h.cutoff - h.n_changes())
            emit_pass("warm")
            return True
        if n_passes >= 22 and shape == "mixed" and "d_over_w" not in done:
            # more slots than workers: a cold pass and a warm pass with D > W.  Most of the slots go to the ask with the
            # fewest feasible workers (they withdraw at once), so the passes stay short: D > W does not make a price war
            done.add("d_over_w")
            all_on()
            T = len(h.asks)
            d = np.where(np.isin(np.arange(T), h.held_asks()[:20]), 2, 1).astype(np.uint32)
            t = int(np.argmin(h.F().sum(axis=1)))
            d[t] = h.n_workers + 10 - (int(d.sum()) - int(d[t]))
            emit_call(("demand", dict(d=d)))
            emit_pass("auction")
            emit_call(g.call("update"))
            emit_pass("warm")
            ones()
            return True
        if n_passes >= 30 and "after_set_asks" not in done:
            # demands above 1, then a table swap: the next pass is one with demand 1, and the export works after it
            done.add("after_set_asks")
            all_on()
            demand_held(6, 3)
            emit_call(g.call("set_asks"))
            emit_pass("auction")
            emit_call(g.restore("own"))
            return True
        if n_passes >= 34 and "back_to_one" not in done:
            # demands above 1, then all 1 under a stored state: certificate, export and restore; then demands again
            done.add("back_to_one")
            slot_state(6, 2)
            ones()
            emit_pass("certificate")
            emit_call(g.restore("own"))
            demand_held(6, 3)
            emit_pass("warm")
            return True
        if n_passes >= 40 and "restore_tracker" not in done:
            # a restore between two incremental passes, a worker resize before an own export, a restore followed by a
            # certificate, and an own restore right after its pass
            done.add("restore_tracker")
            all_on()
            ones()
            emit_pass("auction")
            emit_call(g.restore("own"))
            emit_pass("lean")
            emit_call(g.call("update"))
            emit_call(g.restore("adversarial"))
            if h.eval:   # cut past the last stored first ask (its workers have none now) and append as many asks back
                T = len(h.asks)
                last = int(h.eval_ff[h.eval_ff != NONE].max(initial=0))
                if 0 < last < T:
                    emit_call(("shrink_asks", dict(n=last)))
                    emit_call(g.delta("append_asks", g.ask_rows(T - last, missing=False), n=T, cap=None))
            emit_pass("lean_incr")
            emit_call(g.call("shrink" if h.n_workers >= 2000 else "grow"))
            emit_call(g.restore("own"))     # refused as exported, then trimmed
            emit_call(g.call("caps"))
            emit_call(g.restore("stale"))
            emit_pass("certificate")
            emit_named("move")
            emit_pass("lean_incr")
            emit_pass("warm")
            return True
        if n_passes >= 26 and h.cutoff < 1000 and "freed_decides" not in done:
            # freed slot workers decide the cutoff: cut the demands of held asks, then write unchanged kept rows until the
            # changes without them reach the cutoff (the pass runs cold), or stop where the changes with them reach it
            # (the pass runs warm); for a warm pass and a repair pass
            done.add("freed_decides")
            for kind in ("warm", "repair"):
                for over in (True, False):
                    slot_state(8, 3)
                    emit_call(("demand", dict(d=np.minimum(h.d, 1 + (h.d > 1)).astype(np.uint32))))
                    if h.auc_state and h.removed_held:
                        base = h.n_changes() - h.removed_held
                        write_unchanged(h.cutoff - base - (0 if over else h.removed_held))
                    emit_pass(kind)
            return True
        return False

    def remove(idx):
        emit_call(("remove_asks", dict(idx=rng.permutation(np.asarray(idx, dtype=np.int64)).astype(np.uint32))))

    def insert(before, rows, cap=None):
        emit_call(g.delta("insert_asks", np.ascontiguousarray(rows).copy(), before=np.asarray(before, dtype=np.uint32),
                          cap=cap))
        return np.asarray(before, dtype=np.int64) + np.arange(len(before))

    def flush():
        """The passes a refusal is to be followed by, before a step's own passes."""
        for _ in range(2):
            if follow:
                kind = follow.pop(0)
                if kind in AUCTION:
                    all_on()
                emit_pass(kind)

    def evaluated():
        """A stored evaluation from a lean pass (again after one a missing pattern refused)."""
        flush()
        emit_pass("lean")
        if not h.eval:
            emit_pass("lean")
        return h.eval

    def first_asks():
        """The stored first asks with a row after them, the ones most workers store first."""
        ff = h.eval_ff[h.eval_ff != NONE].astype(np.int64)
        c = np.bincount(ff, minlength=len(h.asks))
        order = np.argsort(-c, kind="stable")
        return [int(t) for t in order[:8] if c[t] > 0 and t + 1 < len(h.asks)]

    def scripted_splice(n_passes):
        """The remove and insert steps every history makes once (each from its pass count on)."""
        s = h.s
        if n_passes >= 3 and "splice_refusals" not in done:
            done.add("splice_refusals")
            for case in SPLICE_REFUSALS:
                emit_call(g.delta("ask_delta_refused", g.ask_rows(2, edge=0), T=len(h.asks), case=case))
            for case in DELTA_REFUSALS:   # each once too (random draws may miss one); rows drawn from nothing random
                emit_call(("ask_delta_refused", dict(rows=s["pool"][:2].copy(), opts=h.opts, own=False, T=len(h.asks),
                                                     case=case)))
            return True
        if n_passes >= 5 and "heir" not in done:
            # remove the asks most workers store first; then one whose heir was disabled, replaced or inserted since
            # the stored evaluation; each before an incremental pass
            done.add("heir")
            for variant in ("plain", "disabled", "replaced", "inserted"):
                if not evaluated() or not first_asks():
                    continue
                first = first_asks()
                t = first[0]
                if variant == "plain":
                    remove(first[:2] + first[:1])
                else:
                    if variant == "disabled":
                        emit_call(("ask_off", dict(idx=np.array([t + 1], dtype=np.uint32))))
                    elif variant == "replaced":
                        emit_call(g.update_asks(np.array([t + 1], dtype=np.uint32), g.ask_rows(1, edge=0)))
                    else:
                        insert([t + 1], g.ask_rows(1, edge=0))
                    remove([t])
                emit_pass("lean_incr")
            return True
        if n_passes >= 7 and "no_heir" not in done:
            # remove a stored first ask with every row after it (and one row before it): its workers store NONE
            done.add("no_heir")
            if evaluated():
                T = len(h.asks)
                ff = h.eval_ff[h.eval_ff != NONE]
                if len(ff):
                    f = int(ff.max())
                    rm = list(range(f, T)) + ([int(rng.integers(0, f))] if f else [])
                    remove(rm)
                    emit_pass("lean_incr")
                    insert(np.full(len(rm), len(h.asks)), g.ask_rows(len(rm), edge=0, missing=False))
            return True
        if n_passes >= 10 and "insert_first" not in done:
            # a row just before a stored first ask that accepts the same workers (the ask's own row)
            done.add("insert_first")
            if evaluated() and first_asks():
                t = first_asks()[0]
                insert([t], h.asks[[t]])
                emit_pass("lean_incr")
            return True
        if n_passes >= 16 and "crossings" not in done:
            # inside one incremental window: rows that turn the fast predicate off, push the feature dictionary past 64
            # and make proximity refuse, inserted and removed again; then each alone before a materialised or
            # proximity pass, and removed before the next
            done.add("crossings")
            if len(h.max0_on()):
                emit_call(("ask_off", dict(idx=h.max0_on().astype(np.uint32))))
            evaluated()
            at = []
            for row in (s["edge"][3:4], s["feature"], s["edge"][0:1]):
                a = int(insert(rng.integers(0, len(h.asks) + 1, 1), row)[0])
                at = [x + (x >= a) for x in at] + [a]
            remove(at)
            emit_pass("lean_incr")
            for row, kinds in ((s["feature"], ("materialized", "materialized")), (s["edge"][3:4], ("materialized",) * 2),
                               (s["edge"][0:1], ("proximity", "proximity"))):
                a = insert(np.sort(rng.integers(0, len(h.asks) + 1, 1)), row)
                emit_pass(kinds[0])
                remove(a)
                emit_pass(kinds[1])
            return True
        if n_passes >= 20 and "splice_chain" not in done:
            # 3 -> 2 on held asks, a removal past them and an insertion at the front (they move up one row), 2 -> 3,
            # then one warm pass: the kept slots chain through the remap
            done.add("splice_chain")
            slot_state(6, 3)
            big = np.flatnonzero(h.d > 1)
            if len(big):
                emit_call(("demand", dict(d=np.where(h.d > 1, 2, h.d).astype(np.uint32))))
                free = np.setdiff1d(np.arange(len(h.asks)), big)
                free = free[free > big.max()] if (free > big.max()).any() else free
                r = int(free[int(rng.integers(0, len(free)))])
                remove([r])
                insert([0], g.ask_rows(1, missing=False))
                d = h.d.copy()
                d[big - (big > r) + 1] = 3
                emit_call(("demand", dict(d=d)))
                if h.cutoff < 1000 and h.auc_state:   # one change past the cutoff, the kept and inserted slots counted
                    write_unchanged(h.cutoff + 1 - h.n_changes())
            emit_pass("warm")
            ones()
            return True
        if n_passes >= 24 and "splice_certificate" not in done:
            # the certificate refuses after a splice until the next auction pass
            done.add("splice_certificate")
            all_on()
            emit_pass("auction")
            remove([int(rng.integers(0, len(h.asks)))])
            emit_pass("certificate")
            emit_pass("auction")
            emit_pass("certificate")
            return True
        if n_passes >= 32 and h.cutoff < 1000 and "splice_held" not in done:
            # a worker shrink below a worker a slot holds, then the removal of held asks of demand > 1: freed slots
            # below and above n_kept; unchanged rows written until removed_held decides the cutoff
            done.add("splice_held")
            for kind, over in (("warm", slot % 2 == 0), ("repair", slot % 2 == 1)):
                slot_state(8, 3)
                if not h.auc_state:
                    continue
                off = ad.offsets(h.d)
                cand = [(int(h.assigned[s_]), int(t)) for t in np.flatnonzero(h.d > 1)
                        for s_ in range(off[t], off[t + 1]) if h.assigned[s_] != NONE]
                high = [c for c in cand if c[0] >= h.n_workers - 200]
                rm = sorted({t for _, t in cand})[:3]
                if high:
                    w, t = max(high)
                    emit_call(("shrink", dict(n=w, rank=rng.permutation(w).astype(np.uint32))))
                    rm = sorted(set(rm[:2]) | {t})
                if rm:
                    remove(rm)
                if h.auc_state and h.removed_held:
                    base = h.n_changes() - h.removed_held
                    write_unchanged(h.cutoff - base - (0 if over else h.removed_held))
                emit_pass(kind)
            ones()
            return True
        return False

    def mine(a, b):
        """An unseen (pass -> pass) pair this slot is to make."""
        return a in PASSES and (a, b) not in seen_pass and (PASSES.index(a) * len(PASSES) + PASSES.index(b)) % n_slots == slot

    follow = []
    extra = [0]                              # the events of the demand and restore steps
    emit_pass("lean_incr")
    while len([e for e in events if e[0] != "probe"]) - extra[0] < n_calls:
        for _ in range(2):                  # what a refusal left, before a scripted step makes a new state
            if follow:
                kind = follow.pop(0)
                if kind in AUCTION:
                    all_on()
                emit_pass(kind)
        if len([e for e in events if e[0] == "pass"]) >= domain_at // 2 and "domain" not in done \
                and h.params != DOMAIN_EDGE:
            done.add("domain")
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
            emit_call(g.restore_refused("domain"))
            emit_pass("warm")                       # refused: the stored state stays
            emit_pass("lean_incr")
            emit_pass("certificate")                # refused too
            emit_call(("update", dict(idx=row, a=old[0], b=old[1], lat=None, lon=None)))
            emit_pass("repair" if rng.random() < 0.5 else "warm")
            emit_call(("auction_params", dict(params=PARAMS[int(rng.integers(0, len(PARAMS)))])))
            continue
        n_passes = len([e for e in events if e[0] == "pass"])
        if scripted(n_passes):
            continue
        if n_passes >= 12 and "b12" not in done:
            # warm or repair after reference passes of both modes, with asks left disabled across them
            done.add("b12")
            all_on()
            emit_pass("auction")
            off = np.union1d(rng.choice(len(h.asks), 5, replace=False), h.max0_on())
            emit_call(("ask_off", dict(idx=off.astype(np.uint32))))
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
            emit_named(names[int(rng.choice(len(names), p=p / p.sum()))])
        if n_passes >= 20 and "b20" not in done:
            done.add("b20")
            # past the cutoff between two reference passes (a full pass under a small PM_TUNE_INCR), and a side column
            emit_pass("lean")
            u = np.unique(rng.choice(h.n_workers, min(h.cutoff + 20, 120), replace=False)).astype(np.uint32)
            a, b = g.rows(len(u))
            emit_call(("update", dict(idx=u, a=a, b=b, lat=None, lon=None)))
            emit_call(g.call("addr_rank"))
            emit_pass("lean_incr")
            continue
        if n_passes >= 26 and "b26" not in done:
            done.add("b26")
            # past the cutoff between two auction passes (a cold PM_AUCTION_WARM pass under a small PM_TUNE_INCR)
            if not h.mask.all():
                emit_call(("ask_on", dict(idx=np.flatnonzero(~h.mask).astype(np.uint32))))
            emit_pass("auction")
            u = np.unique(rng.choice(h.n_workers, min(h.cutoff + 20, 120), replace=False)).astype(np.uint32)
            a, b = g.rows(len(u))
            emit_call(("update", dict(idx=u, a=a, b=b, lat=None, lon=None)))
            emit_pass("warm")
            continue
        if n_passes >= 34 and "b34" not in done:
            done.add("b34")
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
            emit_named(c)
        elif targets and rng.random() < 0.85:
            tw = np.array([0.5 if c in RARE else 1.0 for c, _ in targets])
            c, kind = targets[int(rng.choice(len(targets), p=tw / tw.sum()))]
            if c == "ask_on" and h.mask.all():
                emit_call(g.call("ask_off"))
            if c != "shrink" or h.n_workers >= 2000:
                emit_named(c)
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
            if len(h.max0_on()) and rng.random() < 0.75:
                emit_call(("ask_off", dict(idx=h.max0_on().astype(np.uint32))))
        emit_pass(kind)
    while scripted_demand(1 << 30) or scripted_splice(1 << 30):   # the steps the loop had no room for
        pass
    for c, kind in must:                    # the slot's pairs the loop had no room for
        emit_named(c)
        emit_pass(kind)
        flush()
    for i in range(slot, len(PASSES) ** 2, n_slots):
        a, b = PASSES[i // len(PASSES)], PASSES[i % len(PASSES)]
        if (a, b) not in seen_pass:
            if last_pass != a:
                emit_pass(a)
            emit_pass(b)
    flush()
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
    """(slot assignment, prices, forward rounds, released, (phases, reverse rounds, reverse bids)) of an auction pass,
    all on the twin tables (row t repeated d[t] times; the ask table itself with every demand 1): the oracle's cold
    pass, the reverse checker, the warm checker or the repair checker, from the slot-level stored state."""
    import auction_repair_checker as rp
    import auction_reverse_checker as rc

    S, E, dv = h.params
    ap = h.wb["ext_ask_price"]
    if warm:
        F, cap = h.slot_F(), h.slot_cap()
        if kind == "warm":
            a, p, n, rel = wc.warm(F, ap, cap, S, h.price, h.assigned, h.n_kept, h.changed_rows(), h.changed_slots())
            return a, p, n, len(rel), (0, 0, 0)
        out = rp.repair(F, ap, cap, S, h.price, h.assigned, h.n_kept, h.changed_rows(), h.changed_slots())
        return out["assigned"], out["price"], out["fwd"], len(out["released"]), (1, out["rev"], out["bids"])
    if kind == "reverse":
        a, p, fwd, rev, bids, phases = rc.scaled(h.slot_F(), ap, h.slot_cap(), S, E, dv, reverse_rounds=True)
        return a, p, fwd, 0, (phases, rev, bids)
    a, p, n = orc.soa_auction(h.wa, h.wb, np.repeat(h.asks, h.d), h.opts, h.bits, h.words, h.slot_cap(), S, E, dv,
                              reputation=h.reputation, min_reputation=h.slot_floors())
    return a, p, n, 0, (0, 0, 0)


def expect_result(h: History, a_slots):
    """Every array pm_fetch_result returns after an auction pass whose slot assignment is a_slots: its fold, one group
    per holding ask in ask order, members sorted (with every demand 1, one solo group per held ask)."""
    return ad.result_arrays(a_slots, h.d, h.wb["ext_ask_price"], h.n_workers)


def expect_certificate(h: History):
    """The certificate of the stored slot state on the current tables (per ask row terms weighted by the demands)."""
    return ad.demand_certificate(h.F(), h.wb["ext_ask_price"], h.cap, h.d, h.params[0], h.price, h.assigned)
