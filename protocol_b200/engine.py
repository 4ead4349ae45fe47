"""Python host wrapper over the C ABI (include/prime_match.h).

Mirrors, for the hot path only, the reference's NodeGroupsPlugin surface:
`Engine.match()` is one `try_form_new_groups` pass
(crates/orchestrator/src/plugins/node_groups/mod.rs:478-628) over the resident
worker and ask tables.  All compute happens in the CUDA library; this module is
plumbing (numpy views over pinned/host buffers, error mapping).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import abi
from ._lib import PrimeMatchError, load


def _ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)


class Interner:
    """pm_interner: model-string interning + acceptance table (node.rs:463-484)."""

    def __init__(self):
        self._lib = load()
        self._h = self._lib.pm_interner_create()
        if not self._h:
            raise MemoryError("pm_interner_create failed")

    def close(self):
        if self._h:
            self._lib.pm_interner_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def model(self, s: str) -> int:
        return self._lib.pm_intern_model(self._h, s.encode())

    def pattern(self, s: str) -> int:
        return self._lib.pm_intern_pattern(self._h, s.encode())

    def table(self):
        bits = C.POINTER(C.c_uint32)()
        npat, nmod, words = C.c_uint32(), C.c_uint32(), C.c_uint32()
        rc = self._lib.pm_interner_table(self._h, C.byref(bits), C.byref(npat), C.byref(nmod), C.byref(words))
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, "pm_interner_table")
        n = max(npat.value, 1) * words.value
        arr = np.ctypeslib.as_array(bits, shape=(n,)).copy()
        return arr, npat.value, nmod.value, words.value

    def parse(self, s: str, max_opts: int = 64):
        """ComputeRequirements::from_str -> (ask_row: np.void ASK, opts: np.ndarray GPU_OPT)."""
        ask = abi.PmAsk()
        opts = (abi.PmGpuOpt * max_opts)()
        n = C.c_uint32()
        err = C.create_string_buffer(256)
        rc = self._lib.pm_parse_requirements(s.encode(), self._h, C.byref(ask), opts, max_opts, C.byref(n), err, 256)
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, err.value.decode())
        a = np.zeros(1, dtype=abi.ASK)
        for f in abi.ASK.names:
            a[f] = getattr(ask, f)
        o = np.zeros(n.value, dtype=abi.GPU_OPT)
        for i in range(n.value):
            for f in abi.GPU_OPT.names:
                o[f][i] = getattr(opts[i], f)
        return a[0], o


def sort_configs(min_group_size, has_requirements) -> np.ndarray:
    """Priority order of NodeGroupsPlugin::new_with_policy (mod.rs:150-164)."""
    lib = load()
    mn = np.ascontiguousarray(min_group_size, dtype=np.uint32)
    hr = np.ascontiguousarray(has_requirements, dtype=np.uint8)
    perm = np.empty(len(mn), dtype=np.uint32)
    rc = lib.pm_sort_configs(_ptr(mn), _ptr(hr), len(mn), _ptr(perm))
    if rc != abi.PM_OK:
        raise PrimeMatchError(rc, "pm_sort_configs")
    return perm


@dataclass
class MatchResult:
    worker_group: np.ndarray
    worker_ask: np.ndarray
    group_ask: np.ndarray
    group_off: np.ndarray
    group_members: np.ndarray
    ask_best: np.ndarray
    ask_count: np.ndarray
    stats: dict

    @property
    def n_groups(self) -> int:
        return len(self.group_ask)

    def groups(self):
        """[(ask, [workers...])] in creation order."""
        return [
            (int(self.group_ask[g]), self.group_members[self.group_off[g]:self.group_off[g + 1]].tolist())
            for g in range(self.n_groups)
        ]


class Engine:
    def __init__(self, device: int = 0, cost_tile_bytes: int = 0, timing: bool = False,
                 shard_first: int = 0, shard_count: int = 0, stream: int = 0):
        self._lib = load()
        cfg = abi.PmCfg(abi.PM_ABI_VERSION, device, abi.PM_CFG_TIMING if timing else 0, 0,
                        cost_tile_bytes, shard_first, shard_count, stream or None)
        h = C.c_void_p()
        rc = self._lib.pm_create(C.byref(cfg), C.byref(h))
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, (self._lib.pm_last_error(None) or b"").decode())
        self._h = h
        self.n_workers = 0
        self._auction_workers = 0   # workers of the last auction pass (auction_state)
        self.n_asks = 0

    def close(self):
        if getattr(self, "_h", None):
            self._lib.pm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, (self._lib.pm_last_error(self._h) or b"").decode())

    # ---- tables -----------------------------------------------------------
    def set_asks(self, asks: np.ndarray, opts: np.ndarray):
        asks = np.ascontiguousarray(asks, dtype=abi.ASK)
        opts = np.ascontiguousarray(opts, dtype=abi.GPU_OPT)
        self._check(self._lib.pm_set_asks(self._h, _ptr(asks), len(asks), _ptr(opts), len(opts)))
        self.n_asks = len(asks)

    def set_ask_enabled(self, idx, enabled):
        """Enable (True) or disable (False) the asks idx (pm_set_ask_enabled): a disabled ask behaves as if it were
        absent from the table; result indices stay those of the full table."""
        idx, en = _ask_enabled_args(idx, enabled)
        self._check(self._lib.pm_set_ask_enabled(self._h, _ptr(idx), _ptr(en), len(idx)))

    def update_asks(self, idx, asks: np.ndarray, opts: np.ndarray | None = None):
        """Replace the ask rows idx (pm_update_asks); asks["opt_off"] / ["n_opts"] index `opts`.  A replaced row keeps
        its enabled flag, price cap and reputation floor; the stored evaluation and auction state are kept."""
        idx, asks, opts = _ask_delta_args(idx, asks, opts)
        self._check(self._lib.pm_update_asks(self._h, _ptr(idx), _ptr(asks), len(idx), _ptr(opts), len(opts)))

    def resize_asks(self, n: int, added: np.ndarray | None = None, opts: np.ndarray | None = None):
        """Shrink the ask table to its first n rows, or append rows `added` (options in `opts`) at the lowest
        priorities, enabled, with cap 0 and floor 0 (pm_resize_asks)."""
        added = np.ascontiguousarray(np.zeros(0, dtype=abi.ASK) if added is None else added, dtype=abi.ASK)
        opts = np.ascontiguousarray(np.zeros(0, dtype=abi.GPU_OPT) if opts is None else opts, dtype=abi.GPU_OPT)
        self._check(self._lib.pm_resize_asks(self._h, n, _ptr(added) if len(added) else None, _ptr(opts), len(opts)))
        self.n_asks = n

    def remove_asks(self, idx):
        """Remove the ask rows idx (any order; a repeated index removes its row once); the rows after them move up,
        order kept (pm_remove_asks).  The stored evaluation and auction state are kept, remapped to the new indices."""
        idx = _remove_args(idx)
        self._check(self._lib.pm_remove_asks(self._h, _ptr(idx) if len(idx) else None, len(idx)))
        self.n_asks -= len(np.unique(idx))

    def insert_asks(self, before, asks: np.ndarray, opts: np.ndarray | None = None):
        """Insert rows `asks` (options in `opts`) before the current rows before[i] (non-decreasing, n_asks = append;
        rows with equal before[] keep their order), enabled, with cap 0, floor 0 and demand 1 (pm_insert_asks)."""
        before, asks, opts = _insert_args(before, asks, opts)
        self._check(self._lib.pm_insert_asks(self._h, _ptr(before) if len(before) else None, _ptr(asks) if len(asks) else None,
                                             len(before), _ptr(opts), len(opts)))
        self.n_asks += len(before)

    def set_model_table(self, bits: np.ndarray, n_patterns: int, n_models: int, words: int):
        bits = np.ascontiguousarray(bits, dtype=np.uint32)
        self._check(self._lib.pm_set_model_table(self._h, _ptr(bits), n_patterns, n_models, words))

    def set_workers(self, a: np.ndarray, b: np.ndarray):
        a = np.ascontiguousarray(a, dtype=abi.WORKER_A)
        b = np.ascontiguousarray(b, dtype=abi.WORKER_B)
        assert len(a) == len(b)
        self._check(self._lib.pm_set_worker_count(self._h, len(a)))
        self._check(self._lib.pm_upsert_workers(self._h, _ptr(a), _ptr(b), 0, len(a)))
        self.n_workers = len(a)
        self.sync()

    def upsert_workers(self, a: np.ndarray, b: np.ndarray, first: int = 0, sync: bool = True):
        """a/b must stay alive (and ideally pinned) until sync()."""
        self._check(self._lib.pm_upsert_workers(self._h, _ptr(a), _ptr(b), first, len(a)))
        if sync:
            self.sync()

    def set_locations(self, lat: np.ndarray, lon: np.ndarray):
        lat = np.ascontiguousarray(lat, dtype=np.float64)
        lon = np.ascontiguousarray(lon, dtype=np.float64)
        self._check(self._lib.pm_set_worker_locations(self._h, _ptr(lat), _ptr(lon), 0, len(lat)))
        self.sync()

    def set_addr_rank(self, rank: np.ndarray):
        rank = np.ascontiguousarray(rank, dtype=np.uint32)
        self._check(self._lib.pm_set_worker_addr_rank(self._h, _ptr(rank), 0, len(rank)))
        self.sync()

    def resize_workers(self, n: int):
        self._check(self._lib.pm_resize_workers(self._h, n))
        self.n_workers = n

    def update_workers(self, idx, a, b, lat=None, lon=None):
        """Scatter changed rows into the resident table (pm_update_workers)."""
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        a = np.ascontiguousarray(a, dtype=abi.WORKER_A)
        b = np.ascontiguousarray(b, dtype=abi.WORKER_B)
        la = np.ascontiguousarray(lat, dtype=np.float64) if lat is not None else None
        lo = np.ascontiguousarray(lon, dtype=np.float64) if lon is not None else None
        self._check(self._lib.pm_update_workers(self._h, _ptr(idx), _ptr(a), _ptr(b), _ptr(la) if la is not None else None,
                                                _ptr(lo) if lo is not None else None, len(idx)))
        self.sync()

    def remove_workers(self, idx):
        """Remove the worker rows idx (any order; a repeated index removes its row once); the rows after them move up,
        order kept (pm_remove_workers).  The stored evaluation and auction state are kept, remapped to the new indices."""
        idx = _remove_args(idx)
        self._check(self._lib.pm_remove_workers(self._h, _ptr(idx) if len(idx) else None, len(idx)))
        self.n_workers -= len(np.unique(idx))
        if self._auction_workers:   # the stored auction state follows the splice: one price per current row
            self._auction_workers = self.n_workers

    def insert_workers(self, before, a, b, lat=None, lon=None):
        """Insert rows a[i], b[i] before the current rows before[i] (non-decreasing, n_workers = append; rows with equal
        before[] keep their order), at (lat, lon) or (0, 0), address rank 0 and reputation 0 (pm_insert_workers)."""
        before, a, b, la, lo = _worker_insert_args(before, a, b, lat, lon)
        self._check(self._lib.pm_insert_workers(self._h, _ptr(before) if len(before) else None, _ptr(a) if len(a) else None,
                                                _ptr(b) if len(b) else None, _ptr(la) if la is not None else None,
                                                _ptr(lo) if lo is not None else None, len(before)))
        self.n_workers += len(before)
        if self._auction_workers:
            self._auction_workers = self.n_workers

    def table_version(self) -> int:
        return int(self._lib.pm_table_version(self._h))

    def set_flags(self, idx: np.ndarray, flags: np.ndarray):
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        flags = np.ascontiguousarray(flags, dtype=np.uint32)
        self._check(self._lib.pm_set_flags(self._h, _ptr(idx), _ptr(flags), len(idx)))
        self.sync()

    # ---- north-star extension columns (PM_MODE_AUCTION only) ---------------
    def set_price_caps(self, caps: np.ndarray):
        caps = np.ascontiguousarray(caps, dtype=np.uint32)
        self._check(self._lib.pm_set_ask_price_caps(self._h, _ptr(caps), len(caps)))

    def set_worker_reputation(self, reputation: np.ndarray, first: int = 0):
        """north_star worker column `reputation` (u32 per worker); read by PM_MODE_AUCTION through the per-ask floor."""
        reputation = np.ascontiguousarray(reputation, dtype=np.uint32)
        self._check(self._lib.pm_set_worker_reputation(self._h, _ptr(reputation), first, len(reputation)))

    def set_min_reputation(self, floors: np.ndarray):
        floors = np.ascontiguousarray(floors, dtype=np.uint32)
        self._check(self._lib.pm_set_ask_min_reputation(self._h, _ptr(floors), len(floors)))

    def set_ask_demand(self, demand: np.ndarray):
        """Workers each ask may take in PM_MODE_AUCTION (pm_set_ask_demand; u32 >= 1 per ask, default 1): ask t behaves as
        its row repeated demand[t] times, and the result holds one group per ask with its workers."""
        demand = np.ascontiguousarray(demand, dtype=np.uint32)
        self._check(self._lib.pm_set_ask_demand(self._h, _ptr(demand), len(demand)))

    def set_auction_params(self, cost_scale: int = 1, eps_start: int = 1, eps_div: int = 4):
        self._check(self._lib.pm_set_auction_params(self._h, cost_scale, eps_start, eps_div))

    def auction_state(self, prices: bool = True):
        """The last auction pass (pm_auction_state): (prices i64[n_workers of that pass] or None, started warm, asks
        released by its warm start)."""
        price = np.zeros(self._auction_workers, dtype=np.int64) if prices else None
        warm, released = C.c_uint32(), C.c_uint32()
        self._check(self._lib.pm_auction_state(self._h, _ptr(price) if prices else None, C.byref(warm), C.byref(released)))
        return price, bool(warm.value), int(released.value)

    def auction_reverse_stats(self):
        """The last auction pass (pm_auction_reverse_stats): (eps phases, reverse rounds, reverse bids); all 0 for a pass
        without PM_AUCTION_REVERSE."""
        phases, rounds, bids = C.c_uint32(), C.c_uint32(), C.c_uint64()
        self._check(self._lib.pm_auction_reverse_stats(self._h, C.byref(phases), C.byref(rounds), C.byref(bids)))
        return int(phases.value), int(rounds.value), int(bids.value)

    def auction_certificate(self, ask_bound: bool = False) -> dict:
        """The certificate of the last auction pass's stored prices and assignment against the current tables
        (pm_auction_certificate): cost, bound (a lower bound on the optimum) and gap = cost - bound as Python ints, the
        hold counts, n_slack_over, max_slack, the priced-unowned sum, evals; with ask_bound, the per-ask row terms
        (int64[n_asks])."""
        cert = abi.PmAuctionCert()
        rows = np.zeros(self.n_asks, dtype=np.int64) if ask_bound else None
        self._check(self._lib.pm_auction_certificate(self._h, C.byref(cert), _ptr(rows) if ask_bound else None))
        out = {n: int(getattr(cert, n)) for n in ("n_held", "n_bad_holds", "n_shared", "n_priced_unowned", "n_slack_over",
                                                  "max_slack", "evals")}
        for n in ("cost", "bound", "gap"):
            out[n] = (int(getattr(cert, n + "_hi")) << 64) | int(getattr(cert, n + "_lo"))
        out["priced_unowned_sum"] = (int(cert.priced_unowned_hi) << 64) | int(cert.priced_unowned_lo)
        if ask_bound:
            out["ask_bound"] = rows
        return out

    def auction_assignment(self) -> np.ndarray:
        """The stored auction state's assignment (pm_auction_assignment): uint32[n_asks], the worker each ask holds or
        PM_NONE.  With auction_state()'s prices this is what auction_restore() takes."""
        out = np.zeros(self.n_asks, dtype=np.uint32)
        self._check(self._lib.pm_auction_assignment(self._h, _ptr(out)))
        return out

    def auction_restore(self, price, assigned) -> dict:
        """Audit (price i64[n_workers], assigned u32[n_asks]) against the current tables and make it the stored auction
        state (pm_auction_restore): bad, shared and over-slack holds are dropped, prices kept.  Returns the report."""
        price = np.ascontiguousarray(price, dtype=np.int64)
        assigned = np.ascontiguousarray(assigned, dtype=np.uint32)
        rep = abi.PmAuctionRestoreReport()
        self._check(self._lib.pm_auction_restore(self._h, _ptr(price), len(price), _ptr(assigned), len(assigned), C.byref(rep)))
        self._auction_workers = len(price)
        return {n: int(getattr(rep, n)) for n, _ in rep._fields_}

    def auction_slot_assignment(self) -> np.ndarray:
        """The stored auction state's assignment per slot (pm_auction_slot_assignment): uint32[D], D = sum of the ask
        demands (n_asks without demands), slot s of ask t at sum(demand[:t]) + k; a worker or PM_NONE.  With
        auction_state()'s prices this is what auction_restore_slots() takes."""
        n = C.c_uint32(0)
        self._check(self._lib.pm_auction_slot_assignment(self._h, None, C.byref(n)))
        out = np.zeros(n.value, dtype=np.uint32)
        if n.value:
            self._check(self._lib.pm_auction_slot_assignment(self._h, _ptr(out), C.byref(n)))
        return out

    def auction_restore_slots(self, price, assigned) -> dict:
        """auction_restore() per slot (pm_auction_restore_slots): with demands, what auction_restore does on the engine
        whose ask table repeats row t demand[t] times, with `assigned` (uint32[D]) as that table's assignment; report
        evals = n_asks x n_workers.  Returns the report."""
        price = np.ascontiguousarray(price, dtype=np.int64)
        assigned = np.ascontiguousarray(assigned, dtype=np.uint32)
        rep = abi.PmAuctionRestoreReport()
        self._check(self._lib.pm_auction_restore_slots(self._h, _ptr(price), len(price), _ptr(assigned), len(assigned),
                                                       C.byref(rep)))
        self._auction_workers = len(price)
        return {n: int(getattr(rep, n)) for n, _ in rep._fields_}

    # ---- the pass ---------------------------------------------------------
    def match(self, mode: int = abi.PM_MODE_FIRST_FIT):
        """pm_match.  Auction passes (PM_MODE_AUCTION) take PM_AUCTION_WARM: start from the last auction pass's state,
        releasing only the asks the changes since disturb (a cold pass without a stored state or past the cutoff); with
        PM_AUCTION_WARM | PM_AUCTION_REPAIR the warm pass keeps every stored price, raises the changed rows instead, and
        ends with reverse rounds (auction_reverse_stats: 1 phase).  PM_AUCTION_REVERSE: reverse rounds after every eps
        phase.  See prime_match.h."""
        self._check(self._lib.pm_match(self._h, mode))
        if mode & 0xFF == abi.PM_MODE_AUCTION:
            self._auction_workers = self.n_workers   # the length of the prices auction_state() returns

    def match_local(self, mode: int = abi.PM_MODE_FIRST_FIT):
        self._check(self._lib.pm_match_local(self._h, mode))

    def match_finish(self, mode: int = abi.PM_MODE_FIRST_FIT):
        self._check(self._lib.pm_match_finish(self._h, mode))

    def sync(self):
        self._check(self._lib.pm_stream_sync(self._h))

    def stats(self) -> dict:
        st = abi.PmStats()
        self._check(self._lib.pm_get_stats(self._h, C.byref(st)))
        return st.as_dict()

    def device_buffer(self, which: int):
        p, n = C.c_void_p(), C.c_size_t()
        self._check(self._lib.pm_device_buffer(self._h, which, C.byref(p), C.byref(n)))
        return p.value, n.value

    def cost_tile(self, t0: int, nt: int, n_cols: int | None = None) -> np.ndarray:
        """The materialised int64 cost rows [t0, t0+nt) x this engine's worker range."""
        n_cols = self.n_workers if n_cols is None else n_cols
        out = np.empty((nt, n_cols), dtype=np.int64)
        self._check(self._lib.pm_build_cost_tile(self._h, t0, nt, _ptr(out)))
        return out

    def fetch(self, copy: bool = True) -> MatchResult:
        r = abi.PmResult()
        self._check(self._lib.pm_fetch_result(self._h, C.byref(r)))
        return _result_views(r, copy)

    # ---- multi-GPU, one process per GPU (SURVEY 8e) -------------------------
    def set_shard(self, first: int, count: int):
        self._check(self._lib.pm_set_shard(self._h, first, count))

    def attach_comm(self, comm: "Comm | None"):
        """With a communicator attached, match() evaluates this rank's share of the workers, exchanges once
        (one packed all-gather inside the library) and runs the replicated resolution sweep."""
        self._check(self._lib.pm_attach_comm(self._h, comm._h if comm is not None else None))
        self._comm = comm   # keep it alive


def _ask_enabled_args(idx, enabled):
    """(idx, enabled) as the C call takes them; a scalar `enabled` applies to every index."""
    idx = np.ascontiguousarray(np.atleast_1d(idx), dtype=np.uint32)
    en = np.broadcast_to(np.asarray(enabled, dtype=bool), idx.shape)
    return idx, np.ascontiguousarray(en, dtype=np.uint8)


def _ask_delta_args(idx, asks, opts):
    """(idx, asks, opts) as pm_update_asks takes them; opts None = no option rows."""
    idx = np.ascontiguousarray(np.atleast_1d(idx), dtype=np.uint32)
    asks = np.ascontiguousarray(np.atleast_1d(asks), dtype=abi.ASK)
    opts = np.ascontiguousarray(np.zeros(0, dtype=abi.GPU_OPT) if opts is None else opts, dtype=abi.GPU_OPT)
    return idx, asks, opts


def _insert_args(before, asks, opts):
    """(before, asks, opts) as pm_insert_asks takes them: one row per position (the call reads len(before) rows)."""
    before, asks, opts = _ask_delta_args(before, asks, opts)
    if len(asks) != len(before):
        raise ValueError(f"insert_asks: {len(before)} positions for {len(asks)} rows")
    return before, asks, opts


def _remove_args(idx):
    return np.ascontiguousarray(np.atleast_1d(np.asarray(idx, dtype=np.int64)).astype(np.uint32))


def _worker_insert_args(before, a, b, lat, lon):
    """(before, a, b, lat, lon) as pm_insert_workers takes them: one row per position (the call reads len(before) rows);
    lat / lon None or one value per row."""
    before = np.ascontiguousarray(np.atleast_1d(np.asarray(before, dtype=np.int64)).astype(np.uint32))
    a = np.ascontiguousarray(np.atleast_1d(a), dtype=abi.WORKER_A)
    b = np.ascontiguousarray(np.atleast_1d(b), dtype=abi.WORKER_B)
    la = np.ascontiguousarray(np.atleast_1d(lat), dtype=np.float64) if lat is not None else None
    lo = np.ascontiguousarray(np.atleast_1d(lon), dtype=np.float64) if lon is not None else None
    if len(a) != len(before) or len(b) != len(before):
        raise ValueError(f"insert_workers: {len(before)} positions for {len(a)} / {len(b)} rows")
    if (la is not None and len(la) != len(before)) or (lo is not None and len(lo) != len(before)):
        raise ValueError("insert_workers: lat / lon need one value per inserted row")
    return before, a, b, la, lo


def _result_views(r: "abi.PmResult", copy: bool) -> MatchResult:
    def view(ptr, n, dt):
        if n == 0:
            return np.zeros(0, dtype=dt)
        arr = np.ctypeslib.as_array(ptr, shape=(n,))
        return arr.copy() if copy else arr

    return MatchResult(
        worker_group=view(r.worker_group, r.n_workers, np.uint32),
        worker_ask=view(r.worker_ask, r.n_workers, np.uint32),
        group_ask=view(r.group_ask, r.n_groups, np.uint32),
        group_off=view(r.group_off, r.n_groups + 1, np.uint32),
        group_members=view(r.group_members, r.n_members, np.uint32),
        ask_best=view(r.ask_best, r.n_asks, np.int64),
        ask_count=view(r.ask_count, r.n_asks, np.uint32),
        stats=r.stats.as_dict(),
    )


class Comm:
    """pm_comm: this rank's end of the communicator the sharded pass exchanges through (NCCL inside the library)."""

    @staticmethod
    def unique_id() -> bytes:
        buf = (C.c_uint8 * abi.PM_COMM_ID_BYTES)()
        lib = load()
        rc = lib.pm_comm_unique_id(buf)
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, (lib.pm_last_error(None) or b"").decode())
        return bytes(buf)

    def __init__(self, unique_id: bytes, n_ranks: int, rank: int, device: int):
        self._lib = load()
        assert len(unique_id) == abi.PM_COMM_ID_BYTES
        buf = (C.c_uint8 * abi.PM_COMM_ID_BYTES).from_buffer_copy(unique_id)
        h = C.c_void_p()
        rc = self._lib.pm_comm_create(buf, n_ranks, rank, device, C.byref(h))
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, (self._lib.pm_last_error(None) or b"").decode())
        self._h = h
        self.n_ranks, self.rank = n_ranks, rank

    def close(self):
        if getattr(self, "_h", None):
            self._lib.pm_comm_destroy(self._h)
            self._h = None


class MultiEngine:
    """pm_multi: one process driving several GPUs (the form the orchestrator's single management loop calls)."""

    def __init__(self, devices, cost_tile_bytes: int = 0, timing: bool = False):
        self._lib = load()
        cfg = abi.PmCfg(abi.PM_ABI_VERSION, 0, abi.PM_CFG_TIMING if timing else 0, 0, cost_tile_bytes, 0, 0, None)
        devs = (C.c_int32 * len(devices))(*devices)
        h = C.c_void_p()
        rc = self._lib.pm_multi_create(C.byref(cfg), devs, len(devices), C.byref(h))
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, (self._lib.pm_multi_last_error(None) or b"").decode())
        self._h = h
        self.n = len(devices)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.pm_multi_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, (self._lib.pm_multi_last_error(self._h) or b"").decode())

    def set_asks(self, asks, opts):
        asks = np.ascontiguousarray(asks, dtype=abi.ASK)
        opts = np.ascontiguousarray(opts, dtype=abi.GPU_OPT)
        self._check(self._lib.pm_multi_set_asks(self._h, _ptr(asks), len(asks), _ptr(opts), len(opts)))

    def set_ask_enabled(self, idx, enabled):
        idx, en = _ask_enabled_args(idx, enabled)
        self._check(self._lib.pm_multi_set_ask_enabled(self._h, _ptr(idx), _ptr(en), len(idx)))

    def update_asks(self, idx, asks, opts=None):
        """pm_multi_update_asks: Engine.update_asks on every device."""
        idx, asks, opts = _ask_delta_args(idx, asks, opts)
        self._check(self._lib.pm_multi_update_asks(self._h, _ptr(idx), _ptr(asks), len(idx), _ptr(opts), len(opts)))

    def resize_asks(self, n: int, added=None, opts=None):
        """pm_multi_resize_asks: Engine.resize_asks on every device."""
        added = np.ascontiguousarray(np.zeros(0, dtype=abi.ASK) if added is None else added, dtype=abi.ASK)
        opts = np.ascontiguousarray(np.zeros(0, dtype=abi.GPU_OPT) if opts is None else opts, dtype=abi.GPU_OPT)
        self._check(self._lib.pm_multi_resize_asks(self._h, n, _ptr(added) if len(added) else None, _ptr(opts), len(opts)))

    def remove_asks(self, idx):
        """pm_multi_remove_asks: Engine.remove_asks on every device."""
        idx = _remove_args(idx)
        self._check(self._lib.pm_multi_remove_asks(self._h, _ptr(idx) if len(idx) else None, len(idx)))

    def insert_asks(self, before, asks, opts=None):
        """pm_multi_insert_asks: Engine.insert_asks on every device."""
        before, asks, opts = _insert_args(before, asks, opts)
        self._check(self._lib.pm_multi_insert_asks(self._h, _ptr(before) if len(before) else None,
                                                   _ptr(asks) if len(asks) else None, len(before), _ptr(opts), len(opts)))

    def set_model_table(self, bits, n_patterns, n_models, words):
        bits = np.ascontiguousarray(bits, dtype=np.uint32)
        self._check(self._lib.pm_multi_set_model_table(self._h, _ptr(bits), n_patterns, n_models, words))

    def set_workers(self, a, b):
        a = np.ascontiguousarray(a, dtype=abi.WORKER_A)
        b = np.ascontiguousarray(b, dtype=abi.WORKER_B)
        self._check(self._lib.pm_multi_set_worker_count(self._h, len(a)))
        self._check(self._lib.pm_multi_upsert_workers(self._h, _ptr(a), _ptr(b), 0, len(a)))
        self._check(self._lib.pm_multi_sync(self._h))

    def set_locations(self, lat, lon):
        lat = np.ascontiguousarray(lat, dtype=np.float64)
        lon = np.ascontiguousarray(lon, dtype=np.float64)
        self._check(self._lib.pm_multi_set_worker_locations(self._h, _ptr(lat), _ptr(lon), 0, len(lat)))
        self._check(self._lib.pm_multi_sync(self._h))

    def set_addr_rank(self, rank):
        rank = np.ascontiguousarray(rank, dtype=np.uint32)
        self._check(self._lib.pm_multi_set_worker_addr_rank(self._h, _ptr(rank), 0, len(rank)))
        self._check(self._lib.pm_multi_sync(self._h))

    def upsert_workers(self, a, b, first: int = 0):
        a = np.ascontiguousarray(a, dtype=abi.WORKER_A)
        b = np.ascontiguousarray(b, dtype=abi.WORKER_B)
        self._check(self._lib.pm_multi_upsert_workers(self._h, _ptr(a), _ptr(b), first, len(a)))
        self._check(self._lib.pm_multi_sync(self._h))

    def set_flags(self, idx, flags):
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        flags = np.ascontiguousarray(flags, dtype=np.uint32)
        self._check(self._lib.pm_multi_set_flags(self._h, _ptr(idx), _ptr(flags), len(idx)))
        self._check(self._lib.pm_multi_sync(self._h))

    def resize_workers(self, n: int):
        self._check(self._lib.pm_multi_resize_workers(self._h, n))

    def update_workers(self, idx, a, b, lat=None, lon=None):
        """Scatter changed rows into every device's resident table (pm_multi_update_workers)."""
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        a = np.ascontiguousarray(a, dtype=abi.WORKER_A)
        b = np.ascontiguousarray(b, dtype=abi.WORKER_B)
        la = np.ascontiguousarray(lat, dtype=np.float64) if lat is not None else None
        lo = np.ascontiguousarray(lon, dtype=np.float64) if lon is not None else None
        self._check(self._lib.pm_multi_update_workers(self._h, _ptr(idx), _ptr(a), _ptr(b),
                                                      _ptr(la) if la is not None else None,
                                                      _ptr(lo) if lo is not None else None, len(idx)))
        self._check(self._lib.pm_multi_sync(self._h))

    def remove_workers(self, idx):
        """pm_multi_remove_workers: Engine.remove_workers on every device."""
        idx = _remove_args(idx)
        self._check(self._lib.pm_multi_remove_workers(self._h, _ptr(idx) if len(idx) else None, len(idx)))

    def insert_workers(self, before, a, b, lat=None, lon=None):
        """pm_multi_insert_workers: Engine.insert_workers on every device."""
        before, a, b, la, lo = _worker_insert_args(before, a, b, lat, lon)
        self._check(self._lib.pm_multi_insert_workers(self._h, _ptr(before) if len(before) else None,
                                                      _ptr(a) if len(a) else None, _ptr(b) if len(b) else None,
                                                      _ptr(la) if la is not None else None,
                                                      _ptr(lo) if lo is not None else None, len(before)))

    def table_version(self) -> int:
        """Changes whenever a table call changed a table on any device (pm_multi_table_version)."""
        return int(self._lib.pm_multi_table_version(self._h))

    def match(self, mode: int = abi.PM_MODE_FIRST_FIT):
        self._check(self._lib.pm_multi_match(self._h, mode))

    def fetch(self, copy: bool = True) -> MatchResult:
        r = abi.PmResult()
        self._check(self._lib.pm_multi_fetch_result(self._h, C.byref(r)))
        return _result_views(r, copy)

    def stats(self, i: int = 0) -> dict:
        st = abi.PmStats()
        e = self._lib.pm_multi_engine(self._h, i)
        rc = self._lib.pm_get_stats(e, C.byref(st))
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, "pm_get_stats")
        return st.as_dict()


def pinned_empty(n: int, dtype) -> np.ndarray:
    """numpy array over pm_alloc_pinned memory (freed when the array dies)."""
    lib = load()
    dt = np.dtype(dtype)
    nbytes = max(n * dt.itemsize, 1)
    p = lib.pm_alloc_pinned(nbytes)
    if not p:
        raise MemoryError("pm_alloc_pinned failed")
    buf = (C.c_char * nbytes).from_address(p)
    arr = np.frombuffer(buf, dtype=dt, count=n)

    class _Owner:
        def __init__(self, ptr):
            self.ptr = ptr

        def __del__(self):
            try:
                lib.pm_free_pinned(self.ptr)
            except Exception:
                pass

    # keep the owner alive as long as any view of `buf` lives
    buf._pm_owner = _Owner(p)
    return arr
