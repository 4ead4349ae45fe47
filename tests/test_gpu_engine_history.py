"""One engine through long random histories of every table call, every pass kind and the auction certificate
(tests/engine_history.py), compared after every call with plain references computed from the host mirror: the CPU
oracle for reference passes, the exact auction checkers for auction passes, the certificate restatement for the
certificate, and the mirror's change sets for whether a pass stays incremental or warm (and how many rows an
incremental pass walks).  Every auction pass's pm_fetch_result arrays are the fold of the predicted slot assignment.
Refused calls must return the status the header gives and leave behind what it says: the next pass of each kind shows
it.  After every reference pass, and after every cold auction pass once the ask table or the demands have changed in
place, a fresh engine with the same settings, loaded from the mirror, must return the same arrays; after every cold
auction pass with a demand above 1, a fresh engine loaded with the twin tables (each ask row, cap and floor repeated
d[t] times) must return the same prices, rounds, reverse stats and slot assignment.  Exports and restores are checked
against the mirror's state and restore_checker's audit, and a move continues the history on a fresh engine.  Cost tile
probes between passes compare pm_build_cost_tile with the oracle's cost matrix and change nothing.  The same
histories' reference side also runs on pm_multi (the auction-only calls skipped).

PM_TEST_BIG=1 runs histories three times as long."""
import ctypes
import functools
import os

import numpy as np
import pytest

import auction_certificate as ac
import engine_history as eh
from protocol_b200 import abi
from protocol_b200._lib import PrimeMatchError
from oracle import pm_oracle as orc
from protocol_b200.engine import Engine, MultiEngine

pytestmark = pytest.mark.gpu

FIELDS = ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count")


def new_engine(setting, make=None):
    """An engine created with the setting's PM_TUNE_* knobs (they are read at pm_create)."""
    env = {k: str(v) for k, v in eh.SETTINGS[setting].items()}
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        if make is not None:
            return make(eh.TILE_BYTES.get(setting, 0))
        return Engine(cost_tile_bytes=eh.TILE_BYTES.get(setting, 0))
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def refused(call, statuses):
    """Run `call`; return its PrimeMatchError status, or None when it succeeded."""
    try:
        call()
    except PrimeMatchError as ex:
        assert statuses and ex.status in statuses, f"status {ex.status}, expected {statuses}: {ex}"
        return ex.status
    return None


class Runner:
    def __init__(self, shape, setting):
        self.setting = setting
        self.h = eh.History(shape, eh.cutoff_of(setting))
        self.eng = new_engine(setting)
        eh.load(self.eng, self.h)
        self.counts = {}
        self.deltas = False         # the ask table has changed in place

    def close(self):
        self.eng.close()

    def stored_state_kept(self):
        h = self.h
        if h.auc_state:
            price, _, _ = self.eng.auction_state()
            assert np.array_equal(price, h.price), "a refused call changed the stored auction state"

    # ---- passes
    def reference(self, kind):
        h, eng = self.h, self.eng
        why, statuses = h.refusal(kind)
        plan = h.incremental_plan() if kind in eh.INCREMENTAL else None
        if refused(lambda: eng.match(eh.MODES[kind]), statuses) is not None:
            h.reference_done(False)
            return
        assert why is None, f"{kind}: ran, expected refusal {why}"
        r = eng.fetch()
        want = eh.expect_reference(h, kind)
        for f in FIELDS:
            assert np.array_equal(getattr(r, f), want[f]), f"{kind}: {f} differs from the oracle"
        if "n_bumped" in want:
            assert r.stats["n_bumped"] == want["n_bumped"], (kind, "n_bumped", r.stats["n_bumped"], want["n_bumped"])
        if plan is not None:
            full, n_tiles, en, dis, sure = plan
            T, W = len(h.asks), h.n_workers
            if sure:
                assert r.stats["n_tiles"] == n_tiles, (kind, "n_tiles", r.stats["n_tiles"], n_tiles, full)
            if not full:
                assert r.stats["evals"] <= T * n_tiles + len(en) * W, (kind, r.stats)
                if n_tiles == 0 and not en and not dis:
                    assert r.stats["evals"] == 0, (kind, r.stats)
        fresh = new_engine(self.setting)
        eh.load(fresh, h)
        fresh.match(eh.MODES[kind])
        q = fresh.fetch()
        fresh.close()
        for f in FIELDS:
            assert np.array_equal(getattr(r, f), getattr(q, f)), f"{kind}: {f} differs from a fresh engine's"
        assert r.stats["n_bumped"] == q.stats["n_bumped"], (kind, "n_bumped")
        h.reference_done(True)

    def auction(self, kind):
        h, eng = self.h, self.eng
        why, statuses = h.refusal(kind)
        want_warm, sure = h.warm_plan() if kind in ("warm", "repair") else (False, True)
        if refused(lambda: eng.match(eh.MODES[kind]), statuses) is not None:
            self.stored_state_kept()
            return
        assert why is None, f"{kind}: ran, expected refusal {why}"
        res = eng.fetch()
        price, warm, released = eng.auction_state()
        rs = eng.auction_reverse_stats()
        if not sure:
            want_warm = warm
        a, p, n, rel, wrs = eh.expect_auction(h, kind, want_warm)
        assert warm == want_warm, (kind, "warm", warm)
        want = eh.expect_result(h, a)
        for f in FIELDS:
            assert np.array_equal(getattr(res, f), want[f]), f"{kind}: {f} differs from the checker's fold"
        assert np.array_equal(price, p), f"{kind}: prices differ from the checker"
        assert res.stats["n_rounds"] == n, (kind, "n_rounds", res.stats["n_rounds"], n)
        assert released == rel, (kind, "n_released", released, rel)
        assert rs == wrs, (kind, "reverse stats", rs, wrs)
        if not warm and self.deltas:   # a cold pass after deltas equals a fresh engine's (prime_match.h)
            fresh = new_engine(self.setting)
            eh.load(fresh, h)
            fresh.match(eh.MODES[kind])
            q = fresh.fetch()
            qprice, _, _ = fresh.auction_state()
            qrs = fresh.auction_reverse_stats()
            fresh.close()
            for f in FIELDS:
                assert np.array_equal(getattr(res, f), getattr(q, f)), f"{kind}: {f} differs from a fresh engine's"
            assert np.array_equal(price, qprice) and res.stats["n_rounds"] == q.stats["n_rounds"] and rs == qrs, \
                f"{kind}: prices or rounds differ from a fresh engine's"
        if not warm and (h.d > 1).any():   # the defining rule: the twin table gives the same pass bit for bit
            twin = new_engine(self.setting)
            eh.load(twin, h, twin=True)
            twin.match(eh.MODES[kind])
            q = twin.fetch()
            qprice, _, _ = twin.auction_state()
            qrs = twin.auction_reverse_stats()
            twin.close()
            slots = np.full(int(h.d.sum()), eh.NONE, dtype=np.uint32)
            for s, members in q.groups():
                assert len(members) == 1
                slots[s] = members[0]
            assert np.array_equal(slots, a), f"{kind}: the twin's slot assignment differs"
            assert np.array_equal(price, qprice) and res.stats["n_rounds"] == q.stats["n_rounds"] and rs == qrs, \
                f"{kind}: prices, rounds or reverse stats differ from the twin's"
        h.auction_done(p, a)

    def certificate(self):
        h, eng = self.h, self.eng
        why, statuses = h.refusal("certificate")
        out = {}
        before = self.untouched()
        if refused(lambda: out.update(eng.auction_certificate(ask_bound=True)), statuses) is not None:
            self.stored_state_kept()
            return
        assert why is None, f"certificate: ran, expected refusal {why}"
        self.same(before, self.untouched())
        want = eh.expect_certificate(h)
        for k in ac.FIELDS:
            assert out[k] == want[k], ("certificate", k, out[k], want[k])
        assert np.array_equal(out["ask_bound"], want["ask_bound"])

    # ---- exports and restores
    def export_matches(self, want):
        """The engine's export (pm_auction_assignment, pm_auction_state's prices) equals the mirror's."""
        price, _, _ = self.eng.auction_state()
        assigned = self.eng.auction_assignment()
        assert np.array_equal(price, want[0]) and np.array_equal(assigned, want[1]), "the export differs from the mirror"

    def untouched(self):
        """What a restore and a certificate must leave as they are: pm_fetch_result, pm_get_stats, pm_table_version."""
        try:
            r = self.eng.fetch()
            res = tuple(getattr(r, f).copy() for f in FIELDS)
        except PrimeMatchError:
            res = None
        st = abi.PmStats()
        assert self.eng._lib.pm_get_stats(self.eng._h, ctypes.byref(st)) == abi.PM_OK
        return res, bytes(st), self.eng.table_version()   # pm_get_stats bit for bit (its timings are floats)

    def same(self, a, b):
        """untouched() before and after a restore or a certificate."""
        assert (a[0] is None) == (b[0] is None) and (a[0] is None or all(np.array_equal(x, y) for x, y in zip(a[0], b[0]))), \
            "pm_fetch_result changed"
        if a[1] != b[1]:
            was, now = abi.PmStats.from_buffer_copy(a[1]).as_dict(), abi.PmStats.from_buffer_copy(b[1]).as_dict()
            raise AssertionError(f"pm_get_stats changed: {[(k, was[k], now[k]) for k in was if was[k] != now[k]]}")
        assert a[2] == b[2], ("pm_table_version changed", a[2], b[2])

    def restored(self, eng, report):
        """A restore's report and what the engine reports after it, against the mirror's audit (just applied)."""
        h = self.h
        assert all(report[k] == v for k, v in h.last_report.items()), ("restore report", report, h.last_report)
        price, warm, released = eng.auction_state()
        assert np.array_equal(price, h.price) and not warm and released == 0, "restore: pm_auction_state"
        assert eng.auction_reverse_stats() == (0, 0, 0), "restore: reverse stats"
        assert np.array_equal(eng.auction_assignment(), h.assigned), "restore: the stored assignment"

    def restore(self, x):
        h, eng = self.h, self.eng
        if x["export"] is not None:
            self.export_matches(x["export"])
        before = self.untouched()
        for price, assigned in x["attempts"]:
            st = h.restore_refusal(price, assigned)
            out = {}
            if refused(lambda: out.update(eng.auction_restore(price, assigned)), st) is not None:
                self.stored_state_kept()
                continue
            assert not st, f"restore ({x['variant']}): taken, expected a refusal in {st}"
            h.restore(price, assigned)
            self.restored(eng, out)
            break
        self.same(before, self.untouched())

    def restore_refused(self, x):
        h, eng = self.h, self.eng
        v = eng.table_version()
        if x["export"]:
            assert refused(lambda: eng.auction_assignment(), h.export_refusal()) is not None, (x["case"], "export taken")
        else:
            st = h.restore_refusal(x["price"], x["assigned"])
            assert refused(lambda: eng.auction_restore(x["price"], x["assigned"]), st) is not None, (x["case"], "taken")
        self.stored_state_kept()
        assert eng.table_version() == v, (x["case"], "pm_table_version changed")

    def move(self, x):
        """Export, load a fresh engine from the mirror, restore into it, close the old engine and go on with the new."""
        h = self.h
        self.export_matches(x["export"])
        fresh = new_engine(self.setting)
        eh.load(fresh, h)
        assert not h.restore_refusal(*x["fit"])
        report = fresh.auction_restore(*x["fit"])
        h.restore(*x["fit"])
        h.discard_eval()                    # the fresh engine has no stored evaluation
        self.restored(fresh, report)
        self.eng.close()
        self.eng = fresh

    def probe(self, t0, nt):
        """pm_build_cost_tile over asks [t0, t0 + nt) against the oracle's cost matrix (disabled rows PM_COST_INF)."""
        h = self.h
        if h.pattern_missing():
            assert refused(lambda: self.eng.cost_tile(t0, nt), {abi.PM_E_STATE}) is not None, "probe: ran"
            return
        got = self.eng.cost_tile(t0, nt)
        want = orc.soa_eval_matrix(h.wa, h.wb, h.asks, h.opts, h.bits, h.words, t0, t0 + nt, 0, h.n_workers, threads=8,
                                   want_cost=True, want_rows=False, want_cols=False)["cost"]
        want[~h.mask[t0:t0 + nt]] = eh.INF
        assert np.array_equal(got, want), f"probe [{t0}, {t0 + nt}): cost tile differs from the oracle"

    def step(self, ev):
        if ev[0] == "call":
            name = ev[1][0]
            if name in ("restore", "restore_refused", "move"):
                getattr(self, name)(ev[1][1])
                return
            eh.drive(self.eng, ev[1])
            self.h.apply(ev[1])
            self.deltas |= name in eh.ASK_DELTAS or name == "demand"
            return
        if ev[0] == "probe":
            self.probe(*ev[1])
            return
        kind = ev[1]
        self.counts[kind] = self.counts.get(kind, 0) + 1
        if kind in eh.REFERENCE:
            self.reference(kind)
        elif kind == "certificate":
            self.certificate()
        else:   # the auction kinds, and auction_incr (always refused)
            self.auction(kind)


def replay(shape, setting, events):
    """Run `events` on one engine; an AssertionError names the failing event."""
    r = Runner(shape, setting)
    try:
        for i, ev in enumerate(events):
            try:
                r.step(ev)
            except AssertionError as ex:
                what = ev[1][0] if ev[0] == "call" else ev[1]
                raise AssertionError(f"{shape}/{setting}: event {i} ({ev[0]} {what}): {ex}") from ex
    finally:
        r.close()
    return r.counts


@functools.lru_cache(maxsize=None)
def history(shape, setting):
    """The events of the seeded history of (shape, setting), generated once per session."""
    return eh.generate(shape, eh.seed_of(shape, setting), cutoff=eh.cutoff_of(setting), slot=eh.slot_of(shape, setting),
                       n_slots=eh.N_SLOTS)[0]


@pytest.mark.parametrize("setting", list(eh.SETTINGS))
@pytest.mark.parametrize("shape", eh.SHAPES)
def test_history(shape, setting):
    events = history(shape, setting)
    counts = replay(shape, setting, events)
    assert all(counts.get(k, 0) for k in eh.PASSES), counts


class ReferenceOnly:
    """A MultiEngine behind the drive() calls: the auction's columns (caps, floors, reputation, parameters) are no
    pm_multi calls, and none of them touches what a reference pass reads."""

    def __init__(self, multi, h):
        self.m, self.h = multi, h

    @property
    def n_workers(self):
        return self.h.n_workers

    def __getattr__(self, name):
        if name in ("set_price_caps", "set_min_reputation", "set_worker_reputation", "set_auction_params"):
            return lambda *a, **k: None
        return getattr(self.m, name)


# the auction's columns and calls: no pm_multi calls
MULTI_SKIP = ("reputation", "caps", "floors", "auction_params") + eh.AUCTION_CALLS


def test_history_on_multi():
    """The reference side of every history on one pm_multi over every visible device: worker and ask table calls,
    refused ask deltas (PM_E_INVALID, pm_multi_table_version unchanged), toggles, locations, ranks, table swaps and
    every reference and incremental pass, each pass against the oracle.  The demand, restore and move calls are skipped
    (auction-only, no pm_multi_ form) while the mirror still applies them, which shows that the reference passes ignore
    demands and restores; a move's fresh engine is not modelled (pm_multi keeps its stored evaluation).
    With one device the incremental passes must walk exactly the rows the mirror plans; with more, each rank's share
    moves when the worker table is resized, which the mirror does not model, so only the results are compared."""
    import torch

    devices = list(range(max(1, torch.cuda.device_count())))
    n_ref = 0
    for shape in eh.SHAPES:
        for setting in eh.SETTINGS:
            events = history(shape, setting)
            h = eh.History(shape, eh.cutoff_of(setting))
            m = new_engine(setting, lambda tb: MultiEngine(devices, cost_tile_bytes=tb))
            eng = ReferenceOnly(m, h)
            try:
                eh.load(eng, h)
                for i, ev in enumerate(events):
                    what = f"{shape}/{setting} on {len(devices)} device(s): event {i}"
                    if ev[0] == "call":
                        if ev[1][0] not in MULTI_SKIP:
                            eh.drive(eng, ev[1])
                        if ev[1][0] != "move":
                            h.apply(ev[1])
                        continue
                    if ev[0] != "pass" or ev[1] not in eh.REFERENCE:
                        continue
                    kind = ev[1]
                    why, statuses = h.refusal(kind)
                    plan = h.incremental_plan() if kind in eh.INCREMENTAL else None
                    if refused(lambda: m.match(eh.MODES[kind]), statuses) is not None:
                        h.reference_done(False)
                        continue
                    assert why is None, f"{what}: {kind} ran, expected refusal {why}"
                    r = m.fetch()
                    want = eh.expect_reference(h, kind)
                    for f in FIELDS:
                        assert np.array_equal(getattr(r, f), want[f]), f"{what}: {kind}: {f} differs from the oracle"
                    if plan is not None and len(devices) == 1 and plan[4]:
                        st = m.stats(0)
                        assert st["n_tiles"] == plan[1], (what, kind, "n_tiles", st["n_tiles"], plan[1])
                    h.reference_done(True)
                    n_ref += 1
            finally:
                m.close()
    assert n_ref > 100


def shortened(shape, setting, events):
    """The shortest prefix-and-subset of `events` that still fails (for turning a failing history into a regression
    test): a history fails when replay raises AssertionError; any other exception counts as passing."""
    def fails(evs):
        try:
            replay(shape, setting, evs)
        except AssertionError:
            return True
        except Exception:
            return False
        return False

    n = len(events)
    while n > 1 and fails(events[:n - 1]):
        n -= 1
    return eh.shrink(events[:n], fails)


def test_auction_fills_an_ask_of_max_group_size_zero():
    """The first history finding, shortened to one load and one cold auction pass: PM_MODE_AUCTION's feasibility is
    candidate, compatible, ask_price <= cap and reputation >= floor (prime_match.h); group sizes belong to the
    reference modes.  An ask with max_group_size == 0 and feasible workers bids like any other, as in the oracle's
    auction, while a first-fit pass between auction passes still never fills it, and the certificate and a warm pass
    after that first-fit pass see the auction's rule again."""
    from helpers import groups_equal, load_engine
    from oracle import pm_oracle as orc
    from test_gpu_auction_warm import tables

    t, cap = tables(50, 700, 2)
    F = eh.wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    z = int(np.flatnonzero(F.any(axis=1))[0])
    t["asks"] = t["asks"].copy()
    t["asks"][z]["min_group_size"] = t["asks"][z]["max_group_size"] = 0
    eng = Engine()
    load_engine(eng, t)
    eng.set_price_caps(cap)

    def auction(mode):
        eng.match(mode)
        got = np.full(len(cap), eh.NONE, dtype=np.uint32)
        for ask, members in eng.fetch().groups():
            got[ask] = members[0]
        return got, eng.auction_state()

    want, wprice, _ = orc.soa_auction(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    assert want[z] != eh.NONE
    got, (price, _, _) = auction(abi.PM_MODE_AUCTION)
    assert np.array_equal(got, want) and np.array_equal(price, wprice)
    eng.match(abi.PM_MODE_FIRST_FIT | eh.LEAN)
    r = eng.fetch()
    og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"])
    assert groups_equal(r, og) and not (r.worker_ask == z).any()
    c = eng.auction_certificate(ask_bound=True)
    wc_ = ac.certificate(F, t["wb"]["ext_ask_price"], cap, 1, wprice, want)
    assert all(c[k] == wc_[k] for k in ac.FIELDS) and np.array_equal(c["ask_bound"], wc_["ask_bound"])
    assert c["n_bad_holds"] == 0
    got, (price, warm, released) = auction(eh.WARM)
    assert warm and released == 0 and np.array_equal(got, want) and np.array_equal(price, wprice)
    eng.close()


def test_a_pattern_id_of_all_ones_is_a_missing_pattern():
    """A history finding, shortened to one delta: an option row with pattern_id 0xFFFFFFFF made pm_ask_convert's 32-bit
    pattern row pattern_id + 1 wrap to 0, which reads as "no model pattern", so the table was accepted and the row
    matched any model.  Like any pattern past the model table it now makes every pass, the certificate and the cost
    tile return PM_E_STATE until the row is replaced, while the stored evaluation and auction state follow the header:
    the reference pass that failed discards the evaluation, the refused auction pass keeps the state."""
    h = eh.History("mixed")
    eng = new_engine("default")
    eh.load(eng, h)
    s = h.s
    eng.match(eh.MODES["auction"])
    price, _, _ = eng.auction_state()
    eng.match(eh.MODES["lean_incr"])
    for row in (s["edge"][6:7], s["edge"][5:6]):      # pattern 0xFFFFFFFF, then the first pattern past the table
        eng.update_asks([7], row, s["opts"])
        for call in (lambda: eng.match(eh.MODES["lean_incr"]), lambda: eng.match(eh.MODES["warm"]),
                     lambda: eng.auction_certificate(), lambda: eng.cost_tile(0, 8)):
            assert refused(call, {abi.PM_E_STATE}) == abi.PM_E_STATE
        assert np.array_equal(eng.auction_state()[0], price)
    eng.update_asks([7], h.asks[7:8], s["opts"])
    eng.match(eh.MODES["lean_incr"])
    r = eng.fetch()
    want = eh.expect_reference(h, "lean_incr")
    assert all(np.array_equal(getattr(r, f), want[f]) for f in FIELDS)
    assert r.stats["n_tiles"] == h.n_workers           # the failed pass discarded the stored evaluation
    eng.match(eh.MODES["warm"])
    assert eng.auction_state()[1] == 1                 # the refused auction passes kept the stored state
    eng.close()


def test_restore_and_certificate_leave_the_launch_count():
    """A history finding, shortened to a reference pass and a restore: with an enabled max_group_size 0 ask, a restore
    or a certificate after a reference pass first puts that row back in the auction's form, a launch that counted in
    pm_get_stats' n_launches although the header says neither call changes what pm_get_stats reports."""
    import auction_restore_checker as rs

    r = Runner("mixed", "default")
    h = r.h
    assert len(h.max0_on())
    state = rs.adversarial_state(h.F(), h.wb["ext_ask_price"], h.cap, h.params[0], np.random.default_rng(3), h.params[1])
    try:
        for ev in [("pass", "lean"), ("call", ("restore", dict(variant="adversarial", export=None, attempts=[state]))),
                   ("pass", "lean"), ("pass", "certificate")]:
            r.step(ev)       # the restore and the certificate compare pm_get_stats before and after, bit for bit
    finally:
        r.close()
