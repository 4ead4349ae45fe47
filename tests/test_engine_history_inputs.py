"""The histories of tests/test_gpu_engine_history.py reach what they claim, shown on the CPU over the exact seeds the GPU
file runs: every (table call -> pass kind) and (pass kind -> pass kind) pair, every refusal kind followed by an
incremental and a warm pass, incremental passes after auction passes and certificates, warm and repair passes after
reference passes of both modes with toggles left on across them, the fast/generic and narrow/wide flips inside an
incremental pass's window, and cutoff crossings on both trackers.  And the mirror checked against itself: the oracle's
groups on the enabled asks equal test_gpu_ask_enabled's compaction, and the warm checker with no changes reproduces
the stored state."""
import functools

import numpy as np
import pytest

import auction_warm_checker as wc
import engine_history as eh
from helpers import assert_distance_certificate
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth


@functools.lru_cache(maxsize=None)
def evidence():
    """Generate every history the GPU file runs and record, through the generator's mirror, what each pass saw."""
    ev = dict(call_pass=set(), pass_pass=set(), refusals={}, after_refusal={}, incr_after_auction_cert=0,
              warm_after_both=set(), flips=set(), incr_over=0, warm_over=0, n_passes=0, incr_saw=set(),
              e_rows_over=0, removed_held=set(), removed_held_decides=set(), max0_by=set(), probes_after_auction=0,
              generated={})
    for shape in eh.SHAPES:
        for setting in eh.SETTINGS:
            cutoff = eh.cutoff_of(setting)
            st = dict(last="start", calls=[], pend_incr=[], pend_warm=[], since_eval=dict(auction=0, certificate=0),
                      since_state=dict(ff=0, prox=0, disabled_across=False), max0=None, after_auction=False)

            def observe(h, e, before, st=st, cutoff=cutoff):
                if e[0] == "call":
                    name = e[1][0]
                    st["after_auction"] = False   # a delta puts the rows back in the reference form
                    if before:
                        st["max0"] = len(h.max0_on()) > 0
                        if name == "ask_delta_refused":
                            ev["refusals"]["ask_delta_refused"] = ev["refusals"].get("ask_delta_refused", 0) + 1
                            st["pend_incr"].append("ask_delta_refused")
                            st["pend_warm"].append(("ask_delta_refused", h.auc_state))
                        return
                    st["calls"].append(name)
                    if name in eh.ASK_DELTAS and (len(h.max0_on()) > 0) != st["max0"]:
                        ev["max0_by"].add(name)
                    if name in ("set_asks", "model_table", "set_workers"):
                        st["since_eval"] = dict(auction=0, certificate=0)
                        st["pend_incr"], st["pend_warm"] = [], []
                    if name == "auction_params":
                        st["pend_warm"] = []
                    if not h.auc_state:
                        st["since_state"] = dict(ff=0, prox=0, disabled_across=False)
                    return
                if e[0] == "probe":
                    ev["probes_after_auction"] += st["after_auction"] and len(h.asks[h.asks["max_group_size"] == 0]) > 0
                    return
                kind = e[1]
                st["after_auction"] = False
                ev["n_passes"] += 1
                why, _ = h.refusal(kind)
                if why is not None:
                    ev["refusals"][why] = ev["refusals"].get(why, 0) + 1
                if kind in eh.INCREMENTAL and why is None:
                    full, n_tiles, en, dis, sure = h.incremental_plan()
                    if not full and h.dirty and st["since_eval"]["auction"] and st["since_eval"]["certificate"]:
                        ev["incr_after_auction_cert"] += 1
                    if not full:
                        ev["flips"] |= h.flipped
                        orphans = eh.walked_rows(h.eval_ff, set(), {t for t in dis if t in h.replaced})
                        if orphans and any(h.mask[t] for t in dis if t in h.replaced):
                            ev["incr_saw"].add("replaced_enabled_with_orphans")
                        if any(not h.mask[t] for t in h.replaced):
                            ev["incr_saw"].add("replaced_disabled")
                        if en & h.appended:
                            ev["incr_saw"].add("append")
                        if h.dropped:
                            ev["incr_saw"].add("shrink_dropped_first_asks")
                    if full and h.eval and h.over and cutoff < eh.DEFAULT_CUTOFF:
                        ev["incr_over"] += 1
                    if full and h.eval and not h.over and len(h.dirty) <= cutoff < eh.DEFAULT_CUTOFF:
                        ev["e_rows_over"] += 1
                    for r in st["pend_incr"]:
                        ev["after_refusal"].setdefault(r, set()).add("incremental")
                if kind in ("warm", "repair") and why is None:
                    warm, _ = h.warm_plan()
                    if warm and h.removed_held:
                        ev["removed_held"].add(kind)
                    if h.auc_state and not h.auc_over and h.n_changes() - h.removed_held <= cutoff < h.n_changes():
                        ev["removed_held_decides"].add((kind, warm))
                    ss = st["since_state"]
                    if warm and ss["ff"] and ss["prox"] and ss["disabled_across"]:
                        ev["warm_after_both"].add(kind)
                    if h.auc_state and not warm and h.auc_over and cutoff < eh.DEFAULT_CUTOFF:
                        ev["warm_over"] += 1
                    for r, had_state in st["pend_warm"]:   # warm on the kept state, or cold where there was none
                        if warm == had_state:
                            ev["after_refusal"].setdefault(r, set()).add("warm")
                    st["pend_warm"] = []
                if kind in eh.REFERENCE and why is None:
                    st["pend_incr"] = []               # this pass stores an evaluation: the refusals are behind it
                if kind in ("auction", "reverse") and why is None:
                    st["pend_warm"] = []               # a new stored state
                if why is not None:
                    st["pend_incr"].append(why)
                    st["pend_warm"].append((why, h.auc_state))
                if kind in eh.REFERENCE:
                    if why is None:
                        st["since_state"]["prox" if kind.startswith("proximity") else "ff"] += 1
                        st["since_state"]["disabled_across"] |= bool(h.auc_state and not h.mask.all())
                    st["since_eval"] = dict(auction=0, certificate=0)
                elif kind in eh.AUCTION:
                    st["since_eval"]["auction"] += 1
                    if why is None:
                        st["since_state"] = dict(ff=0, prox=0, disabled_across=False)
                        st["after_auction"] = True
                elif kind == "certificate":
                    st["since_eval"]["certificate"] += 1
                if kind != "auction_incr":
                    ev["call_pass"] |= {(c, kind) for c in st["calls"]}
                    ev["pass_pass"].add((st["last"], kind))
                    st["last"] = kind
                    st["calls"] = []

            ev["generated"][shape, setting] = eh.generate(shape, eh.seed_of(shape, setting), cutoff=cutoff,
                                                          slot=eh.slot_of(shape, setting), n_slots=eh.N_SLOTS,
                                                          observe=observe)
    return ev


def test_every_call_and_pass_pair_occurs():
    ev = evidence()
    missing = [(c, p) for c in eh.CALLS for p in eh.PASSES if (c, p) not in ev["call_pass"]]
    assert not missing, missing
    missing = [(a, b) for a in eh.PASSES for b in eh.PASSES if (a, b) not in ev["pass_pass"]]
    assert not missing, missing


def test_every_refusal_occurs_and_is_followed_by_an_incremental_and_a_warm_pass():
    ev = evidence()
    for r in eh.REFUSALS:
        assert ev["refusals"].get(r, 0) > 0, (r, ev["refusals"])
        assert ev["after_refusal"].get(r, set()) >= {"incremental", "warm"}, (r, ev["after_refusal"].get(r))


def test_incremental_passes_after_auction_passes_and_certificates():
    assert evidence()["incr_after_auction_cert"] > 0


def test_warm_and_repair_passes_after_reference_passes_of_both_modes_and_toggles():
    assert evidence()["warm_after_both"] >= {"warm", "repair"}, evidence()["warm_after_both"]


def test_predicate_and_tile_flips_inside_an_incremental_window():
    assert evidence()["flips"] >= {"fast", "narrow"}, evidence()["flips"]


def test_cutoff_crossings_on_both_trackers():
    ev = evidence()
    assert ev["incr_over"] > 0 and ev["warm_over"] > 0, (ev["incr_over"], ev["warm_over"])


def test_incremental_passes_see_every_ask_delta():
    """Passes that stay incremental after a replaced enabled ask with orphans, a replaced disabled ask, an append, and
    an ask shrink that set stored first asks to NONE."""
    want = {"replaced_enabled_with_orphans", "replaced_disabled", "append", "shrink_dropped_first_asks"}
    assert evidence()["incr_saw"] >= want, evidence()["incr_saw"]


def test_appended_asks_alone_pass_the_cutoff():
    """Under PM_TUNE_INCR=40 an incremental pass goes full because ceil(|E| W / T) passes the cutoff, not the rows."""
    assert evidence()["e_rows_over"] > 0


def test_warm_and_repair_passes_after_removed_held_asks():
    assert evidence()["removed_held"] >= {"warm", "repair"}, evidence()["removed_held"]


def test_removed_held_asks_decide_the_warm_cutoff():
    """Under PM_TUNE_INCR=40 a warm and a repair pass whose changes stay within the cutoff without the removed asks that
    held a worker and pass it with them: both run cold."""
    assert evidence()["removed_held_decides"] >= {("warm", False), ("repair", False)}, evidence()["removed_held_decides"]


MIRROR = ("asks", "mask", "eval_mask", "cap", "floors", "wa", "wb", "lat", "lon", "rank", "reputation", "eval_ff")
TRACKED = ("params", "eval", "dirty", "over", "replaced", "appended", "dropped", "flipped", "auc_state", "auc_w",
           "auc_over", "resized", "rows", "toggled", "n_kept", "cap0", "floors0")


@pytest.mark.parametrize("setting", list(eh.SETTINGS))
@pytest.mark.parametrize("shape", eh.SHAPES)
def test_events_alone_rebuild_the_mirror(shape, setting):
    """The GPU runner rebuilds the mirror from the events alone: replaying them on a fresh History (auction passes
    without their state values) ends with the generator's tables and trackers."""
    events, g = evidence()["generated"][shape, setting]
    h = eh.History(shape, eh.cutoff_of(setting))
    for e in events:
        if e[0] == "call":
            h.apply(e[1])
        elif e[0] == "pass":
            why, _ = h.refusal(e[1])
            if e[1] in eh.REFERENCE:
                h.reference_done(why is None)
            elif e[1] in eh.AUCTION and why is None:
                h.auction_done(None, None)
    for f in MIRROR:
        a, b = getattr(h, f), getattr(g, f)
        assert (a is None and b is None) or np.array_equal(a, b), f
    for f in TRACKED:
        a, b = getattr(h, f), getattr(g, f)
        assert (np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b), f


def test_fast_predicate_flips_through_an_ask_row():
    assert "ask_fast" in evidence()["flips"], evidence()["flips"]


def test_max_group_size_zero_fact_changes_through_every_ask_delta():
    assert evidence()["max0_by"] >= set(eh.ASK_DELTAS), evidence()["max0_by"]


def test_cost_tile_probes_after_auction_passes_with_max0_rows():
    assert evidence()["probes_after_auction"] > 0


def test_a_missing_pattern_is_any_id_past_the_model_table():
    """pattern_id >= n_patterns is missing, 0xFFFFFFFF (whose 32-bit pattern row wraps to 0) included; an option row
    without PM_O_MODEL or an ask without requirements reads no pattern."""
    s = eh.setup("mixed")
    npat = s["npat"]
    asks = np.repeat(s["edge"][5:6], 5).copy()
    opts = np.zeros(4, dtype=s["opts"].dtype)
    opts["present"] = [abi.PM_O_MODEL, abi.PM_O_MODEL, abi.PM_O_MODEL, 0]
    opts["pattern_id"] = [npat - 1, npat, 0xFFFFFFFF, npat]
    asks["opt_off"] = [0, 1, 2, 3, 1]
    asks["flags"][4] = 0
    assert eh.missing_pattern(asks, opts, npat).tolist() == [False, True, True, False, False]


def test_locations_pass_the_distance_certificate():
    pts = synth.CITIES
    assert_distance_certificate(pts[:, 0], pts[:, 1], np.ones(len(pts), dtype=bool))


@pytest.mark.parametrize("shape", eh.SHAPES)
def test_oracle_on_the_enabled_asks_equals_the_compacted_table(shape):
    from test_gpu_ask_enabled import mapped, subset

    h = eh.History(shape)
    rng = np.random.default_rng(5)
    h.mask[rng.choice(len(h.asks), 60, replace=False)] = False
    for kind in ("materialized", "proximity"):
        want = eh.expect_reference(h, kind)
        og = orc.soa_form_groups(h.wa, h.wb, subset(h.asks, h.mask), h.opts, h.bits, h.words, addr_rank=h.rank,
                                 lat=h.lat, lon=h.lon, proximity="banded" if kind == "proximity" else False)
        wg = np.full(h.n_workers, eh.NONE, dtype=np.uint32)
        wk = np.full(h.n_workers, eh.NONE, dtype=np.uint32)
        for g in range(len(og.cfg)):
            m = og.members[og.off[g]:og.off[g + 1]]
            wg[m], wk[m] = g, og.cfg[g]
        ev = orc.soa_eval_matrix(h.wa, h.wb, subset(h.asks, h.mask), h.opts, h.bits, h.words, 0, int(h.mask.sum()), 0,
                                 h.n_workers, threads=8)

        class Sub:
            worker_group, worker_ask, group_ask, group_off, group_members = wg, wk, og.cfg, og.off, og.members
            ask_best, ask_count = ev["row_best"], ev["row_count"]

        got = mapped(Sub, h.mask)
        fields = ["worker_group", "worker_ask", "group_ask", "group_off", "group_members"]
        for f in fields + (["ask_best", "ask_count"] if kind == "materialized" else []):
            assert np.array_equal(got[f], want[f]), (kind, f)
        assert len(want["group_ask"]) > 20


@pytest.mark.parametrize("shape", eh.SHAPES)
def test_warm_checker_without_changes_reproduces_the_stored_state(shape):
    h = eh.History(shape)
    for kind in ("auction", "reverse"):
        a, p, n, _, _ = eh.expect_auction(h, kind, False)
        h.auction_done(p, a)
        wa, wp, _, rel = h.warm(h.params[0])
        assert np.array_equal(wa, a) and np.array_equal(wp, p) and len(rel) == 0
        assert (a != wc.NONE).sum() > 20


@pytest.mark.parametrize("shape", eh.SHAPES)
def test_the_max_group_size_zero_ask_is_filled_by_the_auction_only(shape):
    """Ask z (max_group_size 0) has feasible workers: the auction gives it one, the reference modes none (first fit
    forms its empty group, as for any min_group_size == 0 ask)."""
    h = eh.History(shape)
    z = h.z
    assert h.asks[z]["max_group_size"] == 0 and h.F()[z].sum() > 50
    a, _, _, _, _ = eh.expect_auction(h, "auction", False)
    assert a[z] != eh.NONE
    assert not (eh.expect_reference(h, "lean")["worker_ask"] == z).any()
