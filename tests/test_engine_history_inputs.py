"""The histories of tests/test_gpu_engine_history.py reach what they claim, shown on the CPU over the exact seeds the GPU
file runs: every (table call -> pass kind) and (pass kind -> pass kind) pair, every refusal kind followed by an
incremental and a warm pass, incremental passes after auction passes and certificates, warm and repair passes after
reference passes of both modes with toggles left on across them, the fast/generic and narrow/wide flips inside an
incremental pass's window, and cutoff crossings on both trackers; the demand and restore steps with the property each
claims.  And the mirror checked against itself: the oracle's groups on the enabled asks equal test_gpu_ask_enabled's
compaction, the warm checker with no changes reproduces the stored state, the slot-level mirror with every demand 1 is
the ask-level one, and each of twelve wrong demand, restore, removal or insertion rules changes some prediction of the
same histories.  The removals and insertions: every refused case, incremental passes after every kind of heir, a removed
first ask with no row after it and a row inserted before one, a demand chain through a splice, removed held slots on
both sides of n_kept that decide the warm cutoff, and the certificate refused after a splice until an auction pass."""
import functools

import numpy as np
import pytest

import auction_certificate as ac
import auction_demand as ad
import auction_repair_checker as rp
import auction_warm_checker as wc
import engine_history as eh
import feature_tables as ft
from helpers import assert_distance_certificate
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth


def n_features(h):
    """The feature dictionary's size over the mirror's ask rows (pm_build_argmin_feat runs when it is at most 64)."""
    return len(ft.dictionary(ft.converted(h.asks, h.opts)))


def splice_seen(h, x, st):
    """Before a removal: which heirs it makes (the heir's state since the stored evaluation), whether a stored first
    ask loses every row after it, and on which side of n_kept the workers of the removed slots lie."""
    T = len(h.asks)
    rm = np.unique(x["idx"].astype(np.int64))
    keep = np.setdiff1d(np.arange(T), rm)
    if h.eval:
        stored = set(h.eval_ff[h.eval_ff != eh.NONE].tolist())
        for t, s in zip(rm, np.searchsorted(keep, rm)):
            if int(t) not in stored:
                continue
            if s == len(keep):
                st["splice_saw"].add("no_heir")
                continue
            heir = int(keep[s])
            st["splice_saw"].add("disabled" if not h.mask[heir] else "replaced" if heir in h.replaced
                                 else "appended" if heir in h.appended else "plain")
    if h.auc_state and h.assigned is not None:
        off = ad.offsets(h.d)
        gone = np.concatenate([h.assigned[off[t]:off[t + 1]] for t in rm])
        gone = gone[gone != eh.NONE]
        st["splice_gone"] = (bool((gone < h.n_kept).any()), bool((gone >= h.n_kept).any()))


@functools.lru_cache(maxsize=None)
def evidence():
    """Generate every history the GPU file runs and record, through the generator's mirror, what each pass saw."""
    ev = dict(call_pass=set(), pass_pass=set(), refusals={}, after_refusal={}, incr_after_auction_cert=0,
              warm_after_both=set(), flips=set(), incr_over=0, warm_over=0, n_passes=0, incr_saw=set(),
              e_rows_over=0, removed_held=set(), removed_held_decides=set(), max0_by=set(), probes_after_auction=0,
              generated={}, cases=set(), freed_decides=set(), chain=set(), past_kept=0, d_over_w=set(),
              variants=set(), own_clean=0, move_full=0, restore_incr=0, restore_cert=0, set_asks_export=0,
              cert_back_to_one=0, window=set(), slot_warm=set(), splice_incr=set(), splice_chain=set(),
              splice_held=set(), splice_cert=set(), crossings=set())
    for shape in eh.SHAPES:
        for setting in eh.SETTINGS:
            cutoff = eh.cutoff_of(setting)
            st = dict(last="start", calls=[], pend_incr=[], pend_warm=[], since_eval=dict(auction=0, certificate=0),
                      since_state=dict(ff=0, prox=0, disabled_across=False), max0=None, after_auction=False,
                      splice_saw=set(), window=dict(feats=[], fast=[], max0=[], start=0, start_fast=False))

            def observe(h, e, before, st=st, cutoff=cutoff):
                if e[0] == "call":
                    name = e[1][0]
                    st["after_auction"] = False   # a delta puts the rows back in the reference form
                    x = e[1][1]
                    if before:
                        st["max0"] = len(h.max0_on()) > 0
                        if name in ("ask_delta_refused", "demand_refused", "restore_refused"):
                            ev["refusals"][name] = ev["refusals"].get(name, 0) + 1
                            st["pend_incr"].append(name)
                            st["pend_warm"].append((name, h.auc_state))
                            ev["cases"].add((name, x["case"]))
                        if name == "demand" and h.auc_state:   # removed slots' workers past n_kept
                            o = ad.offsets(h.d)
                            gone = [int(w) for t in range(len(h.d)) for w in
                                    h.assigned[o[t] + min(int(h.d[t]), int(x["d"][t])):o[t + 1]] if w != eh.NONE]
                            ev["past_kept"] += any(w >= h.n_kept for w in gone)
                        if name == "set_asks" and (h.d > 1).any():
                            st["set_asks_d"] = True
                        if name in ("restore", "move"):
                            st["restore_eval"] = h.eval
                        if name == "remove_asks":
                            splice_seen(h, x, st)
                        if name == "insert_asks" and h.eval and set(x["before"].tolist()) & set(h.eval_ff.tolist()):
                            st["splice_saw"].add("insert_before_first")
                        return
                    if name in ("restore", "move") and h.last_report is not None:
                        variant = x.get("variant", "move")
                        ev["variants"].add(variant)
                        if variant == "own" and st["calls"] == [] and st["last"] in eh.AUCTION:
                            ev["own_clean"] += 1
                            assert h.last_report["n_dropped_bad"] + h.last_report["n_dropped_shared"] \
                                + h.last_report["n_dropped_slack"] == 0, h.last_report
                        if variant == "own" and st.get("set_asks_d"):
                            ev["set_asks_export"] += 1
                            st["set_asks_d"] = False
                        st["restored"] = True
                        st["restored_eval"] = st.get("restore_eval", False) and name == "restore"
                        st["moved"] = name == "move"
                    st["calls"].append(name)
                    if name in ("remove_asks", "insert_asks"):   # the facts each splice leaves inside the window
                        w = st["window"]
                        w["feats"].append(n_features(h))
                        w["fast"].append(eh.asks_small(h.asks, h.opts))
                        w["max0"].append(len(h.max0_on()) > 0)
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
                restored, st["restored"] = st.get("restored", False), False
                if kind == "certificate" and why is None:
                    ev["restore_cert"] += restored
                    ev["cert_back_to_one"] += bool(h.dem_kept is not None and (h.d == 1).all())
                if kind in eh.INCREMENTAL and why is None:
                    full = h.incremental_plan()[0]
                    ev["move_full"] += bool(st.get("moved") and full and not h.eval)
                    ev["restore_incr"] += bool(restored and st.get("restored_eval") and h.eval and not full)
                    st["moved"] = False
                spliced = bool({"remove_asks", "insert_asks"} & set(st["calls"]))
                if kind == "certificate" and why == "certificate_asks_resized" and spliced:
                    ev["splice_cert"].add("refused")
                    st["cert_splice"] = True
                elif kind == "certificate" and why is None and st.get("cert_splice") and st["last"] == "auction":
                    ev["splice_cert"].add("ran")
                if kind in ("warm", "repair") and why is None and h.auc_state and not h.auc_over \
                        and st.get("splice_gone") == (True, True) and h.n_changes() - h.removed_held <= cutoff:
                    ev["splice_held"].add((kind, h.n_changes() <= cutoff))
                if kind in ("warm", "repair") and why is None and spliced and h.dem_kept is not None \
                        and (h.dem_kept != np.minimum(h.d_pass, h.d)).any():
                    ev["splice_chain"].add(kind)
                if kind in eh.AUCTION and why is None:
                    st["splice_gone"] = None
                if kind in eh.INCREMENTAL and why is None and not h.incremental_plan()[0]:
                    ev["splice_incr"] |= st["splice_saw"]
                    w = st["window"]
                    if w["feats"]:   # splices inside this incremental pass's window
                        if shape == "wide" and w["start"] <= ft.MAX_FEATURES < max(w["feats"]) \
                                and n_features(h) <= ft.MAX_FEATURES:
                            ev["crossings"].add("past_64_and_back")
                        if w["start_fast"] and not all(w["fast"]) and eh.asks_small(h.asks, h.opts) \
                                and "ask_fast" in h.flipped:
                            ev["crossings"].add("fast_off_and_on")
                        if any(w["max0"]) and not len(h.max0_on()):
                            ev["crossings"].add("max0_on_and_off")
                if kind.startswith("proximity") and why == "proximity_max0" and st["calls"][-1:] == ["insert_asks"]:
                    ev["crossings"].add("proximity_refused")
                    st["prox_splice"] = True
                elif kind.startswith("proximity") and why is None and st.get("prox_splice") \
                        and st["calls"][-1:] == ["remove_asks"]:
                    ev["crossings"].add("proximity_cleared")
                if kind in eh.REFERENCE:
                    st["splice_saw"] = set()
                    if why is None:   # a new stored evaluation: a new window
                        st["window"] = dict(feats=[], fast=[], max0=[], start=n_features(h),
                                            start_fast=eh.asks_small(h.asks, h.opts))
                if kind in eh.AUCTION and why is None:
                    D = int(h.d.sum())
                    warm = h.warm_plan()[0] if kind in ("warm", "repair") else False
                    if D > h.n_workers:
                        ev["d_over_w"].add("warm" if warm else "cold")
                    if warm and (h.d > 1).any():
                        ev["slot_warm"].add(kind)
                    if kind in ("warm", "repair") and h.auc_state and h.dem_kept is not None:
                        if h.removed_held and not h.auc_over and abs(h.n_changes() - h.cutoff) <= h.removed_held \
                                and h.n_changes() - h.removed_held <= h.cutoff:
                            ev["freed_decides"].add((kind, warm))
                        if (h.dem_kept != np.minimum(h.d_pass, h.d)).any():
                            ev["chain"].add(kind)
                        if warm and {"demand", "update_asks", "append_asks", "shrink_asks", "ask_off", "ask_on",
                                     "update"} <= set(st["calls"]):
                            ev["window"].add(kind)
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


MIRROR = ("asks", "mask", "eval_mask", "cap", "floors", "wa", "wb", "lat", "lon", "rank", "reputation", "eval_ff", "d",
          "d_pass", "dem_kept", "price", "assigned")
TRACKED = ("params", "eval", "dirty", "over", "replaced", "appended", "heirs", "dropped", "flipped", "auc_state", "auc_w",
           "auc_over", "resized", "rows", "toggled", "n_kept", "cap0", "floors0", "removed_held")


def rebuild(events, outcomes, h, until=None, on_pass=None):
    """Replay `events` on the mirror h, each auction pass taking the state the generator predicted for it (outcomes);
    on_pass(h, i, kind, why) runs before each pass and may return an outcome to use instead."""
    for i, e in enumerate(events[:until]):
        if e[0] == "call":
            h.apply(e[1])
        elif e[0] == "pass":
            why, _ = h.refusal(e[1])
            got = on_pass(h, i, e[1], why) if on_pass is not None else None
            if e[1] in eh.REFERENCE:
                h.reference_done(why is None)
            elif e[1] in eh.AUCTION and why is None:
                out = got or outcomes[i]
                h.auction_done(out[2], out[1])
    return h


@pytest.mark.parametrize("setting", list(eh.SETTINGS))
@pytest.mark.parametrize("shape", eh.SHAPES)
def test_events_alone_rebuild_the_mirror(shape, setting):
    """The GPU runner rebuilds the mirror from the events alone: replaying them on a fresh History, each auction pass
    storing the state its checker predicted, ends with the generator's tables and trackers, demands, kept slots and
    slot-level state included."""
    events, g = evidence()["generated"][shape, setting]
    h = rebuild(events, g.outcomes, eh.History(shape, eh.cutoff_of(setting)))
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


# ------------------------------------------------------------------ demands and restores
def test_every_demand_and_restore_refusal_occurs():
    cases = evidence()["cases"]
    want = {("demand_refused", c) for c in eh.DEMAND_REFUSALS} | {("restore_refused", c) for c in eh.RESTORE_REFUSALS}
    assert cases >= want, sorted(want - cases)


def test_warm_and_repair_passes_on_slot_states_after_mixed_windows():
    """Warm passes with demands above 1, and passes that stay warm after a window with a demand change, a replaced
    held ask, an append, a shrink, a toggle off and on and written rows."""
    ev = evidence()
    assert ev["slot_warm"] >= {"warm", "repair"} and ev["window"] >= {"warm", "repair"}, (ev["slot_warm"], ev["window"])


def test_freed_slot_workers_decide_the_cutoff():
    """Under PM_TUNE_INCR=40, warm and repair passes whose changes pass the cutoff only with the workers of removed
    slots (cold), and ones they leave within it (warm)."""
    want = {(k, w) for k in ("warm", "repair") for w in (False, True)}
    assert evidence()["freed_decides"] >= want, evidence()["freed_decides"]


def test_demand_chains_and_freed_workers_past_n_kept():
    """A chain of demand changes whose kept slots differ from min(demand at the pass, demand now), and a demand cut
    whose removed slots held a worker a worker shrink had cut off."""
    ev = evidence()
    assert "warm" in ev["chain"] and ev["past_kept"] > 0, (ev["chain"], ev["past_kept"])


def test_more_slots_than_workers():
    assert evidence()["d_over_w"] >= {"cold", "warm"}, evidence()["d_over_w"]


def test_restores_of_every_kind():
    """Own states (one right after its pass, which the audit keeps whole), stale, adversarial and resized ones, a
    move, an export after a table swap with demands, and a certificate after demands back to 1."""
    ev = evidence()
    assert ev["variants"] >= {"own", "stale", "adversarial", "resized", "move"}, ev["variants"]
    assert ev["own_clean"] > 0 and ev["set_asks_export"] > 0 and ev["cert_back_to_one"] > 0


def test_restores_then_incremental_passes_and_certificates():
    """A restore between two incremental passes (the second stays incremental), a certificate right after a restore,
    and a move followed by a full incremental pass (the fresh engine has no stored evaluation)."""
    ev = evidence()
    assert ev["restore_incr"] > 0 and ev["restore_cert"] > 0 and ev["move_full"] > 0, \
        (ev["restore_incr"], ev["restore_cert"], ev["move_full"])


def test_demands_of_one_are_the_ask_level_mirror():
    """With every demand 1 the slot-level mirror is the ask-level one: A0 over slots is A0, the change count, the warm
    and repair predictions, the certificate and the result fold are today's, over a history without demand calls."""
    events, g = evidence()["generated"]["wide", "incr40"]
    events = [e for e in events if not (e[0] == "call" and e[1][0] == "demand")]
    checked = []

    def on_pass(h, i, kind, why):
        assert (h.d == 1).all()
        if kind not in eh.AUCTION or why is not None:
            return None
        S = h.params[0]
        warm = h.warm_plan()[0] if kind in ("warm", "repair") else False
        out = eh.expect_auction(h, kind, warm)
        if warm:
            assert h.changed_slots() == h.changed_asks()
            assert h.n_changes() == len(h.rows) + (h.n_workers - h.n_kept) + len(h.changed_asks()) + h.removed_held
            if kind == "warm":
                a, p, n, rel = h.warm(S)
                assert np.array_equal(a, out[0]) and np.array_equal(p, out[1]) and (n, len(rel)) == out[2:4]
            else:
                r = rp.market_repair(h, S)
                assert np.array_equal(r["assigned"], out[0]) and np.array_equal(r["price"], out[1])
            checked.append(kind)
        a = out[0]
        res = eh.expect_result(h, a)
        held = np.flatnonzero(a != eh.NONE)
        assert np.array_equal(res["group_ask"], held) and np.array_equal(res["group_members"], a[held])
        assert np.array_equal(res["group_off"], np.arange(len(held) + 1))
        assert np.array_equal(res["worker_ask"][a[held]], held) and np.array_equal(res["ask_count"], a != eh.NONE)
        if h.auc_state and not h.resized and h.auc_w == h.n_workers and h.mask.all():
            c1, c2 = eh.expect_certificate(h), ac.market_certificate(h, S, h.price, h.assigned)
            assert all(c1[k] == c2[k] for k in ac.FIELDS) and np.array_equal(c1["ask_bound"], c2["ask_bound"])
        return (warm,) + out

    rebuild(events, g.outcomes, eh.History("wide", eh.cutoff_of("incr40")), on_pass=on_pass)
    assert {"warm", "repair"} <= set(checked), checked


# ---- mutations: each wrong rule must change some prediction of the seeded histories
class CountPastKept(eh.History):
    def _slot_freed(self, gone):           # a removed slot's worker past n_kept counted too
        return int(len(gone))


class NoFreed(eh.History):
    def _slot_freed(self, gone):           # removed slots' workers not counted at all
        return 0


class AllSlotsA0(eh.History):
    def _kept_after(self, new):            # every slot of an ask whose demand changed in A0
        return np.where(new != self.d, 0, super()._kept_after(new))


class PassMin(eh.History):
    def _kept_after(self, new):            # min(demand at the pass, new demand) instead of the chain's minimum
        return np.minimum(self.d_pass, new)


class PriceReset(eh.History):
    def _free_price(self, workers):        # a removed slot's worker back at price 0
        self.price = self.price.copy()
        self.price[workers[workers < len(self.price)].astype(np.int64)] = 0


class KeepChanges(eh.History):
    def _restore_clear(self, price, kept):  # R0 and A0 kept across a restore
        rows, toggled, cap0, floors0 = self.rows, self.toggled, self.cap0, self.floors0
        super()._restore_clear(price, kept)
        self.rows, self.toggled, self.cap0, self.floors0 = rows, toggled, cap0, floors0


class HeirInE(eh.History):
    def split(self):                       # the heir listed in E instead of D
        en, dis = eh.split_toggles(self.mask, self.eval_mask, self.replaced)
        return en | self.heirs, dis


class NoHeir(eh.History):
    def _new_heirs(self, rm, keep):        # the heir not marked at all
        return set()


class RemovedPastKept(eh.History):
    def _removed_freed(self, gone):        # a removed ask's held slots past n_kept counted too
        return int((np.asarray(gone) != eh.NONE).sum())


class InsertedNotA0(eh.History):
    def _inserted_a0(self, at):            # an inserted ask's empty slot not in A0
        return set()


class DemKeptNotRemapped(eh.History):      # the kept slots of a demand chain left at their old indices
    def remove_asks(self, idx):
        k = self.dem_kept
        super().remove_asks(idx)
        if k is not None:
            self.dem_kept = k[:len(self.d)].copy()

    def insert_asks(self, before, rows):
        k = self.dem_kept
        at = super().insert_asks(before, rows)
        if k is not None:
            self.dem_kept = np.concatenate([k, np.ones(len(at), dtype=k.dtype)])
        return at


class SpliceNotResized(eh.History):        # a removal or an insertion leaves the certificate's resize flag
    def remove_asks(self, idx):
        r = self.resized
        super().remove_asks(idx)
        self.resized = r

    def insert_asks(self, before, rows):
        r = self.resized
        at = super().insert_asks(before, rows)
        self.resized = r
        return at


def differs(cls, shape, setting):
    """Replay a seeded history on the true mirror and on a mutated one side by side: does any incremental plan (full or
    not, rows walked), certificate refusal, warm decision, auction prediction (assignment, prices, rounds, n_released)
    or restore report differ?"""
    events, g = evidence()["generated"][shape, setting]
    t, m = eh.History(shape, eh.cutoff_of(setting)), cls(shape, eh.cutoff_of(setting))
    inputs = ("price", "assigned", "n_kept")
    for i, e in enumerate(events):
        if e[0] == "call":
            t.apply(e[1])
            m.apply(e[1])
            if e[1][0] in ("restore", "move") and t.last_report != m.last_report:
                return True
            continue
        if e[0] != "pass":
            continue
        why, _ = t.refusal(e[1])
        if e[1] in eh.INCREMENTAL and why is None and t.incremental_plan()[:2] != m.incremental_plan()[:2]:
            return True
        if e[1] == "certificate" and m.refusal(e[1])[0] != why:
            return True
        if e[1] in eh.REFERENCE:
            t.reference_done(why is None)
            m.reference_done(why is None)
            continue
        if e[1] not in eh.AUCTION or why is not None:
            continue
        out = g.outcomes[i]
        warm = out[0]
        if e[1] in ("warm", "repair") and m.warm_plan()[0] != warm:
            return True
        same = not warm or (all(np.array_equal(getattr(t, f), getattr(m, f)) for f in inputs)
                            and t.changed_rows() == m.changed_rows() and t.changed_slots() == m.changed_slots())
        mine = out if same else (warm,) + eh.expect_auction(m, e[1], warm)
        if not same and not (np.array_equal(mine[1], out[1]) and np.array_equal(mine[2], out[2])
                             and mine[3:] == out[3:]):
            return True
        t.auction_done(out[2], out[1])
        m.auction_done(mine[2], mine[1])
    return False


@pytest.mark.parametrize("cls", [CountPastKept, NoFreed, AllSlotsA0, PassMin, PriceReset, KeepChanges, HeirInE, NoHeir,
                                 RemovedPastKept, InsertedNotA0, DemKeptNotRemapped, SpliceNotResized],
                         ids=lambda c: c.__name__)
def test_a_wrong_rule_changes_a_prediction(cls):
    order = [("mixed", "incr40"), ("wide", "incr40")] + [(sh, st) for sh in eh.SHAPES for st in eh.SETTINGS
                                                         if st != "incr40"]
    assert any(differs(cls, sh, st) for sh, st in order), f"{cls.__name__}: no history tells it from the rule"


# ------------------------------------------------------------------ removals and insertions
def test_every_ask_delta_refusal_occurs():
    cases = evidence()["cases"]
    want = {("ask_delta_refused", c) for c in eh.DELTA_REFUSALS + eh.SPLICE_REFUSALS}
    assert cases >= want, sorted(want - cases)


def test_incremental_passes_walk_every_kind_of_heir():
    """Passes that stay incremental after a removal whose heir was enabled and untouched, disabled, replaced or
    inserted since the stored evaluation, after one that left a stored first ask without a row after it, and after a
    row inserted just before a stored first ask."""
    want = {"plain", "disabled", "replaced", "appended", "no_heir", "insert_before_first"}
    assert evidence()["splice_incr"] >= want, evidence()["splice_incr"]


def test_demand_chains_through_a_splice():
    assert "warm" in evidence()["splice_chain"], evidence()["splice_chain"]


def test_removed_held_slots_on_both_sides_of_n_kept_decide_the_cutoff():
    """Under PM_TUNE_INCR=40, warm and repair passes after removed asks whose slots held workers below and above
    n_kept, which are within the cutoff without the removed holds: cold where those pass it, warm where not, each
    side at least once."""
    held = evidence()["splice_held"]
    assert {k for k, _ in held} == {"warm", "repair"} and {w for _, w in held} == {False, True}, held


def test_the_certificate_waits_for_an_auction_pass_after_a_splice():
    assert evidence()["splice_cert"] >= {"refused", "ran"}, evidence()["splice_cert"]


def test_splices_cross_the_predicate_the_feature_budget_and_proximity_inside_one_window():
    """Inside one incremental window, splices turn the fast predicate off and on again, take the wide tables' current
    rows past 64 features and back, and enable and remove a max_group_size 0 row; a proximity pass right after such an
    insertion is refused and one right after its removal runs."""
    want = {"past_64_and_back", "fast_off_and_on", "max0_on_and_off", "proximity_refused", "proximity_cleared"}
    assert evidence()["crossings"] >= want, evidence()["crossings"]


def test_the_feature_row_takes_the_wide_tables_past_the_budget():
    for shape, n in (("mixed", 46), ("wide", 64)):
        s = eh.setup(shape)
        for k in (0, 1):
            assert len(ft.dictionary(ft.converted(s["asks"][k], s["opts"]))) == n
            with_row = np.concatenate([s["asks"][k], s["feature"]])
            assert len(ft.dictionary(ft.converted(with_row, s["opts"]))) == n + 1 and eh.asks_small(with_row, s["opts"])


@pytest.mark.parametrize("shape", eh.SHAPES)
def test_removing_the_tail_is_a_shrink_and_inserting_at_the_end_an_append(shape):
    """On the mirror, with a stored evaluation, a stored auction state and demands above 1."""
    import copy

    events, g = evidence()["generated"][shape, "default"]
    found = []

    def on_pass(h, i, kind, why):
        if not found and h.eval and h.auc_state and (h.d > 1).any() and h.held_asks()[-1] > len(h.asks) - 10:
            found.append(copy.deepcopy(h))

    rebuild(events, g.outcomes, eh.History(shape), on_pass=on_pass)
    assert found
    a, b = found[0], copy.deepcopy(found[0])
    T = len(a.asks)

    def same():
        for f in MIRROR:
            x, y = getattr(a, f), getattr(b, f)
            assert (x is None and y is None) or np.array_equal(x, y), f
        for f in TRACKED:
            x, y = getattr(a, f), getattr(b, f)
            assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f

    a.remove_asks(np.random.default_rng(1).permutation(np.arange(T - 10, T)))
    b.shrink_asks(T - 10)
    assert b.removed_held
    same()
    rows = a.s["pool"][:4]
    a.insert_asks(np.full(4, T - 10), rows)
    b.append_asks(rows)
    same()
