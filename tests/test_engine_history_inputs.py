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
from protocol_b200 import synth


@functools.lru_cache(maxsize=None)
def evidence():
    """Replay every history the GPU file runs on the mirror alone and record what each pass saw."""
    ev = dict(call_pass=set(), pass_pass=set(), refusals={}, after_refusal={}, incr_after_auction_cert=0,
              warm_after_both=set(), flips=set(), incr_over=0, warm_over=0, n_passes=0)
    for shape in eh.SHAPES:
        for setting in eh.SETTINGS:
            cutoff = eh.cutoff_of(setting)
            events, _ = eh.generate(shape, eh.seed_of(shape, setting), cutoff=cutoff, slot=eh.slot_of(shape, setting),
                                    n_slots=eh.N_SLOTS)
            h = eh.History(shape, cutoff)
            last, calls = "start", []
            # refusals waiting for the next incremental pass on the kept evaluation, and for the next warm pass on
            # the auction state they left (name, whether a stored state existed)
            pend_incr, pend_warm = [], []
            since_eval = dict(auction=0, certificate=0)
            since_state = dict(ff=0, prox=0, disabled_across=False)
            for e in events:
                if e[0] == "call":
                    h.apply(e[1])
                    calls.append(e[1][0])
                    if e[1][0] in ("set_asks", "model_table", "set_workers"):
                        since_eval = dict(auction=0, certificate=0)
                        pend_incr, pend_warm = [], []
                    if e[1][0] == "auction_params":
                        pend_warm = []
                    if not h.auc_state:
                        since_state = dict(ff=0, prox=0, disabled_across=False)
                    continue
                kind = e[1]
                ev["n_passes"] += 1
                why, _ = h.refusal(kind)
                if why is not None:
                    ev["refusals"][why] = ev["refusals"].get(why, 0) + 1
                if kind in eh.INCREMENTAL and why is None:
                    full, n_tiles, en, dis, sure = h.incremental_plan()
                    if not full and h.dirty and since_eval["auction"] and since_eval["certificate"]:
                        ev["incr_after_auction_cert"] += 1
                    if not full:
                        ev["flips"] |= h.flipped
                    if full and h.eval and h.over and cutoff < eh.DEFAULT_CUTOFF:
                        ev["incr_over"] += 1
                    for r in pend_incr:
                        ev["after_refusal"].setdefault(r, set()).add("incremental")
                if kind in ("warm", "repair") and why is None:
                    warm, _ = h.warm_plan()
                    if warm and since_state["ff"] and since_state["prox"] and since_state["disabled_across"]:
                        ev["warm_after_both"].add(kind)
                    if h.auc_state and not warm and h.auc_over and cutoff < eh.DEFAULT_CUTOFF:
                        ev["warm_over"] += 1
                    for r, had_state in pend_warm:   # warm on the kept state, or cold where there was none
                        if warm == had_state:
                            ev["after_refusal"].setdefault(r, set()).add("warm")
                    pend_warm = []
                if kind in eh.REFERENCE and why is None:
                    pend_incr = []               # this pass stores an evaluation: the refusals are behind it
                if kind in ("auction", "reverse") and why is None:
                    pend_warm = []               # a new stored state
                if why is not None:
                    pend_incr.append(why)
                    pend_warm.append((why, h.auc_state))
                if kind in eh.REFERENCE:
                    if why is None:
                        since_state["prox" if kind.startswith("proximity") else "ff"] += 1
                        since_state["disabled_across"] |= bool(h.auc_state and not h.mask.all())
                    h.reference_done(why is None)
                    since_eval = dict(auction=0, certificate=0)
                elif kind in eh.AUCTION:
                    since_eval["auction"] += 1
                    if why is None:
                        h.auction_done(None, None)
                        since_state = dict(ff=0, prox=0, disabled_across=False)
                elif kind == "certificate":
                    since_eval["certificate"] += 1
                if kind != "auction_incr":
                    ev["call_pass"] |= {(c, kind) for c in calls}
                    ev["pass_pass"].add((last, kind))
                    last = kind
                    calls = []
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
