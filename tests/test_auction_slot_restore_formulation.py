"""The per-slot audit of pm_auction_restore_slots (prime_match.h "Auction state restore per slot", DESIGN 4) on the CPU.

The rule: on an engine with demands d the restore is pm_auction_restore on the twin table, which repeats row t d[t]
times, so the slot audit is auction_restore_checker.audit over F[slot_ask] and cap[slot_ask].  Here it is also
restated slot by slot over the ask table (the ask's row term, the slot's hold, ownership recounted over every slot)
and the two agree; it is idempotent; it drops nothing from the final twin states of the warm and repair checkers; on
constructed slot states it drops exactly the holds the rule names (two slots of one ask naming one worker, a worker
named across asks, infeasible holds, over-slack holds, PM_NONE kept as it is); and the warm and repair checkers
started from an audited slot state end within D of scipy's optimum, on it with cost_scale = D + 1."""
import numpy as np
import pytest

import auction_repair_checker as rp
import auction_restore_checker as rs
import auction_warm_checker as wc
from auction_demand import demand_certificate, offsets
from test_auction_restore_formulation import check_audited, check_next_passes
from test_auction_warm_formulation import market

NONE = wc.NONE
DROPS = ("n_dropped_bad", "n_dropped_shared", "n_dropped_slack")


def twin(F, cap, d):
    slot_ask = np.repeat(np.arange(len(d)), d)
    return F[slot_ask], np.asarray(cap)[slot_ask], slot_ask


def slot_audit(F, ap, cap, d, S, price, a_slots):
    """The audit restated per slot over the ask table: slot s of ask t is checked against F[t] and row(t)."""
    T, W = F.shape
    row = demand_certificate(F, ap, cap, d, S, price, a_slots)["ask_bound"]
    off = offsets(d)
    a_slots = np.asarray(a_slots, dtype=np.uint32)
    own = np.bincount(a_slots[a_slots != NONE].astype(np.int64), minlength=W)
    kept = np.full(len(a_slots), NONE, dtype=np.uint32)
    n = dict(n_held=0, n_dropped_bad=0, n_dropped_shared=0, n_dropped_slack=0)
    for t in range(T):
        for s in range(off[t], off[t + 1]):
            w = int(a_slots[s])
            if w == NONE:
                continue
            if not F[t, w]:
                n["n_dropped_bad"] += 1
            elif own[w] > 1:
                n["n_dropped_shared"] += 1
            elif int(ap[w]) * int(S) + int(price[w]) - int(row[t]) > 1:
                n["n_dropped_slack"] += 1
            else:
                kept[s] = w
                n["n_held"] += 1
    return dict(assigned=kept, **n)


def audit_both(F, ap, cap, d, S, price, a_slots):
    """The twin's audit, checked equal to the per-slot restatement; evals of the device's form (T x W)."""
    Fx, capx, _ = twin(F, cap, d)
    out = rs.audit(Fx, ap, capx, S, price, a_slots)
    mine = slot_audit(F, ap, cap, d, S, price, a_slots)
    assert np.array_equal(out["assigned"], mine["assigned"])
    assert all(out[k] == mine[k] for k in ("n_held",) + DROPS)
    assert out["evals"] == len(a_slots) * F.shape[1]   # the twin's D x W; the device reports T x W
    return out


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("S_mode", ["unit", "scaled", "exact"])
def test_adversarial_slot_states(seed, S_mode):
    m = market(25, 120, 30 + seed, floors=seed % 2 == 1)
    rng = np.random.default_rng(300 + seed)
    d = rng.choice([1, 2, 3, 4], len(m.asks)).astype(np.uint32)
    D = int(d.sum())
    S = {"unit": 1, "scaled": 7, "exact": D + 1}[S_mode]
    F, ap = m.F(), m.wb["ext_ask_price"]
    Fx, capx, _ = twin(F, m.cap, d)
    seen = dict.fromkeys(DROPS, 0)
    for _ in range(4):
        eps_start = int(rng.choice([1, 64]))
        price, a = rs.adversarial_state(Fx, ap, capx, S, rng, eps_start)
        assert price.max() <= rs.price_bound(m.cap, S, eps_start)   # the twin's bound is the engine's: same K
        out = audit_both(F, ap, m.cap, d, S, price, a)
        held = int((a != NONE).sum())
        assert out["n_held"] + sum(out[k] for k in DROPS) == held
        assert np.all((out["assigned"] == a) | (out["assigned"] == NONE))
        check_audited(Fx, ap, capx, S, price, out)
        again = audit_both(F, ap, m.cap, d, S, price, out["assigned"])   # idempotent
        assert np.array_equal(again["assigned"], out["assigned"]) and again["n_held"] == out["n_held"]
        assert all(again[k] == 0 for k in DROPS)
        for k in DROPS:
            seen[k] += out[k]
        check_next_passes(Fx, ap, capx, S, price, out["assigned"])   # within D of the optimum, on it with D + 1
    assert all(v > 0 for v in seen.values()), seen


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("S_mode", ["unit", "exact"])
def test_final_twin_states_pass_unchanged(seed, S_mode):
    m = market(30, 140, 40 + seed, floors=seed == 1)
    rng = np.random.default_rng(400 + seed)
    d = rng.choice([1, 2, 4], len(m.asks)).astype(np.uint32)
    D = int(d.sum())
    S = 1 if S_mode == "unit" else D + 1
    F, ap = m.F(), m.wb["ext_ask_price"]
    Fx, capx, _ = twin(F, m.cap, d)
    a, p, _ = wc.cold(Fx, ap, capx, S)
    for kind in ("warm", "repair"):
        pk, ak = p, a
        for _ in range(3):   # a changed row and a changed ask, then the pass from the stored state
            rows = [int(rng.integers(0, Fx.shape[1]))]
            asks = [int(rng.integers(0, D))]
            if kind == "warm":
                ak, pk, _, _ = wc.warm(Fx, ap, capx, S, pk, ak, Fx.shape[1], rows, asks)
            else:
                out = rp.repair(Fx, ap, capx, S, pk, ak, Fx.shape[1], rows, asks)
                ak, pk = out["assigned"], out["price"]
            got = audit_both(F, ap, m.cap, d, S, pk, ak)
            assert np.array_equal(got["assigned"], ak) and got["n_held"] == int((ak != NONE).sum())


def test_constructed_slot_states_drop_what_the_rule_names():
    """From a cold twin state (every hold kept), one change of each kind; the expected drops follow from the rule."""
    m = market(30, 160, 77)
    rng = np.random.default_rng(77)
    d = rng.choice([2, 3, 4], len(m.asks)).astype(np.uint32)
    F, ap = m.F(), m.wb["ext_ask_price"]
    Fx, capx, slot_ask = twin(F, m.cap, d)
    off = offsets(d)
    a, p, _ = wc.cold(Fx, ap, capx, 1)
    base = audit_both(F, ap, m.cap, d, 1, p, a)
    assert np.array_equal(base["assigned"], a) and all(base[k] == 0 for k in DROPS)
    held = np.flatnonzero(a != NONE)
    assert len(held) >= 6

    def expect(a2, bad=(), shared=(), slack=()):
        out = audit_both(F, ap, m.cap, d, 1, p, a2)
        kept = a2.copy()
        kept[list(bad) + list(shared) + list(slack)] = NONE
        assert np.array_equal(out["assigned"], kept)
        assert (out["n_dropped_bad"], out["n_dropped_shared"], out["n_dropped_slack"]) == (len(bad), len(shared), len(slack))
        assert out["n_held"] == int((kept != NONE).sum())

    # PM_NONE: a released slot is simply unheld
    a2 = a.copy()
    a2[held[0]] = NONE
    expect(a2)
    # two slots of one ask naming one worker: both are shared
    t = next(t for t in range(len(d)) if a[off[t]] != NONE)
    a2 = a.copy()
    a2[off[t] + 1] = a[off[t]]
    expect(a2, shared=[off[t], off[t] + 1])
    # a worker named by slots of two asks: both are shared, and a third naming counts too
    s1 = int(held[1])
    s2, s3 = (int(s) for s in [s for s in held if slot_ask[s] != slot_ask[s1]][:2])
    a2 = a.copy()
    a2[s2] = a[s1]
    a2[s3] = a[s1]
    infeasible = [s for s in (s2, s3) if not Fx[s, a[s1]]]
    expect(a2, bad=infeasible, shared=[s1] + [s for s in (s2, s3) if s not in infeasible])
    # an infeasible hold on a worker nobody else names: bad
    free = np.setdiff1d(np.arange(Fx.shape[1]), a[held])
    s = int(held[4])
    w_bad = next(int(w) for w in free if not Fx[s, w])
    a2 = a.copy()
    a2[s] = w_bad
    expect(a2, bad=[s])
    # a feasible, unshared hold far above the slot's row term: over-slack
    row = demand_certificate(F, ap, m.cap, d, 1, p, a)["ask_bound"]
    s, w_hi = next((int(s), int(w)) for s in held[5:] for w in free
                   if Fx[s, w] and int(ap[w]) + int(p[w]) - int(row[slot_ask[s]]) > 1)
    a2 = a.copy()
    a2[s] = w_hi
    expect(a2, slack=[s])
