"""The audit of pm_auction_restore (auction_restore_checker.py, DESIGN 4) on the CPU: the kept holds are feasible,
unshared and eps-complementary slack; the audit is idempotent and drops nothing from the final states of the cold,
eps-scaled, warm and repair checkers; and the warm and repair checkers started from an audited state, adversarial or
stale after table changes, end within T of scipy's optimum (on it with cost_scale = T + 1)."""
import numpy as np
import pytest

import auction_certificate as ac
import auction_repair_checker as rp
import auction_restore_checker as rs
import auction_reverse_checker as rc
import auction_warm_checker as wc
from test_auction_certificate_formulation import cost_of
from test_auction_warm_formulation import market

NONE = wc.NONE


def check_audited(F, ap, cap, S, price, out):
    a = out["assigned"]
    wc.check_feasible_injective(F, a)
    rp.check_held_eps_cs(F, ap, cap, S, price, a)
    c = ac.certificate(F, ap, cap, S, price, a)
    assert c["n_bad_holds"] == c["n_shared"] == 0
    assert all(c["slack"][t] <= 1 for t in np.flatnonzero(a != NONE))   # unheld asks may have slack: they bid next
    assert c["n_held"] == out["n_held"]


def check_next_passes(F, ap, cap, S, price, kept):
    """The warm and the repair checker from the audited state with nothing changed since: within T of the optimum, on
    it with S = T + 1."""
    T, W = F.shape
    opt = rc.optimum(F, ap, cap, S)
    a, p, _, rel = wc.warm(F, ap, cap, S, price, kept, W, [], [])
    out = rp.repair(F, ap, cap, S, price, kept, W, [], [], check=True)
    assert len(out["released"]) == 0
    for a, p in ((a, p), (out["assigned"], out["price"])):
        wc.check_feasible_injective(F, a)
        c = ac.certificate(F, ap, cap, S, p, a)
        assert c["n_priced_unowned"] == 0 and 0 <= c["gap"] <= T
        cost = cost_of(a, ap, cap, S)
        assert opt <= cost <= opt + T
        if S == T + 1:
            assert cost == opt


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("S_mode", ["unit", "scaled", "exact"])
def test_adversarial_states(seed, S_mode):
    m = market(30, 110, 50 + seed, floors=seed % 2 == 1)
    T = len(m.asks)
    S = {"unit": 1, "scaled": 7, "exact": T + 1}[S_mode]
    F, ap = m.F(), m.wb["ext_ask_price"]
    rng = np.random.default_rng(700 + seed)
    seen = dict(n_dropped_bad=0, n_dropped_shared=0, n_dropped_slack=0, priced_unowned=0)
    for _ in range(5):
        eps_start = int(rng.choice([1, 64]))
        price, a = rs.adversarial_state(F, ap, m.cap, S, rng, eps_start)
        assert price.max() <= rs.price_bound(m.cap, S, eps_start)
        out = rs.audit(F, ap, m.cap, S, price, a)
        held = int((a != NONE).sum())
        assert out["n_held"] + out["n_dropped_bad"] + out["n_dropped_shared"] + out["n_dropped_slack"] == held
        assert np.all((out["assigned"] == a) | (out["assigned"] == NONE))
        check_audited(F, ap, m.cap, S, price, out)
        again = rs.audit(F, ap, m.cap, S, price, out["assigned"])    # idempotent
        assert np.array_equal(again["assigned"], out["assigned"]) and again["n_held"] == out["n_held"]
        assert again["n_dropped_bad"] == again["n_dropped_shared"] == again["n_dropped_slack"] == 0
        for k in ("n_dropped_bad", "n_dropped_shared", "n_dropped_slack"):
            seen[k] += out[k]
        seen["priced_unowned"] += ac.certificate(F, ap, m.cap, S, price, out["assigned"])["n_priced_unowned"]
        check_next_passes(F, ap, m.cap, S, price, out["assigned"])
    assert all(v > 0 for v in seen.values()), seen


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("S_mode", ["unit", "exact"])
def test_final_states_of_every_checker_pass_unchanged(seed, S_mode):
    m = market(40, 150, 60 + seed, floors=seed == 1)
    T = len(m.asks)
    S = 1 if S_mode == "unit" else T + 1
    F, ap = m.F(), m.wb["ext_ask_price"]
    states = [m.cold(S)[:2]]
    states.append(rc.scaled(F, ap, m.cap, S, 64, 4, reverse_rounds=True)[:2])
    states.append(rc.scaled(F, ap, m.cap, S, 64, 4, reverse_rounds=False)[:2])   # priced unowned workers: kept as given
    for a, p in states:
        assert p.max(initial=0) <= rs.price_bound(m.cap, S, 64)
        out = rs.audit(F, ap, m.cap, S, p, a)
        assert np.array_equal(out["assigned"], a) and out["n_held"] == int((a != NONE).sum())
    rng = np.random.default_rng(800 + seed)
    for kind in ("warm", "repair"):
        m = market(40, 150, 60 + seed, floors=seed == 1)
        a, p, _ = m.cold(S)
        m.store(p, a)
        for _ in range(3):
            wc.random_step(m, rng)
            if kind == "warm":
                a, p, _, _ = m.warm(S)
            else:
                out = rp.market_repair(m, S)
                a, p = out["assigned"], out["price"]
            m.store(p, a)
            out = rs.market_audit(m, S, p, a)
            assert np.array_equal(out["assigned"], a) and out["n_held"] == int((a != NONE).sum())


@pytest.mark.parametrize("seed", range(4))
def test_stale_states_after_table_changes(seed):
    """A stored state, then random table changes (auction_warm_checker.random_step), then the audit against the new
    tables (rows past a shrink handed over as unheld, prices of added rows 0) and the next passes from it."""
    m = market(35, 130, 90 + seed, floors=seed % 2 == 0)
    T = len(m.asks)
    rng = np.random.default_rng(900 + seed)
    n_audited = n_dropped = 0
    for S in (1, T + 1):
        a, p, _ = m.cold(S)
        m.store(p, a)
        for _ in range(4):
            for _ in range(int(rng.integers(1, 4))):
                wc.random_step(m, rng)
            W = m.n_workers
            price = np.zeros(W, dtype=np.int64)
            k = min(W, len(m.price))
            price[:k] = m.price[:k]
            assigned = np.where(m.assigned < W, m.assigned, NONE).astype(np.uint32)
            F, ap = m.F(), m.wb["ext_ask_price"]
            if price.max(initial=0) > rs.price_bound(m.cap, S):
                continue   # the largest cap went down: the engine refuses such a state (PM_E_INVALID)
            out = rs.audit(F, ap, m.cap, S, price, assigned)
            n_audited += 1
            n_dropped += out["n_dropped_bad"] + out["n_dropped_slack"]
            check_audited(F, ap, m.cap, S, price, out)
            check_next_passes(F, ap, m.cap, S, price, out["assigned"])
            a, p, _, _ = wc.warm(F, ap, m.cap, S, price, out["assigned"], W, [], [])
            m.store(p, a)
    assert n_audited >= 6 and n_dropped > 0
