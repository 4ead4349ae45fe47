"""PM_MODE_AUCTION at the edges of its integer domain on the device, bit for bit against the exact-integer checker
(auction_exact.py): u32 prices, caps, reputations and floors at 0, 2^31 and 2^32 - 1; both sides of the packed-key
switch (every reachable cost below 2^40) and of the packed claim (fewer than 2^23 asks, fewer than 2^24 workers); the
largest admitted cost_scale and eps_start, and the refusal one step past them that leaves the stored state alone;
warm chains and reverse passes at edge values.  Every instance's round count is checked on the CPU first."""
import os

import numpy as np
import pytest

import auction_exact as ex
import auction_warm_checker as wc
from protocol_b200 import abi
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine
from test_auction_exact_checker import U32, feasible, ladder, last_admitted_scale, open_market, tables

pytestmark = pytest.mark.gpu

NONE = ex.NONE
AUC, REV, WARM = abi.PM_MODE_AUCTION, abi.PM_MODE_AUCTION | abi.PM_AUCTION_REVERSE, abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM
TUNES = [0, 2, 8, 64, 128]
MAX_ROUNDS = 20000
EDGE = [0, 1, 0x7FFFFFFF, 0x80000000, U32 - 1, U32]
EDGE_CAP = [0, 0x7FFFFFFF, U32 - 1, U32]
RESULT_LAUNCHES = 2   # pm_stats.n_launches of an auction pass: 6 or 7 per round, then the two kernels that emit the result


def engine(t, cap, tune=0, reputation=None, floors=None):
    if tune:
        os.environ["PM_TUNE_AUCTION"] = str(tune)
    try:
        eng = Engine()
    finally:
        os.environ.pop("PM_TUNE_AUCTION", None)
    eng.set_asks(t["asks"], t["opts"])
    if t["n_patterns"]:
        eng.set_model_table(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    eng.set_workers(t["wa"], t["wb"])
    eng.set_price_caps(cap)
    if reputation is not None:
        eng.set_worker_reputation(reputation)
    if floors is not None:
        eng.set_min_reputation(floors)
    return eng


def run(eng, T, mode):
    eng.match(mode)
    res = eng.fetch()
    got = np.full(T, NONE, dtype=np.uint32)
    for ask, members in res.groups():
        assert len(members) == 1
        got[ask] = members[0]
    price, warm, released = eng.auction_state()
    return got, price, res.stats, warm, released, eng.auction_reverse_stats()


def plan(t, cap, S, eps_start=1, eps_div=4, reverse=False, reputation=None, floors=None, feas=None):
    """The exact checker's cold pass, its round counts bounded on the CPU before any device runs the instance."""
    F = ex.lists_from_matrix(feasible(t, cap, reputation, floors)) if feas is None else feas
    A = ex.Auction(len(cap), F, t["wb"]["ext_ask_price"], cap, S)
    st = A.scaled(eps_start, eps_div, reverse=reverse, max_rounds=MAX_ROUNDS)
    assert st["fwd"] + st["rev"] < MAX_ROUNDS
    return A, st


def check_cold(eng, A, st, S, eps_start=1, eps_div=4, reverse=False):
    eng.set_auction_params(cost_scale=S, eps_start=eps_start, eps_div=eps_div)
    got, price, stats, warm, released, rs = run(eng, A.n_asks, REV if reverse else AUC)
    assert np.array_equal(got, A.assignment())
    assert np.array_equal(price, A.prices(len(price)))
    assert stats["n_rounds"] == st["fwd"]
    assert not warm and released == 0
    assert rs == ((st["phases"], st["rev"], st["bids"]) if reverse else (0, 0, 0))
    return stats


# ---------------------------------------------------------------- u32 edges
def edge_market(seed):
    """40 ordinary workers and every edge price twice; 24 asks, caps mixing the edges with ordinary ones; reputations
    and floors at 0 or 0xFFFFFFFF.  Ordinary prices and caps lie close together, so that no price war outlasts a few
    thousand rounds at cost_scale = T + 1."""
    rng = np.random.default_rng(seed)
    ap = np.concatenate([rng.integers(10, 60, 40), EDGE, EDGE]).astype(np.uint32)
    ap = ap[rng.permutation(len(ap))]
    cap = np.concatenate([rng.integers(20, 80, 12), EDGE_CAP, EDGE_CAP, [U32, U32, 0x80000000, 1]]).astype(np.uint32)
    cap = cap[rng.permutation(len(cap))]
    t, cap = open_market(len(cap), len(ap), ap, cap)
    t["wa"]["flags"][rng.choice(len(ap), 6, replace=False)] = 0   # a few rows are no candidate
    rep = rng.choice(np.array([0, 1, 7, U32], dtype=np.uint32), len(ap))
    floors = rng.choice(np.array([0, 0, 1, U32], dtype=np.uint32), len(cap))
    return t, cap, rep, floors


@pytest.mark.parametrize("tune", TUNES)
@pytest.mark.parametrize("seed", [1, 2])
def test_u32_edges_cold(seed, tune):
    t, cap, rep, floors = edge_market(seed)
    T = len(cap)
    plans = [(S, *plan(t, cap, S, reputation=rep, floors=floors)) for S in (1, T + 1)]
    eng = engine(t, cap, tune=tune, reputation=rep, floors=floors)
    for S, A, st in plans:
        check_cold(eng, A, st, S)
    eng.close()


@pytest.mark.parametrize("tune", [0, 128])
def test_u32_edges_reverse(tune):
    t, cap, rep, floors = edge_market(3)
    T = len(cap)
    A, st = plan(t, cap, T + 1, 1 << 40, 16, reverse=True, reputation=rep, floors=floors)
    assert st["rev"] > 0
    eng = engine(t, cap, tune=tune, reputation=rep, floors=floors)
    check_cold(eng, A, st, T + 1, 1 << 40, 16, reverse=True)
    eng.close()


# ---------------------------------------------------------------- packed keys
def packed_ok(P, K, S, E):
    """pm_auction_decide_packed's rule, restated: every reachable cost below 2^40."""
    lim = 1 << 40
    return S < lim and E < lim and P + K + 2 < (lim - E) // S


def last_packed_scale(P, K, E=1):
    S = max(1, ((1 << 40) - E) // (P + K + 3))
    while packed_ok(P, K, S + 1, E):
        S += 1
    while not packed_ok(P, K, S, E):
        S -= 1
    return S


PACKED_CASES = [   # (ladder prices, caps): scarce rungs whose price climbs to the cap's outside option
    ([1, 2, 3, 0x80000000], [U32, U32, U32 - 1, U32]),
    ([0, 5, 1000, 1001], [1500, 1001, 1500, 2000]),
]


@pytest.mark.parametrize("case", range(len(PACKED_CASES)))
def test_packed_key_boundary(case):
    ap, caps = PACKED_CASES[case]
    t, cap, rep, floors = ladder(ap, caps)
    P, K = max(ap), max(caps)
    S = last_packed_scale(P, K)
    assert packed_ok(P, K, S, 1) and not packed_ok(P, K, S + 1, 1)
    for s, want_packed in ((S, True), (S + 1, False)):
        A, st = plan(t, cap, s, reputation=rep, floors=floors)
        for tune in (0, 128):
            eng = engine(t, cap, tune=tune, reputation=rep, floors=floors)
            stats = check_cold(eng, A, st, s)
            eng.close()
            per_round = 6 if (want_packed and tune == 0) else 7   # the packed claim needs no pm_auction_claim
            assert stats["n_launches"] == per_round * stats["n_rounds"] + RESULT_LAUNCHES, (s, tune)
    # the cost reached: within one scale step of the limit the packed key was built for
    A, _ = plan(t, cap, S, reputation=rep, floors=floors)
    top = max(-A.a[w] + A.price.get(w, 0) for w in A.assigned.values())
    assert top >= (1 << 40) // 2


# ---------------------------------------------------------------- index fields
def sparse_market(T, W, contested):
    """T asks without requirements, W workers of which only the last three are candidates; the last `contested` asks
    have caps that reach them, every other ask has cap 0 (every price is at least 1): one feasible list per contested
    ask, every other ask withdraws in the first round."""
    a = np.zeros(W, dtype=abi.WORKER_A)
    b = np.zeros(W, dtype=abi.WORKER_B)
    b["ext_ask_price"] = 1
    a["flags"][W - 3:] = abi.PM_W_HEALTHY | abi.PM_W_P2P
    b["ext_ask_price"][W - 3:] = [9, 5, 7]
    asks = np.zeros(T, dtype=abi.ASK)
    asks["min_group_size"] = asks["max_group_size"] = 1
    cap = np.zeros(T, dtype=np.uint32)
    cap[T - contested:] = [8, 100, U32][:contested]
    feas = {}
    for k in range(T - contested, T):
        feas[k] = [w for w in range(W - 3, W) if b["ext_ask_price"][w] <= cap[k]]
    t = dict(asks=asks, opts=np.zeros(0, dtype=abi.GPU_OPT), wa=a, wb=b, bits=np.array([U32], dtype=np.uint32),
             n_patterns=0, n_models=0, words=1)
    return t, cap, feas


@pytest.mark.parametrize("T,W,claim_packed", [((1 << 23) - 1, 1000, True), (1 << 23, 1000, False),
                                              (64, (1 << 24) - 1, True), (64, 1 << 24, False)])
def test_index_fields(T, W, claim_packed):
    """The top ask and worker indices of the packed claim ((bid << 23) | (2^23 - 1 - ask)) and of the packed key
    ((-value) << 24 | worker), and one past them."""
    t, cap, feas = sparse_market(T, W, 3)
    A, st = plan(t, cap, 1, feas=feas)
    assert (A.assignment()[T - 3:] != NONE).sum() == 3
    eng = engine(t, cap)
    stats = check_cold(eng, A, st, 1)
    assert stats["n_launches"] == (6 if claim_packed else 7) * stats["n_rounds"] + RESULT_LAUNCHES
    check_cold(eng, A, st, 1, reverse=True)
    eng.close()


# ---------------------------------------------------------------- the top of the domain
DOMAIN_CASES = [
    ([1, 2, (1 << 31) + 3], [U32, U32 - 1, U32], (1 << 31) + 3),
    ([0, 0x7FFFFFFF, 0x80000000, U32 - 1], [U32, 0x80000000, U32, U32 - 1], U32),
    ([5, 6, 1000], [1500, 1499, 1500], 2000),
]


@pytest.mark.parametrize("case", range(len(DOMAIN_CASES)))
@pytest.mark.parametrize("tune", [0, 128])
def test_top_of_the_domain(case, tune):
    ap, caps, P = DOMAIN_CASES[case]
    t, cap, rep, floors = ladder(ap, caps, extra_price=P)
    K = max(caps)
    S = last_admitted_scale(P, K)
    E = (1 << 61) - 1 - (P + K + 2) * (len(caps) + 1)
    A, st = plan(t, cap, S, reputation=rep, floors=floors)
    B, bst = plan(t, cap, len(caps) + 1, E, 1 << 20, reverse=True, reputation=rep, floors=floors)
    eng = engine(t, cap, tune=tune, reputation=rep, floors=floors)
    check_cold(eng, B, bst, len(caps) + 1, E, 1 << 20, reverse=True)
    check_cold(eng, A, st, S)
    # one step past either: pm_match refuses
    for s, e in ((S + 1, 1), (len(caps) + 1, E + 1)):
        eng.set_auction_params(cost_scale=s, eps_start=e)   # (set_auction_params discards the state: pass again)
        with pytest.raises(PrimeMatchError) as exc:
            eng.match(AUC)
        assert exc.value.status == abi.PM_E_INVALID
    eng.set_auction_params(cost_scale=S)
    check_cold(eng, A, st, S)
    for s, e in ((1 << 61, 1), (1, 1 << 61), ((1 << 64) - 1, 1)):   # refused whatever the tables; the state stays
        with pytest.raises(PrimeMatchError) as exc:
            eng.set_auction_params(cost_scale=s, eps_start=e)
        assert exc.value.status == abi.PM_E_INVALID
    assert np.array_equal(eng.auction_state()[0], A.prices(len(t["wa"])))
    eng.close()


@pytest.mark.parametrize("tune", [0, 128])
def test_a_refused_pass_keeps_the_stored_state(tune):
    """A row written past the domain (P from 3 to 0xFFFFFFFF at the largest scale P = 3 admits): every auction pass is
    refused and the stored state is still the one reported; written back, a warm pass starts from that state."""
    t, cap, rep, floors = ladder([1, 2, 3], [100, 100, 100], extra_price=1)
    S = last_admitted_scale(3, 100)
    A, st = plan(t, cap, S, reputation=rep, floors=floors)
    eng = engine(t, cap, tune=tune, reputation=rep, floors=floors)
    check_cold(eng, A, st, S)
    state = eng.auction_state()
    rs = eng.auction_reverse_stats()
    for s, e in ((1 << 61, 1), (1, 1 << 61)):
        with pytest.raises(PrimeMatchError) as exc:
            eng.set_auction_params(cost_scale=s, eps_start=e)
        assert exc.value.status == abi.PM_E_INVALID
    W = len(t["wa"])
    row = np.array([W - 1], dtype=np.uint32)
    b = t["wb"][row].copy()
    b["ext_ask_price"] = U32
    eng.update_workers(row, t["wa"][row], b)
    for mode in (AUC, WARM, REV):
        with pytest.raises(PrimeMatchError) as exc:
            eng.match(mode)
        assert exc.value.status == abi.PM_E_INVALID
    after = eng.auction_state()
    assert np.array_equal(after[0], state[0]) and after[1:] == state[1:] and eng.auction_reverse_stats() == rs
    eng.update_workers(row, t["wa"][row], t["wb"][row])          # back inside: a warm pass from the kept state
    got, price, stats, warm, released, _ = run(eng, len(cap), WARM)
    Wm = ex.Auction(len(cap), ex.lists_from_matrix(feasible(t, cap, rep, floors)), t["wb"]["ext_ask_price"], cap, S)
    wst = Wm.warm(state[0], A.assignment(), W, W, [W - 1], [])
    assert warm and released == wst["released"]
    assert np.array_equal(got, Wm.assignment()) and np.array_equal(price, Wm.prices(W)) and stats["n_rounds"] == wst["fwd"]
    eng.close()


# ---------------------------------------------------------------- warm chains at edge values
def edge_step(m: wc.Market, rng, eng):
    """Write edge prices into a few rows, or edge caps into a few asks."""
    W, T = m.n_workers, len(m.asks)
    if rng.random() < 0.5:
        idx = np.unique(rng.choice(W, 3, replace=False)).astype(np.uint32)
        a, b = m.wa[idx].copy(), m.wb[idx].copy()
        b["ext_ask_price"] = rng.choice(np.array(EDGE, dtype=np.uint32), len(idx))
        m.write(idx, a, b, eng)
    else:
        cap = m.cap.copy()
        idx = rng.choice(T, 2, replace=False)
        cap[idx] = rng.choice(np.array(EDGE_CAP, dtype=np.uint32), len(idx))
        m.set_caps(cap, eng)


def exact_warm(m: wc.Market, S):
    A = ex.Auction(len(m.asks), ex.lists_from_matrix(m.F()), m.wb["ext_ask_price"], m.cap, S)
    st = A.warm(m.price, m.assigned, m.n_kept, m.n_workers, m.changed_rows(), m.changed_asks(), max_rounds=MAX_ROUNDS)
    return A, st


def warm_chain_plan(t, cap, seed, steps, S):
    """The whole chain on the CPU: each step's changes and the exact warm pass after them."""
    m = wc.Market(t, cap)
    A, st = plan(t, cap, S)
    m.store(A.prices(len(t["wa"])), A.assignment())
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(steps):
        edge_step(m, rng, None)
        B, bst = exact_warm(m, S)
        out.append((B.assignment(), B.prices(m.n_workers), bst))
        m.store(B.prices(m.n_workers), B.assignment())
    return A, st, out


@pytest.mark.parametrize("S", [1, 51])
@pytest.mark.parametrize("tune", [0, 128])
def test_warm_chain_at_edge_values(S, tune):
    t, cap = tables(50, 700, 2)
    A, st, want = warm_chain_plan(t, cap, 40 + S, 6, S)
    m = wc.Market(t, cap)
    eng = engine(t, cap, tune=tune)
    check_cold(eng, A, st, S)
    m.store(A.prices(700), A.assignment())
    rng = np.random.default_rng(40 + S)
    for a, p, wst in want:
        edge_step(m, rng, eng)
        got, price, stats, warm, released, _ = run(eng, len(cap), WARM)
        assert warm and released == wst["released"]
        assert np.array_equal(got, a) and np.array_equal(price, p) and stats["n_rounds"] == wst["fwd"]
        m.store(p, a)
    eng.close()
