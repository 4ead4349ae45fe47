"""The collapsed reference (tests/collapsed_oracle.py) against the dense oracle it stands in for.

Every array of Reference.result() and Reference.local() must equal what orc.soa_eval_matrix and orc.soa_form_groups
compute on the whole table, and collapsed_oracle.certificate() must equal auction_certificate.certificate() on the
dense feasibility matrix, field by field and row by row.  The tables cover the three ask kinds, every price column
(sign edges of the packed cost's high word included), wide model catalogues, every kind of non-candidate worker,
max_group_size == 0 rows, duplicated and disabled asks, and shard ranges at the start, middle and end of the table.

At the benchmark's own shapes (cfg3, and cfg5's per-GPU shape) the reference is built in full and held to reach
assertions, so that the GPU comparisons there are not vacuous: every cost tile holds feasible and infeasible asks, the
row minima carry prices and land in dozens of stripes, past the first quarter of the table, and the collapse stays
small enough to build in seconds.
"""
import importlib.util
import os
import time

import numpy as np
import pytest

import auction_certificate as ac
import auction_warm_checker as wc
import collapsed_oracle as co
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE, INF = co.NONE, co.INF
SIGN_EDGES = np.array([0, 1, 0x7FFFFFFE, 0x7FFFFFFF, 0x80000000, 0x80000001, 0xFFFFFFFE, 0xFFFFFFFF], dtype=np.uint32)


def make_table(kind, price, n_models, T, W, seed):
    """Synthetic tables with every edge the collapse must keep apart: assigned workers on top of synth's unhealthy,
    p2p-less, spec-less and memory-less ones, max_group_size == 0 rows, and asks duplicated elsewhere in the table."""
    rng = np.random.default_rng(seed)
    cat = synth.wide_model_catalogue(n_models) if n_models else None
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed, price=None if price == "edges" else price, catalogue=cat)
    a = synth.make_asks(T, kind, seed=synth.SEED_ASKS + seed)
    wa, wb = w.a.copy(), w.b.copy()
    if price == "edges":
        wb["ext_ask_price"] = rng.choice(SIGN_EDGES, W)
    wa["flags"][rng.random(W) < 0.03] |= abi.PM_W_ASSIGNED
    asks = a.asks.copy()
    asks["max_group_size"][rng.random(T) < 0.02] = 0
    dup = rng.choice(T, T // 10, replace=False)
    asks[dup] = asks[rng.choice(T, T // 10)]            # duplicates share their option rows
    bits, npat, nmod, words = orc.model_table(w.model_strings, a.pattern_strings, threads=co.threads())
    return dict(wa=wa, wb=wb, asks=asks, opts=a.opts, bits=bits, n_patterns=npat, n_models=nmod, words=words)


def reference(t, enabled=None):
    return co.Reference(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["n_patterns"], t["n_models"], t["words"],
                        enabled=enabled)


def dense(t, enabled, w0=0, w1=None):
    """The oracle on the whole table: the enabled asks alone (a disabled ask is absent), indices mapped back."""
    W, T = len(t["wa"]), len(t["asks"])
    w1 = W if w1 is None else w1
    idx = np.flatnonzero(enabled).astype(np.uint32)
    sub = t["asks"][idx]
    ev = orc.soa_eval_matrix(t["wa"], t["wb"], sub, t["opts"], t["bits"], t["words"], 0, len(sub), w0, w1,
                             threads=co.threads())
    up = lambda x: np.where(x == NONE, NONE, idx[np.minimum(x, max(len(idx) - 1, 0))] if len(idx) else NONE).astype(np.uint32)
    best = np.full(T, INF, dtype=np.int64)
    cnt = np.zeros(T, dtype=np.uint32)
    best[idx], cnt[idx] = ev["row_best"], ev["row_count"]
    return up(ev["col_first"]), best, cnt, sub, up


CASES = {
    "uniform1_unpriced": ("uniform1", None, 0, 1000, 20000),
    "mixed_loguniform": ("mixed", "loguniform", 0, 3000, 30000),
    "skewed_zipf": ("skewed", "zipf", 0, 3000, 30000),
    "mixed_sign_edges": ("mixed", "edges", 0, 2000, 20000),
    "mixed_200_models": ("mixed", "loguniform", 200, 2000, 20000),
    "skewed_3000_models": ("skewed", "zipf", 3000, 2000, 20000),
    "mixed_100000_models": ("mixed", "zipf", 100_000, 2000, 30000),
}


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("toggled", [False, True], ids=["all_enabled", "disabled_asks"])
def test_collapsed_result_equals_dense(name, toggled):
    kind, price, n_models, T, W = CASES[name]
    seed = 1 + list(CASES).index(name)
    t = make_table(kind, price, n_models, T, W, seed)
    rng = np.random.default_rng(seed + 100)
    enabled = rng.random(T) < 0.7 if toggled else np.ones(T, dtype=bool)
    ref = reference(t, enabled if toggled else None)
    assert ref.P < W // 2 and ref.U < T          # the collapse did collapse
    got = ref.result()
    first, best, cnt, sub, up = dense(t, enabled)
    og = orc.soa_form_groups(t["wa"], t["wb"], sub, t["opts"], t["bits"], t["words"])
    wg = np.full(W, NONE, dtype=np.uint32)
    wg[og.members] = np.arange(len(og.cfg), dtype=np.uint32)
    want = dict(worker_group=wg, worker_ask=first, group_ask=up(og.cfg), group_off=og.off, group_members=og.members,
                ask_best=best, ask_count=cnt)
    for f in co.FIELDS:
        assert np.array_equal(got[f], want[f]), f
    lean = ref.result(ask_stats=False)
    assert (lean["ask_best"] == INF).all() and (lean["ask_count"] == 0).all()
    assert all(np.array_equal(lean[f], got[f]) for f in co.FIELDS[:5])
    # the case is not vacuous: feasible pairs, priced minima, and (sign edges) negative packed costs
    assert (cnt > 0).sum() > T // 4 and len(og.cfg) > W // 10
    if price == "edges":
        assert (best[cnt > 0] < 0).any() and (best[cnt > 0] > 0).any()
    if n_models:
        assert len(np.unique(ref.classes)) < n_models     # the class remap merged model ids


@pytest.mark.parametrize("name", ["mixed_loguniform", "mixed_sign_edges", "mixed_100000_models"])
def test_collapsed_ranges_equal_dense(name):
    """Reference.local over [w0, w0 + n): the first ask over the range, per-ask minimum and count over the range."""
    kind, price, n_models, T, W = CASES[name]
    seed = 1 + list(CASES).index(name)
    t = make_table(kind, price, n_models, T, W, seed)
    enabled = np.random.default_rng(seed).random(T) < 0.8
    ref = reference(t, enabled)
    for w0, n in ((0, W // 3), (W // 2 - 17, W // 4 + 5), (W - 1, 1), (0, W)):
        got = ref.local(w0, n)
        first, best, cnt, _, _ = dense(t, enabled, w0, w0 + n)
        fa = np.full(W, NONE, dtype=np.uint32)
        fa[w0:w0 + n] = first
        assert np.array_equal(got["first_ask"], fa), (w0, n)
        assert np.array_equal(got["ask_best"], best), (w0, n)
        assert np.array_equal(got["ask_count"], cnt), (w0, n)


def test_collapsed_refuses_group_sizes_beyond_solo():
    t = make_table("mixed", None, 0, 50, 500, 9)
    t["asks"]["max_group_size"][3] = 2
    with pytest.raises(ValueError):
        reference(t)


# ------------------------------------------------------------------ the auction certificate, collapsed
def _market(T, W, seed, floors):
    rng = np.random.default_rng(seed)
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed, price="loguniform")
    a = synth.make_asks(T // 4, "mixed", seed=synth.SEED_ASKS + seed)
    asks = a.asks[rng.integers(0, T // 4, T)].copy()          # duplicated rows with different caps
    asks["max_group_size"][rng.random(T) < 0.05] = 0           # a reference-mode clause the certificate ignores
    bits, npat, nmod, words = orc.model_table(w.model_strings, a.pattern_strings)
    cap = rng.integers(5, 400, T).astype(np.uint32)
    rep = fl = None
    if floors:
        rep = rng.integers(0, 6, W).astype(np.uint32)
        fl = np.where(rng.random(T) < 0.5, 0, rng.integers(1, 7, T)).astype(np.uint32)
    return dict(wa=w.a.copy(), wb=w.b.copy(), asks=asks, opts=a.opts, bits=bits, n_patterns=npat, n_models=nmod,
                words=words), cap, rep, fl, rng


def _both(m, cap, S, price, assigned, rep, fl):
    F = wc.feasible(m["wa"], m["wb"], m["asks"], m["opts"], m["bits"], m["words"], cap, rep, fl)
    want = ac.certificate(F, m["wb"]["ext_ask_price"], cap, S, price, assigned)
    got = co.certificate(m["wa"], m["wb"], m["asks"], m["opts"], m["bits"], m["n_patterns"], m["n_models"], m["words"],
                         cap, S, price, assigned, reputation=rep, floors=fl)
    for f in co.CERT_FIELDS:
        assert got[f] == want[f], f
    assert np.array_equal(got["ask_bound"], want["ask_bound"]) and got["slack"] == want["slack"]
    return got


@pytest.mark.parametrize("S,eps_start,floors", [(1, 1, False), (3, 1, True), (5, 64, False), (7, 32, True)],
                         ids=["S1", "S3_floors", "S5_eps_scaled", "S7_eps_scaled_floors"])
def test_collapsed_certificate_equals_dense(S, eps_start, floors):
    T, W = 400, 3000
    m, cap, rep, fl, rng = _market(T, W, 30 + S, floors)
    assigned, price, _ = orc.soa_auction(m["wa"], m["wb"], m["asks"], m["opts"], m["bits"], m["words"], cap, cost_scale=S,
                                         eps_start=eps_start, eps_div=4, reputation=rep, min_reputation=fl)
    c0 = _both(m, cap, S, price, assigned, rep, fl)
    assert c0["n_held"] > T // 4 and c0["n_bad_holds"] == 0
    # stale holds: rows rewritten after the pass (other specs, health, prices), caps lowered under some holds
    held = np.flatnonzero(assigned != NONE)
    wr = assigned[rng.choice(held, 40, replace=False)]
    src = rng.integers(0, W, len(wr))
    m["wa"][wr], m["wb"][wr] = m["wa"][src], m["wb"][src]
    m["wa"]["flags"][wr[:10]] &= ~np.uint32(abi.PM_W_HEALTHY)
    cap2 = cap.copy()
    cap2[held[:20]] = 0
    # shared holds and priced unowned workers
    a2 = assigned.copy()
    a2[held[20:30]] = a2[held[30:40]]
    p2 = price.copy()
    unowned = np.setdiff1d(np.arange(W), a2[a2 != NONE])
    p2[rng.choice(unowned, 50, replace=False)] += rng.integers(1, 1000, 50)
    c1 = _both(m, cap2, S, p2, a2, rep, fl)
    assert c1["n_bad_holds"] > 0 and c1["n_shared"] > 0 and c1["n_priced_unowned"] > 0 and c1["n_slack_over"] > 0


# ------------------------------------------------------------------ reach at the benchmark's shapes
def bench_module():
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def tile_rows(T, W, tile_bytes=8 << 30):
    """Asks per cost tile of a materialised pass (pm_match's tiling): 8 bytes per element over whole 1024-column
    stripes, rounded down to 512-row bands from 1024 rows on."""
    ld = -(-W // 1024) * 1024
    rows = min(max(tile_bytes // (ld * 8), 1), T)
    return rows & ~511 if rows >= 1024 else rows


# workload: (profiles at most, distinct rows at most, price levels among the row minima at least).  The bounds on the
# collapse make a synth change that defeats it fail here, at once.  Under cfg5's Zipf prices every row minimum is at
# the lowest level.
REACH = {"cfg3": (40_000, 15_000, 2), "cfg5": (40_000, 70_000, 1)}


@pytest.mark.parametrize("workload", list(REACH))
def test_reach_at_bench_shapes(workload):
    bench = bench_module()
    w, a, (bits, npat, nmod, words), (T, W, Wg, _) = bench.make_tables(workload, 1)
    t0 = time.perf_counter()
    ref = co.Reference(w.a, w.b, a.asks, a.opts, bits, npat, nmod, words)
    r = ref.result()
    seconds = time.perf_counter() - t0
    max_p, max_u, levels = REACH[workload]
    assert ref.P <= max_p and ref.U <= max_u, (ref.P, ref.U)
    rows = tile_rows(T, W)
    feasible = r["ask_count"] > 0
    n_tiles = -(-T // rows)
    assert n_tiles > 50
    assert all(feasible[s:s + rows].any() for s in range(0, T, rows)), "a cost tile without feasible asks"
    assert all((~feasible[s:s + rows]).any() for s in range(0, T, rows)), "a cost tile without infeasible asks"
    assert (r["ask_best"][feasible] >> 32 > 0).all()                  # every row minimum carries a price
    assert len(np.unique(r["ask_best"][feasible] >> 32)) >= levels
    # The row minima are the cheapest feasible workers, lowest index first: with thousands of workers at the lowest
    # price levels they gather in a few dozen of the 1024-column stripes, reaching past the first quarter of the table.
    # The per-worker first asks are about 15 of the first 34 asks, which between them accept every assignable worker,
    # so at these shapes worker_ask never leaves the first tile; tests/test_gpu_bench_workloads.py disables the first
    # tile's asks to move it out.
    stripes = np.unique((r["ask_best"][feasible] & 0xFFFFFFFF) // 1024)
    assert len(stripes) >= 32 and stripes.max() >= (W // 1024) // 4, stripes
    firsts = np.unique(r["worker_ask"][r["worker_ask"] != NONE])
    assert 8 <= len(firsts) and firsts.max() < rows
    print(f"{workload}: {ref.P} profiles x {ref.U} distinct rows, built and expanded in {seconds:.1f} s; "
          f"row minima in {len(stripes)} stripes, first asks {len(firsts)} distinct")
