"""The incremental pass (PM_INCREMENTAL, pm_kernels.cuh pm_first_ask_rows), restated on the CPU.

1. The per-worker first feasible ask depends on the worker's own row, the ask table and the model table only: over a
   random history of row writes, recomputing just the written rows gives what recomputing every row gives.
2. The kernel's schedule: the asks are cut into chunks of whole 128-row steps, one CTA per (block of 1024 listed
   workers, chunk).  Before each step a CTA publishes its hits (atomicMin into the result, which starts at NONE for
   every listed worker) and stops when each of its workers has a hit of its own, a published hit below the step's first
   row, or is not a candidate.  Whatever order the CTAs run in, the result is the lowest feasible ask."""
import numpy as np
import pytest

from oracle import pm_oracle as orc
from protocol_b200 import abi, synth

NONE = 0xFFFFFFFF
STEP = 128          # kEvalRows: rows staged per step
CTA_COLS = 1024     # kEvalCols: listed workers per CTA
CAND = abi.PM_W_HEALTHY | abi.PM_W_P2P


def tables(n_workers, n_asks, seed):
    w = synth.make_workers(n_workers, seed=synth.SEED_WORKERS + seed)
    a = synth.make_asks(n_asks, "mixed", seed=synth.SEED_ASKS + seed)
    bits, _, _, words = orc.model_table(w.model_strings, a.pattern_strings)
    return w, a, bits, words


def test_recomputing_written_rows_equals_full_recomputation():
    rng = np.random.default_rng(0)
    w, a, bits, words = tables(3000, 150, 1)
    pool = synth.make_workers(2000, seed=synth.SEED_WORKERS + 9)
    wa, wb = w.a.copy(), w.b.copy()
    stored = orc.soa_first_feasible(wa, wb, a.asks, a.opts, bits, words)
    for step in range(30):
        dirty = np.unique(rng.integers(0, len(wa), int(rng.integers(0, 80))))
        src = rng.integers(0, len(pool), len(dirty))
        wa[dirty], wb[dirty] = pool.a[src], pool.b[src]
        flip = dirty[rng.random(len(dirty)) < 0.3]
        wa["flags"][flip] ^= abi.PM_W_ASSIGNED
        if len(dirty):
            stored[dirty] = orc.soa_first_feasible(wa[dirty], wb[dirty], a.asks, a.opts, bits, words)
        full = orc.soa_first_feasible(wa, wb, a.asks, a.opts, bits, words)
        assert np.array_equal(stored, full), f"step {step}"


def chunked_schedule(feasible, cand, chunk, order):
    """pm_first_ask_rows over listed workers whose feasibility rows are `feasible` [T, n], run CTA by CTA in `order`
    (CTAs run concurrently on the device: any order of whole steps must give the same answer; here the CTAs take turns
    one step at a time in the given order).  Returns (first ask per listed worker, pairs evaluated)."""
    T, n = feasible.shape
    gx, gy = -(-n // CTA_COLS), -(-T // chunk)
    result = np.full(n, NONE, dtype=np.int64)
    pairs = 0
    state = {}
    for bx in range(gx):
        for by in range(gy):
            cols = np.arange(bx * CTA_COLS, min(n, (bx + 1) * CTA_COLS))
            state[bx, by] = dict(cols=cols, first=np.full(len(cols), NONE, dtype=np.int64), open=cand[cols].copy(),
                                 r0=by * chunk, end=min(T, (by + 1) * chunk), live=True)
    while any(s["live"] for s in state.values()):
        for key in order(list(state)):
            s = state[key]
            if not s["live"]:
                continue
            if s["r0"] >= s["end"]:
                s["live"] = False
            else:
                hit = s["open"] & (s["first"] != NONE)
                np.minimum.at(result, s["cols"][hit], s["first"][hit])   # publish
                s["open"] &= ~hit
                waiting = s["open"] & ~(result[s["cols"]] < s["r0"])
                if not waiting.any():
                    s["live"] = False
                else:
                    r1 = min(s["end"], s["r0"] + STEP)
                    f = feasible[s["r0"]:r1][:, s["cols"]]
                    rows = np.where(f, np.arange(s["r0"], r1)[:, None], NONE).min(0, initial=NONE)
                    s["first"] = np.minimum(s["first"], rows)
                    pairs += (r1 - s["r0"]) * len(s["cols"])
                    s["r0"] = r1
            if not s["live"]:
                hit = s["open"] & (s["first"] != NONE)
                np.minimum.at(result, s["cols"][hit], s["first"][hit])
                s["open"] &= ~hit
    return result.astype(np.uint32), pairs


def first_row(feasible):
    T = feasible.shape[0]
    return np.where(feasible.any(0), feasible.argmax(0), NONE).astype(np.uint32) if T else np.full(feasible.shape[1], NONE, np.uint32)


@pytest.mark.parametrize("chunk", [STEP, 3 * STEP, 12 * STEP])
@pytest.mark.parametrize("order_name", ["forward", "backward", "shuffled"])
def test_chunked_early_exit_schedule_gives_the_first_ask(chunk, order_name):
    rng = np.random.default_rng(chunk)
    T, n = 1200, 2100
    # hits spread over the whole table: row 0, the last row, rows just before / after chunk starts, and none at all
    feasible = np.zeros((T, n), dtype=bool)
    hit_at = rng.integers(0, T, n)
    hit_at[:50] = 0
    hit_at[50:100] = T - 1
    hit_at[100:150] = min(chunk, T) - 1
    hit_at[150:200] = min(chunk, T - 1)
    feasible[hit_at, np.arange(n)] = True
    feasible |= rng.random((T, n)) < 0.002          # later hits that must not win
    feasible[:, 200:300] = False                    # candidates without any feasible ask
    cand = np.ones(n, dtype=bool)
    cand[300:400] = False                           # not candidates: NONE without touching an ask
    feasible[:, 300:400] &= False                   # (the predicate requires the candidate bit)
    shuffle = np.random.default_rng(1)
    order = {"forward": lambda ks: ks, "backward": lambda ks: ks[::-1],
             "shuffled": lambda ks: [ks[i] for i in shuffle.permutation(len(ks))]}[order_name]
    got, pairs = chunked_schedule(feasible, cand, chunk, order)
    want = first_row(feasible)
    assert np.array_equal(got, want)
    assert (got[200:400] == NONE).all() and (got[:50] == 0).all()
    assert pairs <= T * n


def test_schedule_on_real_tables_and_the_early_exit():
    """The schedule on the oracle's feasibility of synthetic tables: same first asks, and with most workers meeting an
    early ask the walk stops long before T x n pairs."""
    w, a, bits, words = tables(2048, 800, 4)
    ev = np.stack([orc.soa_first_feasible(w.a, w.b, a.asks[t:t + 1], a.opts, bits, words) == 0 for t in range(len(a))])
    cand = (w.a["flags"] & (CAND | abi.PM_W_ASSIGNED)) == CAND
    want = orc.soa_first_feasible(w.a, w.b, a.asks, a.opts, bits, words)
    got, pairs = chunked_schedule(ev, cand, 4 * STEP, lambda ks: ks)
    assert np.array_equal(got, want) and pairs <= ev.size
    hit = want != NONE   # a CTA whose every worker meets some ask stops early
    got, pairs = chunked_schedule(ev[:, hit], cand[hit], 4 * STEP, lambda ks: ks)
    assert np.array_equal(got, want[hit]) and pairs < ev[:, hit].size // 2
