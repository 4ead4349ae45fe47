"""pm_build_argmin's register fold restated in numpy and held against the CPU oracle (no GPU needed).

  * the stripe rank table (pm_stripe_rank): per 1024-column stripe, the columns sorted by (price, column), padding
    columns (at or past nw) last; rank[c] is a column's place, best_of_rank[s * 1024 + rho] the packed
    (price << 32) | (w0 + column) of the column at place rho;
  * the fold: per row and column key = b * 0x8000 + rank[c] with b = 1 when infeasible; lane l of warp j holds the
    columns j * 128 + 4 l .. + 3, takes the least of its 4 keys and the sum of its 4 bits; the warp reduces both
    (min, add); the CTA takes the least key and the sum over its 8 warps.  A row with fewer than 1024 infeasible
    columns merges best_of_rank[least key] into ask_best (min) and 1024 - infeasible into ask_count (sum);
  * first_ask: per column, min over rows t of t | (fail & 2^31), flushed when below 2^31."""
import numpy as np
import pytest

from oracle import pm_oracle as orc
from test_tile_pipeline_formulation import INF, sign_fail_words, tables

NO_RANK = 0x8000


def rank_table(price, nw, ld, w0):
    """price: uint32 [nw] -> (rank uint32 [ld], best_of_rank int64 [ld])"""
    rank = np.empty(ld, dtype=np.uint32)
    best = np.empty(ld, dtype=np.int64)
    for c0 in range(0, ld, 1024):
        cols = np.arange(c0, c0 + 1024)
        pad = cols >= nw
        p = np.where(pad, 0, price[np.minimum(cols, max(nw - 1, 0))]).astype(np.int64)
        order = np.lexsort((cols, p, pad))                 # padding last, then price, then column
        rank[c0 + order] = np.arange(1024, dtype=np.uint32)
        best[c0:c0 + 1024] = np.where(pad[order], INF, (p[order] << 32) | (w0 + cols[order]))
    return rank, best


def fold(feasible, rank, best_of_rank):
    """feasible: bool [T, ld] -> (ask_best, ask_count) as the CTAs leave them"""
    T, ld = feasible.shape
    b = (~feasible).astype(np.uint32)
    key = b * NO_RANK + rank[None, :]
    key = key.reshape(T, ld // 1024, 8, 32, 4)                  # [t, stripe, warp, lane, k]
    bits = b.reshape(T, ld // 1024, 8, 32, 4)
    lane_key, lane_nb = key.min(axis=4), bits.sum(axis=4)
    warp_key, warp_nb = lane_key.min(axis=3), lane_nb.sum(axis=3)
    cta_key, cta_nb = warp_key.min(axis=2), warp_nb.sum(axis=2)  # [t, stripe]
    hit = cta_nb < 1024
    assert (cta_key[hit] < 1024).all() and (cta_key[~hit] >= NO_RANK).all()
    stripe = np.arange(ld // 1024)[None, :]
    packed = np.where(hit, best_of_rank[stripe * 1024 + np.minimum(cta_key, 1023)], INF)
    count = np.where(hit, 1024 - cta_nb, 0)
    return packed.min(axis=1), count.sum(axis=1).astype(np.uint32)


def first_ask(fail, t0):
    t = (t0 + np.arange(fail.shape[0], dtype=np.uint32))[:, None]
    cm = np.min(t | (fail & np.uint32(0x80000000)), axis=0)
    return np.where(cm < 0x80000000, cm, np.uint32(0xFFFFFFFF))


@pytest.mark.parametrize("prices", ["loguniform", "constant", "mod3", "top"])
@pytest.mark.parametrize("T,W,w0", [(37, 1, 0), (64, 1025, 0), (300, 4099, 0), (200, 3000, 1234)])
def test_rank_fold_matches_the_oracle(T, W, w0, prices):
    w, a, bits, words = tables(T, w0 + W, seed=T + W, prices=prices)
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, bits, words, 0, T, w0, w0 + W, want_cost=True)
    feasible_w = ev["cost"] != INF
    ld = -(-W // 1024) * 1024
    feasible = np.zeros((T, ld), dtype=bool)                    # padding columns are never feasible
    feasible[:, :W] = feasible_w

    rank, best_of_rank = rank_table(w.b["ext_ask_price"][w0:w0 + W], W, ld, w0)
    for c0 in range(0, ld, 1024):
        assert np.array_equal(np.sort(rank[c0:c0 + 1024]), np.arange(1024))
    best, cnt = fold(feasible, rank, best_of_rank)
    assert np.array_equal(cnt, ev["row_count"])
    assert np.array_equal(best, ev["row_best"])

    fail = sign_fail_words(feasible_w, np.random.default_rng(T * W))
    assert np.array_equal(first_ask(fail, 0), ev["col_first"])


def test_ties_in_the_last_lane_of_a_stripe():
    """The least price sits only in the last lane of warp 7: rank order is (price, column), so the least column wins."""
    W, T = 3000, 50
    w, a, bits, words = tables(T, W, seed=11, prices="constant")
    price = np.full(W, 900, dtype=np.uint32)
    col = np.arange(W) % 1024
    price[(col >= 1021)] = 7
    w.b["ext_ask_price"] = price
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, bits, words, 0, T, 0, W, want_cost=True)
    ld = 3072
    feasible = np.zeros((T, ld), dtype=bool)
    feasible[:, :W] = ev["cost"] != INF
    rank, best_of_rank = rank_table(price, W, ld, 0)
    assert rank[1021] == 0 and rank[1023] == 2 and rank[2045] == 0
    best, cnt = fold(feasible, rank, best_of_rank)
    assert np.array_equal(cnt, ev["row_count"]) and np.array_equal(best, ev["row_best"])
