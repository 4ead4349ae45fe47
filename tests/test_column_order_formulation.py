"""pm_build_argmin_feat's column order restated in numpy and held against the fold in worker order (no GPU needed).

  * the order (pm_feature_keys + one stable radix sort): the workers of [w0, w0 + nw) sorted by __brevll(F), ties in
    worker order; column c < nw holds worker w0 + perm[c], the padding columns [nw, ld) stay at the end (perm[c] = c);
  * the stripe ranks (pm_stripe_rank with perm): per 1024-column stripe the columns sorted by (price, worker), padding
    last; best_of_rank[s * 1024 + rho] = (price << 32) | (w0 + worker) of the column at place rho;
  * the fold of test_rank_fold_formulation over the permuted columns, and first_ask flushed to first_ask[w0 + perm[c]].
ask_best, ask_count and first_ask must be those of the unpermuted fold, bit for bit.  The layout guard checks what
the order is for: on cfg3-shaped tables nearly every aligned 128-byte block of a row is all infeasible."""
import numpy as np
import pytest

from oracle import pm_oracle as orc
from protocol_b200 import synth
import feature_tables as ft
from test_fast_predicate_formulation import device_bits
from test_rank_fold_formulation import INF, fold, rank_table

NONE = np.uint32(0xFFFFFFFF)


def brev(F, n):
    """__brevll(F) of words whose bits past n are clear: feature i goes to bit 63 - i."""
    out = np.zeros_like(F)
    for i in range(n):
        out |= ((F >> np.uint64(i)) & np.uint64(1)) << np.uint64(63 - i)
    return out


def column_order(F, n, ld):
    """perm [ld]: the stable sort of brev(F) over [0, nw), then the padding columns in place."""
    nw = len(F)
    return np.concatenate([np.argsort(brev(F, n), kind="stable"), np.arange(nw, ld)]).astype(np.int64)


def rank_table_perm(price, perm, nw, ld, w0):
    """price: uint32 [nw] of workers w0 .. -> (rank uint32 [ld], best_of_rank int64 [ld]), columns holding perm"""
    rank = np.empty(ld, dtype=np.uint32)
    best = np.empty(ld, dtype=np.int64)
    for c0 in range(0, ld, 1024):
        cols = np.arange(c0, c0 + 1024)
        pad = cols >= nw
        wk = perm[cols]
        p = np.where(pad, 0, price[np.minimum(wk, max(nw - 1, 0))]).astype(np.int64)
        order = np.lexsort((wk, p, pad))                   # padding last, then price, then worker
        rank[c0 + order] = np.arange(1024, dtype=np.uint32)
        best[c0:c0 + 1024] = np.where(pad[order], INF, (p[order] << 32) | (w0 + wk[order]))
    return rank, best


def column_first(fail, t0):
    """per column, the first ask whose fail word is zero (the kernel's cm = min(t + 2^31 * b)), NONE if none"""
    t = (t0 + np.arange(fail.shape[0], dtype=np.uint32))[:, None]
    cm = np.min(np.where(fail != 0, np.uint32(0x80000000), np.uint32(0)) + t, axis=0)
    return np.where(cm < 0x80000000, cm, NONE)


def features(t, w0, nw):
    conv = ft.converted(t["asks"], t["opts"])
    d = ft.dictionary(conv)
    assert ft.fits(d), f"{len(d)} features"
    tbl, _ = device_bits(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    F = ft.worker_features(t["wa"][w0:w0 + nw], t["wb"][w0:w0 + nw], tbl, d)
    fail = np.stack([ft.feature_fail(F, rs) for rs in ft.requirement_masks(conv, d)])
    return F, len(d), fail


def both_folds(t, w0, nw, t0=0):
    """((ask_best, ask_count, first_ask) in worker order, the same through the column order, perm)"""
    F, n, fail = features(t, w0, nw)
    price = t["wb"]["ext_ask_price"][w0:w0 + nw].astype(np.uint32)
    ld = -(-nw // 1024) * 1024
    T = fail.shape[0]

    def run(perm):
        """perm None: worker order, ranked by (price, column) as pm_stripe_rank without perm"""
        cols = np.arange(ld) if perm is None else perm
        fp = np.full((T, ld), 1, dtype=np.uint32)         # padding columns: never feasible
        fp[:, :nw] = fail[:, cols[:nw]]
        rank, best_of_rank = (rank_table_perm(price, perm, nw, ld, w0) if perm is not None
                              else rank_table(price, nw, ld, w0))
        best, cnt = fold(fp == 0, rank, best_of_rank)
        first = np.full(nw, NONE, dtype=np.uint32)
        first[cols[:nw]] = column_first(fp, t0)[:nw]       # flushed to first_ask[w0 + perm[c]]
        return best, cnt, first

    plain = run(None)
    assert all(np.array_equal(x, y) for x, y in zip(plain, run(np.arange(ld))))   # the identity is worker order
    perm = column_order(F, n, ld)
    return plain, run(perm), perm, fail, price


def direct(fail, price, w0, t0=0):
    """ask_best, ask_count, first_ask straight from the fail words"""
    feas = fail == 0
    packed = (price.astype(np.int64) << 32) | (w0 + np.arange(fail.shape[1], dtype=np.int64))
    best = np.where(feas, packed[None, :], INF).min(axis=1)
    cnt = feas.sum(axis=1).astype(np.uint32)
    anyf = feas.any(axis=0)
    first = np.where(anyf, t0 + feas.argmax(axis=0), NONE).astype(np.uint32)
    return best, cnt, first


def assert_same(a, b):
    for x, y, name in zip(a, b, ("ask_best", "ask_count", "first_ask")):
        assert np.array_equal(x, y), name


@pytest.mark.parametrize("seed,T,W,w0,price_max", [
    (1, 60, 1000, 0, 1 << 30),       # one ragged stripe
    (2, 80, 3000, 0, 3),             # price ties within and across stripes
    (3, 50, 2500, 777, 1),           # every price equal, w0 off a stripe boundary
    (4, 40, 4096, 1024, 5),          # whole stripes, w0 on one
    (5, 70, 1025, 3, 2),             # one column past a stripe
])
def test_column_order_matches_worker_order_on_edge_tables(seed, T, W, w0, price_max):
    t = ft.edge_tables(seed, T, w0 + W, price_max=price_max)
    plain, permuted, perm, fail, price = both_folds(t, w0, W)
    assert not np.array_equal(perm[:W], np.arange(W))      # the order moves columns
    assert_same(permuted, plain)
    assert_same(plain, direct(fail, price, w0))


def test_ties_in_a_stripe_whose_columns_are_out_of_worker_order():
    """Equal least prices on workers whose columns come in the opposite order: (price, worker) picks the least worker,
    not the least column."""
    t = ft.edge_tables(8, 60, 2048, price_max=1 << 20)
    F, n, fail = features(t, 0, 2048)
    perm = column_order(F, n, 2048)
    # two workers of the same stripe whose columns are in the opposite order of their indices, both feasible somewhere
    feas_any = (fail == 0).any(axis=0)
    c = np.nonzero(feas_any[perm[:1024]])[0]
    pairs = [(i, j) for i in c[:64] for j in c[:64] if i < j and perm[i] > perm[j] and
             ((fail[:, perm[i]] == 0) & (fail[:, perm[j]] == 0)).any()]
    assert pairs, "no inverted pair of commonly feasible workers"
    i, j = pairs[0]
    wb = t["wb"].copy()
    wb["ext_ask_price"] = 1000
    wb["ext_ask_price"][[perm[i], perm[j]]] = 5
    t = dict(t, wb=wb)
    plain, permuted, _, fail, price = both_folds(t, 0, 2048)
    assert_same(permuted, plain)
    rows = (fail[:, perm[i]] == 0) & (fail[:, perm[j]] == 0)
    assert (permuted[0][rows] == (5 << 32) | perm[j]).all()


def cfg3_tables(n_workers, n_asks):
    w = synth.make_workers(n_workers, price="loguniform")
    a = synth.make_asks(n_asks, "mixed")
    bits, npat, nmod, words = orc.model_table(w.model_strings, a.pattern_strings)
    return dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words)


@pytest.mark.parametrize("w0,W", [(0, 6000), (1500, 4321)])
def test_column_order_matches_worker_order_on_cfg3_shaped_tables(w0, W):
    t = cfg3_tables(w0 + W, 300)
    plain, permuted, _, fail, price = both_folds(t, w0, W)
    assert_same(permuted, plain)
    assert_same(plain, direct(fail, price, w0))


def test_sorted_columns_leave_rows_in_uniform_infeasible_blocks():
    """The layout the order is for: with cfg3's ask table over 200k of its workers, at least 85 % of a row's aligned
    128-byte blocks (32 columns) are all infeasible, where worker order leaves about a quarter."""
    W, T = 200_000, 100_000
    w = synth.make_workers(W, price="loguniform")
    a = synth.make_asks(T, "mixed")
    bits, npat, nmod, words = orc.model_table(w.model_strings, a.pattern_strings)
    conv = ft.converted(a.asks, a.opts)
    d = ft.dictionary(conv)
    assert ft.fits(d)
    tbl, _ = device_bits(bits, npat, nmod, words)
    F = ft.worker_features(w.a, w.b, tbl, d)
    perm = column_order(F, len(d), W)
    masks = ft.requirement_masks(conv, d)
    rows = np.random.default_rng(0).choice(T, 200, replace=False)
    n = W // 32 * 32

    def uniform_share(order):
        s = 0.0
        for r in rows:
            bad = ft.feature_fail(F[order], masks[r]) != 0
            s += bad[:n].reshape(-1, 32).all(axis=1).mean()
        return s / len(rows)

    sorted_share, worker_share = uniform_share(perm), uniform_share(np.arange(W))
    assert sorted_share >= 0.85, sorted_share
    assert worker_share < 0.5, worker_share
