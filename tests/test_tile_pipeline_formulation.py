"""pm_build_argmin's two reductions restated in numpy and held against the CPU oracle (no GPU needed).

  * first_ask from the build phase: per column, min over rows t of t | (int32(fail) >> 31), where fail is the
    predicate word whose sign bit is set exactly when the worker does not meet the ask;
  * (ask_best, ask_count) from the read-back: per row and 1024-column CTA stripe, lane l folds the words at columns
    j * 128 + 4 l + c (j = 0..7, c = 0..3) in that order into (least word, first column) with a strict "<"; the warp
    takes the least word, then the least column holding it, and the feasible count; the stripes' packed
    (word << 32) | (w0 + column) are merged with min and their counts with a sum."""
import numpy as np
import pytest

from oracle import pm_oracle as orc
from protocol_b200 import synth

INF_WORD = 0x7FFFFFFF          # the 32-bit tile's infeasible word
INF = np.int64(0x7FFFFFFFFFFFFFFF)
NONE = 0xFFFFFFFF


def tables(T, W, seed, prices):
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed, price=None)
    a = synth.make_asks(T, "mixed", seed=synth.SEED_ASKS + seed)
    bits, _, _, words = synth.intern_tables(w, a)
    w.b["ext_ask_price"] = {"loguniform": synth.make_workers(W, seed=seed, price="loguniform").b["ext_ask_price"],
                            "constant": np.full(W, 4242), "mod3": np.arange(W) % 3,
                            "top": np.full(W, 0x7FFFFFFE)}[prices].astype(np.uint32)
    return w, a, bits, words


def sign_fail_words(feasible, rng):
    """Predicate words as the build forms them: any value, with the sign bit set exactly when infeasible."""
    low = rng.integers(0, 1 << 31, feasible.shape, dtype=np.uint32)
    return np.where(feasible, low, low | np.uint32(1 << 31))


def first_ask(fail, t0):
    T = fail.shape[0]
    t = (t0 + np.arange(T, dtype=np.uint32))[:, None]
    s = (fail.view(np.int32) >> 31).view(np.uint32)   # all-ones when infeasible
    return np.min(t | s, axis=0)


def band_reduce(tile, w0):
    """tile: uint32 [T, ld] with ld a multiple of 1024 -> (ask_best, ask_count) as the CTAs' atomics leave them."""
    T, ld = tile.shape
    x = tile.reshape(T, ld // 1024, 8, 32, 4).transpose(0, 1, 3, 2, 4).reshape(T, ld // 1024, 32, 32)   # [t, cta, lane, j*4+c]
    k = np.argmin(x, axis=3)                           # first of the lane's least words: its strict "<" fold
    bw = np.take_along_axis(x, k[..., None], axis=3)[..., 0]
    bc = (k // 4) * 128 + (k % 4) + 4 * np.arange(32)[None, None, :]
    cnt = (x != INF_WORD).sum(axis=(2, 3)).astype(np.uint32)
    wmin = bw.min(axis=2)
    cmin = np.where(bw == wmin[..., None], bc, NONE).min(axis=2)
    col = w0 + 1024 * np.arange(ld // 1024)[None, :] + cmin
    packed = np.where(cnt > 0, (wmin.astype(np.int64) << 32) | col.astype(np.int64), INF)
    return packed.min(axis=1), cnt.sum(axis=1).astype(np.uint32)


@pytest.mark.parametrize("prices", ["loguniform", "constant", "mod3", "top"])
@pytest.mark.parametrize("T,W,w0", [(37, 1, 0), (64, 1025, 0), (300, 4099, 0), (200, 3000, 1234)])
def test_pipeline_reductions_match_the_oracle(T, W, w0, prices):
    w, a, bits, words = tables(T, w0 + W, seed=T + W, prices=prices)
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, bits, words, 0, T, w0, w0 + W, want_cost=True)
    cost = ev["cost"]
    feasible = cost != INF
    ld = -(-W // 1024) * 1024
    tile = np.full((T, ld), INF_WORD, dtype=np.uint32)             # padding columns hold the infeasible word
    tile[:, :W] = np.where(feasible, cost >> 32, INF_WORD).astype(np.uint32)
    assert (tile[:, :W][feasible] < INF_WORD).all()

    fail = sign_fail_words(feasible, np.random.default_rng(T * W))
    assert np.array_equal(first_ask(fail, 0), ev["col_first"])

    best, cnt = band_reduce(tile, w0)
    assert np.array_equal(cnt, ev["row_count"])
    assert np.array_equal(best, ev["row_best"])


def test_first_ask_over_tiles_is_the_min_of_the_tiles():
    """Each tile's CTAs flush their column minima with atomicMin: merging tiles is a min as well."""
    w, a, bits, words = tables(300, 2000, seed=3, prices="mod3")
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, bits, words, 0, 300, 0, 2000, want_cost=True)
    fail = sign_fail_words(ev["cost"] != INF, np.random.default_rng(3))
    parts = [first_ask(fail[t0:t0 + 64], t0) for t0 in range(0, 300, 64)]
    assert np.array_equal(np.minimum.reduce(parts), ev["col_first"])
