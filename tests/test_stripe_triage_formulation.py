"""pm_build_argmin_feat's row triage restated in numpy (no GPU needed).

A CTA owns one 1024-column stripe of its rows: 8 warp blocks, with Fo_j the OR of block j's feature words.  Before any
warp walks a row, the CTA triages it against So, the OR of the 8 Fo_j:
  * stripe-dead: R_o & ~So != 0 for every option o (folded to 32 bits, the least over the options, as the block test).
    Each Fo_j is a subset of So, so every block of the row is dead.  Such a row is
      - SKIP when its map byte is 0xFF: every block already holds the sentinel.  Nothing is stored, no slot written,
        nothing folded, and the byte is left alone;
      - SENTINEL otherwise: each warp whose bit is clear stores the sentinel block, and the byte becomes 0xFF;
  * LIVE: every other row, which runs the block classes (test_block_class_formulation.py).
Stripe-dead is sufficient, not necessary: a row whose blocks are each dead through different features stays LIVE.

The triaged launch must leave the buffer, the map, ask_best, ask_count and first_ask that the classified launch leaves,
through a history of launches.  The count guard keeps what the triage is for: on cfg3-shaped tables, in the second of
two passes, most rows of a CTA have nothing to do."""
import numpy as np

from oracle import pm_oracle as orc
from protocol_b200 import synth
import feature_tables as ft
from test_block_class_formulation import (DEAD, MIXED, ClassBuffer, Pass, block_words, cfg3_like, classify, crafted,
                                          fold32, multi, with_disabled)
from test_column_order_formulation import column_first, column_order
from test_fast_predicate_formulation import device_bits
from test_rank_fold_formulation import fold
from test_tile_write_skip_formulation import BLOCK, STRIPE, S

SKIP, SENTINEL, LIVE = 0, 1, 2


def stripe_words(Fo):
    """So [stripes]: the OR of each stripe's 8 block words"""
    return np.bitwise_or.reduce(Fo.reshape(-1, STRIPE // BLOCK), axis=1)


def stripe_dead(rs, So):
    """bool [stripes] of one row whose options require rs"""
    dead = None
    for R in rs:
        d = fold32(np.uint64(R) & ~So)
        dead = d if dead is None else np.minimum(dead, d)
    return dead != 0


def kinds(dead, byte):
    return np.where(~dead, LIVE, np.where(byte == 0xFF, SKIP, SENTINEL))


class TPass(Pass):
    def __init__(self, t, w0, nw, t0=0):
        super().__init__(t, w0, nw, t0)
        self.So = stripe_words(self.Fo)
        self.sd = np.stack([stripe_dead(rs, self.So) for rs in self.masks])   # [T, stripes]
        self._classified = None

    def classified(self):
        if self._classified is None:
            self._classified = super().classified()
        return self._classified

    def triaged(self):
        """(ask_best, ask_count, first_ask by column) merged and flushed from the LIVE rows' stripes only"""
        live = np.repeat(~self.sd, STRIPE, axis=1)                           # [T, ld]
        best, cnt = fold((self.fp == 0) & live, self.rank, self.best_of_rank)
        return best, cnt, column_first(np.where(live, self.fp, 1), self.t0)


def assert_triage_sound(p):
    """every block of a stripe-dead row is dead, and the LIVE rows alone give the outputs"""
    blocks_dead = (p.cls.reshape(len(p.cls), -1, STRIPE // BLOCK) == DEAD).all(axis=2)
    assert blocks_dead[p.sd].all()
    for x, y, name in zip(p.triaged(), p.classified()[1:], ("ask_best", "ask_count", "first_ask")):
        assert np.array_equal(x, y), name


# ----------------------------------------------------------------- soundness
def test_stripe_dead_rows_have_only_dead_blocks_on_edge_tables():
    seen_multi = seen_live_all_dead = 0
    for seed, T, W, w0 in [(1, 80, 1000, 0), (2, 120, 3000, 0), (3, 90, 2500, 777), (4, 70, 4096, 1024),
                           (5, 100, 1025, 3)]:
        t = ft.edge_tables(seed, T, w0 + W, max_opts=3)
        p = TPass(t, w0, W)
        assert_triage_sound(p)
        seen_multi += int(p.sd[multi(p)].sum())
        blocks_dead = (p.cls.reshape(T, -1, STRIPE // BLOCK) == DEAD).all(axis=2)
        seen_live_all_dead += int((blocks_dead & ~p.sd).sum())
    assert seen_multi > 0, "no multi-option row is stripe-dead"
    assert seen_live_all_dead > 0, "no LIVE stripe-row whose blocks are all dead"


def test_the_gpu_tables_are_triaged_soundly():
    for t, shard in [(cfg3_like(1500, 20077, 61), None), (cfg3_like(1200, 30011, 62), (9001, 12345)),
                     (ft.with_features(ft.edge_tables(63, 900, 6100, max_opts=3), 64), None)]:
        w0, nw = shard if shard is not None else (0, len(t["wa"]))
        p = TPass(t, w0, nw)
        assert_triage_sound(p)
        assert p.sd.any() and (~p.sd).any()
        assert p.ld > p.nw and not p.sd[:, -1].all()      # a padded last stripe, LIVE in some rows


def test_multi_option_rows_are_stripe_dead_only_through_every_option():
    """Per stripe, rows of two options built from So: dead when both need a feature outside So, LIVE when only the
    first does; and a one-option row needing two features that no single block has, dead in every block but LIVE."""
    t, F, d, W = crafted()
    n = len(d)
    ld = -(-W // STRIPE) * STRIPE
    perm = column_order(F, n, ld)
    Fo, Fa = block_words(F, perm, ld)
    So = stripe_words(Fo)
    seen = set()
    for s in range(len(So)):
        fo = Fo[s * 8:(s + 1) * 8]
        out = [i for i in range(n) if not (int(So[s]) >> i) & 1]
        inn = [i for i in range(n) if (int(So[s]) >> i) & 1]
        cases = []
        if out and inn:
            cases.append(("both_miss", [1 << out[0], (1 << out[-1]) | (1 << inn[0])], True))
            cases.append(("first_misses", [1 << out[0], 1 << inn[0]], False))
        split = [(a, b) for a in inn for b in inn if a < b
                 and not any((int(f) >> a) & 1 and (int(f) >> b) & 1 for f in fo)]
        if split:
            a, b = split[0]
            cases.append(("split", [(1 << a) | (1 << b)], False))
        for name, rs, want in cases:
            got = bool(stripe_dead(rs, So[s:s + 1])[0])
            assert got == want, (name, s)
            cls = classify(rs, fo, Fa[s * 8:(s + 1) * 8])
            if got or name == "split":
                assert (cls == DEAD).all(), (name, s)
            seen.add(name)
    assert seen == {"both_miss", "first_misses", "split"}, seen


def test_disabled_asks_are_stripe_dead_everywhere():
    t = cfg3_like(400, 5000, 65)
    on = with_disabled(t)
    conv = ft.converted(t["asks"], t["opts"], on)
    d = ft.dictionary(conv)
    tbl, _ = device_bits(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    F = ft.worker_features(t["wa"], t["wb"], tbl, d)
    ld = -(-len(F) // STRIPE) * STRIPE
    So = stripe_words(block_words(F, column_order(F, len(d), ld), ld)[0])
    masks = ft.requirement_masks(conv, d)
    for i in np.flatnonzero(~on):
        assert stripe_dead(masks[i], So).all()


# ----------------------------------------------------------------- the sentinel map with triaged rows
class TriageBuffer(ClassBuffer):
    """ClassBuffer with the triage: SKIP rows untouched, SENTINEL rows store the sentinel where the map's bit is clear
    and set every bit, LIVE rows take the classified store rule.  Only the map bytes that change are written."""

    def __init__(self, words):
        super().__init__(words)
        self.kinds = np.zeros(3, dtype=np.int64)
        self.byte_writes = 0

    def launch_triaged(self, p, r0, n):
        ld = p.ld
        if not self.valid:
            self.held[:] = 0
            self.valid = True
        nst, nbk = ld // STRIPE, ld // BLOCK
        tile = p.classified()[0][r0:r0 + n]
        cls = p.cls[r0:r0 + n]
        self.full[:n * ld] = np.where(p.fp[r0:r0 + n] != 0, S, p.pc[None, :]).reshape(-1)   # every store
        byte = np.arange(n)[:, None] * nst + np.arange(nst)[None, :]                  # [slot, stripe]
        old = self.held[byte]
        kind = kinds(p.sd[r0:r0 + n], old)
        self.kinds += np.bincount(kind.reshape(-1), minlength=3)
        bit = ((old[:, :, None] >> np.arange(8, dtype=np.uint8)) & 1).reshape(n, nbk)
        k8 = np.repeat(kind, 8, axis=1)
        blocks = tile.reshape(n, nbk, BLOCK)
        sentinel = (cls == DEAD) | ((cls == MIXED) & (blocks == S).all(axis=2))
        store_live = (k8 == LIVE) & ~(sentinel & (bit == 1))
        store_sent = (k8 == SENTINEL) & (bit == 0)
        view = self.mem[:n * ld].reshape(n, nbk, BLOCK)
        view[store_live] = blocks[store_live]
        view[store_sent] = S
        stores = int(store_live.sum() + store_sent.sum())
        self.stores += stores
        self.skipped += n * nbk - stores
        m = (sentinel.reshape(n, nst, 8) << np.arange(8, dtype=np.uint8)).sum(axis=2).astype(np.uint8)
        new = np.where(kind == LIVE, m, np.uint8(0xFF)).astype(np.uint8)
        write = new != old
        self.held[byte[write]] = new[write]
        self.byte_writes += int(write.sum())
        assert not write[kind == SKIP].any()


def test_triaged_launches_leave_what_classified_launches_leave():
    """One history through both buffers: the triaged one must match the classified one, buffer and map, after every
    launch, store for store, and the pass's outputs must equal the classified pass's."""
    t = cfg3_like(700, 6000, 66)
    t = dict(t, wa=t["wa"].copy(), wb=t["wb"].copy())
    rng = np.random.default_rng(5)
    W = len(t["wa"])
    words = 256 * 6144 * 2
    cb, tb = ClassBuffer(words), TriageBuffer(words)

    def run(p, rows):
        assert_triage_sound(p)
        T = p.fp.shape[0]
        for r0 in range(0, T, rows):
            n = min(rows, T - r0)
            cb.launch_classified(p, r0, n)
            tb.launch_triaged(p, r0, n)
            assert np.array_equal(tb.mem, tb.full)
            assert np.array_equal(tb.mem, cb.mem) and np.array_equal(tb.held, cb.held)
            assert tb.stores == cb.stores

    def other_writer(words):   # the same junk into both
        seed = int(rng.integers(1 << 30))
        cb.other_writer(np.random.default_rng(seed), words)
        tb.other_writer(np.random.default_rng(seed), words)

    p = TPass(t, 0, W)
    run(p, 256)                                  # 256, 256, 188: the first pass finds the map zeroed
    run(p, 256)
    run(p, 100)                                  # the rows per tile change: each slot sees other asks
    other_writer(100 * 6144 * 2)
    run(p, 100)
    src = rng.permutation(W)[:1500]              # worker upsert: another column order
    t["wa"][1000:2500], t["wb"][1000:2500] = t["wa"][src], t["wb"][src]
    p = TPass(t, 0, W)
    run(p, 256)
    run(TPass(t, 1234, 2500), 400)               # a shard: ld 6144 -> 3072, w0 off a stripe boundary, a ragged tile
    run(p, 256)
    assert (tb.kinds > 0).all(), tb.kinds          # every kind reached
    assert tb.byte_writes < tb.kinds.sum() - tb.kinds[SKIP]


def test_the_gpu_history_reaches_every_row_kind():
    """test_gpu_stripe_triage's tables through its first passes and the reversal of the asks: SKIP, SENTINEL with a
    partly set byte, and LIVE rows all occur in each launch of 512 rows."""
    t = cfg3_like(1300, 20077, 67)
    W, T = len(t["wa"]), len(t["asks"])
    p = TPass(t, 0, W)
    sd = p.sd
    dead_blocks = (p.cls == DEAD).reshape(T, -1, 8)
    m = (dead_blocks << np.arange(8, dtype=np.uint8)).sum(axis=2).astype(np.uint8)
    rev = sd[::-1]
    held = np.zeros((512, sd.shape[1]), dtype=np.uint8)
    for second, (s, mm) in enumerate([(sd, m), (rev, m[::-1])]):
        for r0 in range(0, T, 512):
            n = min(512, T - r0)
            old = held[:n].copy()
            kind = np.where(~s[r0:r0 + n], LIVE, np.where(old == 0xFF, SKIP, SENTINEL))
            if second:
                partly = (kind == SENTINEL) & (old != 0)
                assert (kind == SKIP).any() and (kind == LIVE).any() and partly.any(), r0
            held[:n] = np.where(kind == LIVE, mm[r0:r0 + n], 0xFF)


# ----------------------------------------------------------------- the count guard
def test_most_stripe_rows_are_skipped_on_cfg3_shaped_tables():
    """200k workers x 20k asks at 5120 rows per tile slot, the second of two passes: 75.2 % of the stripe-rows SKIP
    when this was written."""
    W, T, rows = 200_000, 20_000, 5120
    w = synth.make_workers(W, price="loguniform")
    a = synth.make_asks(T, "mixed")
    bits, npat, nmod, words = orc.model_table(w.model_strings, a.pattern_strings)
    conv = ft.converted(a.asks, a.opts)
    d = ft.dictionary(conv)
    assert ft.fits(d)
    tbl, _ = device_bits(bits, npat, nmod, words)
    F = ft.worker_features(w.a, w.b, tbl, d)
    ld = -(-W // STRIPE) * STRIPE
    Fo, Fa = block_words(F, column_order(F, len(d), ld), ld)
    So = stripe_words(Fo)
    keys = {}
    rk = np.array([keys.setdefault(tuple(rs), len(keys)) for rs in ft.requirement_masks(conv, d)])
    sd = np.stack([stripe_dead(list(k), So) for k in keys])[rk]                     # [T, stripes]
    dead_blocks = np.stack([classify(list(k), Fo, Fa) == DEAD for k in keys])[rk]   # [T, blocks]; mixed ignored
    m = (dead_blocks.reshape(T, -1, 8) << np.arange(8, dtype=np.uint8)).sum(axis=2).astype(np.uint8)
    held = np.zeros((rows, ld // STRIPE), dtype=np.uint8)
    counts = np.zeros(3)
    for second in (False, True):
        for r0 in range(0, T, rows):
            n = min(rows, T - r0)
            kind = kinds(sd[r0:r0 + n], held[:n])
            if second:
                counts += np.bincount(kind.reshape(-1), minlength=3)
            held[:n] = np.where(kind == LIVE, m[r0:r0 + n], 0xFF)
    skip, sent, live = counts / counts.sum()
    assert skip >= 0.70, (skip, sent, live)
    assert live <= 0.20, (skip, sent, live)
