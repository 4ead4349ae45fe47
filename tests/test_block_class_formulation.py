"""pm_build_argmin_feat's block classes restated in numpy (no GPU needed).

A warp's block of a row is its 128 columns of the sorted column order.  With Fo / Fa the OR / AND of the block's feature
words F (padding columns: F = 0) and kmin its least stripe rank, the kernel decides a row's block before any
per-column work:
  * dead: R_o & ~Fo != 0 for every option o.  Every column fails every option (F_c is a subset of Fo): every word the
    sentinel, slot (kNoRank, 128), no first ask; the store only when the sentinel map's bit is clear;
  * full: R_o & ~Fa == 0 for some option o.  Every column meets it (Fa is a subset of F_c): every word the column's
    price, slot (kmin, 0), every column's first ask min(cm, t); always stored;
  * mixed: the per-column evaluation.
Both tests fold to 32 bits and take the least over the options, as the per-column fail word does.

The classified pass must give the tile, ask_best, ask_count and first_ask of the per-column pass; inside the sentinel
map's buffer model (test_tile_write_skip_formulation.Buffer) it must leave the fully written buffer after every launch.
The reach checks hold the GPU test's tables to what they are for, and the count guard keeps what the classes are for:
on cfg3-shaped tables nearly every block is decided without per-column work."""
import numpy as np
import pytest

from oracle import pm_oracle as orc
from protocol_b200 import synth
import feature_tables as ft
from test_column_order_formulation import column_first, column_order, direct, features, rank_table_perm
from test_fast_predicate_formulation import device_bits
from test_rank_fold_formulation import INF, NO_RANK, fold
from test_tile_write_skip_formulation import BLOCK, STRIPE, S, Buffer

DEAD, FULL, MIXED = 0, 1, 2
NONE = np.uint32(0xFFFFFFFF)
LO = np.uint64(0xFFFFFFFF)


def fold32(x):
    return ((x & LO) | (x >> np.uint64(32))).astype(np.uint32)


def block_words(F, perm, ld):
    """(Fo, Fa) uint64 [ld / 128] of the sorted columns; padding columns have F = 0"""
    Fs = np.zeros(ld, dtype=np.uint64)
    Fs[:len(F)] = F[perm[:len(F)]]
    b = Fs.reshape(-1, BLOCK)
    return np.bitwise_or.reduce(b, axis=1), np.bitwise_and.reduce(b, axis=1)


def classify(rs, Fo, Fa):
    """class [blocks] of one row whose options require rs"""
    dead = full = None
    for R in rs:
        d, f = fold32(np.uint64(R) & ~Fo), fold32(np.uint64(R) & ~Fa)
        dead = d if dead is None else np.minimum(dead, d)
        full = f if full is None else np.minimum(full, f)
    return np.where(dead != 0, DEAD, np.where(full == 0, FULL, MIXED))


class Pass:
    """One pass over workers [w0, w0 + nw) of t in the sorted column order, t0 the first ask."""

    def __init__(self, t, w0, nw, t0=0):
        self.F, n, self.fail = features(t, w0, nw)            # fail [T, nw] in worker order
        self.nw, self.w0, self.t0 = nw, w0, t0
        self.ld = ld = -(-nw // STRIPE) * STRIPE
        self.perm = column_order(self.F, n, ld)
        self.price = t["wb"]["ext_ask_price"][w0:w0 + nw].astype(np.uint32)
        self.rank, self.best_of_rank = rank_table_perm(self.price, self.perm, nw, ld, w0)
        self.Fo, self.Fa = block_words(self.F, self.perm, ld)
        conv = ft.converted(t["asks"], t["opts"])
        self.masks = ft.requirement_masks(conv, ft.dictionary(conv))
        self.cls = np.stack([classify(rs, self.Fo, self.Fa) for rs in self.masks])   # [T, blocks]
        T = len(self.masks)
        self.fp = np.ones((T, ld), dtype=np.uint32)            # per-column fail words, padding never feasible
        self.fp[:, :nw] = self.fail[:, self.perm[:nw]]
        self.pc = np.zeros(ld, dtype=np.uint32)                # per-column price, the null worker's 0 on padding
        self.pc[:nw] = self.price[self.perm[:nw]]

    def per_column(self):
        """(tile, ask_best, ask_count, first_ask by column) of the per-column evaluation"""
        tile = np.where(self.fp != 0, S, self.pc[None, :])
        best, cnt = fold(self.fp == 0, self.rank, self.best_of_rank)
        return tile, best, cnt, column_first(self.fp, self.t0)

    def classified(self):
        """The same four outputs as the kernel forms them: dead and full blocks from their constants only."""
        T, ld = self.fp.shape
        nbk = ld // BLOCK
        blk_fp = self.fp.reshape(T, nbk, BLOCK)
        blk_pc = self.pc.reshape(nbk, BLOCK)
        blk_rank = self.rank.reshape(nbk, BLOCK)
        kmin = blk_rank.min(axis=1)
        tile = np.empty((T, nbk, BLOCK), dtype=np.uint32)
        key = np.empty((T, nbk), dtype=np.uint32)
        nb = np.empty((T, nbk), dtype=np.uint32)
        cm = np.full((nbk, BLOCK), NONE, dtype=np.uint32)
        for r in range(T):
            c = self.cls[r]
            d, f, m = c == DEAD, c == FULL, c == MIXED
            t = np.uint32(self.t0 + r)
            tile[r, d] = S
            key[r, d], nb[r, d] = NO_RANK, BLOCK
            tile[r, f] = blk_pc[f]
            key[r, f], nb[r, f] = kmin[f], 0
            cm[f] = np.minimum(cm[f], t)
            b = (blk_fp[r, m] != 0).astype(np.uint32)
            tile[r, m] = np.where(b != 0, S, blk_pc[m])
            key[r, m] = (b * NO_RANK + blk_rank[m]).min(axis=1)
            nb[r, m] = b.sum(axis=1)
            cm[m] = np.minimum(cm[m], b * np.uint32(0x80000000) + t)
        # the end-of-CTA merge over each stripe's 8 warp slots
        ck, cn = key.reshape(T, -1, 8).min(axis=2), nb.reshape(T, -1, 8).sum(axis=2)
        hit = cn < STRIPE
        stripe = np.arange(ld // STRIPE)[None, :]
        best = np.where(hit, self.best_of_rank[stripe * STRIPE + np.minimum(ck, STRIPE - 1)], INF).min(axis=1)
        cnt = np.where(hit, STRIPE - cn, 0).sum(axis=1).astype(np.uint32)
        cm = cm.reshape(-1)
        return tile.reshape(T, ld), best, cnt, np.where(cm < 0x80000000, cm, NONE)

    def by_worker(self, first_by_column):
        out = np.full(self.nw, NONE, dtype=np.uint32)
        out[self.perm[:self.nw]] = first_by_column[:self.nw]
        return out


def assert_classified_equals_per_column(t, w0, nw, t0=0):
    p = Pass(t, w0, nw, t0)
    want, got = p.per_column(), p.classified()
    for x, y, name in zip(got, want, ("tile", "ask_best", "ask_count", "first_ask")):
        assert np.array_equal(x, y), name
    best, cnt, first = direct(p.fail, p.price, w0, t0)
    assert np.array_equal(got[1], best) and np.array_equal(got[2], cnt)
    assert np.array_equal(p.by_worker(got[3]), first)
    return p


def multi(p):
    return np.array([len(rs) > 1 for rs in p.masks])


def reach(p):
    """(classes present, classes present on multi-option rows, the last real column's block holds padding)"""
    mo = multi(p)
    return set(np.unique(p.cls)), set(np.unique(p.cls[mo])), p.nw % BLOCK != 0


# ----------------------------------------------------------------- tables the GPU test runs (test_gpu_block_class.py)
def cfg3_like(n_asks, n_workers, seed_shift):
    """bench.py's cfg3 generators (log-uniform prices, mixed asks) at another seed"""
    w = synth.make_workers(n_workers, seed=synth.SEED_WORKERS + seed_shift, price="loguniform")
    a = synth.make_asks(n_asks, "mixed", seed=synth.SEED_ASKS + seed_shift)
    bits, npat, nmod, words = orc.model_table(w.model_strings, a.pattern_strings)
    return dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words)


def with_disabled(t, every=7):
    """enable flags for t's asks, every `every`-th one disabled (a disabled ask requires the never bit)"""
    on = np.ones(len(t["asks"]), dtype=bool)
    on[::every] = False
    return on


def gpu_tables():
    """name -> (tables, shard or None); every one reaches all three classes, on multi-option rows too"""
    return {
        "cfg3_like": (cfg3_like(1500, 20077, 61), None),
        "cfg3_like_shard": (cfg3_like(1200, 30011, 62), (9001, 12345)),
        "edge_64": (ft.with_features(ft.edge_tables(63, 900, 6100, max_opts=3), 64), None),
    }


# ----------------------------------------------------------------- soundness and equality
@pytest.mark.parametrize("seed,T,W,w0", [
    (1, 80, 1000, 0),         # one ragged stripe
    (2, 120, 3000, 0),
    (3, 90, 2500, 777),       # w0 off a stripe boundary
    (4, 70, 4096, 1024),      # whole stripes
    (5, 100, 1025, 3),        # one column past a stripe
])
def test_classified_pass_equals_per_column_on_edge_tables(seed, T, W, w0):
    t = ft.edge_tables(seed, T, w0 + W, max_opts=3)
    assert_classified_equals_per_column(t, w0, W)


def test_classified_pass_equals_per_column_at_64_features():
    t = ft.with_features(ft.edge_tables(21, 400, 5000), 64)
    p = assert_classified_equals_per_column(t, 0, 5000)
    assert len(p.Fo) and ft.n_features(t) == 64


@pytest.mark.parametrize("name", ["cfg3_like", "cfg3_like_shard", "edge_64"])
def test_classified_pass_equals_per_column_on_the_gpu_tables(name):
    t, shard = gpu_tables()[name]
    w0, nw = shard if shard is not None else (0, len(t["wa"]))
    p = assert_classified_equals_per_column(t, w0, nw, t0=0)
    got, mo, padded = reach(p)
    assert got == {DEAD, FULL, MIXED} and mo == {DEAD, FULL, MIXED}, (got, mo)
    assert padded, "the last real column's block holds no padding"
    assert (p.cls[:, -1] == DEAD).all() or p.ld - p.nw < BLOCK


def test_shard_tiles_with_a_ragged_last_stripe_and_a_later_first_ask():
    t = cfg3_like(300, 9000, 64)
    assert_classified_equals_per_column(t, 2345, 4321, t0=1000)


def crafted():
    """Two-option asks whose options miss different features of a block: dead only through both of them, and full only
    through the second.  Built on a table whose sorted blocks each hold workers of two kinds."""
    t = ft.edge_tables(31, 60, 3000, max_opts=1)
    t = dict(t, asks=t["asks"].copy(), opts=t["opts"].copy())
    W = len(t["wa"])
    conv = ft.converted(t["asks"], t["opts"])
    d = ft.dictionary(conv)
    tbl, _ = device_bits(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    F = ft.worker_features(t["wa"], t["wb"], tbl, d)
    return t, F, d, W


def test_multi_option_rows_decided_through_every_option():
    """Per block, the class of an ask with options {R1, R2} is what every column's min over its options gives, where
    R1 and R2 each take one feature from outside Fa: dead when both miss Fo, full when R2 alone lies in Fa."""
    t, F, d, W = crafted()
    ld = -(-W // STRIPE) * STRIPE
    perm = column_order(F, len(d), ld)
    Fo, Fa = block_words(F, perm, ld)
    n = len(d)
    allb = np.uint64((1 << n) - 1)
    seen = set()
    for j in range(len(Fo)):
        out_o = [i for i in range(n) if not (int(Fo[j]) >> i) & 1]    # features no column of the block has
        mix = [i for i in range(n) if (int(Fo[j]) >> i) & 1 and not (int(Fa[j]) >> i) & 1]   # some columns have
        inside = int(Fa[j]) & int(allb)
        cases = []
        if len(out_o) >= 2:
            cases.append(("dead", [1 << out_o[0], 1 << out_o[1]], DEAD))
        if out_o and mix:
            cases.append(("mixed", [1 << out_o[0], 1 << mix[0]], None))
        if out_o and inside:
            cases.append(("full", [1 << out_o[0], inside], FULL))
        if len(mix) >= 2:
            cases.append(("two_mixed", [1 << mix[0], 1 << mix[1]], None))
        for name, rs, want in cases:
            c = classify(rs, Fo[j:j + 1], Fa[j:j + 1])[0]
            Fs = np.zeros(BLOCK, dtype=np.uint64)
            cols = np.arange(j * BLOCK, (j + 1) * BLOCK)
            real = cols < W
            Fs[real] = F[perm[cols[real]]]
            fail = ft.feature_fail(Fs, rs)
            if c == DEAD:
                assert (fail != 0).all(), name
            elif c == FULL:
                assert (fail == 0).all(), name
            if want is not None:
                assert c == want, (name, j)
            seen.add((name, int(c)))
    assert ("dead", DEAD) in seen and ("full", FULL) in seen
    assert ("mixed", MIXED) in seen          # the first option alone would have made the block dead


def test_disabled_asks_are_dead_everywhere():
    t = cfg3_like(400, 5000, 65)
    on = with_disabled(t)
    conv = ft.converted(t["asks"], t["opts"], on)
    d = ft.dictionary(conv)
    tbl, _ = device_bits(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    F = ft.worker_features(t["wa"], t["wb"], tbl, d)
    ld = -(-len(F) // STRIPE) * STRIPE
    Fo, Fa = block_words(F, column_order(F, len(d), ld), ld)
    masks = ft.requirement_masks(conv, d)
    for i in np.flatnonzero(~on):
        assert (classify(masks[i], Fo, Fa) == DEAD).all()


def test_padding_blocks_are_dead_and_padded_blocks_never_full():
    t = ft.edge_tables(9, 300, 1100)   # 1100 workers: 1024 + 76 real columns in the second stripe
    p = Pass(t, 0, 1100)
    last = (p.nw - 1) // BLOCK
    assert (p.cls[:, last + 1:] == DEAD).all()
    assert (p.cls[:, last] != FULL).all()
    assert p.Fa[last] == 0


# ----------------------------------------------------------------- the sentinel map with classified blocks
class ClassBuffer(Buffer):
    """Buffer with the kernel's store rule on classified blocks: a dead block is stored when its map bit is clear, a
    full one always, a mixed one unless all its words are the sentinel and the bit is set."""

    def __init__(self, words):
        super().__init__(words)
        self.classes = []   # per launch: (slots, block index within the slot, class)

    def launch_classified(self, p, r0, n):
        ld = p.ld
        if not self.valid:
            self.held[:] = 0
            self.valid = True
        tile = p.classified()[0][r0:r0 + n]
        cls = p.cls[r0:r0 + n]
        self.full[:n * ld] = np.where(p.fp[r0:r0 + n] != 0, S, p.pc[None, :]).reshape(-1)   # every store
        blocks = tile.reshape(n, ld // BLOCK, BLOCK)
        sentinel = (cls == DEAD) | ((cls == MIXED) & (blocks == S).all(axis=2))
        off = np.arange(n)[:, None] * ld + np.arange(ld // BLOCK)[None, :] * BLOCK
        byte, bit = off // STRIPE, (off // BLOCK) % 8
        held = (self.held[byte] >> bit) & 1
        store = ~(sentinel & (held == 1))
        view = self.mem[:n * ld].reshape(n, ld // BLOCK, BLOCK)
        view[store] = blocks[store]
        self.stores += int(store.sum())
        self.skipped += int((~store).sum())
        m = (sentinel.reshape(n, ld // STRIPE, 8) << np.arange(8, dtype=np.uint8)).sum(axis=2).astype(np.uint8)
        self.held[byte[:, ::8]] = m
        self.classes.append((ld, cls.copy()))

    def run_pass(self, p, rows_per_tile):
        T = p.fp.shape[0]
        for r0 in range(0, T, rows_per_tile):
            self.launch_classified(p, r0, min(rows_per_tile, T - r0))
            assert np.array_equal(self.mem, self.full)


def dead_full_dead(classes):
    """some slot's block went dead -> full -> dead over three consecutive launches of one ld"""
    for (l0, a), (l1, b), (l2, c) in zip(classes, classes[1:], classes[2:]):
        if l0 == l1 == l2:
            n = min(len(a), len(b), len(c))
            if ((a[:n] == DEAD) & (b[:n] == FULL) & (c[:n] == DEAD)).any():
                return True
    return False


def test_classified_stores_leave_the_fully_written_buffer():
    t = cfg3_like(700, 6000, 66)
    t = dict(t, wa=t["wa"].copy(), wb=t["wb"].copy())
    rng = np.random.default_rng(5)
    W = len(t["wa"])
    buf = ClassBuffer(256 * 6144 * 2)
    p = Pass(t, 0, W)
    buf.run_pass(p, 256)                         # 256, 256, 188: the first pass finds the map zeroed
    buf.run_pass(p, 256)
    buf.run_pass(p, 100)                         # the rows per tile change: each slot sees other asks
    buf.other_writer(rng, 100 * 6144 * 2)
    buf.run_pass(p, 100)
    src = rng.permutation(W)[:1500]              # worker upsert: another column order
    t["wa"][1000:2500], t["wb"][1000:2500] = t["wa"][src], t["wb"][src]
    p = Pass(t, 0, W)
    buf.run_pass(p, 256)
    buf.run_pass(Pass(t, 1234, 2500), 400)      # a shard: ld 6144 -> 3072
    buf.run_pass(p, 256)
    assert buf.skipped > buf.stores / 4, (buf.skipped, buf.stores)
    assert dead_full_dead(buf.classes)


# ----------------------------------------------------------------- the count guard
def cfg3_class_shares(W, T):
    """(dead, full, mixed) shares of the warp blocks of one pass over cfg3-shaped tables"""
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
    counts = np.zeros(3)
    seen = {}
    for rs in ft.requirement_masks(conv, d):
        k = tuple(rs)
        if k not in seen:
            seen[k] = np.bincount(classify(rs, Fo, Fa), minlength=3)
        counts += seen[k]
    return counts / counts.sum()


def test_nearly_every_block_is_decided_on_cfg3_shaped_tables():
    """200k workers x 20k asks: 88.2 % of the blocks dead and 1.5 % mixed when this was written."""
    dead, full, mixed = cfg3_class_shares(200_000, 20_000)
    assert dead >= 0.85, dead
    assert mixed <= 0.03, mixed
    assert full > 0.05, full
