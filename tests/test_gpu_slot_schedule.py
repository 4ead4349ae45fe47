"""pm_build_argmin_feat's slot schedule and its `priced` map on hardware.  A pass of four tiles or more takes its asks
in the scheduled order (the final writers last, the others sorted by their first option's requirement mask) and skips
the stores of blocks that already hold the sentinel or this pass's column prices; the outputs must be the natural
order's, and the buffer (PM_BUF_COST_TILE) what the natural order leaves.

One engine and its PM_TUNE_BUILD=8 twin go through a history (test_gpu_tile_write_skip.History): after every pass the
outputs are held against the twin's and the read-back buffer against the natural order's tiles.  The history covers a
price-only worker upsert (the column order stays, the prices in the priced blocks change: the map must be zeroed at the
pass start), an upsert that reorders the columns, another writer of the buffer, disabled asks, a sharded range and a
shrink below one tile; the tables' asks include multi-option ones."""
import numpy as np
import pytest

from test_gpu_narrow_tile import assert_same, tables
from test_gpu_tile_overlap import tile_bytes
from test_gpu_tile_write_skip import History, expected_tile

pytestmark = pytest.mark.gpu

ROWS = 128


def check_pass(h, narrow=True):
    h.run_pass(narrow)
    T = len(h.t["asks"])
    _, _, ld = h.range()
    rows = min(h.cost_tile_bytes // (ld * 8), T)   # rows are sized at 8 B per element of the padded row
    assert h.e.stats()["n_tiles"] == -(-T // rows), "the launches per pass changed"


def full_blocks(h):
    w0, nw, _ = h.range()
    tile = expected_tile(h.twin, h.t, w0, nw)
    return int((tile != 0x7FFFFFFF).reshape(len(tile), -1, 128).all(axis=2).sum())


def test_the_scheduled_passes_leave_the_natural_tile():
    t = tables(900, 5000, 43)
    W, T = len(t["wa"]), len(t["asks"])
    assert (t["asks"]["n_opts"] > 1).any(), "no multi-option asks"
    h = History(t, tile_bytes(W, ROWS))   # 8 tiles of 128 rows, the last ragged (4)
    h.cost_tile_bytes = tile_bytes(W, ROWS)
    rng = np.random.default_rng(11)
    try:
        check_pass(h)
        check_pass(h)
        assert full_blocks(h) > 0, "no block holds prices: the priced map is not exercised"
        # a price-only upsert: same features, so the same column order; new prices in every priced block
        a, b = 300, 4300
        nb = h.t["wb"][a:b].copy()
        nb["ext_ask_price"] = nb["ext_ask_price"] + 1 + rng.integers(0, 5, b - a).astype(nb["ext_ask_price"].dtype)
        na = h.t["wa"][a:b].copy()
        h.both(lambda x: x.upsert_workers(na, nb, a))
        h.t["wb"][a:b] = nb
        check_pass(h)
        check_pass(h)
        # workers rewritten with other workers' contents: the column order changes
        src = rng.permutation(W)[:1500]
        na, nb = h.t["wa"][src].copy(), h.t["wb"][src].copy()
        h.both(lambda x: x.upsert_workers(na, nb, 700))
        h.t["wa"][700:2200], h.t["wb"][700:2200] = na, nb
        check_pass(h)
        # another writer: the export's int64 rows over the start of the buffer
        h.export()
        check_pass(h)
        # disabled asks: their rows are infeasible everywhere; then enabled again
        off = np.sort(rng.choice(T, 200, replace=False)).astype(np.uint32)
        h.both(lambda x: x.set_ask_enabled(off, False))
        check_pass(h)
        h.both(lambda x: x.set_ask_enabled(off, True))
        check_pass(h)
        # a sharded range: ld 5120 -> 3072 (213 rows per tile, 5 tiles), w0 off a stripe boundary
        h.shard = (1234, 2500)
        h.both(lambda x: x.set_shard(*h.shard))
        check_pass(h)
        check_pass(h)
        h.shard = None
        h.both(lambda x: x.set_shard(0, 0))
        check_pass(h)
        # exactly 7 tiles, then fewer asks than one tile
        h.both(lambda x: x.resize_asks(896))
        h.t["asks"] = h.t["asks"][:896].copy()
        check_pass(h)
        h.both(lambda x: x.resize_asks(100))
        h.t["asks"] = h.t["asks"][:100].copy()
        check_pass(h)
        check_pass(h)
        assert h.n_checked == 14
    finally:
        h.close()
    assert_same(h.t, tile_bytes(W, ROWS))
