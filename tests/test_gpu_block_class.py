"""pm_build_argmin_feat's block classes on hardware: a warp decides its block of a row as dead (every word the sentinel)
or full (every word the column's price) from the OR and AND of its columns' feature words, and evaluates per column
only a mixed block (test_block_class_formulation.py).  Every table here has blocks of all three classes, on
multi-option rows too, and a last real block that holds padding (checked on the CPU by that file).

One engine and its PM_TUNE_BUILD=8 twin (the int64 tile, per-column evaluation in worker order) go through passes and
table calls (test_gpu_tile_write_skip.History).  After every materialised pass every output equals the twin's and the
CPU oracle's, and the cost buffer read back through PM_BUF_COST_TILE equals the expected tile: repeated passes over a
warm sentinel map, a worker upsert that reorders the columns, disabled asks, an incremental pass in between and a
sharded range."""
import numpy as np
import pytest

from protocol_b200 import abi
from test_block_class_formulation import gpu_tables, with_disabled
from test_gpu_feature_predicate import FEAT, kernel_of
from test_gpu_narrow_tile import assert_oracle
from test_gpu_tile_overlap import tile_bytes
from test_gpu_tile_write_skip import History

pytestmark = pytest.mark.gpu

INCR = abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS | abi.PM_INCREMENTAL


class Checked(History):
    """History that also holds each pass of the engine against the CPU oracle while every ask is enabled."""

    enabled = True

    def outputs(self, x):
        arr, res = super().outputs(x)
        if x is self.e and self.enabled:
            w0, nw, _ = self.range()
            fa, best, cnt = arr
            assert_oracle(self.t, (fa.view(np.uint32), best, cnt.view(np.uint32)), w0, w0 + nw)
        return arr, res


@pytest.mark.parametrize("name", ["cfg3_like", "edge_64"])
def test_block_classes_through_a_history(name):
    t, _ = gpu_tables()[name]
    W, T = len(t["wa"]), len(t["asks"])
    assert kernel_of(t) == {FEAT}
    h = Checked(t, tile_bytes(W, 512))   # tiles of 512 rows: a slot sees other asks from tile to tile
    rng = np.random.default_rng(11)
    try:
        for _ in range(3):                   # the first pass writes every block, the next ones find the map warm
            h.run_pass()
        # workers rewritten with other workers' contents: other F runs, another column order
        src = rng.permutation(W)[:W // 4]
        na, nb = h.t["wa"][src].copy(), h.t["wb"][src].copy()
        nb["ext_ask_price"] = rng.integers(1, 1 << 24, len(src))
        first = W // 3
        h.both(lambda x: x.upsert_workers(na, nb, first))
        h.t["wa"][first:first + len(src)], h.t["wb"][first:first + len(src)] = na, nb
        h.run_pass()
        h.run_pass()
        # an incremental pass (the fused lean path) after another upsert; the tile and its map are left alone
        src = rng.permutation(W)[:500]
        na, nb = h.t["wa"][src].copy(), h.t["wb"][src].copy()
        h.both(lambda x: x.upsert_workers(na, nb, 77))
        h.t["wa"][77:577], h.t["wb"][77:577] = na, nb
        h.both(lambda x: x.match(INCR))
        a, b = h.e.fetch(), h.twin.fetch()
        assert np.array_equal(a.worker_ask, b.worker_ask) and np.array_equal(a.group_members, b.group_members)
        h.run_pass()
        # disabled asks require the never bit: dead in every block
        on = with_disabled(h.t)
        off = np.flatnonzero(~on).astype(np.uint32)
        h.both(lambda x: x.set_ask_enabled(off, False))
        h.enabled = False
        h.run_pass()
        h.run_pass()
        h.both(lambda x: x.set_ask_enabled(off, True))
        h.enabled = True
        h.run_pass()
        assert h.n_checked == 9
    finally:
        h.close()


def test_block_classes_on_a_sharded_range():
    t, (w0, nw) = gpu_tables()["cfg3_like_shard"]
    h = Checked(t, tile_bytes(nw, 512))
    try:
        h.shard = (w0, nw)
        h.both(lambda x: x.set_shard(w0, nw))
        for _ in range(3):
            h.run_pass()
        h.shard = None                       # the whole table: ld and the rows per tile change under the map
        h.both(lambda x: x.set_shard(0, 0))
        h.run_pass()
        h.shard = (w0, nw)
        h.both(lambda x: x.set_shard(w0, nw))
        h.run_pass()
        assert h.n_checked == 5
    finally:
        h.close()
