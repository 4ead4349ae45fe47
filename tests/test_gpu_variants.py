"""The kernel variants real swarms select, which the 16-model synthetic catalogue never reaches (VERDICT r1, A10).

GpuSpecs.model is a free-form NVML string that the reference normalises and substring-matches
(crates/shared/src/models/node.rs:463-484), so a permissionless pool has far more than 32 distinct models:

  * > 32 models, table <= 2048 words  -> acceptance rows in shared memory, one word PER WORKER  (BITS = 1)
  * table > 2048 words                -> acceptance rows read from global memory              (BITS = 0)
  * an ask with more OR-options than the shared-memory stage holds (384) -> eval_row_global
  * option rows that point at the last pattern rows of the table

In every test the acceptance table is computed TWICE — by the oracle from the strings with the reference's model
clause (oracle.model_table) and by the product's interner — the two are diffed, the oracle's goes to the oracle and
the product's to the engine.  Both predicate forms (generic, fast) and both evaluation paths run.
"""
import os

import numpy as np
import pytest

from helpers import groups_equal
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200.engine import Engine, Interner

pytestmark = pytest.mark.gpu

MAT, FUSED, LEAN = abi.PM_PATH_MATERIALIZED, abi.PM_PATH_FUSED, abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS
EXTRA_PATTERNS = ["mi300x", "b200", "quadro", "rev3", "sxm,nvl", "geforce rtx 4090 ti", "tesla", "pcie", "h100 80gb",
                  "instinct", "rtx a6000,l40s", "hbm3"]


def product_table(model_strings, pattern_strings):
    it = Interner()
    for i, m in enumerate(model_strings):
        assert it.model(m) == i
    for i, p in enumerate(pattern_strings):
        assert it.pattern(p) == i
    out = it.table()
    it.close()
    return out


def wide_tables(n_asks, n_workers, n_models, n_patterns, seed_shift=0, last_rows=False):
    cat = synth.wide_model_catalogue(n_models)
    w = synth.make_workers(n_workers, seed=synth.SEED_WORKERS + seed_shift, catalogue=cat)
    a = synth.make_asks(n_asks, "mixed", seed=synth.SEED_ASKS + seed_shift)
    pats = list(synth.PATTERN_CATALOGUE) + EXTRA_PATTERNS
    while len(pats) < n_patterns:   # patterns that single out one family/revision: sparse rows
        k = len(pats)
        pats.append(f"rev{k % 40},{cat[(k * 37) % len(cat)][0].lower()},zz{k}")   # the last piece only makes the string unique
    a.pattern_strings = pats[:n_patterns]
    # spread the asks' model clauses over the whole pattern table (and, if asked, pin some to its last rows)
    has_model = (a.opts["present"] & abi.PM_O_MODEL) != 0
    pid = (synth.splitmix64(synth.SEED_ASKS + seed_shift, len(a.opts), 21) % np.uint64(n_patterns)).astype(np.uint32)
    if last_rows:
        tail = np.arange(len(a.opts)) % 5 == 0
        pid[tail] = n_patterns - 1 - (np.arange(len(a.opts))[tail] % 3)
    a.opts["pattern_id"][has_model] = pid[has_model]
    obits, npat, nmod, words = orc.model_table(w.model_strings, a.pattern_strings)
    pbits, p_npat, p_nmod, p_words = product_table(w.model_strings, a.pattern_strings)
    assert (npat, nmod, words) == (p_npat, p_nmod, p_words)
    assert np.array_equal(obits, pbits), "product interner and the reference's model clause disagree"
    return w, a, obits, pbits, npat, nmod, words


def run_all_paths(w, a, obits, pbits, npat, nmod, words, expect_bits, check_cost_rows=64):
    T, W = len(a), len(w)
    og = orc.soa_form_groups(w.a, w.b, a.asks, a.opts, obits, words)
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, obits, words, 0, T, 0, W, threads=8)
    dwords = max((nmod + 30) // 31, 1)            # the device keeps 31 models per acceptance word
    bits_rows_words = (npat + 1) * dwords
    got_bits = 2 if (bits_rows_words <= 2048 and dwords == 1) else 1 if bits_rows_words <= 2048 else 0
    assert got_bits == expect_bits, f"table shape selects BITS={got_bits}, the test is meant for BITS={expect_bits}"
    for generic in ("0", "1"):
        os.environ["PM_TUNE_GENERIC"] = generic   # read at pm_create
        try:
            eng = Engine(cost_tile_bytes=1 << 20)
        finally:
            os.environ.pop("PM_TUNE_GENERIC", None)
        eng.set_asks(a.asks, a.opts)
        eng.set_model_table(pbits, npat, nmod, words)
        eng.set_workers(w.a, w.b)
        for path in (MAT, FUSED, LEAN):
            eng.match(abi.PM_MODE_FIRST_FIT | path)
            res = eng.fetch()
            assert groups_equal(res, og), f"groups differ (generic={generic}, path={path:#x})"
            if path != LEAN:
                assert np.array_equal(res.ask_best, ev["row_best"]) and np.array_equal(res.ask_count, ev["row_count"])
        n = min(check_cost_rows, T)
        cost = eng.cost_tile(T - n, n)
        ref = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, obits, words, T - n, T, 0, W, threads=8, want_cost=True)["cost"]
        assert np.array_equal(cost, ref)
        eng.close()


def test_200_models_acceptance_rows_in_shared_memory():
    """200 distinct model strings, 7 words per row, 113 rows: BITS = 1."""
    t = wide_tables(700, 6000, n_models=200, n_patterns=112, seed_shift=1)
    run_all_paths(*t, expect_bits=1)


def test_3000_models_acceptance_rows_in_global_memory():
    """3000 models x 112 patterns = 10.6k words > 2048: BITS = 0; option rows pinned to the table's last rows."""
    t = wide_tables(700, 6000, n_models=3000, n_patterns=112, seed_shift=2, last_rows=True)
    run_all_paths(*t, expect_bits=0)


def test_100k_models():
    """100 000 distinct model strings (3125 words per row)."""
    t = wide_tables(260, 20000, n_models=100_000, n_patterns=40, seed_shift=3, last_rows=True)
    run_all_paths(*t, expect_bits=0)


@pytest.mark.parametrize("n_models,n_patterns", [(100_000, 24), (3000, 30), (3000, 31), (70_000, 12)])
def test_wide_catalogue_few_patterns_worker_major_acceptance(n_models, n_patterns):
    """More model strings than the shared-memory table holds, at most 30 patterns: the fast kernels turn the acceptance
    table around (one word per WORKER over all patterns, pm_worker_nacc; EvalParams::nacc) instead of one global-memory
    lookup per (row, worker) pair.  30 patterns is the last size that fits (31 rows with row 0), 31 falls back to the
    global-memory table; the generic predicate always uses the table as it is.  Same groups, per-ask minima and cost rows
    as the oracle on every path."""
    t = wide_tables(500, 9000, n_models=n_models, n_patterns=n_patterns, seed_shift=11 + n_patterns, last_rows=True)
    run_all_paths(*t, expect_bits=0)


def test_few_models_many_patterns_still_uniform_word():
    """<= 32 models but many patterns: one warp-uniform word per row (BITS = 2), rows near the end of the table."""
    t = wide_tables(400, 5000, n_models=30, n_patterns=900, seed_shift=4, last_rows=True)
    run_all_paths(*t, expect_bits=2)


def many_option_requirement(n_opts, feasible_every, pats):
    parts = []
    for k in range(n_opts):
        parts.append(f"gpu:count={3 if k % feasible_every else [1, 2, 4, 8][(k // feasible_every) % 4]}")   # no worker has 3 GPUs
        if k % 3 == 0:
            parts.append(f"gpu:model={pats[k % len(pats)]}")
        if k % 4 == 1:
            parts.append(f"gpu:memory_mb_min={16000 + (k % 7) * 8000}")
    return ";".join(parts)


BIG_ASKS = {40: 500, 41: 384, 42: 385, 170: 1200, 299: 400}   # ask -> OR-options; the stage holds 384


def many_option_tables(n_models):
    """300 ordinary asks over 5000 workers, with the asks of BIG_ASKS replaced by ones with that many OR-options:
    (workers, asks, oracle table, product table, n_patterns, n_models, words)."""
    cat = synth.wide_model_catalogue(n_models)
    w = synth.make_workers(5000, seed=synth.SEED_WORKERS + 9, catalogue=cat)
    base = synth.make_asks(300, "mixed", seed=synth.SEED_ASKS + 9)
    pats = list(synth.PATTERN_CATALOGUE) + EXTRA_PATTERNS
    it = Interner()
    for i, m in enumerate(w.model_strings):
        assert it.model(m) == i
    for i, p in enumerate(pats):
        assert it.pattern(p) == i
    rows, opts = [], []
    for t in range(300):
        if t in BIG_ASKS:
            row, o = it.parse(many_option_requirement(BIG_ASKS[t], 97 if t != 41 else 50, pats), max_opts=2048)
            assert len(o) == BIG_ASKS[t]
        else:
            row, o = base.asks[t].copy(), base.opts[int(base.asks["opt_off"][t]):int(base.asks["opt_off"][t]) + int(base.asks["n_opts"][t])]
        row = row.copy()
        row["opt_off"] = sum(len(x) for x in opts)
        row["min_group_size"] = row["max_group_size"] = 1
        rows.append(row)
        opts.append(o)
    a = synth.Asks(asks=np.array(rows, dtype=abi.ASK), opts=np.concatenate(opts).astype(abi.GPU_OPT), pattern_strings=pats)
    pbits, npat, nmod, words = it.table()
    it.close()
    obits, o_npat, o_nmod, o_words = orc.model_table(w.model_strings, pats)
    assert (npat, nmod, words) == (o_npat, o_nmod, o_words) and np.array_equal(obits, pbits)
    return w, a, obits, pbits, npat, nmod, words


@pytest.mark.parametrize("n_models", [16, 200], ids=["uniform_word", "per_worker_word"])
def test_asks_with_more_options_than_the_stage_holds(n_models):
    """One ask with 500 OR-options (eval_row_global), neighbours with exactly 384 and 385, between ordinary asks."""
    w, a, obits, pbits, npat, nmod, words = many_option_tables(n_models)
    # the big asks must not be trivially empty or trivially full
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, obits, words, 0, 300, 0, 5000, threads=8)
    for t in BIG_ASKS:
        assert 0 < ev["row_count"][t] < 4500
    run_all_paths(w, a, obits, pbits, npat, nmod, words, expect_bits=2 if n_models <= 31 else 1, check_cost_rows=300)
