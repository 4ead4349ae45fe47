"""Group formation under the reference's DEFAULT policy, ProximityOptimizationPolicy{enabled:true}
(crates/orchestrator/src/plugins/node_groups/mod.rs:85-89, 524-552, 218-255), on the all-SM cooperative sweep
(pm_proximity_grid.cuh, the default) and on the single-CTA sweep it replaced (PM_TUNE_PROX=2): groups, creation order
and member order equal the CPU checker's on every shape the sweep has a special path for — ties everywhere (city
clusters, one point), scattered coordinates, nobody located, groups larger than one selection pass (16), empty
groups (min 0), long hand-downs between configurations (ordered compaction), solo configurations after grouped ones.
The edges of the coordinate space (EDGES: poles, antimeridian, antipodes, latitudes beyond ±90) run on both, and the
grid sweep's latitude pruning must switch off where the latitude bound fails.
Past the first stride (thousands of configurations, hand-downs across the shared-memory limit, seed-parallel batches on
many CTAs, selections in several chunks of 16): tests/test_gpu_proximity_sweeps.py.
"""
import math
import os

import numpy as np
import pytest

from helpers import CERT_GAP_ANTIPODE_KM, CERT_GAP_KM, assert_distance_certificate, groups_equal, load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200.engine import Engine, Interner

pytestmark = pytest.mark.gpu

KERNELS = [("0", "grid"), ("2", "single_cta")]
EDGES = ["polar", "antimeridian", "antipodal", "beyond_90"]
R_KM = 6371.0
KM_PER_DEG = R_KM * np.pi / 180.0


def _unit(lat, lon):
    la, lo = np.radians(lat), np.radians(lon)
    return np.stack([np.cos(la) * np.cos(lo), np.cos(la) * np.sin(lo), np.sin(la)], -1)


def _near_ties(pts, margin=3.0):
    """(i, j, k): from point i, points j and k lie closer in distance than the certificate allows (times `margin`;
    f64 here, the 50-digit certificate decides)."""
    u = _unit(pts[:, 0], pts[:, 1])
    d = R_KM * np.arctan2(np.linalg.norm(np.cross(u[:, None], u[None]), axis=-1), u @ u.T)
    out = []
    for i in range(len(pts)):
        order = np.argsort(d[i])
        order = order[order != i]
        row = d[i, order]
        need = np.where(row[1:] > np.pi * R_KM - 1.0, CERT_GAP_ANTIPODE_KM, CERT_GAP_KM) * margin
        out += [(i, int(order[c]), int(order[c + 1])) for c in np.nonzero(np.diff(row) < need)[0]]
    return out


def _thin(pts, n_special):
    """Drop background points (all but the first n_special) until no near-tie is left."""
    while True:
        drop = set()
        for i, j, k in _near_ties(pts):
            victim = max(j, k) if max(j, k) >= n_special else i    # a tie between special points: drop the viewer
            assert victim >= n_special, f"placement bug: {pts[j]} and {pts[k]} tie from {pts[i]}"
            drop.add(victim)
        if not drop:
            return pts
        pts = np.delete(pts, sorted(drop), axis=0)


def _draw_groups(rng, n_points, make):
    """Groups of points from make(rng, points so far) (None: draw again), each redrawn while it ties with the ones
    before, until there are n_points."""
    pts = np.zeros((0, 2))
    while len(pts) < n_points:
        grp = make(rng, len(pts))
        if grp is not None and not _near_ties(np.concatenate([pts, grp])):
            pts = np.concatenate([pts, grp])
    return pts


def _antipodal_trios(rng, n, n_over):
    """n (seed, its exact antipode, a point 2-9 m from the antipode), the first n_over of them pairs for which glibc's
    haversine rounds `a` above 1."""
    def trio(rng, have):
        lat, lon = float(rng.uniform(-60, 60)), float(rng.uniform(-180, 180))
        if have < 3 * n_over and _restated_a(lat, lon, -lat, lon + 180.0) <= 1.0:
            return None
        m = float(rng.uniform(2.0, 9.0))
        return np.array([(lat, lon), (-lat, lon + 180.0), (-lat + m * 1e-3 / KM_PER_DEG, lon + 180.0)])
    return _draw_groups(rng, 3 * n, trio)


def _beyond_90_traps(rng, n):
    """n (seed, its nearest neighbour 1 km north written beyond ±90: over 4 000 km away by R·|Δlatitude|)."""
    def trap(rng, have):
        lat, lon = float(rng.uniform(-70, 70)), float(rng.uniform(-180, 180))
        return np.array([(lat, lon), _as_beyond_90(lat + 1.0 / KM_PER_DEG, lon)])
    return _draw_groups(rng, 2 * n, trap)


def _sphere(rng, n, lat_lo=-90.0, lat_hi=90.0):
    """n places uniform by area between two latitudes."""
    z = rng.uniform(np.sin(np.radians(lat_lo)), np.sin(np.radians(lat_hi)), n)
    return np.stack([np.degrees(np.arcsin(z)), rng.uniform(-180, 180, n)], 1)


def _restated_a(lat1, lon1, lat2, lon2):
    k = 3.14159265358979323846264338327950288 / 180.0
    s1, s2 = math.sin((lat2 - lat1) * k / 2.0), math.sin((lon2 - lon1) * k / 2.0)
    return s1 * s1 + math.cos(lat1 * k) * math.cos(lat2 * k) * (s2 * s2)


def _as_beyond_90(lat, lon):
    """The same place with its latitude written beyond ±90."""
    return math.copysign(180.0, lat) - lat, lon + 180.0


def edge_points(where, rng):
    """(points as written, how many of the first ones are `special`): ~256 distinct places at one edge of the
    coordinate space.  Special points go to one worker each (no duplicate can stand between a seed and them), the
    rest are shared by several workers (position ties)."""
    special = []
    if where == "polar":
        special = [(90.0, 0.0), (-90.0, 37.0)]                      # each pole under one longitude only
        for pole in (1.0, -1.0):
            for lon in rng.uniform(-180, 180, 5):                    # candidates on a seed's meridian
                special += [(pole * (90.0 - float(x)), float(lon)) for x in rng.uniform(0.02, 4.0, 5)]
        bg = np.concatenate([_sphere(rng, 100, 86.0, 90.0), _sphere(rng, 100, -90.0, -86.0)])
    elif where == "antimeridian":
        bg = []
        for lat in rng.uniform(-75, 75, 8):                          # clusters across ±180 ...
            true_lon = 180.0 + rng.uniform(-1.5, 1.5, 30)
            wrap = rng.random(30) < 0.5                              # ... written as 179.9 or -180.1, 180.2 or -179.8
            bg += list(zip(lat + rng.uniform(-1.0, 1.0, 30), np.where(wrap, true_lon - 360.0, true_lon)))
        bg = np.array(bg)
    elif where == "antipodal":
        special = [tuple(p) for p in _antipodal_trios(rng, 12, 9)]
        bg = _sphere(rng, 200)
    else:
        assert where == "beyond_90"
        special = [tuple(p) for p in _beyond_90_traps(rng, 24)]
        bg = _sphere(rng, 200)
        for i in np.nonzero(rng.random(len(bg)) < 0.35)[0]:
            bg[i] = _as_beyond_90(*bg[i])
    return _thin(np.concatenate([np.array(special, dtype=np.float64).reshape(-1, 2), bg]), len(special)), len(special)


def swarm(n_workers, where, seed_shift=0):
    w = synth.make_workers(n_workers, seed=synth.SEED_WORKERS + seed_shift, with_addresses=n_workers <= 30000)
    rng = np.random.default_rng(seed_shift + 1)
    lat, lon = w.lat.copy(), w.lon.copy()
    if where == "scattered":      # distinct points: no near-ties between different libm's at kilometre scale
        lat = lat + rng.normal(0, 3.0, len(lat)).clip(-20, 20)
        lon = lon + rng.normal(0, 5.0, len(lon))
    elif where == "one_point":
        lat[:] = 45.5
        lon[:] = -73.5
    elif where == "nowhere":
        w.a["flags"] &= ~np.uint32(abi.PM_W_HAS_LOC)
    elif where in EDGES:
        pts, n_special = edge_points(where, rng)
        located = np.nonzero(w.a["flags"] & abi.PM_W_HAS_LOC)[0]
        pick = rng.integers(n_special, len(pts), len(w))
        cand = located[(w.a["flags"][located] & (abi.PM_W_HEALTHY | abi.PM_W_P2P | abi.PM_W_ASSIGNED))
                       == (abi.PM_W_HEALTHY | abi.PM_W_P2P)]
        pick[cand[:n_special]] = np.arange(n_special)              # the first located candidates: one special point each
        lat, lon = pts[pick, 0].copy(), pts[pick, 1].copy()
    else:
        assert where == "cities"
    w.lat, w.lon = lat, lon
    return w


def tables_for(w, a):
    bits, npat, nmod, words = synth.intern_tables(w, a)
    return dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words,
                lat=w.lat, lon=w.lon)


def custom_asks(rows):
    """[(requirement string | None, min, max)] in priority order -> synth.Asks."""
    it = Interner()
    for i, m in enumerate(m for m, _ in synth.MODEL_CATALOGUE):
        assert it.model(m) == i
    for i, p in enumerate(synth.PATTERN_CATALOGUE):
        assert it.pattern(p) == i
    asks, opts = [], []
    for req, mn, mx in rows:
        if req is None:
            row, o = np.zeros(1, dtype=abi.ASK)[0], np.zeros(0, dtype=abi.GPU_OPT)
        else:
            row, o = it.parse(req)
        row = row.copy()
        row["opt_off"] = sum(len(x) for x in opts)
        row["min_group_size"], row["max_group_size"] = mn, mx
        asks.append(row)
        opts.append(o)
    it.close()
    allo = np.concatenate(opts).astype(abi.GPU_OPT) if sum(map(len, opts)) else np.zeros(0, dtype=abi.GPU_OPT)
    return synth.Asks(asks=np.array(asks, dtype=abi.ASK), opts=allo, pattern_strings=list(synth.PATTERN_CATALOGUE))


def run(kernel, w, a, checker="banded"):
    """Engine groups on `kernel` == the checker's.  An input of at most 512 distinct points (all but "scattered", whose
    thousands of points allow no tie-free certificate) must first pass the distance certificate: a difference is then
    a kernel bug, not two libm's rounding a near-tie differently."""
    if len(np.unique(np.stack([w.lat, w.lon], 1), axis=0)) <= 512:
        assert_distance_certificate(w.lat, w.lon, (w.a["flags"] & abi.PM_W_HAS_LOC) != 0)
    t = tables_for(w, a)
    os.environ["PM_TUNE_PROX"] = kernel   # read at pm_create
    try:
        eng = Engine(timing=True)
    finally:
        os.environ.pop("PM_TUNE_PROX", None)
    load_engine(eng, t, addr_rank=w.addr_rank, locations=True)
    eng.match(abi.PM_MODE_PROXIMITY)
    res = eng.fetch()
    eng.match(abi.PM_MODE_PROXIMITY)            # a second pass on the same engine reuses every buffer
    res2 = eng.fetch()
    eng.close()
    og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], addr_rank=w.addr_rank,
                             lat=t["lat"], lon=t["lon"], proximity=checker)
    assert groups_equal(res, og), f"groups differ: engine {res.n_groups} vs checker {len(og)}"
    assert groups_equal(res2, og)
    wg = np.full(len(w), abi.PM_NONE, dtype=np.uint32)
    for g in range(len(og.cfg)):
        wg[og.members[og.off[g]:og.off[g + 1]]] = g
    assert np.array_equal(res.worker_group, wg)
    return res, og


@pytest.mark.parametrize("kernel", [k for k, _ in KERNELS], ids=[n for _, n in KERNELS])
@pytest.mark.parametrize("where", ["cities", "scattered", "one_point", "nowhere"] + EDGES)
def test_mixed_group_sizes(kernel, where):
    sizes = [(1, 1), (2, 2), (2, 4), (3, 3), (4, 8), (1, 3), (0, 2), (2, 5), (0, 1)]
    w = swarm(4000, where, seed_shift=7)
    a = synth.make_asks(120, "mixed", seed=synth.SEED_ASKS + 7, group_sizes=sizes)
    res, og = run(kernel, w, a, checker=True if where == "nowhere" else "banded")
    assert res.n_groups > 50


@pytest.mark.parametrize("kernel", [k for k, _ in KERNELS], ids=[n for _, n in KERNELS])
@pytest.mark.parametrize("where", EDGES)
def test_pairs_at_coordinate_edges(kernel, where):
    """Everybody competes for pairs, so the seed-parallel batches with their latitude pruning (grid) run.  The first
    located candidates hold one special point each: under "beyond_90" every other seed's nearest neighbour is 1 km
    away but written beyond ±90, more than 4 000 km away by R·|Δlatitude| — a sweep that kept pruning by latitude
    would pass it over."""
    w = swarm(4000, where, seed_shift=5)
    a = custom_asks([(None, 2, 2), (None, 1, 1)])
    res, og = run(kernel, w, a)
    assert (np.diff(res.group_off) == 2).sum() > 1500
    if where == "beyond_90":
        special = set(np.nonzero((np.abs(w.lat) > 90) & (w.a["flags"] & abi.PM_W_HAS_LOC != 0))[0].tolist())
        pairs = [og.members[og.off[g]:og.off[g + 1]].tolist() for g in range(len(og.cfg)) if og.off[g + 1] - og.off[g] == 2]
        held = sum(1 for p in pairs if abs(w.lat[p[0]] - w.lat[p[1]]) * KM_PER_DEG > 1000.0
                   and haversine_pair(w, p) < 1.001 and special & set(p))
        assert held >= 10          # the traps were sprung: pairs 1 km apart, thousands of km apart by latitude


def haversine_pair(w, p):
    return orc.haversine_km(w.lat[p[0]], w.lon[p[0]], w.lat[p[1]], w.lon[p[1]])


@pytest.mark.parametrize("kernel", [k for k, _ in KERNELS], ids=[n for _, n in KERNELS])
def test_antipode_ranks_before_no_location(kernel):
    """A seed's exact antipode is the farthest place there is, R·π, but still nearer than a candidate without a
    location (f64::MAX).  Each configuration holds one seed, its exact antipode, a point metres from that antipode and
    two unlocated workers; groups of three take the two antipodal points.  For most seeds rounding pushes haversine's
    `a` above 1 with glibc, where an unclamped sqrt(1 - a) is NaN — which ranks nowhere."""
    w = synth.make_workers(16 * 5, seed=synth.SEED_WORKERS + 41, with_addresses=True, healthy_frac=1.0)
    full = (abi.PM_W_HAS_SPECS | abi.PM_W_HAS_GPU | abi.PM_W_HAS_GPU_COUNT | abi.PM_W_HAS_GPU_MEM | abi.PM_W_HAS_GPU_MODEL
            | abi.PM_W_HAS_CPU | abi.PM_W_HAS_CPU_CORES | abi.PM_W_HAS_RAM | abi.PM_W_HAS_STORAGE | abi.PM_W_HEALTHY | abi.PM_W_P2P
            | abi.PM_W_HAS_LOC)
    trios = _antipodal_trios(np.random.default_rng(41), 16, 12)
    assert sum(_restated_a(*trios[3 * t], *trios[3 * t + 1]) > 1.0 for t in range(16)) >= 12
    for t in range(16):
        rows = slice(5 * t, 5 * t + 5)
        w.a["gpu_count"][rows] = 100 + t
        w.a["flags"][rows] = full
        w.a["flags"][5 * t + 3: 5 * t + 5] &= ~np.uint32(abi.PM_W_HAS_LOC)
        w.lat[rows] = [*trios[3 * t: 3 * t + 3, 0], 0.0, 0.0]
        w.lon[rows] = [*trios[3 * t: 3 * t + 3, 1], 0.0, 0.0]
    a = custom_asks([(f"gpu:count={100 + t}", 3, 3) for t in range(16)])
    res, og = run(kernel, w, a, checker=True)
    assert len(og) == 16
    for g in range(16):
        mem = og.members[og.off[g]:og.off[g + 1]]
        assert np.all(w.a["flags"][mem] & abi.PM_W_HAS_LOC)     # the antipodal points, not the unlocated workers


@pytest.mark.parametrize("kernel", [k for k, _ in KERNELS], ids=[n for _, n in KERNELS])
@pytest.mark.parametrize("where", ["cities", "scattered"] + EDGES)
def test_groups_larger_than_one_selection_pass(kernel, where):
    """max - 1 > 16 neighbours: several selection passes (and barriers) per group; min close to max leaves tails."""
    w = swarm(6000, where, seed_shift=3)
    a = custom_asks([("gpu:count=8", 30, 40), ("gpu:count=4", 17, 17), ("gpu:count=2", 18, 35), (None, 20, 33), (None, 2, 19)])
    res, og = run(kernel, w, a)
    sizes = np.diff(res.group_off)
    assert sizes.max() >= 35 and res.stats["n_bumped"] > 0


@pytest.mark.parametrize("kernel", [k for k, _ in KERNELS], ids=[n for _, n in KERNELS])
def test_long_hand_down_between_configurations(kernel):
    """A configuration that cannot reach its minimum hands ALL its candidates down (hundreds: the list of the next
    configuration is rebuilt by ordered compaction), a pair configuration leaves one, and a solo configuration with
    min 0 takes the rest and adds its empty group."""
    w = swarm(9000, "cities", seed_shift=11)
    n8 = int(((w.a["gpu_count"] == 8) & ((w.a["flags"] & 3) == 3) & ((w.a["flags"] & abi.PM_W_HAS_SPECS) != 0)).sum())
    assert n8 > 600
    a = custom_asks([("gpu:count=8", n8 + 50, n8 + 60),      # never forms: every 8-GPU candidate is handed down
                     ("gpu:count=8;gpu:model=H100", 3, 3),
                     ("gpu:count=8", 2, 2),
                     ("gpu:count=4", 2, 7),
                     (None, 0, 1)])
    res, og = run(kernel, w, a)
    assert res.stats["n_bumped"] >= n8 and (np.diff(res.group_off) == 0).sum() == 1


@pytest.mark.parametrize("kernel", [k for k, _ in KERNELS], ids=[n for _, n in KERNELS])
def test_pairs_then_solo_at_100k_nodes(kernel):
    """The host benchmark's shape (tools/host_bench.cpp: pair-h100 2..2 + solo 1..1, default policy) at 100 000 nodes."""
    w = swarm(100_000, "cities", seed_shift=0)
    a = custom_asks([("gpu:count=8;gpu:count=4", 2, 2), (None, 1, 1)])   # 35 % of the candidates compete for pairs
    res, og = run(kernel, w, a)
    print(f"\n[proximity {dict(KERNELS)[kernel]}] 100k nodes: {res.n_groups} groups, ms_resolve = {res.stats['ms_resolve']:.2f}, "
          f"batches = {res.stats['n_tiles']}, groups formed in batches = {res.stats['n_rounds']}, one at a time = {res.stats['n_build_launches']}")
    assert (np.diff(res.group_off) == 2).sum() > 10_000


@pytest.mark.skipif(os.environ.get("PM_TEST_BIG") != "1", reason="1M-node timing run (PM_TEST_BIG=1): ~1 min of CPU checker")
def test_pairs_then_solo_at_1m_nodes():
    """1M nodes, every fourth an 8-GPU node competing for pair groups (the case the single-CTA sweep is slowest on)."""
    w = swarm(1_000_000, "cities", seed_shift=0)
    a = custom_asks([("gpu:count=8;gpu:count=4", 2, 2), (None, 1, 1)])
    res, og = run("0", w, a)
    print(f"\n[proximity grid] 1M nodes: {res.n_groups} groups ({int((np.diff(res.group_off) == 2).sum())} pairs), "
          f"ms_resolve = {res.stats['ms_resolve']:.1f}, batches = {res.stats['n_tiles']}, groups formed in batches = {res.stats['n_rounds']}, "
          f"one at a time = {res.stats['n_build_launches']}")
