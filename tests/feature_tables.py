"""The feature predicate of pm_build_argmin_feat (csrc/pm_kernels.cuh FeatDict, pm_feature_collect / _asks / _workers)
restated in numpy over the fast predicate's converted rows (test_fast_predicate_formulation.convert_ask), and random
tables that reach every feature kind at its edge values.  Shared by the CPU formulation test and the GPU test."""
import numpy as np

from protocol_b200 import abi
from test_fast_predicate_formulation import U, convert_ask, device_bits, workers_reg

KEY, COUNT, MODEL, MEM_LO, MEM_HI, TOT_LO, TOT_HI, CORES, RAM, STORAGE = range(10)
MAX_FEATURES = 64
CAND_KEY, NEVER_KEY = 10, 11   # key bits every dictionary holds
OPEN_HI = 0x7FFFFFFF           # an upper bound every fast-domain operand meets: no feature
INF = np.int64(0x7FFFFFFFFFFFFFFF)


def converted(asks, opts, enabled=None):
    """Per ask (cpu, ram, storage, [DevOptF rows]); a disabled ask carries the never bit in every row."""
    out = []
    for t, a in enumerate(asks):
        cpu, ram, sto, rows = convert_ask(a, opts)
        if enabled is not None and not enabled[t]:
            rows = [dict(r, m=r["m"] | 1 << NEVER_KEY, v=r["v"] | 1 << NEVER_KEY) for r in rows]
        out.append((cpu, ram, sto, rows))
    return out


def ask_features(cpu, ram, sto):
    return [(k, v) for k, v in ((CORES, cpu), (RAM, ram), (STORAGE, sto)) if v]


def opt_features(r):
    f = [(KEY, j) for j in range(13) if r["m"] >> j & 1]
    if r["m"] >> 13:
        f.append((COUNT, (r["v"] >> 13) & 0xFFFF))
    if r["prow"]:
        f.append((MODEL, r["prow"]))
    for k, v, on in ((MEM_LO, r["mem_lo"], r["mem_lo"] > 0), (MEM_HI, r["mem_hi"], r["mem_hi"] < OPEN_HI),
                     (TOT_LO, r["tot_lo"], r["tot_lo"] > 0), (TOT_HI, r["tot_hi"], r["tot_hi"] < OPEN_HI)):
        if on:
            f.append((k, v))
    return f


def dictionary(conv):
    """[(kind, value)] in bit order: kinds in order, values increasing; the candidate and never bits always."""
    vals = {k: set() for k in range(10)}
    vals[KEY] |= {CAND_KEY, NEVER_KEY}
    for cpu, ram, sto, rows in conv:
        for k, v in ask_features(cpu, ram, sto):
            vals[k].add(v)
        for r in rows:
            for k, v in opt_features(r):
                vals[k].add(v)
    return [(k, v) for k in range(10) for v in sorted(vals[k])]


def fits(d):
    return len(d) <= MAX_FEATURES


def worker_features(wa, wb, tbl, d):
    """F per worker, uint64: bit i = the worker meets feature d[i]."""
    w = workers_reg(wa, wb)
    fl = wa["flags"].astype(np.uint32)
    count_eff = np.where((fl & U(abi.PM_W_HAS_GPU_COUNT)) != 0, wa["gpu_count"], 0).astype(np.uint32)
    keep = w["tot_keep"] != 0
    F = np.zeros(len(wa), dtype=np.uint64)
    for i, (k, v) in enumerate(d):
        b = {KEY: lambda: (w["key"] >> U(v)) & U(1) != 0,
             COUNT: lambda: count_eff == v,
             MODEL: lambda: (tbl[v, w["mword"]] & w["mmask"]) != 0,
             MEM_LO: lambda: w["mem_eff"] >= v,
             MEM_HI: lambda: w["mem_eff"] <= v,
             TOT_LO: lambda: ~keep | (w["tot"] >= v),
             TOT_HI: lambda: ~keep | (w["tot"] <= v),
             CORES: lambda: w["cores"] >= v,
             RAM: lambda: w["ram"] >= v,
             STORAGE: lambda: w["storage"] >= v}[k]()
        F |= b.astype(np.uint64) << np.uint64(i)
    return F


def requirement_masks(conv, d):
    """Per ask the list of R_o (uint64): the option's features with the ask's scalar clauses OR-ed in."""
    bit = {kv: 1 << i for i, kv in enumerate(d)}
    out = []
    for cpu, ram, sto, rows in conv:
        s = 0
        for kv in ask_features(cpu, ram, sto):
            s |= bit[kv]
        rs = []
        for r in rows:
            m = s
            for kv in opt_features(r):
                m |= bit[kv]
            rs.append(m)
        out.append(rs)
    return out


def feature_fail(F, rs):
    """The kernel's fail word per worker: min over the options of (R_o & ~F) folded to 32 bits; non-zero = infeasible."""
    u = None
    for R in rs:
        x = np.uint64(R) & ~F
        x32 = ((x & np.uint64(0xFFFFFFFF)) | (x >> np.uint64(32))).astype(np.uint32)
        u = x32 if u is None else np.minimum(u, x32)
    return u


def feature_cost_matrix(t, enabled=None):
    """The packed int64 cost of every (ask, worker) pair from the feature predicate (raises when it does not fit)."""
    conv = converted(t["asks"], t["opts"], enabled)
    d = dictionary(conv)
    assert fits(d), f"{len(d)} features"
    tbl, _ = device_bits(t["bits"], t["n_patterns"], t["n_models"], t["words"])
    F = worker_features(t["wa"], t["wb"], tbl, d)
    price = t["wb"]["ext_ask_price"].astype(np.int64)
    feas_cost = (price << 32) | np.arange(len(t["wa"]), dtype=np.int64)
    out = np.empty((len(conv), len(t["wa"])), dtype=np.int64)
    for i, rs in enumerate(requirement_masks(conv, d)):
        out[i] = np.where(feature_fail(F, rs) != 0, INF, feas_cost)
    return out


def n_features(t):
    return len(dictionary(converted(t["asks"], t["opts"])))


MEM = [0, 1, 2, 24000, 40000, 80000, 0x7FFFFFFE]
TOT = [0, 1, 2, 100000, 320000, 0x7FFFFFFE]
SCALAR = [0, 1, 2, 8, 64, 0x7FFFFFFE]


def edge_tables(seed, n_asks, n_workers, n_models=40, n_patterns=6, max_opts=3, price_max=1 << 30):
    """Random tables in the fast domain whose thresholds and operands include 0, 1 and 0x7FFFFFFE, lo == hi, empty
    memory and total-memory intervals, workers without count or memory, OR-options next to scalar clauses, asks
    without options and max_group_size == 0 asks."""
    rng = np.random.default_rng(seed)
    wa = np.zeros(n_workers, dtype=abi.WORKER_A)
    wb = np.zeros(n_workers, dtype=abi.WORKER_B)
    has = [abi.PM_W_HAS_SPECS, abi.PM_W_HAS_GPU, abi.PM_W_HAS_GPU_COUNT, abi.PM_W_HAS_GPU_MEM, abi.PM_W_HAS_GPU_MODEL,
           abi.PM_W_HAS_CPU, abi.PM_W_HAS_CPU_CORES, abi.PM_W_HAS_RAM, abi.PM_W_HAS_STORAGE]
    for i in range(n_workers):
        f = abi.PM_W_HEALTHY * (rng.random() > .05) | abi.PM_W_P2P * (rng.random() > .03) | abi.PM_W_ASSIGNED * (rng.random() < .03)
        for h in has:
            f |= h * (rng.random() > .12)
        c = int(rng.choice([0, 1, 2, 4, 8, 3]))
        m = int(rng.choice(MEM))
        if c and m * c >= 1 << 31:
            m = (0x7FFFFFFF // c) if rng.random() < .5 else 40000
        wa[i] = (c, m, int(rng.integers(0, n_models)), f)
        wb[i] = tuple(int(rng.choice(SCALAR)) for _ in range(3)) + (int(rng.integers(0, price_max)),)
    asks = np.zeros(n_asks, dtype=abi.ASK)
    opts = []
    for t in range(n_asks):
        fl = abi.PM_A_HAS_REQ * (rng.random() > .08)
        for b in (abi.PM_A_REQ_CPU, abi.PM_A_REQ_CPU_CORES, abi.PM_A_REQ_RAM, abi.PM_A_REQ_STORAGE):
            fl |= b * (rng.random() < .35)
        k = int(rng.integers(0, max_opts + 1))
        mx = int(rng.choice([1, 1, 1, 3, 0]))
        asks[t] = (fl, k, len(opts), int(rng.choice(SCALAR)), int(rng.choice(SCALAR)), int(rng.choice(SCALAR)),
                   0 if mx == 0 else 1, mx)
        for _ in range(k):
            pr = 0
            for b in (abi.PM_O_COUNT, abi.PM_O_MODEL, abi.PM_O_MEM, abi.PM_O_MEM_MIN, abi.PM_O_MEM_MAX, abi.PM_O_TOT_MIN,
                      abi.PM_O_TOT_MAX):
                pr |= b * (rng.random() < .35)
            lo = int(rng.choice(MEM))
            hi = lo if rng.random() < .2 else int(rng.choice(MEM))   # lo == hi, and lo > hi: an empty interval
            tlo = int(rng.choice(TOT))
            thi = tlo if rng.random() < .2 else int(rng.choice(TOT))
            opts.append((pr, int(rng.choice([0, 1, 2, 4, 8])), int(rng.choice(MEM)), lo, hi, tlo, thi,
                         int(rng.integers(0, n_patterns))))
    words = (n_models + 31) // 32
    bits = rng.integers(0, 1 << 32, size=(n_patterns, words), dtype=np.uint64).astype(np.uint32)
    if n_models % 32:
        bits[:, -1] &= np.uint32((1 << (n_models % 32)) - 1)
    return dict(asks=asks, opts=np.array(opts, dtype=abi.GPU_OPT), wa=wa, wb=wb, bits=bits.reshape(-1),
                n_patterns=n_patterns, n_models=n_models, words=words)


def with_features(t, n, first=100_000):
    """t with asks appended, each requiring cpu cores at a new threshold, until the dictionary has exactly n features."""
    asks = list(t["asks"])
    v = first
    while True:
        cur = n_features(dict(t, asks=np.array(asks, dtype=abi.ASK)))
        if cur >= n:
            break
        asks.append((abi.PM_A_HAS_REQ | abi.PM_A_REQ_CPU | abi.PM_A_REQ_CPU_CORES, 0, 0, v, 0, 0, 1, 1))
        v += 1
    out = dict(t, asks=np.array(asks, dtype=abi.ASK))
    assert n_features(out) == n, (n_features(out), n)
    return out
