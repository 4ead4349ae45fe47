"""ctypes binding of the CPU oracle (oracle/pm_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and the
cpu_baseline / --impl reference legs of bench.py.  Never by protocol_b200/.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpm_oracle.so")
_lib = None

ORC_HAS_SPECS, ORC_HAS_GPU, ORC_HAS_GPU_COUNT, ORC_HAS_GPU_MODEL, ORC_HAS_GPU_MEM = 1, 2, 4, 8, 16
ORC_HAS_CPU, ORC_HAS_CPU_CORES, ORC_HAS_RAM, ORC_HAS_STORAGE = 32, 64, 128, 256
ORC_HAS_P2P, ORC_HAS_LOC, ORC_ASSIGNED = 512, 1024, 2048
DISCOVERED, WAITING, HEALTHY, UNHEALTHY, DEAD, EJECTED, BANNED, LOWBALANCE = range(8)
PM_NONE = 0xFFFFFFFF
AUCTION_REFUSED = 0xFFFFFFFF   # orc_soa_auction(_rep) outside the engine's integer domain


class OrcNode(C.Structure):
    _fields_ = [
        ("has", C.c_uint32), ("status", C.c_uint32),
        ("gpu_count", C.c_uint32), ("gpu_mem_mb", C.c_uint32), ("cpu_cores", C.c_uint32),
        ("ram_mb", C.c_uint32), ("storage_gb", C.c_uint32), ("pad", C.c_uint32),
        ("gpu_model", C.c_char_p), ("address", C.c_char_p),
        ("lat", C.c_double), ("lon", C.c_double),
    ]


class OrcSolo(C.Structure):
    _fields_ = [("id", C.c_char_p), ("node", C.c_uint32), ("has_task", C.c_uint32)]


class OrcConfig(C.Structure):
    _fields_ = [("name", C.c_char_p), ("min_group_size", C.c_uint64), ("max_group_size", C.c_uint64),
                ("req", C.c_void_p)]


def build(force: bool = False) -> str:
    src = [os.path.join(_HERE, f) for f in ("pm_oracle.cpp", "pm_oracle.h")]
    src.append(os.path.join(os.path.dirname(_HERE), "include", "prime_match.h"))
    stale = (not os.path.exists(LIB_PATH)) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in src)
    if force or stale:
        subprocess.run(["make", "-C", _HERE, "-B", "libpm_oracle.so"], check=True, capture_output=True)
    return LIB_PATH


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        build()
    lib = C.CDLL(LIB_PATH)
    u32, vp, cp, sz, i32 = C.c_uint32, C.c_void_p, C.c_char_p, C.c_size_t, C.c_int
    P = C.POINTER
    sig = {
        "orc_req_parse": (vp, [cp, C.c_char_p, sz]),
        "orc_req_free": (None, [vp]),
        "orc_req_n_gpu": (u32, [vp]),
        "orc_req_gpu_u32": (i32, [vp, u32, i32, P(u32)]),
        "orc_req_gpu_model": (cp, [vp, u32]),
        "orc_req_scalar": (i32, [vp, i32, P(u32)]),
        "orc_meets": (i32, [P(OrcNode), vp]),
        "orc_node_compatible": (i32, [P(OrcNode), vp]),
        "orc_model_matches": (i32, [cp, cp]),
        "orc_haversine_km": (C.c_double, [C.c_double] * 4),
        "orc_sort_configs": (None, [P(OrcConfig), u32, vp]),
        "orc_available_configs": (u32, [P(OrcConfig), vp, u32, vp]),
        "orc_sort_nodes_by_status": (None, [vp, u32, vp]),
        "orc_form_groups": (vp, [P(OrcNode), u32, P(OrcConfig), u32, i32]),
        "orc_groups_free": (None, [vp]),
        "orc_groups_count": (u32, [vp]),
        "orc_groups_members_total": (u32, [vp]),
        "orc_groups_cfg": (P(u32), [vp]),
        "orc_groups_off": (P(u32), [vp]),
        "orc_groups_members": (P(u32), [vp]),
        "orc_groups_evals": (C.c_uint64, [vp]),
        "orc_merge_solo_groups": (vp, [P(OrcNode), u32, P(OrcSolo), u32, P(OrcConfig), u32, i32, i32, i32]),
        "orc_newest_task": (u32, [vp, u32]),
        "orc_sort_tasks": (None, [vp, u32, vp]),
        "orc_idx_in_group": (C.c_int64, [P(cp), u32, cp]),
        "orc_soa_compatible": (i32, [vp, vp, vp, vp, vp, u32]),
        "orc_soa_form_groups": (vp, [vp, vp, u32, vp, u32, vp, vp, u32, vp, vp, vp, i32]),
        "orc_soa_auction": (u32, [vp, vp, u32, vp, u32, vp, vp, u32, vp, C.c_uint64, C.c_uint64, u32, vp, vp]),
        "orc_soa_auction_rep": (u32, [vp, vp, u32, vp, u32, vp, vp, u32, vp, vp, vp, C.c_uint64, C.c_uint64, u32, vp, vp]),
        "orc_model_table": (None, [P(cp), u32, P(cp), u32, u32, u32, vp]),
        "orc_soa_first_feasible": (None, [vp, vp, u32, vp, u32, vp, vp, u32, u32, vp]),
        "orc_soa_eval_matrix": (C.c_uint64, [vp, vp, vp, vp, vp, u32, u32, u32, u32, u32, u32, vp, vp, vp, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


# ---------------------------------------------------------------- requirement strings
class Req:
    """Parsed ComputeRequirements (node.rs:180-374).  Raises ValueError on Err."""

    FIELDS = {"count": 0, "memory_mb": 1, "memory_mb_min": 2, "memory_mb_max": 3,
              "total_memory_min": 4, "total_memory_max": 5}

    def __init__(self, s: str):
        lib = load()
        err = C.create_string_buffer(256)
        self._h = lib.orc_req_parse(s.encode(), err, 256)
        if not self._h:
            raise ValueError(err.value.decode())
        self._lib = lib

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.orc_req_free(self._h)
            self._h = None

    @property
    def handle(self):
        return self._h

    def n_gpu(self) -> int:
        return self._lib.orc_req_n_gpu(self._h)

    def gpu(self, opt: int, name: str):
        if name == "model":
            m = self._lib.orc_req_gpu_model(self._h, opt)
            return None if m is None else m.decode()
        v = C.c_uint32()
        ok = self._lib.orc_req_gpu_u32(self._h, opt, self.FIELDS[name], C.byref(v))
        return v.value if ok else None

    def scalar(self, name: str):
        v = C.c_uint32()
        rc = self._lib.orc_req_scalar(self._h, {"cpu_cores": 0, "ram_mb": 1, "storage_gb": 2}[name], C.byref(v))
        return v.value if rc == 1 else None

    def has_cpu(self) -> bool:
        return self._lib.orc_req_scalar(self._h, 0, None) != -1


def make_node(address: str = "0x0", status: int = HEALTHY, p2p: bool = True, specs: bool = True,
              gpu_count=None, gpu_model=None, gpu_mem=None, gpu_present=None, cpu_cores=None,
              cpu_present=None, ram=None, storage=None, location=None, assigned: bool = False) -> OrcNode:
    """Mirror of the reference tests' create_compute_specs / create_test_node helpers
    (node.rs:626-657, node_groups/tests.rs:24-56)."""
    n = OrcNode()
    has = 0
    if specs:
        has |= ORC_HAS_SPECS
        if gpu_present is None:
            gpu_present = gpu_count is not None or gpu_model is not None or gpu_mem is not None
        if gpu_present:
            has |= ORC_HAS_GPU
            if gpu_count is not None:
                has |= ORC_HAS_GPU_COUNT
                n.gpu_count = gpu_count
            if gpu_model is not None:
                has |= ORC_HAS_GPU_MODEL
                n.gpu_model = gpu_model.encode()
            if gpu_mem is not None:
                has |= ORC_HAS_GPU_MEM
                n.gpu_mem_mb = gpu_mem
        if cpu_present is None:
            cpu_present = cpu_cores is not None
        if cpu_present:
            has |= ORC_HAS_CPU
            if cpu_cores is not None:
                has |= ORC_HAS_CPU_CORES
                n.cpu_cores = cpu_cores
        if ram is not None:
            has |= ORC_HAS_RAM
            n.ram_mb = ram
        if storage is not None:
            has |= ORC_HAS_STORAGE
            n.storage_gb = storage
    if p2p:
        has |= ORC_HAS_P2P
    if assigned:
        has |= ORC_ASSIGNED
    if location is not None:
        has |= ORC_HAS_LOC
        n.lat, n.lon = location
    n.has = has
    n.status = status
    n.address = address.encode()
    return n


def meets(node: OrcNode, req: Req) -> bool:
    return bool(load().orc_meets(C.byref(node), req.handle))


def node_compatible(node: OrcNode, req: Req | None) -> bool:
    return bool(load().orc_node_compatible(C.byref(node), req.handle if req else None))


def model_matches(spec: str, req: str) -> bool:
    return bool(load().orc_model_matches(spec.encode(), req.encode()))


def haversine_km(lat1, lon1, lat2, lon2) -> float:
    return load().orc_haversine_km(lat1, lon1, lat2, lon2)


def _configs(cfgs):
    """cfgs: list of (name, min, max, Req|None) -> ctypes array (keeps Req alive via caller)."""
    arr = (OrcConfig * max(len(cfgs), 1))()
    for i, (name, mn, mx, req) in enumerate(cfgs):
        arr[i].name = name.encode()
        arr[i].min_group_size = mn
        arr[i].max_group_size = mx
        arr[i].req = req.handle if req is not None else None
    return arr


def sort_configs(cfgs) -> list:
    arr = _configs(cfgs)
    perm = np.empty(len(cfgs), dtype=np.uint32)
    load().orc_sort_configs(arr, len(cfgs), perm.ctypes.data)
    return perm.tolist()


def available_configs(sorted_cfgs, enabled) -> list:
    arr = _configs(sorted_cfgs)
    en = np.ascontiguousarray(enabled, dtype=np.uint8)
    out = np.empty(len(sorted_cfgs), dtype=np.uint32)
    k = load().orc_available_configs(arr, en.ctypes.data, len(sorted_cfgs), out.ctypes.data)
    return out[:k].tolist()


def sort_nodes_by_status(status) -> list:
    st = np.ascontiguousarray(status, dtype=np.uint32)
    perm = np.empty(len(st), dtype=np.uint32)
    load().orc_sort_nodes_by_status(st.ctypes.data, len(st), perm.ctypes.data)
    return perm.tolist()


class Groups:
    def __init__(self, handle):
        lib = load()
        g = lib.orc_groups_count(handle)
        m = lib.orc_groups_members_total(handle)
        self.cfg = np.ctypeslib.as_array(lib.orc_groups_cfg(handle), shape=(g,)).copy() if g else np.zeros(0, np.uint32)
        self.off = np.ctypeslib.as_array(lib.orc_groups_off(handle), shape=(g + 1,)).copy()
        self.members = np.ctypeslib.as_array(lib.orc_groups_members(handle), shape=(m,)).copy() if m else np.zeros(0, np.uint32)
        self.evals = int(lib.orc_groups_evals(handle))
        lib.orc_groups_free(handle)

    def __len__(self):
        return len(self.cfg)

    def as_list(self):
        return [(int(self.cfg[g]), self.members[self.off[g]:self.off[g + 1]].tolist()) for g in range(len(self.cfg))]


def form_groups(nodes, cfgs, proximity: bool) -> Groups:
    """Faithful try_form_new_groups.  nodes: list[OrcNode]; cfgs: available configs in priority order."""
    arr = (OrcNode * max(len(nodes), 1))(*nodes)
    carr = _configs(cfgs)
    h = load().orc_form_groups(arr, len(nodes), carr, len(cfgs), 1 if proximity else 0)
    return Groups(h)


def merge_solo_groups(nodes, solos, cfgs, proximity=True, task_switching_enabled=True, prefer_larger_groups=True) -> Groups:
    """Faithful try_merge_solo_groups.  solos: list of (group id, node index, has_task)."""
    arr = (OrcNode * max(len(nodes), 1))(*nodes)
    sarr = (OrcSolo * max(len(solos), 1))()
    for i, (gid, node, has_task) in enumerate(solos):
        sarr[i].id, sarr[i].node, sarr[i].has_task = gid.encode(), node, int(has_task)
    carr = _configs(cfgs)
    h = load().orc_merge_solo_groups(arr, len(nodes), sarr, len(solos), carr, len(cfgs), int(proximity),
                                     int(task_switching_enabled), int(prefer_larger_groups))
    return Groups(h)


def newest_task(created_at) -> int:
    ca = np.ascontiguousarray(created_at, dtype=np.int64)
    return load().orc_newest_task(ca.ctypes.data, len(ca))


def sort_tasks(created_at) -> list:
    ca = np.ascontiguousarray(created_at, dtype=np.int64)
    perm = np.empty(len(ca), dtype=np.uint32)
    load().orc_sort_tasks(ca.ctypes.data, len(ca), perm.ctypes.data)
    return perm.tolist()


def idx_in_group(members, addr: str) -> int:
    arr = (C.c_char_p * max(len(members), 1))(*[m.encode() for m in members])
    return load().orc_idx_in_group(arr, len(members), addr.encode())


# ---------------------------------------------------------------- SoA side
def soa_compatible(a_row, b_row, ask_row, opts, bits, words) -> bool:
    a = np.ascontiguousarray(a_row).reshape(1)
    b = np.ascontiguousarray(b_row).reshape(1)
    k = np.ascontiguousarray(ask_row).reshape(1)
    opts = np.ascontiguousarray(opts)
    bits = np.ascontiguousarray(bits, dtype=np.uint32)
    return bool(load().orc_soa_compatible(a.ctypes.data, b.ctypes.data, k.ctypes.data, opts.ctypes.data,
                                          bits.ctypes.data, words))


def soa_form_groups(a, b, asks, opts, bits, words, addr_rank=None, lat=None, lon=None, proximity=False) -> Groups:
    """proximity: False (first fit), True (the reference's loop restated) or "banded" (same groups, latitude-pruned)."""
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    asks = np.ascontiguousarray(asks); opts = np.ascontiguousarray(opts)
    bits = np.ascontiguousarray(bits, dtype=np.uint32)
    ar = np.ascontiguousarray(addr_rank, dtype=np.uint32) if addr_rank is not None else None
    la = np.ascontiguousarray(lat, dtype=np.float64) if lat is not None else None
    lo = np.ascontiguousarray(lon, dtype=np.float64) if lon is not None else None
    h = load().orc_soa_form_groups(a.ctypes.data, b.ctypes.data, len(a), asks.ctypes.data, len(asks),
                                   opts.ctypes.data, bits.ctypes.data, words,
                                   ar.ctypes.data if ar is not None else None,
                                   la.ctypes.data if la is not None else None,
                                   lo.ctypes.data if lo is not None else None,
                                   2 if proximity == "banded" else (1 if proximity else 0))
    return Groups(h)


def soa_eval_matrix(a, b, asks, opts, bits, words, t0, t1, w0, w1, threads=1,
                    want_cost=False, want_rows=True, want_cols=True):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    asks = np.ascontiguousarray(asks); opts = np.ascontiguousarray(opts)
    bits = np.ascontiguousarray(bits, dtype=np.uint32)
    nt, nw = t1 - t0, w1 - w0
    cost = np.empty((nt, nw), dtype=np.int64) if want_cost else None
    rb = np.empty(nt, dtype=np.int64) if want_rows else None
    rc = np.empty(nt, dtype=np.uint32) if want_rows else None
    cf = np.empty(nw, dtype=np.uint32) if want_cols else None
    evals = load().orc_soa_eval_matrix(
        a.ctypes.data, b.ctypes.data, asks.ctypes.data, opts.ctypes.data, bits.ctypes.data, words,
        t0, t1, w0, w1, threads,
        cost.ctypes.data if cost is not None else None, rb.ctypes.data if rb is not None else None,
        rc.ctypes.data if rc is not None else None, cf.ctypes.data if cf is not None else None)
    return {"evals": int(evals), "cost": cost, "row_best": rb, "row_count": rc, "col_first": cf}


def model_table(model_strings, pattern_strings, threads=8):
    """(bits, n_patterns, n_models, words) in pm_set_model_table's layout, from the oracle's own model clause."""
    nm, npat = len(model_strings), len(pattern_strings)
    words = max((nm + 31) // 32, 1)
    bits = np.zeros(max(npat, 1) * words, dtype=np.uint32)
    ms = (C.c_char_p * max(nm, 1))(*[m.encode() for m in model_strings])
    ps = (C.c_char_p * max(npat, 1))(*[p.encode() for p in pattern_strings])
    load().orc_model_table(ms, nm, ps, npat, words, threads, bits.ctypes.data)
    return bits, npat, nm, words


def soa_first_feasible(a, b, asks, opts, bits, words, threads=8):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    asks = np.ascontiguousarray(asks); opts = np.ascontiguousarray(opts)
    bits = np.ascontiguousarray(bits, dtype=np.uint32)
    out = np.empty(len(a), dtype=np.uint32)
    load().orc_soa_first_feasible(a.ctypes.data, b.ctypes.data, len(a), asks.ctypes.data, len(asks), opts.ctypes.data,
                                  bits.ctypes.data, words, threads, out.ctypes.data)
    return out


def soa_auction(a, b, asks, opts, bits, words, price_cap, cost_scale=1, eps_start=1, eps_div=4, reputation=None,
                min_reputation=None):
    """EXTENSION self-oracle (no reference counterpart): returns (ask_worker u32[T], worker_price i64[W], rounds).
    reputation u32[W] / min_reputation u32[T] (north-star column, optional): feasible only if reputation >= floor.
    ValueError outside the engine's integer domain, (max ask_price + max cap + 2) * cost_scale + eps_start >= 2^61."""
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    asks = np.ascontiguousarray(asks); opts = np.ascontiguousarray(opts)
    bits = np.ascontiguousarray(bits, dtype=np.uint32)
    cap = np.ascontiguousarray(price_cap, dtype=np.uint32)
    rep = None if reputation is None else np.ascontiguousarray(reputation, dtype=np.uint32)
    floor = None if min_reputation is None else np.ascontiguousarray(min_reputation, dtype=np.uint32)
    assert rep is None or len(rep) == len(a)
    assert floor is None or len(floor) == len(asks)
    out = np.empty(len(asks), dtype=np.uint32)
    price = np.empty(len(a), dtype=np.int64)
    rounds = load().orc_soa_auction_rep(a.ctypes.data, b.ctypes.data, len(a), asks.ctypes.data, len(asks), opts.ctypes.data,
                                        bits.ctypes.data, words, cap.ctypes.data, None if rep is None else rep.ctypes.data,
                                        None if floor is None else floor.ctypes.data, cost_scale, eps_start, eps_div,
                                        out.ctypes.data, price.ctypes.data)
    if rounds == AUCTION_REFUSED:
        raise ValueError("soa_auction: (max ask_price + max cap + 2) * cost_scale + eps_start must stay below 2^61")
    return out, price, rounds


# ---- node ids: Address::from_str + Address::to_string (alloy-primitives 1.1.0, pinned in the reference's Cargo.lock; the
# crate is not part of the reference repository).  Restated from the published algorithms: Keccak-f[1600] as in the Keccak
# reference (state A[x][y], steps theta, rho, pi, chi, iota written out), Keccak-256 = rate 1088, padding 0x01 .. 0x80;
# EIP-55: hex letter i is upper case iff nibble i of keccak256(lower-case hex digits) >= 8.  Pinned by the vectors of
# EIP-55 itself and keccak256("") (tests/test_oracle_kat.py).  Pure Python: inputs are 40 bytes.
_KECCAK_RC = []


def _keccak_round_constants():
    if _KECCAK_RC:
        return _KECCAK_RC
    r = 1                                   # LFSR x^8 + x^6 + x^5 + x^4 + 1
    for _ in range(24):
        rc = 0
        for j in range(7):
            if r & 1:
                rc |= 1 << ((1 << j) - 1)
            r = ((r << 1) ^ ((r >> 7) * 0x71)) & 0xFF
        _KECCAK_RC.append(rc)
    return _KECCAK_RC


def keccak256(data: bytes) -> bytes:
    M64 = (1 << 64) - 1
    rol = lambda v, n: ((v << n) | (v >> (64 - n))) & M64 if n else v
    rate = 136
    msg = bytearray(data)
    msg.append(0x01)
    while len(msg) % rate:
        msg.append(0)
    msg[-1] |= 0x80
    A = [[0] * 5 for _ in range(5)]         # A[x][y]
    rc = _keccak_round_constants()
    for off in range(0, len(msg), rate):
        for i in range(rate // 8):
            A[i % 5][i // 5] ^= int.from_bytes(msg[off + 8 * i: off + 8 * i + 8], "little")
        for rnd in range(24):
            C = [A[x][0] ^ A[x][1] ^ A[x][2] ^ A[x][3] ^ A[x][4] for x in range(5)]
            D = [C[(x - 1) % 5] ^ rol(C[(x + 1) % 5], 1) for x in range(5)]
            A = [[A[x][y] ^ D[x] for y in range(5)] for x in range(5)]
            B = [[0] * 5 for _ in range(5)]
            x, y = 1, 0
            B[0][0] = A[0][0]
            for t in range(24):             # rho offsets (t+1)(t+2)/2 along the pi orbit of (1, 0)
                B[y][(2 * x + 3 * y) % 5] = rol(A[x][y], ((t + 1) * (t + 2) // 2) % 64)
                x, y = y, (2 * x + 3 * y) % 5
            A = [[B[x][y] ^ ((~B[(x + 1) % 5][y]) & B[(x + 2) % 5][y] & M64) for y in range(5)] for x in range(5)]
            A[0][0] ^= rc[rnd]
    out = b"".join(A[i % 5][i // 5].to_bytes(8, "little") for i in range(4))
    return out


def eip55(address: str):
    """`Address::from_str(address)?.to_string()`: None when the string is not 40 hex digits (optional 0x)."""
    h = address[2:] if address[:2] in ("0x", "0X") else address
    if len(h) != 40 or any(c not in "0123456789abcdefABCDEF" for c in h):
        return None
    low = h.lower()
    digest = keccak256(low.encode()).hex()
    return "0x" + "".join(c.upper() if c in "abcdef" and int(digest[i], 16) >= 8 else c for i, c in enumerate(low))
