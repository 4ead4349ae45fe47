"""Python mirror of include/prime_match.h: constants, ctypes structs, numpy dtypes."""
from __future__ import annotations

import ctypes as C

import numpy as np

PM_ABI_VERSION = 1
PM_NONE = 0xFFFFFFFF
PM_COST_INF = 0x7FFFFFFFFFFFFFFF

PM_COMM_ID_BYTES = 128
PM_OK, PM_E_INVALID, PM_E_CUDA, PM_E_NO_DEVICE = 0, -1, -2, -3
PM_E_STATE, PM_E_NOMEM, PM_E_UNSUPPORTED, PM_E_PARSE = -4, -5, -6, -7

# pm_worker_flag
PM_W_HEALTHY = 1 << 0
PM_W_P2P = 1 << 1
PM_W_ASSIGNED = 1 << 2
PM_W_HAS_SPECS = 1 << 3
PM_W_HAS_GPU = 1 << 4
PM_W_HAS_GPU_COUNT = 1 << 5
PM_W_HAS_GPU_MEM = 1 << 6
PM_W_HAS_GPU_MODEL = 1 << 7
PM_W_HAS_CPU = 1 << 8
PM_W_HAS_CPU_CORES = 1 << 9
PM_W_HAS_RAM = 1 << 10
PM_W_HAS_STORAGE = 1 << 11
PM_W_HAS_LOC = 1 << 12

# pm_ask_flag
PM_A_HAS_REQ = 1 << 0
PM_A_REQ_CPU = 1 << 1
PM_A_REQ_CPU_CORES = 1 << 2
PM_A_REQ_RAM = 1 << 3
PM_A_REQ_STORAGE = 1 << 4

# pm_opt_present
PM_O_COUNT = 1 << 0
PM_O_MODEL = 1 << 1
PM_O_MEM = 1 << 2
PM_O_MEM_MIN = 1 << 3
PM_O_MEM_MAX = 1 << 4
PM_O_TOT_MIN = 1 << 5
PM_O_TOT_MAX = 1 << 6

PM_CFG_TIMING = 1 << 0

PM_MODE_FIRST_FIT, PM_MODE_PROXIMITY, PM_MODE_AUCTION, PM_MODE_PROXIMITY_MERGE = 0, 1, 2, 3
PM_PATH_MATERIALIZED, PM_PATH_FUSED, PM_NO_ASK_STATS = 0, 1 << 8, 1 << 9
PM_INCREMENTAL = 1 << 10   # re-evaluate only the worker rows written since the stored evaluation (prime_match.h)
PM_AUCTION_WARM = 1 << 11  # PM_MODE_AUCTION: start from the last auction pass's prices and assignment (prime_match.h)
PM_AUCTION_REVERSE = 1 << 12  # PM_MODE_AUCTION: end every eps phase with reverse rounds (prime_match.h)
PM_AUCTION_REPAIR = 1 << 13  # with PM_AUCTION_WARM: keep the stored prices, raise the changed rows, end with reverse rounds

PM_BUF_WORKER_FIRST_ASK, PM_BUF_ASK_BEST, PM_BUF_ASK_COUNT, PM_BUF_COST_TILE = 0, 1, 2, 3

WORKER_A = np.dtype([("gpu_count", "<u4"), ("gpu_mem_mb", "<u4"), ("model_id", "<u4"), ("flags", "<u4")])
WORKER_B = np.dtype([("cpu_cores", "<u4"), ("ram_mb", "<u4"), ("storage_gb", "<u4"), ("ext_ask_price", "<u4")])
ASK = np.dtype([
    ("flags", "<u4"), ("n_opts", "<u4"), ("opt_off", "<u4"), ("cpu_cores", "<u4"),
    ("ram_mb", "<u4"), ("storage_gb", "<u4"), ("min_group_size", "<u4"), ("max_group_size", "<u4"),
])
GPU_OPT = np.dtype([
    ("present", "<u4"), ("count", "<u4"), ("memory_mb", "<u4"), ("memory_mb_min", "<u4"),
    ("memory_mb_max", "<u4"), ("total_memory_min", "<u4"), ("total_memory_max", "<u4"), ("pattern_id", "<u4"),
])
assert WORKER_A.itemsize == 16 and WORKER_B.itemsize == 16 and ASK.itemsize == 32 and GPU_OPT.itemsize == 32


class PmAsk(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ASK.names]


class PmGpuOpt(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in GPU_OPT.names]


class PmCfg(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32), ("device", C.c_int32), ("flags", C.c_uint32), ("reserved0", C.c_uint32),
        ("cost_tile_bytes", C.c_uint64), ("shard_first", C.c_uint32), ("shard_count", C.c_uint32),
        ("stream", C.c_void_p),
    ]


class PmStats(C.Structure):
    _fields_ = [
        ("evals", C.c_uint64), ("cost_bytes_written", C.c_uint64), ("cost_bytes_read", C.c_uint64),
        ("n_tiles", C.c_uint32), ("n_launches", C.c_uint32), ("n_bumped", C.c_uint32), ("n_rounds", C.c_uint32),
        ("ms_build", C.c_float), ("ms_argmin", C.c_float), ("ms_fused", C.c_float), ("ms_resolve", C.c_float),
        ("ms_total", C.c_float), ("n_build_launches", C.c_uint32), ("n_argmin_launches", C.c_uint32),
        ("n_fused_launches", C.c_uint32), ("ms_exchange", C.c_float), ("exchange_bytes", C.c_uint64),
    ]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class PmAuctionCert(C.Structure):
    """pm_auction_cert: 128-bit quantities as (signed high, low) 64-bit halves."""
    _fields_ = [
        ("cost_hi", C.c_int64), ("cost_lo", C.c_uint64), ("bound_hi", C.c_int64), ("bound_lo", C.c_uint64),
        ("gap_hi", C.c_int64), ("gap_lo", C.c_uint64), ("n_held", C.c_uint32), ("n_bad_holds", C.c_uint32),
        ("n_shared", C.c_uint32), ("n_priced_unowned", C.c_uint32), ("n_slack_over", C.c_uint32),
        ("reserved", C.c_uint32), ("max_slack", C.c_int64), ("priced_unowned_lo", C.c_uint64),
        ("priced_unowned_hi", C.c_uint64), ("evals", C.c_uint64),
    ]


class PmAuctionRestoreReport(C.Structure):
    """pm_auction_restore_report."""
    _fields_ = [
        ("n_held", C.c_uint32), ("n_dropped_bad", C.c_uint32), ("n_dropped_shared", C.c_uint32),
        ("n_dropped_slack", C.c_uint32), ("evals", C.c_uint64),
    ]


class PmResult(C.Structure):
    _fields_ = [
        ("n_workers", C.c_uint32), ("n_asks", C.c_uint32), ("n_groups", C.c_uint32), ("n_members", C.c_uint32),
        ("worker_group", C.POINTER(C.c_uint32)), ("worker_ask", C.POINTER(C.c_uint32)),
        ("group_ask", C.POINTER(C.c_uint32)), ("group_off", C.POINTER(C.c_uint32)),
        ("group_members", C.POINTER(C.c_uint32)), ("ask_best", C.POINTER(C.c_int64)),
        ("ask_count", C.POINTER(C.c_uint32)), ("stats", PmStats),
    ]


# every symbol include/prime_match.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "pm_abi_version",
    "pm_interner_create", "pm_interner_destroy", "pm_intern_model", "pm_intern_pattern", "pm_interner_table",
    "pm_parse_requirements", "pm_sort_configs", "pm_address_canonical",
    "pm_create", "pm_destroy", "pm_last_error", "pm_alloc_pinned", "pm_free_pinned",
    "pm_set_asks", "pm_set_ask_enabled", "pm_update_asks", "pm_resize_asks", "pm_remove_asks", "pm_insert_asks", "pm_set_model_table", "pm_set_worker_count", "pm_upsert_workers",
    "pm_set_worker_locations", "pm_set_worker_addr_rank", "pm_set_flags",
    "pm_set_ask_price_caps", "pm_set_auction_params", "pm_set_worker_reputation", "pm_set_ask_min_reputation",
    "pm_set_ask_demand",
    "pm_auction_state", "pm_auction_reverse_stats", "pm_auction_certificate", "pm_auction_assignment", "pm_auction_restore",
    "pm_auction_slot_assignment", "pm_auction_restore_slots",
    "pm_match", "pm_fetch_result", "pm_get_stats", "pm_build_cost_tile",
    "pm_match_local", "pm_match_finish", "pm_device_buffer", "pm_stream_sync", "pm_set_shard",
    "pm_resize_workers", "pm_update_workers", "pm_remove_workers", "pm_insert_workers", "pm_table_version", "pm_create_sibling",
    "pm_comm_unique_id", "pm_comm_create", "pm_comm_destroy", "pm_attach_comm",
    "pm_multi_create", "pm_multi_destroy", "pm_multi_size", "pm_multi_engine", "pm_multi_last_error",
    "pm_multi_set_asks", "pm_multi_set_ask_enabled", "pm_multi_update_asks", "pm_multi_resize_asks", "pm_multi_remove_asks", "pm_multi_insert_asks", "pm_multi_set_model_table", "pm_multi_set_worker_count", "pm_multi_upsert_workers",
    "pm_multi_set_worker_locations", "pm_multi_set_worker_addr_rank", "pm_multi_set_flags",
    "pm_multi_resize_workers", "pm_multi_update_workers", "pm_multi_remove_workers", "pm_multi_insert_workers", "pm_multi_sync", "pm_multi_table_version",
    "pm_multi_match", "pm_multi_fetch_result",
    "pm_plugin_create", "pm_plugin_create_multi", "pm_plugin_destroy", "pm_plugin_last_error", "pm_plugin_add_config", "pm_plugin_seal_configs",
    "pm_plugin_enable_configuration", "pm_plugin_upsert_node", "pm_plugin_set_node_status", "pm_plugin_sync_discovery", "pm_plugin_sync_discovery_json", "pm_plugin_get_node", "pm_plugin_add_task",
    "pm_plugin_delete_task", "pm_plugin_record_upload", "pm_plugin_try_form_new_groups", "pm_plugin_try_merge_solo_groups", "pm_plugin_get_node_group", "pm_plugin_get_all_groups", "pm_plugin_get_group_by_id", "pm_plugin_handle_group_not_found", "pm_plugin_restore_group", "pm_plugin_export_tables", "pm_plugin_redis_writeback",
    "pm_scheduler_get_task_for_node",
]


class PmPluginPolicy(C.Structure):
    _fields_ = [("task_switching_enabled", C.c_uint8), ("prefer_larger_groups", C.c_uint8),
                ("proximity_enabled", C.c_uint8), ("canonical_addresses", C.c_uint8)]


class PmKv(C.Structure):
    _fields_ = [("key", C.c_char_p), ("value", C.c_char_p)]


class PmTaskDesc(C.Structure):
    _fields_ = [
        ("id", C.c_char_p), ("name", C.c_char_p), ("image", C.c_char_p), ("created_at", C.c_int64),
        ("env_vars", C.POINTER(PmKv)), ("n_env_vars", C.c_uint32), ("has_env_vars", C.c_int32),
        ("cmd", C.POINTER(C.c_char_p)), ("n_cmd", C.c_uint32), ("has_cmd", C.c_int32),
        ("volume_mounts", C.POINTER(PmKv)), ("n_volume_mounts", C.c_uint32), ("has_volume_mounts", C.c_int32),
        ("scheduling", C.c_int32),
        ("allowed_topologies", C.POINTER(C.c_char_p)), ("n_allowed_topologies", C.c_uint32),
    ]


class PmNodeDesc(C.Structure):
    _fields_ = [
        ("address", C.c_char_p), ("status", C.c_uint32), ("p2p_id", C.c_char_p), ("spec_flags", C.c_uint32),
        ("gpu_count", C.c_uint32), ("gpu_mem_mb", C.c_uint32), ("gpu_model", C.c_char_p),
        ("cpu_cores", C.c_uint32), ("ram_mb", C.c_uint32), ("storage_gb", C.c_uint32),
        ("has_location", C.c_int32), ("lat", C.c_double), ("lon", C.c_double),
        ("ip_address", C.c_char_p), ("port", C.c_uint16), ("reserved", C.c_uint16),
        ("last_status_change_ms", C.c_int64),
    ]


class PmDiscoveryNode(C.Structure):
    _fields_ = [
        ("node", PmNodeDesc), ("ip_address", C.c_char_p), ("port", C.c_uint16),
        ("is_validated", C.c_uint8), ("is_active", C.c_uint8), ("is_provider_whitelisted", C.c_uint8),
        ("is_blacklisted", C.c_uint8), ("has_latest_balance", C.c_uint8), ("latest_balance_is_zero", C.c_uint8),
        ("last_updated_ms", C.c_int64),
    ]
