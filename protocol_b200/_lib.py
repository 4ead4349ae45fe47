"""ctypes loader for libprime_match.so (the C ABI of include/prime_match.h).

The product has no CPU fallback: if the shared library is missing this raises,
and if no H100 is visible pm_create returns PM_E_NO_DEVICE which Engine turns
into an exception.
"""
from __future__ import annotations

import ctypes as C
import os

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libprime_match.so")
_lib = None


class PrimeMatchError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"prime_match status {status}: {message}")
        self.status = status


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: run `python -m protocol_b200.build` (needs nvcc). "
            "There is no CPU fallback for the matching engine."
        )
    lib = C.CDLL(LIB_PATH)
    u32, i32, vp, cp, sz = C.c_uint32, C.c_int, C.c_void_p, C.c_char_p, C.c_size_t
    P = C.POINTER
    sig = {
        "pm_abi_version": (u32, []),
        "pm_interner_create": (vp, []),
        "pm_interner_destroy": (None, [vp]),
        "pm_intern_model": (u32, [vp, cp]),
        "pm_intern_pattern": (u32, [vp, cp]),
        "pm_interner_table": (i32, [vp, P(P(u32)), P(u32), P(u32), P(u32)]),
        "pm_parse_requirements": (i32, [cp, vp, P(abi.PmAsk), P(abi.PmGpuOpt), u32, P(u32), C.c_char_p, sz]),
        "pm_sort_configs": (i32, [vp, vp, u32, vp]),
        "pm_address_canonical": (i32, [C.c_char_p, vp]),
        "pm_create": (i32, [P(abi.PmCfg), P(vp)]),
        "pm_destroy": (None, [vp]),
        "pm_last_error": (cp, [vp]),
        "pm_alloc_pinned": (vp, [sz]),
        "pm_free_pinned": (None, [vp]),
        "pm_set_asks": (i32, [vp, vp, u32, vp, u32]),
        "pm_set_ask_enabled": (i32, [vp, vp, vp, u32]),
        "pm_update_asks": (i32, [vp, vp, vp, u32, vp, u32]),
        "pm_resize_asks": (i32, [vp, u32, vp, vp, u32]),
        "pm_remove_asks": (i32, [vp, vp, u32]),
        "pm_insert_asks": (i32, [vp, vp, vp, u32, vp, u32]),
        "pm_set_model_table": (i32, [vp, vp, u32, u32, u32]),
        "pm_set_worker_count": (i32, [vp, u32]),
        "pm_upsert_workers": (i32, [vp, vp, vp, u32, u32]),
        "pm_set_worker_locations": (i32, [vp, vp, vp, u32, u32]),
        "pm_set_worker_addr_rank": (i32, [vp, vp, u32, u32]),
        "pm_set_flags": (i32, [vp, vp, vp, u32]),
        "pm_set_ask_price_caps": (i32, [vp, vp, u32]),
        "pm_set_worker_reputation": (i32, [vp, vp, u32, u32]),
        "pm_set_ask_min_reputation": (i32, [vp, vp, u32]),
        "pm_set_ask_demand": (i32, [vp, vp, u32]),
        "pm_set_auction_params": (i32, [vp, C.c_uint64, C.c_uint64, u32]),
        "pm_auction_state": (i32, [vp, vp, P(u32), P(u32)]),
        "pm_auction_reverse_stats": (i32, [vp, P(u32), P(u32), P(C.c_uint64)]),
        "pm_auction_certificate": (i32, [vp, P(abi.PmAuctionCert), vp]),
        "pm_auction_assignment": (i32, [vp, vp]),
        "pm_auction_restore": (i32, [vp, vp, u32, vp, u32, P(abi.PmAuctionRestoreReport)]),
        "pm_auction_slot_assignment": (i32, [vp, vp, P(u32)]),
        "pm_auction_restore_slots": (i32, [vp, vp, u32, vp, u32, P(abi.PmAuctionRestoreReport)]),
        "pm_match": (i32, [vp, u32]),
        "pm_fetch_result": (i32, [vp, P(abi.PmResult)]),
        "pm_get_stats": (i32, [vp, P(abi.PmStats)]),
        "pm_build_cost_tile": (i32, [vp, u32, u32, vp]),
        "pm_match_local": (i32, [vp, u32]),
        "pm_match_finish": (i32, [vp, u32]),
        "pm_device_buffer": (i32, [vp, u32, P(vp), P(sz)]),
        "pm_stream_sync": (i32, [vp]),
        "pm_set_shard": (i32, [vp, u32, u32]),
        "pm_resize_workers": (i32, [vp, u32]),
        "pm_update_workers": (i32, [vp, vp, vp, vp, vp, vp, u32]),
        "pm_remove_workers": (i32, [vp, vp, u32]),
        "pm_insert_workers": (i32, [vp, vp, vp, vp, vp, vp, u32]),
        "pm_table_version": (C.c_uint64, [vp]),
        "pm_create_sibling": (i32, [vp, P(vp)]),
        "pm_comm_unique_id": (i32, [vp]),
        "pm_comm_create": (i32, [vp, u32, u32, C.c_int32, P(vp)]),
        "pm_comm_destroy": (None, [vp]),
        "pm_attach_comm": (i32, [vp, vp]),
        "pm_multi_create": (i32, [P(abi.PmCfg), P(C.c_int32), u32, P(vp)]),
        "pm_multi_destroy": (None, [vp]),
        "pm_multi_size": (u32, [vp]),
        "pm_multi_engine": (vp, [vp, u32]),
        "pm_multi_last_error": (cp, [vp]),
        "pm_multi_set_asks": (i32, [vp, vp, u32, vp, u32]),
        "pm_multi_set_ask_enabled": (i32, [vp, vp, vp, u32]),
        "pm_multi_update_asks": (i32, [vp, vp, vp, u32, vp, u32]),
        "pm_multi_resize_asks": (i32, [vp, u32, vp, vp, u32]),
        "pm_multi_remove_asks": (i32, [vp, vp, u32]),
        "pm_multi_insert_asks": (i32, [vp, vp, vp, u32, vp, u32]),
        "pm_multi_set_model_table": (i32, [vp, vp, u32, u32, u32]),
        "pm_multi_set_worker_count": (i32, [vp, u32]),
        "pm_multi_upsert_workers": (i32, [vp, vp, vp, u32, u32]),
        "pm_multi_set_worker_locations": (i32, [vp, vp, vp, u32, u32]),
        "pm_multi_set_worker_addr_rank": (i32, [vp, vp, u32, u32]),
        "pm_multi_set_flags": (i32, [vp, vp, vp, u32]),
        "pm_multi_resize_workers": (i32, [vp, u32]),
        "pm_multi_update_workers": (i32, [vp, vp, vp, vp, vp, vp, u32]),
        "pm_multi_remove_workers": (i32, [vp, vp, u32]),
        "pm_multi_insert_workers": (i32, [vp, vp, vp, vp, vp, vp, u32]),
        "pm_multi_sync": (i32, [vp]),
        "pm_multi_table_version": (C.c_uint64, [vp]),
        "pm_multi_match": (i32, [vp, u32]),
        "pm_multi_fetch_result": (i32, [vp, P(abi.PmResult)]),
        "pm_plugin_create": (i32, [vp, P(abi.PmPluginPolicy), P(vp)]),
        "pm_plugin_create_multi": (i32, [vp, P(abi.PmPluginPolicy), P(vp)]),
        "pm_plugin_destroy": (None, [vp]),
        "pm_plugin_last_error": (cp, [vp]),
        "pm_plugin_add_config": (i32, [vp, cp, u32, u32, cp]),
        "pm_plugin_seal_configs": (i32, [vp]),
        "pm_plugin_enable_configuration": (i32, [vp, cp, i32]),
        "pm_plugin_upsert_node": (i32, [vp, P(abi.PmNodeDesc)]),
        "pm_plugin_set_node_status": (i32, [vp, cp, u32]),
        "pm_plugin_sync_discovery": (i32, [vp, vp, u32, C.c_int64, u32, P(u32)]),
        "pm_plugin_sync_discovery_json": (i32, [vp, cp, sz, C.c_int64, u32, P(u32)]),
        "pm_plugin_get_node": (i32, [vp, cp, C.c_char_p, sz]),
        "pm_plugin_add_task": (i32, [vp, P(abi.PmTaskDesc)]),
        "pm_plugin_delete_task": (i32, [vp, cp]),
        "pm_plugin_record_upload": (i32, [vp, cp, cp, cp]),
        "pm_plugin_try_form_new_groups": (i32, [vp, P(u32)]),
        "pm_plugin_try_merge_solo_groups": (i32, [vp, P(u32)]),
        "pm_plugin_get_node_group": (i32, [vp, cp, C.c_char_p, sz]),
        "pm_plugin_get_all_groups": (i32, [vp, C.c_char_p, sz]),
        "pm_plugin_get_group_by_id": (i32, [vp, cp, C.c_char_p, sz]),
        "pm_plugin_handle_group_not_found": (i32, [vp, cp, cp, P(u32)]),
        "pm_plugin_export_tables": (i32, [vp, vp, vp, vp, vp, vp, u32, P(u32)]),
        "pm_plugin_restore_group": (i32, [vp, cp, cp, P(C.c_char_p), u32, cp, C.c_int64]),
        "pm_plugin_redis_writeback": (i32, [vp, C.c_char_p, sz]),
        "pm_scheduler_get_task_for_node": (i32, [vp, cp, C.c_char_p, sz]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
