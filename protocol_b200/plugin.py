"""Python face of the host mirror (csrc/pm_plugin.cpp): same names and argument meaning as the
reference's NodeGroupsPlugin / Scheduler for this path, so tests read like
crates/orchestrator/src/plugins/node_groups/tests.rs and scheduler/mod.rs tests."""
from __future__ import annotations

import ctypes as C
import json
import uuid
from dataclasses import dataclass, field

from . import abi
from ._lib import PrimeMatchError, load
from .engine import MultiEngine


class NodeStatus:  # crates/orchestrator/src/models/node.rs:74-85
    Discovered, WaitingForHeartbeat, Healthy, Unhealthy, Dead, Ejected, Banned, LowBalance = range(8)


@dataclass
class GpuSpecs:  # shared/src/models/node.rs:72-78
    count: int | None = None
    model: str | None = None
    memory_mb: int | None = None


@dataclass
class ComputeSpecs:  # node.rs:25-35
    gpu: GpuSpecs | None = None
    cpu_cores: int | None = None
    cpu_present: bool | None = None
    ram_mb: int | None = None
    storage_gb: int | None = None


@dataclass
class NodeGroupConfiguration:  # node_groups/mod.rs:30-37
    name: str
    min_group_size: int
    max_group_size: int
    compute_requirements: str | None = None


@dataclass
class Task:  # shared/src/models/task.rs:162-184 (fields on the path)
    name: str = ""
    image: str = ""
    id: str = field(default_factory=lambda: str(uuid.uuid4()))
    env_vars: dict | None = None
    cmd: list | None = None
    created_at: int = 0
    volume_mounts: list | None = None          # [(host_path, container_path)]
    allowed_topologies: list | None = None     # scheduling_config.plugins["node_groups"]["allowed_topologies"]
    scheduling: int | None = None              # override: 0 None, 1 no node_groups entry, 2 no allowed_topologies


@dataclass
class OrchestratorNode:  # orchestrator/src/models/node.rs:10-37 (fields on the path)
    address: str
    status: int = NodeStatus.Healthy
    p2p_id: str | None = "test_p2p_id"
    compute_specs: ComputeSpecs | None = None
    location: tuple | None = None
    ip_address: str = ""
    port: int = 0
    last_status_change_ms: int | None = None


@dataclass
class DiscoveryNode:  # shared/src/models/node.rs:552-570 (fields the monitor reads)
    id: str
    ip_address: str = "127.0.0.1"
    port: int = 8080
    compute_specs: ComputeSpecs | None = None
    is_validated: bool = False
    is_active: bool = False
    is_provider_whitelisted: bool = False
    is_blacklisted: bool = False
    last_updated_ms: int | None = None
    location: tuple | None = None
    latest_balance: int | None = None


def _b(s):
    return s.encode() if s is not None else None


class NodeGroupsPlugin:
    """NodeGroupsPlugin::new_with_policy (mod.rs:129-175).  `engine` is an Engine, a MultiEngine (the formation pass
    then runs on all of its GPUs) or None (no group formation).  Close the plugin before its engine."""

    def __init__(self, configuration_templates, engine=None, task_switching_enabled=True,
                 prefer_larger_groups=True, proximity_enabled=True, canonical_addresses=False):
        self._lib = load()
        pol = abi.PmPluginPolicy(int(task_switching_enabled), int(prefer_larger_groups), int(proximity_enabled), int(canonical_addresses))
        h = C.c_void_p()
        self._engine = engine
        if isinstance(engine, MultiEngine):
            create, name = self._lib.pm_plugin_create_multi, "pm_plugin_create_multi"
        else:
            create, name = self._lib.pm_plugin_create, "pm_plugin_create"
        rc = create(engine._h if engine is not None else None, C.byref(pol), C.byref(h))
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, name)
        self._h = h
        for c in configuration_templates:
            self._check(self._lib.pm_plugin_add_config(self._h, c.name.encode(), c.min_group_size, c.max_group_size,
                                                       _b(c.compute_requirements)))
        self._check(self._lib.pm_plugin_seal_configs(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.pm_plugin_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != abi.PM_OK:
            raise PrimeMatchError(rc, (self._lib.pm_plugin_last_error(self._h) or b"").decode())

    def _json(self, fn, *args, cap=1 << 20):
        buf = C.create_string_buffer(cap)
        self._check(fn(self._h, *args, buf, cap))
        return json.loads(buf.value.decode())

    # ---- stores ------------------------------------------------------------
    @staticmethod
    def _fill_specs(d, s, location):
        f = 0
        if s is not None:
            f |= abi.PM_W_HAS_SPECS
            if s.gpu is not None:
                f |= abi.PM_W_HAS_GPU
                if s.gpu.count is not None:
                    f |= abi.PM_W_HAS_GPU_COUNT
                    d.gpu_count = s.gpu.count
                if s.gpu.model is not None:
                    f |= abi.PM_W_HAS_GPU_MODEL
                    d.gpu_model = s.gpu.model.encode()
                if s.gpu.memory_mb is not None:
                    f |= abi.PM_W_HAS_GPU_MEM
                    d.gpu_mem_mb = s.gpu.memory_mb
            cpu_present = s.cpu_present if s.cpu_present is not None else s.cpu_cores is not None
            if cpu_present:
                f |= abi.PM_W_HAS_CPU
                if s.cpu_cores is not None:
                    f |= abi.PM_W_HAS_CPU_CORES
                    d.cpu_cores = s.cpu_cores
            if s.ram_mb is not None:
                f |= abi.PM_W_HAS_RAM
                d.ram_mb = s.ram_mb
            if s.storage_gb is not None:
                f |= abi.PM_W_HAS_STORAGE
                d.storage_gb = s.storage_gb
        d.spec_flags = f
        if location is not None:
            d.has_location = 1
            d.lat, d.lon = location

    def add_node(self, node: OrchestratorNode):
        d = abi.PmNodeDesc()
        d.address = node.address.encode()
        d.status = node.status
        d.p2p_id = _b(node.p2p_id)
        d.ip_address = node.ip_address.encode()
        d.port = node.port
        d.last_status_change_ms = node.last_status_change_ms or 0
        self._fill_specs(d, node.compute_specs, node.location)
        self._check(self._lib.pm_plugin_upsert_node(self._h, C.byref(d)))

    def sync_discovery(self, discovery_nodes, now_ms: int, max_healthy_nodes_with_same_endpoint: int = 1) -> int:
        """DiscoveryMonitor::get_nodes (discovery/monitor.rs:422-435) for one fetch."""
        arr = (abi.PmDiscoveryNode * max(len(discovery_nodes), 1))()
        for i, dn in enumerate(discovery_nodes):
            d = arr[i]
            d.node.address = dn.id.encode()
            self._fill_specs(d.node, dn.compute_specs, dn.location)
            d.ip_address = dn.ip_address.encode()
            d.port = dn.port
            d.is_validated, d.is_active = int(dn.is_validated), int(dn.is_active)
            d.is_provider_whitelisted, d.is_blacklisted = int(dn.is_provider_whitelisted), int(dn.is_blacklisted)
            d.has_latest_balance = int(dn.latest_balance is not None)
            d.latest_balance_is_zero = int(dn.latest_balance == 0)
            d.last_updated_ms = -1 if dn.last_updated_ms is None else dn.last_updated_ms
        n_new = C.c_uint32()
        self._check(self._lib.pm_plugin_sync_discovery(self._h, arr, len(discovery_nodes), now_ms,
                                                       max_healthy_nodes_with_same_endpoint, C.byref(n_new)))
        return n_new.value

    def sync_discovery_json(self, body: str, now_ms: int, max_healthy_nodes_with_same_endpoint: int = 1) -> int:
        """The body of `GET {discovery}/api/pool/{id}` (discovery/monitor.rs:109-193)."""
        raw = body.encode()
        n_new = C.c_uint32()
        self._check(self._lib.pm_plugin_sync_discovery_json(self._h, raw, len(raw), now_ms,
                                                            max_healthy_nodes_with_same_endpoint, C.byref(n_new)))
        return n_new.value

    def get_node(self, address: str):
        return self._json(self._lib.pm_plugin_get_node, address.encode())

    def update_node_status(self, address: str, status: int):
        """NodeStore::update_node_status followed by StatusUpdatePlugin::handle_status_change."""
        self._check(self._lib.pm_plugin_set_node_status(self._h, address.encode(), status))

    def add_task(self, task: Task):
        d = abi.PmTaskDesc()
        keep = []
        d.id, d.name, d.image, d.created_at = task.id.encode(), task.name.encode(), task.image.encode(), task.created_at
        if task.env_vars is not None:
            arr = (abi.PmKv * max(len(task.env_vars), 1))()
            for i, (k, v) in enumerate(task.env_vars.items()):
                arr[i].key, arr[i].value = k.encode(), v.encode()
            d.env_vars, d.n_env_vars, d.has_env_vars = arr, len(task.env_vars), 1
            keep.append(arr)
        if task.cmd is not None:
            arr = (C.c_char_p * max(len(task.cmd), 1))(*[c.encode() for c in task.cmd])
            d.cmd, d.n_cmd, d.has_cmd = arr, len(task.cmd), 1
            keep.append(arr)
        if task.volume_mounts is not None:
            arr = (abi.PmKv * max(len(task.volume_mounts), 1))()
            for i, (h, c) in enumerate(task.volume_mounts):
                arr[i].key, arr[i].value = h.encode(), c.encode()
            d.volume_mounts, d.n_volume_mounts, d.has_volume_mounts = arr, len(task.volume_mounts), 1
            keep.append(arr)
        if task.allowed_topologies is not None:
            arr = (C.c_char_p * max(len(task.allowed_topologies), 1))(*[t.encode() for t in task.allowed_topologies])
            d.allowed_topologies, d.n_allowed_topologies, d.scheduling = arr, len(task.allowed_topologies), 3
            keep.append(arr)
        else:
            d.scheduling = task.scheduling or 0
        self._check(self._lib.pm_plugin_add_task(self._h, C.byref(d)))

    def delete_task(self, task_id: str):
        self._check(self._lib.pm_plugin_delete_task(self._h, task_id.encode()))

    def record_upload(self, address: str, group_id: str, file_name: str):
        self._check(self._lib.pm_plugin_record_upload(self._h, address.encode(), group_id.encode(), file_name.encode()))

    def enable_configuration(self, name: str):
        self._check(self._lib.pm_plugin_enable_configuration(self._h, name.encode(), 1))

    def disable_configuration(self, name: str):
        self._check(self._lib.pm_plugin_enable_configuration(self._h, name.encode(), 0))

    # ---- the path ------------------------------------------------------------
    def try_form_new_groups(self) -> int:
        n = C.c_uint32()
        self._check(self._lib.pm_plugin_try_form_new_groups(self._h, C.byref(n)))
        return n.value

    def try_merge_solo_groups(self) -> int:
        n = C.c_uint32()
        self._check(self._lib.pm_plugin_try_merge_solo_groups(self._h, C.byref(n)))
        return n.value

    def get_node_group(self, address: str):
        return self._json(self._lib.pm_plugin_get_node_group, address.encode())

    def get_all_groups(self):
        return self._json(self._lib.pm_plugin_get_all_groups)

    def get_group_by_id(self, group_id: str):
        """mod.rs:1046-1055."""
        return self._json(self._lib.pm_plugin_get_group_by_id, group_id.encode())

    def validate_group_exists(self, group_id: str) -> bool:
        """mod.rs:1067-1070."""
        return self.get_group_by_id(group_id) is not None

    def handle_group_not_found(self, group_id: str, task_id: str) -> bool:
        """mod.rs:1073-1119: True when an idle group took the orphaned task."""
        n = C.c_uint32()
        self._check(self._lib.pm_plugin_handle_group_not_found(self._h, group_id.encode(), task_id.encode(), C.byref(n)))
        return bool(n.value)

    def export_tables(self):
        """The SoA tables a management pass uploads: dict(a, b, lat, lon, addr_rank) of numpy arrays, canonical row order."""
        import numpy as np

        n = C.c_uint32()
        self._check(self._lib.pm_plugin_export_tables(self._h, None, None, None, None, None, 0, C.byref(n)))
        w = n.value
        a = np.zeros(w, dtype=abi.WORKER_A)
        b = np.zeros(w, dtype=abi.WORKER_B)
        lat, lon, rank = np.zeros(w), np.zeros(w), np.zeros(w, dtype=np.uint32)
        self._check(self._lib.pm_plugin_export_tables(self._h, a.ctypes.data, b.ctypes.data, lat.ctypes.data, lon.ctypes.data,
                                                      rank.ctypes.data, w, C.byref(n)))
        return dict(a=a, b=b, lat=lat, lon=lon, addr_rank=rank)

    def restore_group(self, group_id: str, configuration_name: str, nodes, task_id: str | None = None,
                      created_at_ms: int = -1):
        """A NodeGroup read back from Redis at start-up (node_group:<id>, group_task:<id>)."""
        arr = (C.c_char_p * max(len(nodes), 1))(*[n.encode() for n in nodes])
        self._check(self._lib.pm_plugin_restore_group(self._h, group_id.encode(), configuration_name.encode(), arr, len(nodes),
                                                      _b(task_id), created_at_ms))

    def redis_writeback(self):
        """[[cmd, key, ...], ...] in the reference's key formats (mod.rs:25-28, 299-322)."""
        return self._json(self._lib.pm_plugin_redis_writeback, cap=1 << 24)


class Scheduler:
    """Scheduler::new(store, plugins) + get_task_for_node (scheduler/mod.rs:14-74).  The plugin chain is
    [NodeGroupsPlugin] when the plugin has configurations, else the default [NewestTaskPlugin]."""

    def __init__(self, plugin: NodeGroupsPlugin):
        self.plugin = plugin

    def get_task_for_node(self, address: str):
        r = self.plugin._json(self.plugin._lib.pm_scheduler_get_task_for_node, address.encode())
        return r["current_task"]
