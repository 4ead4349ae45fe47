// pm_plugin.cpp — host-side mirror of the reference's plugin interface for this path,
// on top of the C-ABI engine (no GPU code here, and no CPU evaluation of the
// feasibility predicate: group formation always goes through pm_match).
//
// Mirrors (names, argument meaning, error behaviour):
//   NodeGroupsPlugin::new_with_policy      crates/orchestrator/src/plugins/node_groups/mod.rs:129-175
//   get_available_configurations           mod.rs:399-418
//   try_form_new_groups                    mod.rs:478-628     (-> pm_match)
//   get_node_group / get_idx_in_group      mod.rs:324-337, 424-434
//   get_current_group_task / assign_task_to_group   mod.rs:436-476
//   dissolve_group / handle_status_change  mod.rs:1423-1487, status_update_impl.rs:8-39
//   on_task_created / on_task_deleted      mod.rs:1224-1325
//   NodeGroupsPlugin::filter_tasks         node_groups/scheduler_impl.rs:11-210
//   NewestTaskPlugin::filter_tasks         plugins/newest_task/mod.rs:8-19
//   Scheduler::get_task_for_node           scheduler/mod.rs:26-74
//   TaskStore::get_all_tasks ordering      store/domains/task_store.rs:57-82
//   NodeStore::get_nodes ordering          store/domains/node_store.rs:163-209
// Redis is replaced by in-process tables (the engine's tables are "a cache of
// Redis", SURVEY 5); the reference's random choices follow the determinisation
// rules of SURVEY 8c (newest applicable task; group id = running counter).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <map>
#include <mutex>
#include <set>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/prime_match.h"
#include "pm_guard.hpp"
#include "pm_json.hpp"

namespace {

enum NodeStatus : uint32_t {  // crates/orchestrator/src/models/node.rs:74-85
  kDiscovered = 0, kWaitingForHeartbeat = 1, kHealthy = 2, kUnhealthy = 3,
  kDead = 4, kEjected = 5, kBanned = 6, kLowBalance = 7
};

int status_class(uint32_t st) {  // node_store.rs:195-206
  if (st == kHealthy) return 0;
  if (st == kDiscovered) return 1;
  if (st == kDead) return 3;
  return 2;
}

struct Config {
  std::string name;
  uint32_t min_group_size = 0, max_group_size = 0;
  bool has_requirements = false;
  pm_ask ask{};
  std::vector<pm_gpu_opt> opts;
};

struct TaskRec {
  std::string id, name, image;
  int64_t created_at = 0;
  bool has_env = false, has_cmd = false, has_mounts = false;
  std::vector<std::pair<std::string, std::string>> env, mounts;
  std::vector<std::string> cmd;
  int scheduling = 0;  // pm_task_desc::scheduling
  std::vector<std::string> topologies;
};

struct NodeRec {
  std::string address;
  std::string ip_address;
  uint16_t port = 0;
  int64_t last_status_change_ms = -1;  // Option<DateTime<Utc>>
  int64_t first_seen_ms = -1;
  uint32_t status = kDiscovered;
  bool has_p2p = false;
  std::string p2p_id;
  pm_worker_a a{};
  pm_worker_b b{};
  bool has_loc = false;
  double lat = 0, lon = 0;
  uint64_t sync_gen = 0;               // the discovery fetch that last touched the node (de-dup by id within a fetch)
  bool grouped = false;                // mirrors node_to_group.count(address): read by the table snapshot
  bool dirty = false;                  // changed since the engine's resident copy of its row was written
};

struct Group {  // NodeGroup, mod.rs:63-69
  std::string id;
  std::vector<std::string> nodes;  // BTreeSet<String> order
  std::string configuration_name;
  int64_t created_at_ms = 0;       // chrono::Utc::now() at creation (mod.rs:575)
};

std::string replace_all(std::string s, const std::string& from, const std::string& to) {
  if (from.empty()) return s;
  size_t pos = 0;
  while ((pos = s.find(from, pos)) != std::string::npos) {
    s.replace(pos, from.size(), to);
    pos += to.size();
  }
  return s;
}

void json_str(std::string& out, const std::string& s) {
  out += '"';
  for (unsigned char c : s) {
    switch (c) {
      case '"': out += "\\\""; break;
      case '\\': out += "\\\\"; break;
      case '\n': out += "\\n"; break;
      case '\r': out += "\\r"; break;
      case '\t': out += "\\t"; break;
      default:
        if (c < 0x20) {
          char b[8];
          std::snprintf(b, sizeof b, "\\u%04x", c);
          out += b;
        } else {
          out += char(c);
        }
    }
  }
  out += '"';
}

// the topology predicate of scheduler_impl.rs:44-59 == mod.rs:1138-1163
bool task_applicable(const TaskRec& t, const std::string& configuration_name) {
  if (t.scheduling != 3) return true;  // None / no node_groups plugin / no allowed_topologies
  return std::find(t.topologies.begin(), t.topologies.end(), configuration_name) != t.topologies.end();
}

// Where the formation pass runs: one engine, or a pm_multi (table calls reach every device, the pass is sharded).
struct Device {
  pm_engine* engine = nullptr;
  pm_multi* multi = nullptr;

  explicit operator bool() const { return engine || multi; }
  pm_engine* first() const { return multi ? pm_multi_engine(multi, 0) : engine; }   // home of the merge pass's sibling
  const char* last_error() const { return multi ? pm_multi_last_error(multi) : pm_last_error(engine); }
  uint64_t table_version() const { return multi ? pm_multi_table_version(multi) : pm_table_version(engine); }
  int set_asks(const pm_ask* a, uint32_t n, const pm_gpu_opt* o, uint32_t no) const {
    return multi ? pm_multi_set_asks(multi, a, n, o, no) : pm_set_asks(engine, a, n, o, no);
  }
  int set_ask_enabled(const uint32_t* idx, const uint8_t* on, uint32_t n) const {
    return multi ? pm_multi_set_ask_enabled(multi, idx, on, n) : pm_set_ask_enabled(engine, idx, on, n);
  }
  int set_model_table(const uint32_t* bits, uint32_t npat, uint32_t nmod, uint32_t words) const {
    return multi ? pm_multi_set_model_table(multi, bits, npat, nmod, words) : pm_set_model_table(engine, bits, npat, nmod, words);
  }
  int set_worker_count(uint32_t n) const { return multi ? pm_multi_set_worker_count(multi, n) : pm_set_worker_count(engine, n); }
  int resize_workers(uint32_t n) const { return multi ? pm_multi_resize_workers(multi, n) : pm_resize_workers(engine, n); }
  int update_workers(const uint32_t* idx, const pm_worker_a* a, const pm_worker_b* b, const double* lat, const double* lon,
                     uint32_t n) const {
    return multi ? pm_multi_update_workers(multi, idx, a, b, lat, lon, n) : pm_update_workers(engine, idx, a, b, lat, lon, n);
  }
  int set_worker_locations(const double* lat, const double* lon, uint32_t first_row, uint32_t n) const {
    return multi ? pm_multi_set_worker_locations(multi, lat, lon, first_row, n) : pm_set_worker_locations(engine, lat, lon, first_row, n);
  }
  int sync() const { return multi ? pm_multi_sync(multi) : pm_stream_sync(engine); }
  int match(uint32_t mode) const { return multi ? pm_multi_match(multi, mode) : pm_match(engine, mode); }
  int fetch_result(pm_result* r) const { return multi ? pm_multi_fetch_result(multi, r) : pm_fetch_result(engine, r); }
};

}  // namespace

struct pm_plugin {
  Device dev;   // not owned
  pm_plugin_policy policy{};
  pm_interner* interner = nullptr;
  std::string err;
  std::shared_mutex mu;  // guards the tables below: exclusive for every update, shared for the read-only heartbeat path
  std::mutex loop_mu;  // serialises management passes (the reference runs them in one tokio task)

  std::vector<Config> templates;  // sorted at seal (mod.rs:150-164)
  bool sealed = false;
  std::set<std::string> available;  // "available_node_group_configs"

  std::vector<NodeRec> nodes;  // insertion order stands in for SMEMBERS order
  std::unordered_map<std::string, size_t> node_index;

  std::vector<TaskRec> tasks;  // RPUSH order (task_store.rs:41)
  std::unordered_map<std::string, size_t> task_pos;   // id -> first position in `tasks` (a heartbeat resolves its claim in O(1))
  // heartbeat fast path (SURVEY 8f-2): the reference re-reads and re-filters every task on every
  // heartbeat (scheduler/mod.rs:27, scheduler_impl.rs:42-61: O(T*K) string compares); here the
  // task a fresh group of a configuration would claim is cached until the task list changes
  std::unordered_map<std::string, std::string> claim_cache;  // configuration name -> task id ("" = none)
  bool claim_cache_valid = false;
  bool newest_valid = false;   // NewestTaskPlugin's choice, valid until the task list changes
  size_t newest_pos = 0;
  const TaskRec* task_for_configuration(const std::string& configuration_name) {
    if (!claim_cache_valid) {
      claim_cache.clear();
      claim_cache_valid = true;
    }
    auto it = claim_cache.find(configuration_name);
    if (it == claim_cache.end()) {
      const TaskRec* chosen = nullptr;  // NewestTask rule over the desc-sorted list: last maximum
      for (const TaskRec* t : all_tasks())
        if (task_applicable(*t, configuration_name) && (!chosen || t->created_at >= chosen->created_at)) chosen = t;
      it = claim_cache.emplace(configuration_name, chosen ? chosen->id : std::string()).first;
    }
    return it->second.empty() ? nullptr : find_task(it->second);
  }

  std::map<std::string, Group> groups;                      // node_group:<id>
  std::unordered_map<std::string, std::string> node_to_group;  // node_to_group
  std::unordered_map<std::string, std::string> group_task;     // group_task:<id>
  uint64_t next_group_id = 1;
  std::set<std::string> upload_keys;                           // "upload:<node>:<group>:<file>" (storage route)
  // (ip, port) -> number of Healthy nodes: replaces the per-node full scan of
  // count_healthy_nodes_with_same_endpoint (discovery/monitor.rs:218-234, Theta(N^2) per sync)
  std::unordered_map<std::string, uint32_t> healthy_at;
  // The engine keeps the worker table between management passes (rows in table order: candidates are all Healthy,
  // so their relative order equals the canonical status-sorted order of node_store.rs:195-206); a pass uploads only
  // the rows touched since the previous one.  `resident_version` detects anybody else using the engine in between.
  std::vector<uint32_t> dirty_list;
  uint32_t resident_rows = 0;
  uint64_t resident_version = ~0ull;
  // The configurations on the engine: every sealed one, in the order available_configurations() puts them when all are
  // enabled (the sealed order stably re-sorted by min_group_size desc), uploaded with the worker table; a pass then
  // sends only the enable flags that changed (pm_set_ask_enabled), which keeps the engine's stored evaluation.  A
  // stable sort of a subset is the same subset of the stable sort of the whole, so the enabled ones keep the priority
  // order available_configurations() gives them.
  std::vector<uint32_t> resident_cfgs;   // indices into templates
  std::vector<uint8_t> resident_on;      // the flags the engine holds, per resident_cfgs entry
  uint32_t resident_npat = ~0u, resident_nmod = ~0u;
  pm_engine* merge_engine = nullptr;   // solo-group merging works on its own small table: a sibling engine, created on demand
  void touch(size_t i) {
    if (!nodes[i].dirty) { nodes[i].dirty = true; dirty_list.push_back((uint32_t)i); }
  }
  uint64_t sync_gen = 0;
  uint64_t sync_skipped = 0;   // discovery entries without id / ip, skipped (the reference logs them)
  // BTreeSet<String> rank of every node's address: addresses never change and nodes are only appended, so the ranks
  // are recomputed only when the table has grown since the last management pass
  std::vector<uint32_t> addr_rank_cache;
  size_t addr_rank_n = 0;

  static std::string endpoint_key(const std::string& ip, uint16_t port) { return ip + ":" + std::to_string(port); }
  void index_remove(const NodeRec& n) {
    if (n.status != kHealthy) return;
    auto it = healthy_at.find(endpoint_key(n.ip_address, n.port));
    if (it != healthy_at.end() && it->second) --it->second;
  }
  void index_add(const NodeRec& n) {
    if (n.status == kHealthy) ++healthy_at[endpoint_key(n.ip_address, n.port)];
  }
  // NodeStore::update_node_status (node_store.rs:284-305) + handle_status_change
  void set_status(NodeRec& n, uint32_t status, int64_t now_ms) {
    index_remove(n);
    n.status = status;
    n.last_status_change_ms = now_ms;
    index_add(n);
    touch(size_t(&n - nodes.data()));
    if (status == kDead || status == kLowBalance) {
      auto g = node_to_group.find(n.address);
      if (g != node_to_group.end()) {
        const std::string gid = g->second;
        dissolve(gid);
      }
    }
  }

  int fail(int st, const std::string& m) {
    err = m;
    return st;
  }

  std::vector<const TaskRec*> all_tasks() const {  // get_all_tasks: stable sort created_at desc
    std::vector<const TaskRec*> v;
    for (const auto& t : tasks) v.push_back(&t);
    std::stable_sort(v.begin(), v.end(), [](const TaskRec* a, const TaskRec* b) { return a->created_at > b->created_at; });
    return v;
  }
  const TaskRec* find_task(const std::string& id) const {
    auto it = task_pos.find(id);
    return it == task_pos.end() ? nullptr : &tasks[it->second];
  }
  void reindex_tasks() {
    task_pos.clear();
    for (size_t i = 0; i < tasks.size(); ++i) task_pos.emplace(tasks[i].id, i);   // first occurrence of an id counts
  }

  std::vector<const Config*> available_configurations() const {  // mod.rs:399-418
    std::vector<const Config*> v;
    for (const auto& c : templates)
      if (available.count(c.name)) v.push_back(&c);
    std::stable_sort(v.begin(), v.end(), [](const Config* a, const Config* b) { return a->min_group_size > b->min_group_size; });
    return v;
  }

  // node_to_group with the per-node mirror bit kept in step
  void map_node(const std::string& addr, const std::string& gid) {
    node_to_group[addr] = gid;
    auto it = node_index.find(addr);
    if (it != node_index.end()) { nodes[it->second].grouped = true; touch(it->second); }
  }
  void unmap_node(const std::string& addr) {
    node_to_group.erase(addr);
    auto it = node_index.find(addr);
    if (it != node_index.end()) { nodes[it->second].grouped = false; touch(it->second); }
  }

  void dissolve(const std::string& group_id) {  // mod.rs:1423-1487
    auto it = groups.find(group_id);
    if (it == groups.end()) return;
    for (const auto& n : it->second.nodes) unmap_node(n);
    group_task.erase(group_id);
    groups.erase(it);
  }

  // get_current_group_task, mod.rs:436-469 (a claim on a deleted task is garbage-collected)
  const TaskRec* current_group_task(const std::string& group_id) {
    auto it = group_task.find(group_id);
    if (it == group_task.end()) return nullptr;
    if (const TaskRec* t = find_task(it->second)) return t;
    group_task.erase(it);
    return nullptr;
  }
};

extern "C" {

// Address::from_str + to_string at the boundary (policy.canonical_addresses): the string every table is keyed by.
// `keep` owns the canonical form; returns nullptr when the policy is on and the string is not an address.
static const char* canon_address(const pm_plugin* p, const char* address, char (&keep)[43]) {
  if (!p->policy.canonical_addresses) return address;
  return pm_address_canonical(address, keep) == PM_OK ? keep : nullptr;
}
#define PM_CANON(var)                                                                      \
  char var##_canon[43];                                                                    \
  var = canon_address(p, var, var##_canon);                                                \
  if (!var) return p->fail(PM_E_INVALID, "not an address (policy.canonical_addresses)")

static int plugin_create(Device dev, const pm_plugin_policy* policy, pm_plugin** out) {
  pm_plugin* p = new (std::nothrow) pm_plugin;
  if (!p) return PM_E_NOMEM;
  p->dev = dev;
  if (policy) p->policy = *policy;
  else {  // TaskSwitchingPolicy::default / ProximityOptimizationPolicy::default, mod.rs:85-98
    p->policy.task_switching_enabled = 1;
    p->policy.prefer_larger_groups = 1;
    p->policy.proximity_enabled = 1;
  }
  p->interner = pm_interner_create();
  *out = p;
  return PM_OK;
}

int pm_plugin_create(pm_engine* engine, const pm_plugin_policy* policy, pm_plugin** out) try {
  if (!out) return PM_E_INVALID;
  Device dev;
  dev.engine = engine;
  return plugin_create(dev, policy, out);
} catch (...) { return pm_guard_rc(); }

int pm_plugin_create_multi(pm_multi* multi, const pm_plugin_policy* policy, pm_plugin** out) try {
  if (!out || !multi) return PM_E_INVALID;
  Device dev;
  dev.multi = multi;
  return plugin_create(dev, policy, out);
} catch (...) { return pm_guard_rc(); }

void pm_plugin_destroy(pm_plugin* p) {
  if (!p) return;
  pm_interner_destroy(p->interner);
  if (p->merge_engine) pm_destroy(p->merge_engine);
  delete p;
}

const char* pm_plugin_last_error(const pm_plugin* p) { return p ? p->err.c_str() : ""; }

int pm_plugin_add_config(pm_plugin* p, const char* name, uint32_t min_group_size, uint32_t max_group_size,
                         const char* requirements) try {
  if (!p || !name) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  if (p->sealed) return p->fail(PM_E_STATE, "configurations are sealed");
  for (const auto& c : p->templates)
    if (c.name == name) return p->fail(PM_E_INVALID, "Configuration names must be unique");       // mod.rs:142-144
  if (max_group_size < min_group_size) return p->fail(PM_E_INVALID, "Plugin configuration is invalid");  // :145-147
  Config c;
  c.name = name;
  c.min_group_size = min_group_size;
  c.max_group_size = max_group_size;
  if (requirements) {  // deserialize_compute_requirements, mod.rs:39-52
    c.has_requirements = true;
    c.opts.resize(64);
    uint32_t n = 0;
    char err[256] = {0};
    int rc = pm_parse_requirements(requirements, p->interner, &c.ask, c.opts.data(), 64, &n, err, sizeof err);
    if (rc != PM_OK) return p->fail(rc, err);
    c.opts.resize(n);
  }
  c.ask.min_group_size = min_group_size;
  c.ask.max_group_size = max_group_size;
  p->templates.push_back(std::move(c));
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_plugin_seal_configs(pm_plugin* p) try {
  if (!p) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  const uint32_t n = (uint32_t)p->templates.size();
  std::vector<uint32_t> mn(n), perm(n);
  std::vector<uint8_t> hr(n);
  for (uint32_t i = 0; i < n; ++i) {
    mn[i] = p->templates[i].min_group_size;
    hr[i] = p->templates[i].has_requirements;
  }
  if (n) {
    int rc = pm_sort_configs(mn.data(), hr.data(), n, perm.data());
    if (rc != PM_OK) return p->fail(rc, "pm_sort_configs");
    std::vector<Config> sorted;
    for (uint32_t i = 0; i < n; ++i) sorted.push_back(std::move(p->templates[perm[i]]));
    p->templates.swap(sorted);
  }
  p->sealed = true;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_plugin_enable_configuration(pm_plugin* p, const char* name, int enable) try {  // mod.rs:1328-1346
  if (!p || !name) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  if (enable) p->available.insert(name);
  else p->available.erase(name);
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_plugin_upsert_node(pm_plugin* p, const pm_node_desc* d) try {
  if (!p || !d || !d->address) return PM_E_INVALID;
  const char* address = d->address;
  PM_CANON(address);
  std::lock_guard<std::shared_mutex> lk(p->mu);
  NodeRec* r;
  auto it = p->node_index.find(address);
  if (it == p->node_index.end()) {
    p->node_index.emplace(address, p->nodes.size());
    p->nodes.emplace_back();
    r = &p->nodes.back();
    r->address = address;
    r->grouped = p->node_to_group.count(r->address) != 0;   // a restored group may name a node before it is stored
  } else {
    r = &p->nodes[it->second];
  }
  p->index_remove(*r);
  r->status = d->status;
  r->has_p2p = d->p2p_id != nullptr;
  r->p2p_id = d->p2p_id ? d->p2p_id : "";
  if (d->ip_address) r->ip_address = d->ip_address;
  r->port = d->port;
  if (d->last_status_change_ms) r->last_status_change_ms = d->last_status_change_ms;
  const uint32_t keep = PM_W_HAS_SPECS | PM_W_HAS_GPU | PM_W_HAS_GPU_COUNT | PM_W_HAS_GPU_MEM | PM_W_HAS_GPU_MODEL |
                        PM_W_HAS_CPU | PM_W_HAS_CPU_CORES | PM_W_HAS_RAM | PM_W_HAS_STORAGE;
  r->a.flags = d->spec_flags & keep;
  r->a.gpu_count = d->gpu_count;
  r->a.gpu_mem_mb = d->gpu_mem_mb;
  r->a.model_id = (d->spec_flags & PM_W_HAS_GPU_MODEL) && d->gpu_model ? pm_intern_model(p->interner, d->gpu_model) : 0;
  r->b.cpu_cores = d->cpu_cores;
  r->b.ram_mb = d->ram_mb;
  r->b.storage_gb = d->storage_gb;
  r->b.ext_ask_price = 0;
  // a location the distance function cannot use (NaN / infinite coordinates) is no location
  r->has_loc = d->has_location != 0 && std::isfinite(d->lat) && std::isfinite(d->lon);
  r->lat = r->has_loc ? d->lat : 0.0;
  r->lon = r->has_loc ? d->lon : 0.0;
  p->index_add(*r);
  p->touch(size_t(r - p->nodes.data()));
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// StatusUpdatePlugin::handle_status_change (plugins/mod.rs:23-34 -> status_update_impl.rs:8-39)
int pm_plugin_set_node_status(pm_plugin* p, const char* address, uint32_t status) try {
  if (!p || !address) return PM_E_INVALID;
  PM_CANON(address);
  std::lock_guard<std::shared_mutex> lk(p->mu);
  auto it = p->node_index.find(address);
  if (it == p->node_index.end()) return p->fail(PM_E_INVALID, "unknown node");
  p->set_status(p->nodes[it->second], status, (int64_t)std::time(nullptr) * 1000);
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// DiscoveryMonitor::get_nodes -> sync_single_node_with_discovery (discovery/monitor.rs:236-435):
// reconcile the validated nodes reported by the discovery service into the node table.
}  // extern "C"

// One fetch may be applied in several chunks (the JSON path releases the table lock between them, as the
// reference awaits between nodes).  "Remove duplicates based on node ID" (:203-210): a node carries the number of
// the fetch that last touched it; ids of this fetch that were not stored are kept in `unstored`.
// The caller holds p->mu.
struct ExistingView {   // the fields of the snapshot the reference keeps testing against
  uint32_t status;
  int64_t last_status_change_ms;
  bool has_loc;
};
static int sync_discovery_chunk(pm_plugin* p, const pm_discovery_node* dn, uint32_t n, int64_t now_ms,
                                uint32_t max_healthy_nodes_with_same_endpoint, uint32_t* n_new, uint64_t gen,
                                std::unordered_set<std::string>& unstored) {
  std::string addr, ip, key;   // reused: no allocation per node once grown
  for (uint32_t i = 0; i < n; ++i) {
    const pm_discovery_node& d = dn[i];
    // a node the monitor cannot use is logged and skipped; the rest of the fetch still applies (monitor.rs:425-429)
    if (!d.node.address || !d.ip_address) { ++p->sync_skipped; continue; }
    if (!d.is_validated) continue;                       // fetch keeps validated nodes only
    addr.assign(d.node.address);
    if (p->policy.canonical_addresses) {   // node.id.parse::<Address>()? fails: this node is logged and skipped (monitor.rs:240,425-429)
      char c[43];
      if (pm_address_canonical(addr.c_str(), c) != PM_OK) { ++p->sync_skipped; continue; }
      addr.assign(c);
    }
    ip.assign(d.ip_address);
    auto it = p->node_index.find(addr);
    const bool exists = it != p->node_index.end();
    if (exists) {
      NodeRec& e = p->nodes[it->second];
      if (e.sync_gen == gen) continue;                   // a second entry with this id in the same fetch
      e.sync_gen = gen;
    } else if (!unstored.empty() && unstored.count(addr)) {
      continue;
    }
    // count_healthy_nodes_with_same_endpoint (:218-234) through the endpoint index
    uint32_t same = 0;
    {
      key.assign(ip);
      key += ':';
      key += std::to_string(d.port);
      auto h = p->healthy_at.find(key);
      if (h != p->healthy_at.end()) same = h->second;
      if (exists) {
        const NodeRec& e = p->nodes[it->second];
        if (e.status == kHealthy && e.ip_address == ip && e.port == d.port && same) --same;
      }
    }
    if (exists) {
      NodeRec& node = p->nodes[it->second];
      const ExistingView existing{node.status, node.last_status_change_ms, node.has_loc};
      if (same > 0 && existing.status != kHealthy) {     // :254-268
        p->set_status(node, kDead, now_ms);
        continue;
      }
      if (d.is_validated && !d.is_provider_whitelisted) p->set_status(node, kEjected, now_ms);          // :270-281
      if (d.is_validated && d.is_provider_whitelisted && existing.status == kEjected)                   // :285-299
        p->set_status(node, kDead, now_ms);
      if (!d.is_active && existing.status == kHealthy) {                                                 // :300-338
        const bool should_mark_inactive =
            existing.last_status_change_ms < 0 || (now_ms - existing.last_status_change_ms) > 5 * 60 * 1000;
        if (should_mark_inactive) p->set_status(node, d.is_provider_whitelisted ? kDead : kEjected, now_ms);
      }
      if (node.ip_address != ip) {                       // existing.ip_address: nothing above changes it     // :340-348
        p->index_remove(node);
        node.ip_address = ip;
        p->index_add(node);
      }
      if (!existing.has_loc && d.node.has_location && std::isfinite(d.node.lat) && std::isfinite(d.node.lon)) {   // :349-362
        node.has_loc = true;
        node.lat = d.node.lat;
        node.lon = d.node.lon;
        p->touch(it->second);
      }
      if (existing.status == kDead && existing.last_status_change_ms >= 0 && d.last_updated_ms >= 0 &&
          existing.last_status_change_ms < d.last_updated_ms) {                                          // :364-389
        const uint32_t keep = PM_W_HAS_SPECS | PM_W_HAS_GPU | PM_W_HAS_GPU_COUNT | PM_W_HAS_GPU_MEM | PM_W_HAS_GPU_MODEL |
                              PM_W_HAS_CPU | PM_W_HAS_CPU_CORES | PM_W_HAS_RAM | PM_W_HAS_STORAGE;
        node.a.flags = d.node.spec_flags & keep;
        node.a.gpu_count = d.node.gpu_count;
        node.a.gpu_mem_mb = d.node.gpu_mem_mb;
        node.a.model_id = (d.node.spec_flags & PM_W_HAS_GPU_MODEL) && d.node.gpu_model ? pm_intern_model(p->interner, d.node.gpu_model) : 0;
        node.b.cpu_cores = d.node.cpu_cores;
        node.b.ram_mb = d.node.ram_mb;
        node.b.storage_gb = d.node.storage_gb;
        p->set_status(node, kDiscovered, now_ms);
      }
      if (d.has_latest_balance && d.latest_balance_is_zero) p->set_status(node, kLowBalance, now_ms);    // :391-402
    } else {
      if (same >= max_healthy_nodes_with_same_endpoint) {                                                // :405-415
        unstored.insert(addr);
        continue;
      }
      NodeRec node;                                      // OrchestratorNode::from(DiscoveryNode), models/node.rs:46-66
      node.address = addr;
      node.ip_address = ip;
      node.port = d.port;
      node.status = kDiscovered;
      node.has_p2p = false;                              // p2p_id: None until the first heartbeat
      node.first_seen_ms = now_ms;
      node.sync_gen = gen;
      const uint32_t keep = PM_W_HAS_SPECS | PM_W_HAS_GPU | PM_W_HAS_GPU_COUNT | PM_W_HAS_GPU_MEM | PM_W_HAS_GPU_MODEL |
                            PM_W_HAS_CPU | PM_W_HAS_CPU_CORES | PM_W_HAS_RAM | PM_W_HAS_STORAGE;
      node.a.flags = d.node.spec_flags & keep;
      node.a.gpu_count = d.node.gpu_count;
      node.a.gpu_mem_mb = d.node.gpu_mem_mb;
      node.a.model_id = (d.node.spec_flags & PM_W_HAS_GPU_MODEL) && d.node.gpu_model ? pm_intern_model(p->interner, d.node.gpu_model) : 0;
      node.b.cpu_cores = d.node.cpu_cores;
      node.b.ram_mb = d.node.ram_mb;
      node.b.storage_gb = d.node.storage_gb;
      node.has_loc = d.node.has_location != 0 && std::isfinite(d.node.lat) && std::isfinite(d.node.lon);
      node.lat = node.has_loc ? d.node.lat : 0.0;
      node.lon = node.has_loc ? d.node.lon : 0.0;
      node.grouped = p->node_to_group.count(addr) != 0;
      p->node_index.emplace(addr, p->nodes.size());
      p->nodes.push_back(std::move(node));
      p->touch(p->nodes.size() - 1);
      if (n_new) ++*n_new;
    }
  }
  return PM_OK;
}

extern "C" {

int pm_plugin_sync_discovery(pm_plugin* p, const pm_discovery_node* dn, uint32_t n, int64_t now_ms,
                             uint32_t max_healthy_nodes_with_same_endpoint, uint32_t* n_new) try {
  if (!p || (n && !dn)) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  if (n_new) *n_new = 0;
  std::unordered_set<std::string> unstored;
  return sync_discovery_chunk(p, dn, n, now_ms, max_healthy_nodes_with_same_endpoint, n_new, ++p->sync_gen, unstored);
} catch (...) { return pm_guard_rc(); }

}  // extern "C"

namespace {

bool json_u32(const pmjson::Value* v, uint32_t* out) {   // Option<u32>
  if (!v || v->kind != pmjson::Value::Number || v->num < 0 || v->num > 4294967295.0) return false;
  if (v->num != (double)(uint32_t)v->num) return false;   // 1.5 is not a u32 (serde rejects it; here the field reads as None)
  *out = (uint32_t)v->num;
  return true;
}
bool json_bool(const pmjson::Value* v, bool dflt) { return (v && v->kind == pmjson::Value::Bool) ? v->b : dflt; }

// chrono DateTime<Utc> serde form (RFC 3339) -> unix milliseconds; -1 when absent/unparsable
int64_t rfc3339_ms(const pmjson::Value* v) {
  if (!v || v->kind != pmjson::Value::String) return -1;
  int Y, M, D, h, m;
  double sec;
  if (std::sscanf(v->str.c_str(), "%d-%d-%dT%d:%d:%lf", &Y, &M, &D, &h, &m, &sec) != 6) return -1;
  std::tm t{};
  t.tm_year = Y - 1900; t.tm_mon = M - 1; t.tm_mday = D; t.tm_hour = h; t.tm_min = m; t.tm_sec = 0;
  const std::time_t base = timegm(&t);
  int64_t ms = (int64_t)base * 1000 + (int64_t)(sec * 1000.0 + 0.5);
  // numeric offset ("+02:00"); 'Z' means none
  const std::string& s = v->str;
  const size_t tpos = s.find('T');
  const size_t sign = s.find_first_of("+-", tpos == std::string::npos ? 0 : tpos);
  if (sign != std::string::npos) {
    int oh = 0, om = 0;
    if (std::sscanf(s.c_str() + sign + 1, "%d:%d", &oh, &om) >= 1) ms -= (s[sign] == '+' ? 1 : -1) * (int64_t)(oh * 60 + om) * 60000;
  }
  return ms;
}

// One DiscoveryNode of the wire format, reduced to what the monitor reads (owning copies of the strings).
struct DiscRec {
  std::string id, ip, model;
  uint32_t port = 0, flags = 0, gpu_count = 0, gpu_mem_mb = 0, cpu_cores = 0, ram_mb = 0, storage_gb = 0;
  bool has_loc = false, validated = false, active = false, whitelisted = false, blacklisted = false;
  bool has_balance = false, balance_zero = false;
  double lat = 0, lon = 0;
  int64_t last_updated_ms = -1;
};

struct KeyView {   // an object key, compared in place
  const char* p;
  size_t n;
  bool operator==(const char* s) const { return std::strlen(s) == n && std::memcmp(p, s, n) == 0; }
};

// Walks the object at the cursor (after its '{'): `on_key(key)` must consume the value and returns false on malformed
// input.  Returns false on malformed JSON.
template <class F>
bool walk_object(pmjson::Parser& ps, std::string& scratch, F&& on_key) {
  if (ps.consume('}')) return true;
  for (;;) {
    KeyView k;
    if (!ps.read_key(&scratch, &k.p, &k.n) || !ps.consume(':')) return false;
    if (!on_key(k)) return false;
    if (ps.consume(',')) continue;
    return ps.consume('}');
  }
}

// compute_specs (shared/src/models/node.rs:128-178): typed read, unknown members (gpu.indices, cpu.model, storage_path ...)
// are skipped in place.  Anything but an object (null) means "no specs".  First occurrence of a key counts.
bool read_specs(pmjson::Parser& ps, DiscRec& d, uint32_t* flags, std::string& key, pmjson::Value& tmp) {
  if (ps.peek() != '{') return ps.skip_value(2);
  ps.consume('{');
  uint32_t f = PM_W_HAS_SPECS, seen = 0;
  const bool ok = walk_object(ps, key, [&](const KeyView& k) {
    if (k == "gpu" && !(seen & 1u)) {
      seen |= 1u;
      if (ps.peek() != '{') return ps.skip_value(3);
      ps.consume('{');
      f |= PM_W_HAS_GPU;
      uint32_t gseen = 0;
      std::string gkey;
      return walk_object(ps, gkey, [&](const KeyView& g) {
        if (g == "count" && !(gseen & 1u)) { gseen |= 1u; tmp = pmjson::Value(); if (!ps.read_value(&tmp)) return false; if (json_u32(&tmp, &d.gpu_count)) f |= PM_W_HAS_GPU_COUNT; return true; }
        if (g == "memory_mb" && !(gseen & 2u)) { gseen |= 2u; tmp = pmjson::Value(); if (!ps.read_value(&tmp)) return false; if (json_u32(&tmp, &d.gpu_mem_mb)) f |= PM_W_HAS_GPU_MEM; return true; }
        if (g == "model" && !(gseen & 4u)) {
          gseen |= 4u;
          tmp = pmjson::Value();
          if (!ps.read_value(&tmp)) return false;
          if (tmp.kind == pmjson::Value::String) { f |= PM_W_HAS_GPU_MODEL; d.model = std::move(tmp.str); }
          return true;
        }
        return ps.skip_value(4);
      });
    }
    if (k == "cpu" && !(seen & 2u)) {
      seen |= 2u;
      if (ps.peek() != '{') return ps.skip_value(3);
      ps.consume('{');
      f |= PM_W_HAS_CPU;
      bool cseen = false;
      std::string ckey;
      return walk_object(ps, ckey, [&](const KeyView& c) {
        if (c == "cores" && !cseen) { cseen = true; tmp = pmjson::Value(); if (!ps.read_value(&tmp)) return false; if (json_u32(&tmp, &d.cpu_cores)) f |= PM_W_HAS_CPU_CORES; return true; }
        return ps.skip_value(4);
      });
    }
    if (k == "ram_mb" && !(seen & 4u)) { seen |= 4u; tmp = pmjson::Value(); if (!ps.read_value(&tmp)) return false; if (json_u32(&tmp, &d.ram_mb)) f |= PM_W_HAS_RAM; return true; }
    if (k == "storage_gb" && !(seen & 8u)) { seen |= 8u; tmp = pmjson::Value(); if (!ps.read_value(&tmp)) return false; if (json_u32(&tmp, &d.storage_gb)) f |= PM_W_HAS_STORAGE; return true; }
    return ps.skip_value(3);
  });
  *flags = f;
  return ok;
}

// location (node.rs:25-44): latitude and longitude must both be numbers
bool read_location(pmjson::Parser& ps, DiscRec& d, std::string& key, pmjson::Value& tmp) {
  if (ps.peek() != '{') return ps.skip_value(2);
  ps.consume('{');
  bool have_la = false, have_lo = false, seen_la = false, seen_lo = false;
  double la = 0, lo = 0;
  const bool ok = walk_object(ps, key, [&](const KeyView& k) {
    if (k == "latitude" && !seen_la) { seen_la = true; tmp = pmjson::Value(); if (!ps.read_value(&tmp)) return false; if (tmp.kind == pmjson::Value::Number) { have_la = true; la = tmp.num; } return true; }
    if (k == "longitude" && !seen_lo) { seen_lo = true; tmp = pmjson::Value(); if (!ps.read_value(&tmp)) return false; if (tmp.kind == pmjson::Value::Number) { have_lo = true; lo = tmp.num; } return true; }
    return ps.skip_value(3);
  });
  if (ok && have_la && have_lo) { d.has_loc = true; d.lat = la; d.lon = lo; }
  return ok;
}

// Reads one node object at the parser's cursor.  Only the fields the monitor uses are materialised;
// everything else is skipped without building it.  Duplicate keys: the first occurrence counts.
bool read_discovery_node(pmjson::Parser& ps, DiscRec* out, std::string* err) {
  enum { kId, kIp, kPort, kSpecs, kLoc, kValidated, kActive, kWhitelisted, kBlacklisted, kLastUpdated, kBalance, kNumKeys };
  static const char* const kNames[kNumKeys] = {"id", "ip_address", "port", "compute_specs", "location", "is_validated", "is_active",
                                               "is_provider_whitelisted", "is_blacklisted", "last_updated", "latest_balance"};
  auto bad = [&]() {
    *err = "discovery JSON: " + (ps.error().empty() ? std::string("invalid JSON") : ps.error());
    return false;
  };
  DiscRec& d = *out;
  d = DiscRec();
  if (ps.peek() != '{') {   // an element that is not an object has no id
    if (!ps.skip_value(2)) return bad();
    *err = "discovery JSON: node without id / ip_address";
    return false;
  }
  ps.consume('{');
  pmjson::Value vals[kNumKeys];   // scalars only (compute_specs and location are read in place)
  pmjson::Value tmp;
  uint32_t have = 0, flags = 0;
  std::string key, sub;
  const bool ok = walk_object(ps, key, [&](const KeyView& k) {
    int j = -1;
    for (int q = 0; q < kNumKeys; ++q)
      if (!(have & (1u << q)) && k == kNames[q]) { j = q; break; }
    if (j < 0) return ps.skip_value(2);
    have |= 1u << j;
    if (j == kSpecs) return read_specs(ps, d, &flags, sub, tmp);
    if (j == kLoc) return read_location(ps, d, sub, tmp);
    return ps.read_value(&vals[j]);
  });
  if (!ok) return bad();
  auto get = [&](int k) -> pmjson::Value* { return (have & (1u << k)) ? &vals[k] : nullptr; };
  pmjson::Value* id = get(kId);
  pmjson::Value* ip = get(kIp);
  if (!id || id->kind != pmjson::Value::String || !ip || ip->kind != pmjson::Value::String) {
    *err = "discovery JSON: node without id / ip_address";
    return false;
  }
  d.id = std::move(id->str);
  d.ip = std::move(ip->str);
  json_u32(get(kPort), &d.port);
  d.port &= 0xFFFFu;
  d.flags = flags;
  d.validated = json_bool(get(kValidated), false);
  d.active = json_bool(get(kActive), false);
  d.whitelisted = json_bool(get(kWhitelisted), false);   // #[serde(default)]
  d.blacklisted = json_bool(get(kBlacklisted), false);
  d.last_updated_ms = rfc3339_ms(get(kLastUpdated));
  const pmjson::Value* bal = get(kBalance);                // Option<U256>
  if (bal && !bal->is_null()) {
    d.has_balance = true;
    const std::string& t = bal->str;   // decimal, hex quantity ("0x0") or a JSON number
    bool zero = !t.empty();
    for (size_t k = (t.rfind("0x", 0) == 0 ? 2 : 0); k < t.size(); ++k)
      if (t[k] != '0') zero = false;
    d.balance_zero = zero;
  }
  return true;
}

// streams the elements of the array at the cursor into `recs`
bool read_discovery_array(pmjson::Parser& ps, std::vector<DiscRec>* recs, std::string* err) {
  if (!ps.consume('[')) { *err = "discovery JSON: no node array"; return false; }
  if (ps.consume(']')) return true;
  for (;;) {
    recs->emplace_back();
    if (!read_discovery_node(ps, &recs->back(), err)) return false;
    if (ps.consume(',')) continue;
    if (ps.consume(']')) return true;
    *err = "discovery JSON: invalid JSON";
    return false;
  }
}

}  // namespace

extern "C" {

// The discovery service's wire format: `{"success":true,"data":[DiscoveryNode,...]}` (or a bare
// array), DiscoveryNode = flattened Node + flags (shared/src/models/node.rs:10-23, 552-570).
// (f-1) ingest: the body is read in one streaming pass — no document tree, unknown fields skipped in place —
// into compact records (nothing is applied if the body does not parse, like `response.json()` failing in the
// reference), which then go through the monitor's per-node logic in chunks, the table lock released in between.
int pm_plugin_sync_discovery_json(pm_plugin* p, const char* json, size_t len, int64_t now_ms,
                                  uint32_t max_healthy_nodes_with_same_endpoint, uint32_t* n_new) try {
  if (!p || !json) return PM_E_INVALID;
  if (n_new) *n_new = 0;
  std::vector<DiscRec> recs;
  recs.reserve(len / 384 + 1);   // a node of the wire format is several hundred bytes
  std::string err;
  {
    pmjson::Parser ps(json, len);
    bool ok = true, found = false;
    const char c = ps.peek();
    if (c == '[') {
      found = true;
      ok = read_discovery_array(ps, &recs, &err);
    } else if (c == '{') {
      ps.consume('{');
      if (!ps.consume('}')) {
        std::string key;
        for (;;) {
          if (!ps.read_string(&key) || !ps.consume(':')) { ok = false; break; }
          if (key == "data" && !found) {
            found = true;
            if (ps.peek() != '[') { ok = false; err = "discovery JSON: no node array"; break; }
            if (!read_discovery_array(ps, &recs, &err)) { ok = false; break; }
          } else if (!ps.skip_value(1)) {
            ok = false;
            break;
          }
          if (ps.consume(',')) continue;
          if (ps.consume('}')) break;
          ok = false;
          break;
        }
      }
    } else {
      ok = ps.skip_value();   // a scalar document: well-formed or not, it holds no node array
      if (ok && ps.at_end()) err = "discovery JSON: no node array";
      if (ok && !ps.at_end()) err = "discovery JSON: trailing characters after JSON value";
      ok = false;
    }
    if (ok && !ps.at_end()) { ok = false; err = "discovery JSON: trailing characters after JSON value"; }
    if (ok && !found) { ok = false; err = "discovery JSON: no node array"; }
    if (!ok) {
      std::lock_guard<std::shared_mutex> lk(p->mu);
      return p->fail(PM_E_PARSE, err.empty() ? (ps.error().empty() ? "discovery JSON: invalid JSON" : "discovery JSON: " + ps.error()) : err);
    }
  }
  std::unordered_set<std::string> unstored;
  uint64_t gen;
  {
    std::lock_guard<std::shared_mutex> lk(p->mu);
    gen = ++p->sync_gen;
    if (p->node_index.empty()) {   // first fetch: no rehashing or table moves while the chunks go in
      p->node_index.reserve(recs.size());
      p->nodes.reserve(recs.size());
    }
  }
  constexpr size_t kChunk = 8192;
  std::vector<pm_discovery_node> nodes(std::min(recs.size(), kChunk));
  for (size_t base = 0; base < recs.size(); base += kChunk) {
    const size_t n = std::min(kChunk, recs.size() - base);
    for (size_t i = 0; i < n; ++i) {
      const DiscRec& r = recs[base + i];
      pm_discovery_node& d = nodes[i];
      std::memset(&d, 0, sizeof d);
      d.node.address = r.id.c_str();
      d.ip_address = r.ip.c_str();
      d.port = (uint16_t)r.port;
      d.node.spec_flags = r.flags;
      d.node.gpu_count = r.gpu_count;
      d.node.gpu_mem_mb = r.gpu_mem_mb;
      d.node.gpu_model = (r.flags & PM_W_HAS_GPU_MODEL) ? r.model.c_str() : nullptr;
      d.node.cpu_cores = r.cpu_cores;
      d.node.ram_mb = r.ram_mb;
      d.node.storage_gb = r.storage_gb;
      d.node.has_location = r.has_loc;
      d.node.lat = r.lat;
      d.node.lon = r.lon;
      d.is_validated = r.validated;
      d.is_active = r.active;
      d.is_provider_whitelisted = r.whitelisted;
      d.is_blacklisted = r.blacklisted;
      d.last_updated_ms = r.last_updated_ms;
      d.has_latest_balance = r.has_balance;
      d.latest_balance_is_zero = r.balance_zero;
    }
    std::lock_guard<std::shared_mutex> lk(p->mu);
    const int rc = sync_discovery_chunk(p, nodes.data(), (uint32_t)n, now_ms, max_healthy_nodes_with_same_endpoint, n_new, gen, unstored);
    if (rc != PM_OK) return rc;
  }
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// node as the /nodes route would show it (fields on this path): JSON or null
int pm_plugin_get_node(pm_plugin* p, const char* address, char* buf, size_t len) try {
  if (!p || !address) return PM_E_INVALID;
  PM_CANON(address);
  std::lock_guard<std::shared_mutex> lk(p->mu);
  auto it = p->node_index.find(address);
  std::string out = "null";
  if (it != p->node_index.end()) {
    static const char* kNames[] = {"Discovered", "WaitingForHeartbeat", "Healthy", "Unhealthy", "Dead", "Ejected", "Banned", "LowBalance"};
    const NodeRec& n = p->nodes[it->second];
    out = "{\"address\":";
    json_str(out, n.address);
    out += ",\"ip_address\":";
    json_str(out, n.ip_address);
    out += ",\"port\":" + std::to_string(n.port);
    out += std::string(",\"status\":\"") + kNames[n.status & 7] + "\"";
    out += ",\"first_seen_ms\":" + (n.first_seen_ms < 0 ? std::string("null") : std::to_string(n.first_seen_ms));
    out += ",\"last_status_change_ms\":" + (n.last_status_change_ms < 0 ? std::string("null") : std::to_string(n.last_status_change_ms));
    out += std::string(",\"has_location\":") + (n.has_loc ? "true" : "false");
    out += std::string(",\"has_compute_specs\":") + ((n.a.flags & PM_W_HAS_SPECS) ? "true" : "false");
    out += ",\"ram_mb\":" + std::to_string(n.b.ram_mb);
    // the SoA row the engine will see (presence bits of include/prime_match.h, interned model id)
    out += ",\"spec_flags\":" + std::to_string(n.a.flags) + ",\"gpu_count\":" + std::to_string(n.a.gpu_count);
    out += ",\"gpu_mem_mb\":" + std::to_string(n.a.gpu_mem_mb) + ",\"model_id\":" + std::to_string(n.a.model_id);
    out += ",\"cpu_cores\":" + std::to_string(n.b.cpu_cores) + ",\"storage_gb\":" + std::to_string(n.b.storage_gb);
    char ll[96];
    std::snprintf(ll, sizeof ll, ",\"lat\":%.17g,\"lon\":%.17g}", n.has_loc ? n.lat : 0.0, n.has_loc ? n.lon : 0.0);
    out += ll;
  }
  if (!buf || len < out.size() + 1) return p->fail(PM_E_NOMEM, "output buffer too small");
  std::memcpy(buf, out.c_str(), out.size() + 1);
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_plugin_add_task(pm_plugin* p, const pm_task_desc* d) try {
  if (!p || !d || !d->id) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  TaskRec t;
  t.id = d->id;
  t.name = d->name ? d->name : "";
  t.image = d->image ? d->image : "";
  t.created_at = d->created_at;
  t.has_env = d->has_env_vars != 0;
  for (uint32_t i = 0; i < d->n_env_vars; ++i) t.env.emplace_back(d->env_vars[i].key, d->env_vars[i].value);
  t.has_cmd = d->has_cmd != 0;
  for (uint32_t i = 0; i < d->n_cmd; ++i) t.cmd.emplace_back(d->cmd[i]);
  t.has_mounts = d->has_volume_mounts != 0;
  for (uint32_t i = 0; i < d->n_volume_mounts; ++i) t.mounts.emplace_back(d->volume_mounts[i].key, d->volume_mounts[i].value);
  t.scheduling = d->scheduling;
  for (uint32_t i = 0; i < d->n_allowed_topologies; ++i) t.topologies.emplace_back(d->allowed_topologies[i]);
  // on_task_created: enable the configuration of every allowed topology (mod.rs:1224-1243)
  if (t.scheduling == 3)
    for (const auto& topo : t.topologies) p->available.insert(topo);
  p->task_pos.emplace(t.id, p->tasks.size());
  p->tasks.push_back(std::move(t));
  p->claim_cache_valid = false;
  p->newest_valid = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_plugin_delete_task(pm_plugin* p, const char* id) try {  // TaskStore::delete_task + on_task_deleted
  if (!p || !id) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  auto it = std::find_if(p->tasks.begin(), p->tasks.end(), [&](const TaskRec& t) { return t.id == id; });
  if (it == p->tasks.end()) return PM_OK;
  TaskRec gone = *it;
  p->tasks.erase(it);
  p->reindex_tasks();
  p->claim_cache_valid = false;
  p->newest_valid = false;
  // dissolve every group working on the task (mod.rs:1259-1291)
  std::vector<std::string> doomed;
  for (const auto& kv : p->group_task)
    if (kv.second == gone.id) doomed.push_back(kv.first);
  for (const auto& gid : doomed) p->dissolve(gid);
  // disable topologies with no remaining task (mod.rs:1295-1320)
  if (gone.scheduling == 3)
    for (const auto& topo : gone.topologies) {
      bool remaining = false;
      for (const auto& t : p->tasks)
        if (t.scheduling == 3 && std::find(t.topologies.begin(), t.topologies.end(), topo) != t.topologies.end()) remaining = true;
      if (!remaining) p->available.erase(topo);
    }
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

}  // extern "C"

// The node table as the engine's SoA tables (SURVEY 8 A21 / 8f-1: ingest -> columnar): rows in the canonical order of
// node_store.get_nodes() (stable status-class sort, node_store.rs:195-206), the candidate flags of mod.rs:492-497,
// locations, and every row's BTreeSet<String> address rank.  The caller holds the table lock exclusively.
struct TableSnapshot {
  std::vector<pm_worker_a> wa;
  std::vector<pm_worker_b> wb;
  std::vector<double> lat, lon;
  std::vector<uint32_t> arank;
  std::vector<uint32_t> row_node;   // row -> index in pm_plugin::nodes (stable: nodes are never removed)
};
static void build_table_snapshot(pm_plugin* p, TableSnapshot* s) {
  const uint32_t W = (uint32_t)p->nodes.size();
  if (p->addr_rank_n != W) {
    std::vector<uint32_t> by_addr(W);
    for (uint32_t i = 0; i < W; ++i) by_addr[i] = i;
    std::sort(by_addr.begin(), by_addr.end(), [&](uint32_t a, uint32_t b) { return p->nodes[a].address < p->nodes[b].address; });
    p->addr_rank_cache.resize(W);
    for (uint32_t i = 0; i < W; ++i) p->addr_rank_cache[by_addr[i]] = i;
    p->addr_rank_n = W;
  }
  // stable sort by status class = four buckets filled in table order
  uint32_t start[5] = {0, 0, 0, 0, 0};
  for (uint32_t i = 0; i < W; ++i) ++start[status_class(p->nodes[i].status) + 1];
  for (int c = 0; c < 4; ++c) start[c + 1] += start[c];
  s->wa.resize(W); s->wb.resize(W); s->lat.resize(W); s->lon.resize(W); s->arank.resize(W); s->row_node.resize(W);
  for (uint32_t i = 0; i < W; ++i) {
    const NodeRec& n = p->nodes[i];
    const uint32_t r = start[status_class(n.status)]++;
    s->wa[r] = n.a;
    s->wb[r] = n.b;
    uint32_t f = n.a.flags;
    if (n.status == kHealthy) f |= PM_W_HEALTHY;                         // mod.rs:494
    if (n.has_p2p) f |= PM_W_P2P;                                        // :495
    if (n.grouped) f |= PM_W_ASSIGNED;                                   // :496 (get_node_group is Some)
    if (n.has_loc) f |= PM_W_HAS_LOC;
    s->wa[r].flags = f;
    s->lat[r] = n.lat;
    s->lon[r] = n.lon;
    s->arank[r] = p->addr_rank_cache[i];
    s->row_node[r] = i;
  }
}

extern "C" {

// The SoA tables a management pass would upload, for callers that keep their own device copy and for inspection.
// Arrays may be NULL (skipped); capacity is in rows; *n_rows receives the row count (PM_E_NOMEM when it does not fit).
int pm_plugin_export_tables(pm_plugin* p, pm_worker_a* a, pm_worker_b* b, double* lat, double* lon, uint32_t* addr_rank,
                            uint32_t capacity, uint32_t* n_rows) try {
  if (!p) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  const uint32_t W = (uint32_t)p->nodes.size();
  if (n_rows) *n_rows = W;
  if ((a || b || lat || lon || addr_rank) && capacity < W) return p->fail(PM_E_NOMEM, "pm_plugin_export_tables: capacity too small");
  if (!(a || b || lat || lon || addr_rank)) return PM_OK;
  TableSnapshot s;
  build_table_snapshot(p, &s);
  if (a && W) std::memcpy(a, s.wa.data(), (size_t)W * sizeof(pm_worker_a));
  if (b && W) std::memcpy(b, s.wb.data(), (size_t)W * sizeof(pm_worker_b));
  if (lat && W) std::memcpy(lat, s.lat.data(), (size_t)W * sizeof(double));
  if (lon && W) std::memcpy(lon, s.lon.data(), (size_t)W * sizeof(double));
  if (addr_rank && W) std::memcpy(addr_rank, s.arank.data(), (size_t)W * sizeof(uint32_t));
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// try_form_new_groups (mod.rs:478-628): the evaluation and the allocation run on the GPU.
//
// The worker table stays RESIDENT on the engine between passes, rows in table (insertion) order — every candidate is
// Healthy, so the candidates' relative order is the canonical order of the status-sorted node list
// (node_store.rs:195-206) and the groups are the same — and a pass sends only the rows touched since the previous one
// (status changes, new group members, new nodes): the reference re-reads and re-parses every node per pass.  Every
// sealed configuration travels once, with a full upload; after that a pass sends only the enable flags that changed
// (task events toggle configurations), and the model table only when the interner changed.  Members of a group are put in
// BTreeSet<String> order here at publication (the address strings are at hand), so no address ranks travel at all.
int pm_plugin_try_form_new_groups(pm_plugin* p, uint32_t* n_formed) try {
  if (!p) return PM_E_INVALID;
  if (n_formed) *n_formed = 0;
  std::lock_guard<std::mutex> loop_lk(p->loop_mu);
  // ---- phase 1 (tables locked): what changed since the previous pass
  uint32_t W = 0, mode = PM_MODE_FIRST_FIT;
  bool full = false, send_asks = false, send_bits = false;
  std::vector<uint32_t> idx;
  std::vector<pm_worker_a> ua;
  std::vector<pm_worker_b> ub;
  std::vector<double> ulat, ulon;
  std::vector<std::string> cfg_names;   // per engine ask (every sealed configuration)
  std::vector<uint32_t> toggle_idx;
  std::vector<uint8_t> toggle_on;
  std::vector<pm_ask> asks;
  std::vector<pm_gpu_opt> opts;
  std::vector<uint32_t> bits_copy;
  uint32_t npat = 0, nmod = 0, words = 1;
  {
    std::lock_guard<std::shared_mutex> lk(p->mu);
    if (!p->dev) return p->fail(PM_E_NO_DEVICE, "no engine attached: group formation has no CPU path");
    if (!p->sealed) return p->fail(PM_E_STATE, "configurations not sealed");
    W = (uint32_t)p->nodes.size();
    full = p->dev.table_version() != p->resident_version || p->resident_rows > W;
    auto row_of = [&](uint32_t i, pm_worker_a* a, pm_worker_b* b, double* la, double* lo) {
      const NodeRec& n = p->nodes[i];
      *a = n.a;
      *b = n.b;
      uint32_t f = n.a.flags;
      if (n.status == kHealthy) f |= PM_W_HEALTHY;                         // mod.rs:494
      if (n.has_p2p) f |= PM_W_P2P;                                        // :495
      if (n.grouped) f |= PM_W_ASSIGNED;                                   // :496 (get_node_group is Some)
      if (n.has_loc) f |= PM_W_HAS_LOC;
      a->flags = f;
      *la = n.lat;
      *lo = n.lon;
    };
    if (full) {
      idx.resize(W); ua.resize(W); ub.resize(W); ulat.resize(W); ulon.resize(W);
      for (uint32_t i = 0; i < W; ++i) {
        idx[i] = i;
        row_of(i, &ua[i], &ub[i], &ulat[i], &ulon[i]);
        p->nodes[i].dirty = false;
      }
    } else {
      const size_t nd = p->dirty_list.size();
      idx.resize(nd); ua.resize(nd); ub.resize(nd); ulat.resize(nd); ulon.resize(nd);
      for (size_t k = 0; k < nd; ++k) {
        const uint32_t i = p->dirty_list[k];
        idx[k] = i;
        row_of(i, &ua[k], &ub[k], &ulat[k], &ulon[k]);
        p->nodes[i].dirty = false;
      }
    }
    p->dirty_list.clear();
    send_asks = full;
    if (send_asks) {
      const uint32_t C = (uint32_t)p->templates.size();
      p->resident_cfgs.resize(C);
      for (uint32_t i = 0; i < C; ++i) p->resident_cfgs[i] = i;
      std::stable_sort(p->resident_cfgs.begin(), p->resident_cfgs.end(), [&](uint32_t x, uint32_t y) {
        return p->templates[x].min_group_size > p->templates[y].min_group_size;
      });
      p->resident_on.assign(C, 1);   // pm_set_asks enables every ask
      for (uint32_t i : p->resident_cfgs) {
        const Config& c = p->templates[i];
        pm_ask a = c.ask;
        a.opt_off = (uint32_t)opts.size();
        a.min_group_size = c.min_group_size;
        a.max_group_size = c.max_group_size;
        opts.insert(opts.end(), c.opts.begin(), c.opts.end());
        asks.push_back(a);
      }
    }
    for (uint32_t j = 0; j < (uint32_t)p->resident_cfgs.size(); ++j) {
      const Config& c = p->templates[p->resident_cfgs[j]];
      cfg_names.push_back(c.name);
      const uint8_t on = p->available.count(c.name) ? 1 : 0;   // get_available_configurations, mod.rs:399-418
      if (on != p->resident_on[j]) {
        toggle_idx.push_back(j);
        toggle_on.push_back(on);
        p->resident_on[j] = on;
      }
    }
    const uint32_t* bits = nullptr;
    int rc = pm_interner_table(p->interner, &bits, &npat, &nmod, &words);
    if (rc != PM_OK) return p->fail(rc, "pm_interner_table");
    send_bits = full || npat != p->resident_npat || nmod != p->resident_nmod;   // rows and columns are only ever added
    if (send_bits) bits_copy.assign(bits, bits + (size_t)std::max<uint32_t>(npat, 1) * words);
    p->resident_npat = npat;
    p->resident_nmod = nmod;
    // the pass needs the per-worker first feasible configuration only: evaluate and reduce on chip, skip the per-ask
    // statistics (same groups as the materialised pass, ~20 MB of DRAM traffic instead of 16 B per pair)
    mode = (p->policy.proximity_enabled ? PM_MODE_PROXIMITY : PM_MODE_FIRST_FIT) | PM_PATH_FUSED | PM_NO_ASK_STATS;
    // resident tables: the engine re-evaluates only the rows this pass sends (a full upload re-evaluates everything)
    if (!full) mode |= PM_INCREMENTAL;
    p->resident_version = ~0ull;  // not valid again until this pass has put its rows on the device
  }
  // ---- phase 2 (tables unlocked: heartbeats keep being served): the pass on the GPU
  const Device& dev = p->dev;
  auto chk = [&](int r, const char* what) {
    if (r != PM_OK) {
      const char* m = dev.last_error();
      std::lock_guard<std::shared_mutex> lk(p->mu);
      p->err = std::string(what) + ": " + (m ? m : "");
    }
    return r;
  };
  int rc;
  if (send_asks && (rc = chk(dev.set_asks(asks.data(), (uint32_t)asks.size(), opts.data(), (uint32_t)opts.size()), "pm_set_asks"))) return rc;
  if (!toggle_idx.empty() &&
      (rc = chk(dev.set_ask_enabled(toggle_idx.data(), toggle_on.data(), (uint32_t)toggle_idx.size()), "pm_set_ask_enabled")))
    return rc;
  if (send_bits && (rc = chk(dev.set_model_table(bits_copy.data(), npat, nmod, words), "pm_set_model_table"))) return rc;
  if (full) {
    if ((rc = chk(dev.set_worker_count(W), "pm_set_worker_count"))) return rc;
  } else if (W != p->resident_rows) {
    if ((rc = chk(dev.resize_workers(W), "pm_resize_workers"))) return rc;
  }
  if (!idx.empty()) {
    if ((rc = chk(dev.update_workers(idx.data(), ua.data(), ub.data(), ulat.data(), ulon.data(), (uint32_t)idx.size()), "pm_update_workers"))) return rc;
    if ((rc = chk(dev.sync(), "pm_stream_sync"))) return rc;   // staging vectors are read asynchronously
  } else if (full) {   // an empty table still needs its location columns for the proximity mode
    if ((rc = chk(dev.set_worker_locations(nullptr, nullptr, 0, 0), "pm_set_worker_locations"))) return rc;
  }
  p->resident_rows = W;
  const uint64_t version_after_upload = dev.table_version();
  if ((rc = chk(dev.match(mode), "pm_match"))) return rc;
  pm_result res{};
  if ((rc = chk(dev.fetch_result(&res), "pm_fetch_result"))) return rc;

  // ---- phase 3 (tables locked): publish the groups (create_group_atomically, mod.rs:299-322, 568-581)
  std::lock_guard<std::shared_mutex> lk(p->mu);
  p->resident_version = version_after_upload;
  uint32_t formed = 0;
  for (uint32_t g = 0; g < res.n_groups; ++g) {
    Group grp;
    grp.configuration_name = cfg_names[res.group_ask[g]];
    grp.created_at_ms = (int64_t)std::time(nullptr) * 1000;
    bool stale = false;   // a member joined another group while the pass ran
    for (uint32_t m = res.group_off[g]; m < res.group_off[g + 1]; ++m) {
      const std::string& addr = p->nodes[res.group_members[m]].address;   // row == index in the node table; nodes are never removed
      if (p->node_to_group.count(addr)) stale = true;
      grp.nodes.push_back(addr);
    }
    if (stale) continue;
    std::sort(grp.nodes.begin(), grp.nodes.end());                         // NodeGroup.nodes: BTreeSet<String> (mod.rs:63-69)
    char idbuf[32];
    std::snprintf(idbuf, sizeof idbuf, "%llx", (unsigned long long)p->next_group_id++);  // format!("{:x}", ..)
    grp.id = idbuf;
    for (const auto& n : grp.nodes) p->map_node(n, grp.id);
    p->groups.emplace(grp.id, std::move(grp));
    ++formed;
  }
  if (n_formed) *n_formed = formed;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// try_merge_solo_groups (mod.rs:631-971).  Compatibility of the solo groups' nodes with each
// configuration, and the batch selection, run on the engine over a temporary table that holds only
// those nodes in get_all_groups() order (sorted by id, mod.rs:1040).
static int merge_pass(pm_plugin* p, const std::vector<const Config*>& configs, const std::vector<std::string>& all_solo_ids,
                      std::vector<std::pair<const Config*, std::vector<std::string>>>* merged /* (config, solo group ids) */) {
  // A solo group whose node is not in the node table (a group restored from the stored keys before its node was
  // synced) is compatible with nothing: find_compatible_solo_groups looks the node up and takes a miss as
  // `false` (mod.rs:733-741, node_specs.get(..).unwrap_or(false)).  It stays out of the engine's table.
  std::vector<std::string> solo_ids;
  solo_ids.reserve(all_solo_ids.size());
  for (const auto& gid : all_solo_ids) {
    const auto g = p->groups.find(gid);
    if (g == p->groups.end() || g->second.nodes.empty()) continue;
    if (p->node_index.find(g->second.nodes[0]) == p->node_index.end()) continue;
    solo_ids.push_back(gid);
  }
  if (solo_ids.size() < 2) return PM_OK;
  const uint32_t W = (uint32_t)solo_ids.size();
  std::vector<pm_worker_a> wa(W);
  std::vector<pm_worker_b> wb(W);
  std::vector<double> lat(W), lon(W);
  // (no address ranks: execute_group_merge puts the merged group's nodes in BTreeSet order from the strings themselves)
  std::vector<const NodeRec*> recs(W);
  for (uint32_t i = 0; i < W; ++i) {
    const Group& g = p->groups.at(solo_ids[i]);
    const NodeRec& n = p->nodes[p->node_index.at(g.nodes[0])];
    recs[i] = &n;
    wa[i] = n.a;
    wb[i] = n.b;
    // find_compatible_solo_groups (mod.rs:712-749) looks at compute specs only
    wa[i].flags = n.a.flags | PM_W_HEALTHY | PM_W_P2P | (n.has_loc ? PM_W_HAS_LOC : 0u);
    lat[i] = n.lat;
    lon[i] = n.lon;
  }

  const bool prox = p->policy.proximity_enabled != 0;
  std::vector<pm_ask> asks;
  std::vector<pm_gpu_opt> opts;
  std::vector<const Config*> ask_cfg;
  for (const Config* c : configs) {
    if (c->max_group_size < 2) continue;          // a batch of one group is never beneficial (mod.rs:868)
    pm_ask a = c->ask;
    a.opt_off = (uint32_t)opts.size();
    // first-fit batches are cut like formation chunks; a tail merges iff it has >= max(min, 2) groups
    a.min_group_size = prox ? c->min_group_size : std::max<uint32_t>(c->min_group_size, 2);
    a.max_group_size = c->max_group_size;
    opts.insert(opts.end(), c->opts.begin(), c->opts.end());
    asks.push_back(a);
    ask_cfg.push_back(c);
  }
  if (asks.empty()) return PM_OK;
  const uint32_t* bits = nullptr;
  uint32_t npat = 0, nmod = 0, words = 1;
  int rc = pm_interner_table(p->interner, &bits, &npat, &nmod, &words);
  if (rc != PM_OK) return p->fail(rc, "pm_interner_table");
  // merging works on its own small table (the nodes of solo groups only): a sibling engine, so that the formation
  // pass's resident worker table stays where it is.  Over a pm_multi it is device 0's: the table is small.
  if (!p->merge_engine) {
    rc = pm_create_sibling(p->dev.first(), &p->merge_engine);
    if (rc != PM_OK) return p->fail(rc, "pm_create_sibling");
  }
  pm_engine* const eng = p->merge_engine;
  auto chk = [&](int r, const char* what) {
    if (r != PM_OK) {
      const char* m = pm_last_error(eng);
      p->err = std::string(what) + ": " + (m ? m : "");
    }
    return r;
  };
  if ((rc = chk(pm_set_asks(eng, asks.data(), (uint32_t)asks.size(), opts.data(), (uint32_t)opts.size()), "pm_set_asks"))) return rc;
  if ((rc = chk(pm_set_model_table(eng, bits, npat, nmod, words), "pm_set_model_table"))) return rc;
  if ((rc = chk(pm_set_worker_count(eng, W), "pm_set_worker_count"))) return rc;
  if ((rc = chk(pm_upsert_workers(eng, wa.data(), wb.data(), 0, W), "pm_upsert_workers"))) return rc;
  if ((rc = chk(pm_set_worker_locations(eng, lat.data(), lon.data(), 0, W), "pm_set_worker_locations"))) return rc;
  if ((rc = chk(pm_stream_sync(eng), "pm_stream_sync"))) return rc;
  if ((rc = chk(pm_match(eng, (prox ? PM_MODE_PROXIMITY_MERGE : PM_MODE_FIRST_FIT) | PM_PATH_FUSED | PM_NO_ASK_STATS), "pm_match"))) return rc;
  pm_result res{};
  if ((rc = chk(pm_fetch_result(eng, &res), "pm_fetch_result"))) return rc;
  for (uint32_t g = 0; g < res.n_groups; ++g) {
    std::vector<std::string> ids;
    for (uint32_t m = res.group_off[g]; m < res.group_off[g + 1]; ++m) ids.push_back(solo_ids[res.group_members[m]]);
    merged->emplace_back(ask_cfg[res.group_ask[g]], std::move(ids));
  }
  return PM_OK;
}

int pm_plugin_try_merge_solo_groups(pm_plugin* p, uint32_t* n_merged) try {
  if (!p) return PM_E_INVALID;
  std::lock_guard<std::mutex> loop_lk(p->loop_mu);
  std::lock_guard<std::shared_mutex> lk(p->mu);   // solo groups are few: the whole merge pass stays under the table lock
  if (n_merged) *n_merged = 0;
  if (!p->dev) return p->fail(PM_E_NO_DEVICE, "no engine attached: merging has no CPU path");
  auto solo_list = [&]() {
    std::vector<std::string> ids;  // std::map iterates in id order == get_all_groups() order
    for (const auto& kv : p->groups)
      if (kv.second.nodes.size() == 1) ids.push_back(kv.first);
    return ids;
  };
  {
    size_t n_solo = 0;
    for (const auto& kv : p->groups)
      if (kv.second.nodes.size() == 1 && ++n_solo >= 2) break;
    if (n_solo < 2) return PM_OK;                                  // mod.rs:640-644
  }
  if (!p->policy.task_switching_enabled) return PM_OK;            // should_switch_tasks, mod.rs:263-265
  const auto configs = p->available_configurations();

  // execute_group_merge (mod.rs:876-971)
  auto apply = [&](const Config* cfg, const std::vector<std::string>& ids) {
    Group merged;
    char idbuf[32];
    std::snprintf(idbuf, sizeof idbuf, "%llx", (unsigned long long)p->next_group_id++);
    merged.id = idbuf;
    merged.configuration_name = cfg->name;
    merged.created_at_ms = (int64_t)std::time(nullptr) * 1000;
    for (const auto& gid : ids) merged.nodes.push_back(p->groups.at(gid).nodes[0]);
    std::sort(merged.nodes.begin(), merged.nodes.end());           // BTreeSet<String>
    // find_best_task_for_group (mod.rs:1122-1189), determinised to the NewestTask rule
    const TaskRec* chosen = p->task_for_configuration(cfg->name);
    for (const auto& gid : ids) p->dissolve(gid);
    for (const auto& n : merged.nodes) p->map_node(n, merged.id);
    if (chosen) p->group_task[merged.id] = chosen->id;              // SET NX on a fresh key
    p->groups.emplace(merged.id, std::move(merged));
    if (n_merged) ++*n_merged;
  };

  if (p->policy.prefer_larger_groups) {
    std::vector<std::pair<const Config*, std::vector<std::string>>> merged;
    int rc = merge_pass(p, configs, solo_list(), &merged);
    if (rc != PM_OK) return rc;
    for (const auto& m : merged) apply(m.first, m.second);
  } else {
    // a batch that contains a group holding a task is refused and ends the configuration
    // (mod.rs:277-287, :704): one pass per configuration, truncated at the first such batch
    for (const Config* c : configs) {
      const auto solos = solo_list();
      if (solos.size() < 2) break;
      std::vector<std::pair<const Config*, std::vector<std::string>>> merged;
      int rc = merge_pass(p, {c}, solos, &merged);
      if (rc != PM_OK) return rc;
      for (const auto& m : merged) {
        bool tasked = false;
        for (const auto& gid : m.second)
          if (p->current_group_task(gid)) tasked = true;
        if (tasked) break;
        apply(m.first, m.second);
      }
    }
  }
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

static void group_json(const pm_plugin* p, const Group& g, std::string& out) {
  out += "{\"id\":";
  json_str(out, g.id);
  out += ",\"nodes\":[";
  for (size_t i = 0; i < g.nodes.size(); ++i) {
    if (i) out += ',';
    json_str(out, g.nodes[i]);
  }
  out += "],\"configuration_name\":";
  json_str(out, g.configuration_name);
  auto it = p->group_task.find(g.id);
  out += ",\"task_id\":";
  if (it == p->group_task.end()) out += "null";
  else json_str(out, it->second);
  out += '}';
}

static int emit(pm_plugin* p, const std::string& s, char* buf, size_t len) {
  if (!buf || len < s.size() + 1) return p->fail(PM_E_NOMEM, "output buffer too small");
  std::memcpy(buf, s.c_str(), s.size() + 1);
  return PM_OK;
}

// the key the storage route writes per requested upload (consumed by scheduler_impl.rs:131-157)
int pm_plugin_record_upload(pm_plugin* p, const char* address, const char* group_id, const char* file_name) try {
  if (!p || !address || !group_id || !file_name) return PM_E_INVALID;
  PM_CANON(address);
  std::lock_guard<std::shared_mutex> lk(p->mu);
  p->upload_keys.insert(std::string("upload:") + address + ":" + group_id + ":" + file_name);
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// get_node_group (mod.rs:324-337): JSON NodeGroup or "null"
int pm_plugin_get_node_group(pm_plugin* p, const char* address, char* buf, size_t len) try {
  if (!p || !address) return PM_E_INVALID;
  PM_CANON(address);
  std::lock_guard<std::shared_mutex> lk(p->mu);
  std::string out = "null";
  auto it = p->node_to_group.find(address);
  if (it != p->node_to_group.end()) {
    auto g = p->groups.find(it->second);
    if (g != p->groups.end()) {
      out.clear();
      group_json(p, g->second, out);
    }
  }
  return emit(p, out, buf, len);
} catch (...) { return pm_guard_rc(); }

// get_all_groups (mod.rs:1006-1044): sorted by id
int pm_plugin_get_all_groups(pm_plugin* p, char* buf, size_t len) try {
  if (!p) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  std::string out = "[";
  bool first = true;
  for (const auto& kv : p->groups) {
    if (!first) out += ',';
    first = false;
    group_json(p, kv.second, out);
  }
  out += ']';
  return emit(p, out, buf, len);
} catch (...) { return pm_guard_rc(); }

// get_group_by_id (mod.rs:1046-1055): JSON NodeGroup or "null"
int pm_plugin_get_group_by_id(pm_plugin* p, const char* group_id, char* buf, size_t len) try {
  if (!p || !group_id) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  std::string out = "null";
  auto g = p->groups.find(group_id);
  if (g != p->groups.end()) {
    out.clear();
    group_json(p, g->second, out);
  }
  return emit(p, out, buf, len);
} catch (...) { return pm_guard_rc(); }

// handle_group_not_found (mod.rs:1073-1119): walk get_all_groups() (id order); the first group without a
// current task takes the orphaned one (assign_task_to_group = SET NX, mod.rs:471-476).  Finding none is not
// an error (the reference logs a warning and returns Ok).
int pm_plugin_handle_group_not_found(pm_plugin* p, const char* group_id, const char* task_id, uint32_t* reassigned) try {
  if (!p || !group_id || !task_id) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  if (reassigned) *reassigned = 0;
  for (const auto& kv : p->groups) {
    if (p->current_group_task(kv.first)) continue;
    if (p->group_task.count(kv.first)) continue;   // SET NX lost
    p->group_task[kv.first] = task_id;
    if (reassigned) *reassigned = 1;
    break;
  }
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// Start-up: a group as the reference stored it (create_group_atomically, mod.rs:299-322) goes back into the tables.
int pm_plugin_restore_group(pm_plugin* p, const char* id, const char* configuration_name, const char* const* nodes,
                            uint32_t n_nodes, const char* task_id, int64_t created_at_ms) try {
  if (!p || !id || !*id || !configuration_name || (n_nodes && !nodes)) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  if (p->groups.count(id)) return p->fail(PM_E_STATE, std::string("pm_plugin_restore_group: group exists: ") + id);
  Group g;
  g.id = id;
  g.configuration_name = configuration_name;
  g.created_at_ms = created_at_ms < 0 ? (int64_t)std::time(nullptr) * 1000 : created_at_ms;
  for (uint32_t i = 0; i < n_nodes; ++i) {
    if (!nodes[i]) return p->fail(PM_E_INVALID, "pm_plugin_restore_group: null node");
    const char* node = nodes[i];
    PM_CANON(node);
    if (p->node_to_group.count(node)) return p->fail(PM_E_STATE, std::string("pm_plugin_restore_group: node already grouped: ") + node);
    g.nodes.emplace_back(node);
  }
  for (size_t i = 0; i < g.nodes.size(); ++i)
    for (size_t j = i + 1; j < g.nodes.size(); ++j)
      if (g.nodes[i] == g.nodes[j]) return p->fail(PM_E_INVALID, "pm_plugin_restore_group: node listed twice");
  std::sort(g.nodes.begin(), g.nodes.end());   // NodeGroup.nodes is a BTreeSet<String>: whatever order the JSON had, it iterates sorted
  // ids this library makes are format!("{:x}", counter): keep the counter ahead of any such id
  {
    unsigned long long v = 0;
    bool hex = g.id.size() <= 16;
    for (char ch : g.id) {
      if (ch >= '0' && ch <= '9') v = (v << 4) | (unsigned)(ch - '0');
      else if (ch >= 'a' && ch <= 'f') v = (v << 4) | (unsigned)(ch - 'a' + 10);
      else { hex = false; break; }
    }
    if (hex && v >= p->next_group_id) p->next_group_id = v + 1;
  }
  for (const auto& n : g.nodes) p->map_node(n, g.id);
  if (task_id && *task_id) p->group_task[g.id] = task_id;
  p->groups.emplace(g.id, std::move(g));
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// The keys a drop-in must leave in Redis for /groups, /nodes, storage routes and the metrics sync to
// keep working unchanged (mod.rs:25-28, 299-322, 471-476): a JSON array of commands
//   ["SET","node_group:<id>","<NodeGroup json>"], ["SADD","orchestrator:groups_index","<id>"],
//   ["HSET","node_to_group","<node>","<id>"], ["SET","group_task:<id>","<task id>"],
//   ["SADD","available_node_group_configs","<name>"].
int pm_plugin_redis_writeback(pm_plugin* p, char* buf, size_t len) try {
  if (!p) return PM_E_INVALID;
  std::lock_guard<std::shared_mutex> lk(p->mu);
  std::string out = "[";
  bool first = true;
  auto cmd = [&](std::initializer_list<std::string> parts) {
    if (!first) out += ',';
    first = false;
    out += '[';
    bool f2 = true;
    for (const auto& s : parts) {
      if (!f2) out += ',';
      f2 = false;
      json_str(out, s);
    }
    out += ']';
  };
  for (const auto& kv : p->groups) {
    const Group& g = kv.second;
    // serde shape of NodeGroup (mod.rs:63-69); created_at as chrono's RFC 3339
    std::string j = "{\"id\":";
    json_str(j, g.id);
    j += ",\"nodes\":[";
    for (size_t i = 0; i < g.nodes.size(); ++i) {
      if (i) j += ',';
      json_str(j, g.nodes[i]);
    }
    j += "],\"created_at\":";
    {
      std::time_t secs = (std::time_t)(g.created_at_ms / 1000);
      std::tm tmv{};
      gmtime_r(&secs, &tmv);
      char tb[64];
      std::snprintf(tb, sizeof tb, "%04d-%02d-%02dT%02d:%02d:%02d.%03dZ", tmv.tm_year + 1900, tmv.tm_mon + 1, tmv.tm_mday,
                    tmv.tm_hour, tmv.tm_min, tmv.tm_sec, (int)(g.created_at_ms % 1000));
      json_str(j, tb);
    }
    j += ",\"configuration_name\":";
    json_str(j, g.configuration_name);
    j += '}';
    cmd({"SET", "node_group:" + g.id, j});
    cmd({"SADD", "orchestrator:groups_index", g.id});
    for (const auto& n : g.nodes) cmd({"HSET", "node_to_group", n, g.id});
    auto t = p->group_task.find(g.id);
    if (t != p->group_task.end()) cmd({"SET", "group_task:" + g.id, t->second});
  }
  for (const auto& name : p->available) cmd({"SADD", "available_node_group_configs", name});
  out += ']';
  if (!buf || len < out.size() + 1) return p->fail(PM_E_NOMEM, "output buffer too small");
  std::memcpy(buf, out.c_str(), out.size() + 1);
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

namespace {

struct Expanded {
  const TaskRec* task = nullptr;
  std::vector<std::pair<std::string, std::string>> env, mounts;
  std::vector<std::string> cmd;
  bool has_env = false, has_cmd = false, has_mounts = false;
};

enum FilterResult { kNoTask = 0, kHasTask = 1, kNeedsUpdate = 2 };

// NodeGroupsPlugin::filter_tasks, scheduler_impl.rs:11-210.
// read_only (the caller holds the table lock shared): nothing is written; a heartbeat whose answer would need a write
// — claiming a task for an idle group (SET NX), dropping a claim on a deleted task — reports kNeedsUpdate and is
// served again under the exclusive lock.  A group that holds a live claim (the steady state) never needs one.
FilterResult node_groups_filter(pm_plugin* p, const std::string& addr, Expanded* out, bool read_only) {
  auto ng = p->node_to_group.find(addr);
  if (ng == p->node_to_group.end()) return kNoTask;          // "Node is not in a group, skipping all tasks"
  auto git = p->groups.find(ng->second);
  if (git == p->groups.end()) return kNoTask;
  const Group& group = git->second;
  auto pos = std::find(group.nodes.begin(), group.nodes.end(), addr);  // get_idx_in_group, mod.rs:424-434
  if (pos == group.nodes.end()) return kNoTask;
  const size_t idx = size_t(pos - group.nodes.begin());

  const TaskRec* current = nullptr;
  if (read_only) {
    auto claim = p->group_task.find(group.id);
    if (claim == p->group_task.end()) {
      if (p->tasks.empty()) return kNoTask;
      // an idle group with no applicable task (allowed_topologies excludes its configuration) writes nothing either:
      // answer from the cached choice under the shared lock, escalate only when a claim would be written
      if (p->claim_cache_valid) {
        auto cc = p->claim_cache.find(group.configuration_name);
        if (cc != p->claim_cache.end() && cc->second.empty()) return kNoTask;
      }
      return kNeedsUpdate;
    }
    current = p->find_task(claim->second);
    if (!current) return kNeedsUpdate;                       // stale claim: collected under the exclusive lock
  } else {
    current = p->current_group_task(group.id);
    if (!current) {
      if (p->tasks.empty()) return kNoTask;
      // reference: filter by allowed_topologies then IteratorRandom::choose (scheduler_impl.rs:42-70);
      // determinised to the NewestTask rule (max_by_key over the desc-sorted list = LAST maximum)
      const TaskRec* chosen = p->task_for_configuration(group.configuration_name);
      if (!chosen) return kNoTask;
      if (!p->group_task.count(group.id)) p->group_task[group.id] = chosen->id;   // SET NX, mod.rs:471-476
      current = p->current_group_task(group.id);
      if (!current) return kNoTask;
    }
  }

  const std::string idx_s = std::to_string(idx), size_s = std::to_string(group.nodes.size());
  const std::string& next_addr = group.nodes[(idx + 1) % group.nodes.size()];
  std::string next_p2p;
  auto ni = p->node_index.find(next_addr);
  if (ni != p->node_index.end()) next_p2p = p->nodes[ni->second].p2p_id;
  // SCAN upload:<node>:<group>:*  (scheduler_impl.rs:131-157); LAST_FILE_IDX = count.saturating_sub(1)
  size_t n_up = 0;
  {
    const std::string prefix = "upload:" + addr + ":" + group.id + ":";
    for (auto it = p->upload_keys.lower_bound(prefix); it != p->upload_keys.end() && it->compare(0, prefix.size(), prefix) == 0; ++it) ++n_up;
  }
  const std::string total_upload = std::to_string(n_up), last_file_idx = std::to_string(n_up ? n_up - 1 : 0);
  auto expand = [&](std::string v) {
    v = replace_all(v, "${GROUP_INDEX}", idx_s);
    v = replace_all(v, "${GROUP_SIZE}", size_s);
    v = replace_all(v, "${NEXT_P2P_ADDRESS}", next_p2p);
    v = replace_all(v, "${GROUP_ID}", group.id);
    v = replace_all(v, "${TOTAL_UPLOAD_COUNT}", total_upload);
    v = replace_all(v, "${LAST_FILE_IDX}", last_file_idx);
    return v;
  };
  out->task = current;
  out->env = current->env;   // env_vars.unwrap_or_default()
  bool have_gi = false;
  for (auto& kv : out->env)
    if (kv.first == "GROUP_INDEX") { kv.second = idx_s; have_gi = true; }
  if (!have_gi) out->env.emplace_back("GROUP_INDEX", idx_s);
  for (auto& kv : out->env) kv.second = expand(kv.second);
  out->has_env = true;
  out->has_cmd = current->has_cmd;
  for (const auto& a : current->cmd) out->cmd.push_back(expand(a));
  out->has_mounts = current->has_mounts;
  for (const auto& m : current->mounts)
    out->mounts.emplace_back(replace_all(m.first, "${GROUP_ID}", group.id), replace_all(m.second, "${GROUP_ID}", group.id));
  return kHasTask;
}

void task_json(const Expanded& e, std::string& out) {
  const TaskRec& t = *e.task;
  out += "{\"name\":"; json_str(out, t.name);
  out += ",\"id\":"; json_str(out, t.id);
  out += ",\"image\":"; json_str(out, t.image);
  out += ",\"env_vars\":";
  if (!e.has_env) out += "null";
  else {
    out += '{';
    for (size_t i = 0; i < e.env.size(); ++i) {
      if (i) out += ',';
      json_str(out, e.env[i].first); out += ':'; json_str(out, e.env[i].second);
    }
    out += '}';
  }
  out += ",\"cmd\":";
  if (!e.has_cmd) out += "null";
  else {
    out += '[';
    for (size_t i = 0; i < e.cmd.size(); ++i) { if (i) out += ','; json_str(out, e.cmd[i]); }
    out += ']';
  }
  out += ",\"created_at\":" + std::to_string(t.created_at);
  out += ",\"volume_mounts\":";
  if (!e.has_mounts) out += "null";
  else {
    out += '[';
    for (size_t i = 0; i < e.mounts.size(); ++i) {
      if (i) out += ',';
      out += "{\"host_path\":"; json_str(out, e.mounts[i].first);
      out += ",\"container_path\":"; json_str(out, e.mounts[i].second); out += '}';
    }
    out += ']';
  }
  out += '}';
}

}  // namespace

// Scheduler::get_task_for_node (scheduler/mod.rs:26-74).  Writes the heartbeat payload
// {"current_task": Task|null} (crates/shared/src/models/heartbeat.rs:7-22).
// builds {"current_task": ...} for one heartbeat.  Returns kNeedsUpdate only when read_only.
static FilterResult heartbeat_answer(pm_plugin* p, const std::string& addr, bool read_only, std::string* out_json) {
  Expanded e;
  FilterResult have = kNoTask;
  if (!p->templates.empty()) {  // plugin chain = [NodeGroupsPlugin]
    have = node_groups_filter(p, addr, &e, read_only);
    if (have == kNeedsUpdate) return have;
  } else if (!p->tasks.empty()) {  // Scheduler::new pushes NewestTaskPlugin when no plugin is configured
    // max_by_key over get_all_tasks() (stable sort, created_at desc) = the LAST task of the newest timestamp in
    // store order; cached until the task list changes
    if (!p->newest_valid) {
      if (read_only) return kNeedsUpdate;
      size_t best = 0;
      for (size_t i = 1; i < p->tasks.size(); ++i)
        if (p->tasks[i].created_at >= p->tasks[best].created_at) best = i;
      p->newest_pos = best;
      p->newest_valid = true;
    }
    const TaskRec* chosen = &p->tasks[p->newest_pos];
    e.task = chosen;
    e.env = chosen->env; e.has_env = chosen->has_env;
    e.cmd = chosen->cmd; e.has_cmd = chosen->has_cmd;
    e.mounts = chosen->mounts; e.has_mounts = chosen->has_mounts;
    have = kHasTask;
  }
  std::string& out = *out_json;
  out = "{\"current_task\":";
  if (have == kNoTask) {
    out += "null}";
    return kNoTask;
  }
  // scheduler/mod.rs:34-70: ${TASK_ID}, ${NODE_ADDRESS} (+ ${TIMESTAMP} in volume mounts)
  const std::string& tid = e.task->id;
  auto expand = [&](std::string v) { return replace_all(replace_all(v, "${TASK_ID}", tid), "${NODE_ADDRESS}", addr); };
  if (e.has_env) for (auto& kv : e.env) kv.second = expand(kv.second);
  if (e.has_cmd) for (auto& a : e.cmd) a = expand(a);
  if (e.has_mounts) {
    const std::string ts = std::to_string((long long)std::time(nullptr));
    for (auto& m : e.mounts) {
      m.first = replace_all(expand(m.first), "${TIMESTAMP}", ts);
      m.second = replace_all(expand(m.second), "${TIMESTAMP}", ts);
    }
  }
  task_json(e, out);
  out += '}';
  return kHasTask;
}

// Heartbeats take the table lock SHARED and answer from what is there (group, claim, task); only a heartbeat that has
// to write — the first one of an idle group, a claim on a deleted task, a cold NewestTask cache — repeats under the
// exclusive lock.  Every table update elsewhere in this file is exclusive.
int pm_scheduler_get_task_for_node(pm_plugin* p, const char* address, char* buf, size_t len) try {
  if (!p || !address) return PM_E_INVALID;
  PM_CANON(address);
  const std::string addr(address);
  std::string out;
  {
    std::shared_lock<std::shared_mutex> rd(p->mu);
    if (heartbeat_answer(p, addr, /*read_only=*/true, &out) != kNeedsUpdate && buf && len >= out.size() + 1) {
      std::memcpy(buf, out.c_str(), out.size() + 1);
      return PM_OK;
    }
  }
  std::lock_guard<std::shared_mutex> lk(p->mu);
  heartbeat_answer(p, addr, /*read_only=*/false, &out);
  return emit(p, out, buf, len);
} catch (...) { return pm_guard_rc(); }

}  // extern "C"
