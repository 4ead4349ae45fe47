// pm_oracle.cpp — CPU ORACLE.  TEST INFRASTRUCTURE, NOT PRODUCT CODE.
// See pm_oracle.h for scope, provenance and the determinisation rules.
// Every function cites the reference lines (PrimeIntellect-ai/protocol @ 1bb7f87c)
// it restates.  Abbreviations:
//   node.rs = crates/shared/src/models/node.rs
//   ng/mod.rs = crates/orchestrator/src/plugins/node_groups/mod.rs
// Build: see oracle/Makefile (-O2 -ffp-contract=off: Rust does not contract
// a*b+c into FMA, and haversine ordering must match a stock Linux build).
#include "pm_oracle.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <optional>
#include <set>
#include <string>
#include <thread>
#include <vector>
#include <queue>

namespace {

using u32 = uint32_t;
using u64 = uint64_t;
template <class T> using Opt = std::optional<T>;

// ---------------------------------------------------------------- model types
// node.rs:58-70
struct GpuRequirements {
  Opt<u32> count;
  Opt<std::string> model;
  Opt<u32> memory_mb, memory_mb_min, memory_mb_max, total_memory_min, total_memory_max;
};
// node.rs:153-157
struct CpuSpecs {
  Opt<u32> cores;
};
// node.rs:49-56
struct ComputeRequirements {
  std::vector<GpuRequirements> gpu;
  Opt<CpuSpecs> cpu;
  Opt<u32> ram_mb, storage_gb;
};
// node.rs:72-78
struct GpuSpecs {
  Opt<u32> count;
  Opt<std::string> model;
  Opt<u32> memory_mb;
};
// node.rs:25-35
struct ComputeSpecs {
  Opt<GpuSpecs> gpu;
  Opt<CpuSpecs> cpu;
  Opt<u32> ram_mb, storage_gb;
};

// ------------------------------------------------------------- string helpers
// Rust str::trim() strips Unicode White_Space; requirement strings are ASCII
// (env/JSON config), so ASCII whitespace is restated here.
bool is_ws(unsigned char c) { return c == ' ' || (c >= 0x09 && c <= 0x0d); }
std::string trim(const std::string& s) {
  size_t b = 0, e = s.size();
  while (b < e && is_ws((unsigned char)s[b])) ++b;
  while (e > b && is_ws((unsigned char)s[e - 1])) --e;
  return s.substr(b, e - b);
}
// str::to_lowercase restricted to ASCII (model names are ASCII).
std::string to_lowercase(std::string s) {
  for (auto& c : s)
    if (c >= 'A' && c <= 'Z') c = char(c - 'A' + 'a');
  return s;
}
std::string replace_char(std::string s, char from, const char* to) {
  std::string out;
  for (char c : s) {
    if (c == from) out += to;
    else out += c;
  }
  return out;
}
bool contains(const std::string& hay, const std::string& needle) {
  return hay.find(needle) != std::string::npos;
}
// str::parse::<u32>(): optional leading '+', then one or more ASCII digits, no
// whitespace, overflow is an error.
bool parse_u32(const std::string& s, u32* out) {
  size_t i = 0;
  if (!s.empty() && s[0] == '+') i = 1;
  if (i >= s.size()) return false;
  u64 v = 0;
  for (; i < s.size(); ++i) {
    if (s[i] < '0' || s[i] > '9') return false;
    v = v * 10 + u64(s[i] - '0');
    if (v > 0xFFFFFFFFull) return false;
  }
  *out = u32(v);
  return true;
}

// ------------------------------------------------------------------- parser
// ComputeRequirements::from_str, node.rs:180-374.
// Returns false and sets err on Err(..).  The two `.unwrap()`s on a bad number
// inside the min/max cross-checks (node.rs:250,275,295,315) would panic in the
// reference; they are reported as errors here.
bool parse_requirements(const std::string& s, ComputeRequirements* out, std::string* err) {
  ComputeRequirements requirements;
  GpuRequirements current;
  bool gpu_spec_started = false;

  size_t pos = 0;
  while (pos <= s.size()) {  // s.split(';')
    size_t semi = s.find(';', pos);
    std::string part = trim(s.substr(pos, semi == std::string::npos ? std::string::npos : semi - pos));
    pos = (semi == std::string::npos) ? s.size() + 1 : semi + 1;
    if (part.empty()) continue;

    size_t eq = part.find('=');  // splitn(2, '=')
    if (eq == std::string::npos) {
      *err = "Invalid key-value pair format: '" + part + "'";
      return false;
    }
    std::string key = trim(part.substr(0, eq));
    std::string value = trim(part.substr(eq + 1));
    u32 v = 0;
    auto need_u32 = [&](const char* k) {
      if (!parse_u32(value, &v)) {
        *err = std::string("Invalid ") + k + " value '" + value + "'";
        return false;
      }
      return true;
    };

    if (key == "gpu:count") {  // node.rs:203-216
      if (gpu_spec_started && current.count.has_value()) {
        requirements.gpu.push_back(current);
        current = GpuRequirements{};
      }
      gpu_spec_started = true;
      if (!need_u32("gpu:count")) return false;
      current.count = v;
    } else if (key == "gpu:model") {  // node.rs:217-222
      gpu_spec_started = true;
      current.model = value;
    } else if (key == "gpu:memory_mb") {  // node.rs:223-238
      gpu_spec_started = true;
      if (current.memory_mb_min || current.memory_mb_max) {
        *err = "Cannot specify both exact memory and min/max memory";
        return false;
      }
      if (!need_u32("gpu:memory_mb")) return false;
      current.memory_mb = v;
    } else if (key == "gpu:memory_mb_min") {  // node.rs:239-262
      gpu_spec_started = true;
      if (current.memory_mb) {
        *err = "Cannot specify both exact memory and min/max memory";
        return false;
      }
      if (current.memory_mb_max) {
        if (!need_u32("gpu:memory_mb_min")) return false;  // reference: unwrap() panic
        if (*current.memory_mb_max < v) {
          *err = "Invalid gpu:memory_mb_min value '" + value + "': min value is greater than max value";
          return false;
        }
      }
      if (!need_u32("gpu:memory_mb_min")) return false;
      current.memory_mb_min = v;
    } else if (key == "gpu:memory_mb_max") {  // node.rs:263-287
      gpu_spec_started = true;
      if (current.memory_mb) {
        *err = "Cannot specify both exact memory and min/max memory";
        return false;
      }
      if (current.memory_mb_min) {
        if (!need_u32("gpu:memory_mb_max")) return false;
        if (*current.memory_mb_min > v) {
          *err = "Invalid gpu:memory_mb_max value '" + value + "': max value is less than min value";
          return false;
        }
      }
      if (!need_u32("gpu:memory_mb_max")) return false;
      current.memory_mb_max = v;
    } else if (key == "gpu:total_memory_min") {  // node.rs:289-308
      gpu_spec_started = true;
      if (current.total_memory_max) {
        if (!need_u32("gpu:total_memory_min")) return false;
        if (*current.total_memory_max < v) {
          *err = "Invalid gpu:total_memory_min value '" + value + "': min value is greater than max value";
          return false;
        }
      }
      if (!need_u32("gpu:total_memory_min")) return false;
      current.total_memory_min = v;
    } else if (key == "gpu:total_memory_max") {  // node.rs:309-328
      gpu_spec_started = true;
      if (current.total_memory_min) {
        if (!need_u32("gpu:total_memory_max")) return false;
        if (*current.total_memory_min > v) {
          *err = "Invalid gpu:total_memory_max value '" + value + "': max value is less than min value";
          return false;
        }
      }
      if (!need_u32("gpu:total_memory_max")) return false;
      current.total_memory_max = v;
    } else if (key == "cpu:cores") {  // node.rs:330-338
      if (!need_u32("cpu:cores")) return false;
      CpuSpecs cpu = requirements.cpu.value_or(CpuSpecs{});
      cpu.cores = v;
      requirements.cpu = cpu;
    } else if (key == "ram_mb") {  // node.rs:341-347
      if (!need_u32("ram_mb")) return false;
      requirements.ram_mb = v;
    } else if (key == "storage_gb") {  // node.rs:348-354
      if (!need_u32("storage_gb")) return false;
      requirements.storage_gb = v;
    } else {  // node.rs:355
      *err = "Unknown requirement key: '" + key + "'";
      return false;
    }
  }
  // node.rs:359-370
  if (gpu_spec_started &&
      (current.count || current.model || current.memory_mb || current.memory_mb_min ||
       current.memory_mb_max || current.total_memory_min || current.total_memory_max)) {
    requirements.gpu.push_back(current);
  }
  *out = requirements;
  return true;
}

// -------------------------------------------------------------------- meets
// node.rs:463-484 (model clause of GpuSpecs::meets)
bool model_matches(const std::string& spec_model, const std::string& req_model) {
  std::string normalized_spec = replace_char(to_lowercase(spec_model), ' ', "_");
  size_t pos = 0;
  while (pos <= req_model.size()) {  // req_model.split(',')
    size_t comma = req_model.find(',', pos);
    std::string m = req_model.substr(pos, comma == std::string::npos ? std::string::npos : comma - pos);
    pos = (comma == std::string::npos) ? req_model.size() + 1 : comma + 1;
    std::string normalized_req = replace_char(to_lowercase(trim(m)), ' ', "_");
    std::string spec_no_underscore = replace_char(normalized_spec, '_', "");
    std::string req_no_underscore = replace_char(normalized_req, '_', "");
    if (contains(normalized_spec, normalized_req) || contains(normalized_req, normalized_spec) ||
        contains(spec_no_underscore, req_no_underscore) ||
        contains(req_no_underscore, spec_no_underscore))
      return true;
  }
  return false;
}

// GpuSpecs::meets, node.rs:443-527
bool gpu_meets(const GpuSpecs& self, const GpuRequirements& requirement) {
  if (requirement.count) {  // :447-461
    u32 req_count = *requirement.count;
    if (!self.count) {
      if (req_count > 0) return false;
    } else if (*self.count != req_count) {
      return false;
    }
  }
  if (requirement.model) {  // :463-484
    if (!(self.model && model_matches(*self.model, *requirement.model))) return false;
  }
  if (requirement.memory_mb) {  // :487-491  is_none_or(spec < req)
    if (!self.memory_mb || *self.memory_mb < *requirement.memory_mb) return false;
  }
  if (requirement.memory_mb_min) {  // :494-498
    if (!self.memory_mb || *self.memory_mb < *requirement.memory_mb_min) return false;
  }
  if (requirement.memory_mb_max) {  // :499-503
    if (!self.memory_mb || *self.memory_mb > *requirement.memory_mb_max) return false;
  }
  if (requirement.total_memory_min && self.count && self.memory_mb) {  // :506-513
    u32 total_memory = *self.count * *self.memory_mb;                  // wraps (release build)
    if (total_memory < *requirement.total_memory_min) return false;
  }
  if (requirement.total_memory_max && self.count && self.memory_mb) {  // :515-522
    u32 total_memory = *self.count * *self.memory_mb;
    if (total_memory > *requirement.total_memory_max) return false;
  }
  return true;
}

// CpuSpecs::meets, node.rs:529-541
bool cpu_meets(const CpuSpecs& self, const CpuSpecs& requirement) {
  if (requirement.cores) {
    if (!self.cores || *self.cores < *requirement.cores) return false;
  }
  return true;
}

// ComputeSpecs::meets, node.rs:377-441 (the info!/debug! logging is omitted)
bool specs_meet(const ComputeSpecs& self, const ComputeRequirements& requirements) {
  if (requirements.cpu) {  // :381-393
    if (!(self.cpu && cpu_meets(*self.cpu, *requirements.cpu))) return false;
  }
  if (requirements.ram_mb) {  // :396-404
    if (!self.ram_mb || *self.ram_mb < *requirements.ram_mb) return false;
  }
  if (requirements.storage_gb) {  // :407-418
    if (!self.storage_gb || *self.storage_gb < *requirements.storage_gb) return false;
  }
  if (!requirements.gpu.empty()) {  // :420-435
    if (!self.gpu) return false;
    bool any = false;
    for (const auto& req_gpu : requirements.gpu)
      if (gpu_meets(*self.gpu, req_gpu)) {
        any = true;
        break;
      }
    if (!any) return false;
  }
  return true;
}

struct Location {
  double latitude, longitude;
};
// crates/orchestrator/src/models/node.rs:10-37 (fields on the path only)
struct Node {
  std::string address;
  u32 status;
  bool has_p2p, assigned;
  Opt<ComputeSpecs> compute_specs;
  Opt<Location> location;
  u32 index;  // input row
};

Node node_from_c(const orc_node& n, u32 index) {
  Node out;
  out.address = n.address ? n.address : "";
  out.status = n.status;
  out.has_p2p = (n.has & ORC_HAS_P2P) != 0;
  out.assigned = (n.has & ORC_ASSIGNED) != 0;
  out.index = index;
  if (n.has & ORC_HAS_SPECS) {
    ComputeSpecs s;
    if (n.has & ORC_HAS_GPU) {
      GpuSpecs g;
      if (n.has & ORC_HAS_GPU_COUNT) g.count = n.gpu_count;
      if (n.has & ORC_HAS_GPU_MODEL) g.model = std::string(n.gpu_model ? n.gpu_model : "");
      if (n.has & ORC_HAS_GPU_MEM) g.memory_mb = n.gpu_mem_mb;
      s.gpu = g;
    }
    if (n.has & ORC_HAS_CPU) {
      CpuSpecs c;
      if (n.has & ORC_HAS_CPU_CORES) c.cores = n.cpu_cores;
      s.cpu = c;
    }
    if (n.has & ORC_HAS_RAM) s.ram_mb = n.ram_mb;
    if (n.has & ORC_HAS_STORAGE) s.storage_gb = n.storage_gb;
    out.compute_specs = s;
  }
  if (n.has & ORC_HAS_LOC) out.location = Location{n.lat, n.lon};
  return out;
}

// ng/mod.rs:206-215
bool is_node_compatible_with_config(const ComputeRequirements* reqs, const Node& node) {
  if (reqs && node.compute_specs) return specs_meet(*node.compute_specs, *reqs);
  if (!reqs) return true;
  return false;
}

// ng/mod.rs:218-231.  f64::to_radians is `self * (PI / 180.0)`; powi(2) is x*x.
double calculate_distance(const Location& loc1, const Location& loc2) {
  const double EARTH_RADIUS_KM = 6371.0;
  const double RADS_PER_DEG = 3.14159265358979323846264338327950288 / 180.0;
  double lat1_rad = loc1.latitude * RADS_PER_DEG;
  double lat2_rad = loc2.latitude * RADS_PER_DEG;
  double delta_lat = (loc2.latitude - loc1.latitude) * RADS_PER_DEG;
  double delta_lon = (loc2.longitude - loc1.longitude) * RADS_PER_DEG;
  double s1 = std::sin(delta_lat / 2.0);
  double s2 = std::sin(delta_lon / 2.0);
  double a = s1 * s1 + std::cos(lat1_rad) * std::cos(lat2_rad) * (s2 * s2);
  // determinisation rule 7: rounding can push a out of [0, 1], its exact range for any real latitudes — above 1 for
  // (near-)antipodal points, below 0 for one place written twice with a latitude beyond ±90 (the cosine product is
  // then negative and a is a difference).  sqrt of a negative is NaN, and the reference's stable sort with
  // partial_cmp(..).unwrap_or(Equal) is then no total order (its result depends on the sort's internal comparison
  // sequence; handing std::stable_sort a comparator that is no strict weak order is undefined behaviour).  a is
  // clamped into [0, 1] here and on the device.
  if (a > 1.0) a = 1.0;
  if (a < 0.0) a = 0.0;
  double c = 2.0 * std::atan2(std::sqrt(a), std::sqrt(1.0 - a));
  return EARTH_RADIUS_KM * c;
}

// ng/mod.rs:234-255.  Stable; missing location => f64::MAX; comparator
// recomputes both distances on every call, as the reference does.
void sort_nodes_by_proximity(const Node& reference_node, std::vector<const Node*>& nodes) {
  if (!reference_node.location) return;
  const Location& ref = *reference_node.location;
  std::stable_sort(nodes.begin(), nodes.end(), [&](const Node* a, const Node* b) {
    double dist_a = a->location ? calculate_distance(ref, *a->location) : 1.7976931348623157e308;
    double dist_b = b->location ? calculate_distance(ref, *b->location) : 1.7976931348623157e308;
    return dist_a < dist_b;  // partial_cmp(..).unwrap_or(Equal) == Less
  });
}

// node_store.rs:195-206 status classes: Healthy < Discovered < (others) < Dead
int status_class(u32 st) {
  if (st == ORC_HEALTHY) return 0;
  if (st == ORC_DISCOVERED) return 1;
  if (st == ORC_DEAD) return 3;
  return 2;
}

}  // namespace

struct orc_req {
  ComputeRequirements r;
};

struct orc_groups {
  std::vector<u32> cfg, off, members;
  u64 evals = 0;
};

extern "C" {

orc_req* orc_req_parse(const char* s, char* err, size_t err_len) {
  ComputeRequirements r;
  std::string e;
  if (!parse_requirements(s ? s : "", &r, &e)) {
    if (err && err_len) {
      std::snprintf(err, err_len, "%s", e.c_str());
    }
    return nullptr;
  }
  auto* out = new orc_req;
  out->r = r;
  return out;
}
void orc_req_free(orc_req* r) { delete r; }
uint32_t orc_req_n_gpu(const orc_req* r) { return u32(r->r.gpu.size()); }
int orc_req_gpu_u32(const orc_req* r, uint32_t opt, int field, uint32_t* val) {
  if (opt >= r->r.gpu.size()) return 0;
  const GpuRequirements& g = r->r.gpu[opt];
  const Opt<u32>* f = nullptr;
  switch (field) {
    case 0: f = &g.count; break;
    case 1: f = &g.memory_mb; break;
    case 2: f = &g.memory_mb_min; break;
    case 3: f = &g.memory_mb_max; break;
    case 4: f = &g.total_memory_min; break;
    case 5: f = &g.total_memory_max; break;
    default: return 0;
  }
  if (!f->has_value()) return 0;
  if (val) *val = **f;
  return 1;
}
const char* orc_req_gpu_model(const orc_req* r, uint32_t opt) {
  if (opt >= r->r.gpu.size() || !r->r.gpu[opt].model) return nullptr;
  return r->r.gpu[opt].model->c_str();
}
int orc_req_scalar(const orc_req* r, int field, uint32_t* val) {
  const Opt<u32>* f = nullptr;
  if (field == 0) {
    if (!r->r.cpu) return -1;
    f = &r->r.cpu->cores;
  } else if (field == 1) {
    f = &r->r.ram_mb;
  } else if (field == 2) {
    f = &r->r.storage_gb;
  } else {
    return 0;
  }
  if (!f->has_value()) return 0;
  if (val) *val = **f;
  return 1;
}

int orc_meets(const orc_node* node, const orc_req* req) {
  Node n = node_from_c(*node, 0);
  if (!n.compute_specs) return 0;
  return specs_meet(*n.compute_specs, req->r) ? 1 : 0;
}
int orc_node_compatible(const orc_node* node, const orc_req* req) {
  Node n = node_from_c(*node, 0);
  return is_node_compatible_with_config(req ? &req->r : nullptr, n) ? 1 : 0;
}
int orc_model_matches(const char* spec_model, const char* req_model) {
  return model_matches(spec_model, req_model) ? 1 : 0;
}
double orc_haversine_km(double lat1, double lon1, double lat2, double lon2) {
  return calculate_distance(Location{lat1, lon1}, Location{lat2, lon2});
}

// ng/mod.rs:150-164
void orc_sort_configs(const orc_config* cfgs, uint32_t n, uint32_t* perm_out) {
  std::vector<u32> p(n);
  for (u32 i = 0; i < n; ++i) p[i] = i;
  std::stable_sort(p.begin(), p.end(), [&](u32 ia, u32 ib) {
    const orc_config& a = cfgs[ia];
    const orc_config& b = cfgs[ib];
    if (a.min_group_size != b.min_group_size) return b.min_group_size < a.min_group_size;
    // (Some, None) => Less ; (None, Some) => Greater ; else Equal
    return (a.req != nullptr) && (b.req == nullptr);
  });
  for (u32 i = 0; i < n; ++i) perm_out[i] = p[i];
}

// ng/mod.rs:399-418
uint32_t orc_available_configs(const orc_config* sorted_templates, const uint8_t* enabled,
                               uint32_t n, uint32_t* idx_out) {
  std::vector<u32> p;
  for (u32 i = 0; i < n; ++i)
    if (enabled[i]) p.push_back(i);
  std::stable_sort(p.begin(), p.end(), [&](u32 a, u32 b) {
    return sorted_templates[b].min_group_size < sorted_templates[a].min_group_size;
  });
  for (size_t i = 0; i < p.size(); ++i) idx_out[i] = p[i];
  return u32(p.size());
}

// node_store.rs:195-206
void orc_sort_nodes_by_status(const uint32_t* status, uint32_t n, uint32_t* perm_out) {
  std::vector<u32> p(n);
  for (u32 i = 0; i < n; ++i) p[i] = i;
  std::stable_sort(p.begin(), p.end(),
                   [&](u32 a, u32 b) { return status_class(status[a]) < status_class(status[b]); });
  for (u32 i = 0; i < n; ++i) perm_out[i] = p[i];
}

// try_form_new_groups, ng/mod.rs:478-628 — faithful loop structure.
orc_groups* orc_form_groups(const orc_node* c_nodes, uint32_t n_nodes, const orc_config* cfgs,
                            uint32_t n_cfgs, int proximity) {
  auto* out = new orc_groups;
  out->off.push_back(0);

  // node_store.get_nodes(): stable status-class sort (node_store.rs:195-206)
  std::vector<Node> nodes_in;
  nodes_in.reserve(n_nodes);
  for (u32 i = 0; i < n_nodes; ++i) nodes_in.push_back(node_from_c(c_nodes[i], i));
  std::vector<const Node*> nodes;
  for (auto& n : nodes_in) nodes.push_back(&n);
  std::stable_sort(nodes.begin(), nodes.end(), [](const Node* a, const Node* b) {
    return status_class(a->status) < status_class(b->status);
  });

  // :492-497
  std::vector<const Node*> healthy_nodes;
  for (const Node* n : nodes)
    if (n->status == ORC_HEALTHY && n->has_p2p && !n->assigned) healthy_nodes.push_back(n);

  size_t total_available = healthy_nodes.size();  // :503

  for (u32 ci = 0; ci < n_cfgs; ++ci) {  // :505
    const orc_config& config = cfgs[ci];
    const ComputeRequirements* reqs = config.req ? &config.req->r : nullptr;
    while (total_available >= config.min_group_size) {  // :507
      size_t initial_available = total_available;

      std::vector<const Node*> compatible_nodes;  // :511-515
      for (const Node* n : healthy_nodes) {
        ++out->evals;
        if (is_node_compatible_with_config(reqs, *n)) compatible_nodes.push_back(n);
      }
      if (compatible_nodes.size() < config.min_group_size) break;  // :517

      std::set<std::string> available_nodes;  // BTreeSet<String>
      std::vector<std::string> nodes_to_remove;

      if (proximity) {  // :524-552
        const Node* seed = nullptr;
        for (const Node* n : compatible_nodes)
          if (n->location) {
            seed = n;
            break;
          }
        if (!seed && !compatible_nodes.empty()) seed = compatible_nodes.front();
        if (seed) {
          available_nodes.insert(seed->address);
          nodes_to_remove.push_back(seed->address);
          std::vector<const Node*> remaining_compatible;
          for (const Node* n : compatible_nodes)
            if (n->address != seed->address) remaining_compatible.push_back(n);
          sort_nodes_by_proximity(*seed, remaining_compatible);
          for (const Node* n : remaining_compatible) {
            if (available_nodes.size() >= config.max_group_size) break;
            available_nodes.insert(n->address);
            nodes_to_remove.push_back(n->address);
          }
        }
      } else {  // :553-561
        for (const Node* n : compatible_nodes) {
          if (available_nodes.size() >= config.max_group_size) break;
          available_nodes.insert(n->address);
          nodes_to_remove.push_back(n->address);
        }
      }

      if (available_nodes.size() < config.min_group_size) break;  // :564

      // :569-581 create group (id = running counter; created_at omitted)
      out->cfg.push_back(ci);
      for (const std::string& addr : available_nodes) {
        // map the address back to the input row (first match, as a hash map would)
        for (const Node* n : healthy_nodes)
          if (n->address == addr) {
            out->members.push_back(n->index);
            break;
          }
      }
      out->off.push_back(u32(out->members.size()));

      // :585 healthy_nodes.retain(|n| !nodes_to_remove.contains(addr))
      std::vector<const Node*> kept;
      for (const Node* n : healthy_nodes) {
        bool rm = false;
        for (const std::string& a : nodes_to_remove)
          if (a == n->address) {
            rm = true;
            break;
          }
        if (!rm) kept.push_back(n);
      }
      healthy_nodes.swap(kept);
      total_available = healthy_nodes.size();

      if (total_available == initial_available) break;  // :606
    }
  }
  return out;
}

void orc_groups_free(orc_groups* g) { delete g; }
uint32_t orc_groups_count(const orc_groups* g) { return u32(g->cfg.size()); }
uint32_t orc_groups_members_total(const orc_groups* g) { return u32(g->members.size()); }
const uint32_t* orc_groups_cfg(const orc_groups* g) { return g->cfg.data(); }
const uint32_t* orc_groups_off(const orc_groups* g) { return g->off.data(); }
const uint32_t* orc_groups_members(const orc_groups* g) { return g->members.data(); }
uint64_t orc_groups_evals(const orc_groups* g) { return g->evals; }

// try_merge_solo_groups / try_merge_groups_for_config / find_compatible_solo_groups /
// attempt_group_merge / is_merge_beneficial / should_switch_tasks, ng/mod.rs:631-873, 257-296.
orc_groups* orc_merge_solo_groups(const orc_node* c_nodes, uint32_t n_nodes, const orc_solo* c_solos,
                                  uint32_t n_solos, const orc_config* cfgs, uint32_t n_cfgs,
                                  int proximity, int task_switching_enabled, int prefer_larger_groups) {
  auto* out = new orc_groups;
  out->off.push_back(0);
  std::vector<Node> nodes;
  for (u32 i = 0; i < n_nodes; ++i) nodes.push_back(node_from_c(c_nodes[i], i));
  struct Solo { std::string id; u32 node; bool has_task; };
  std::vector<Solo> all;  // get_all_groups(): sorted by id (:1040); only solo groups matter here
  for (u32 i = 0; i < n_solos; ++i) all.push_back({c_solos[i].id, c_solos[i].node, c_solos[i].has_task != 0});
  std::sort(all.begin(), all.end(), [](const Solo& a, const Solo& b) { return a.id < b.id; });
  if (all.size() < 2) return out;  // :640-644

  for (u32 ci = 0; ci < n_cfgs; ++ci) {  // :654-661, current_groups refreshed per configuration
    const orc_config& config = cfgs[ci];
    const ComputeRequirements* reqs = config.req ? &config.req->r : nullptr;
    // find_compatible_solo_groups (:712-749): specs only, no health/p2p filter
    std::vector<Solo> remaining;
    for (const Solo& g : all) {
      ++out->evals;
      if (is_node_compatible_with_config(reqs, nodes[g.node])) remaining.push_back(g);
    }
    if (remaining.size() < config.min_group_size) continue;  // :687-690
    while (remaining.size() >= config.min_group_size) {       // :694
      // attempt_group_merge (:752-860)
      std::vector<const Solo*> merge_batch;
      std::set<std::string> total_nodes;
      auto in_batch = [&](const Solo* g) {
        for (const Solo* b : merge_batch)
          if (b->id == g->id) return true;
        return false;
      };
      if (proximity) {
        const Solo* seed = nullptr;
        for (const Solo& g : remaining)
          if (nodes[g.node].location) { seed = &g; break; }
        if (seed) {
          merge_batch.push_back(seed);
          total_nodes.insert(nodes[seed->node].address);
          const Location& sl = *nodes[seed->node].location;
          std::vector<std::pair<double, const Solo*>> with_distance;
          for (const Solo& g : remaining)
            if (g.id != seed->id && nodes[g.node].location)
              with_distance.push_back({calculate_distance(sl, *nodes[g.node].location), &g});
          std::stable_sort(with_distance.begin(), with_distance.end(),
                           [](const auto& a, const auto& b) { return a.first < b.first; });
          for (const auto& dg : with_distance) {
            if (total_nodes.size() + 1 <= config.max_group_size) {
              merge_batch.push_back(dg.second);
              total_nodes.insert(nodes[dg.second->node].address);
              if (total_nodes.size() >= config.max_group_size) break;
            }
          }
        }
      }
      if (merge_batch.empty() ||
          (total_nodes.size() < config.max_group_size && total_nodes.size() < config.min_group_size)) {  // :823-848
        if (total_nodes.size() < config.min_group_size) {
          merge_batch.clear();
          total_nodes.clear();
        }
        for (const Solo& g : remaining) {
          if (!in_batch(&g) && total_nodes.size() + 1 <= config.max_group_size) {
            merge_batch.push_back(&g);
            total_nodes.insert(nodes[g.node].address);
            if (total_nodes.size() >= config.max_group_size) break;
          }
        }
      }
      // is_merge_beneficial (:863-873) + should_switch_tasks (:257-296)
      bool ok = merge_batch.size() >= 2 && total_nodes.size() >= 2 && task_switching_enabled;
      if (ok && !prefer_larger_groups)
        for (const Solo* g : merge_batch)
          if (g->has_task) ok = false;
      if (!ok) break;  // :704
      out->cfg.push_back(ci);
      for (const std::string& addr : total_nodes)
        for (const Solo* g : merge_batch)
          if (nodes[g->node].address == addr) { out->members.push_back(g->node); break; }
      out->off.push_back(u32(out->members.size()));
      std::set<std::string> used;
      for (const Solo* g : merge_batch) used.insert(g->id);
      std::vector<Solo> next;
      for (const Solo& g : remaining)
        if (!used.count(g.id)) next.push_back(g);
      remaining.swap(next);
      // the merged groups leave `all` (they are no longer solo groups in the next get_all_groups())
      std::vector<Solo> all_next;
      for (const Solo& g : all)
        if (!used.count(g.id)) all_next.push_back(g);
      all.swap(all_next);
    }
  }
  return out;
}

// newest_task/mod.rs:8-19; Iterator::max_by_key returns the LAST maximum.
uint32_t orc_newest_task(const int64_t* created_at, uint32_t n) {
  if (n == 0) return PM_NONE;
  u32 best = 0;
  for (u32 i = 1; i < n; ++i)
    if (created_at[i] >= created_at[best]) best = i;
  return best;
}

// task_store.rs:79
void orc_sort_tasks(const int64_t* created_at, uint32_t n, uint32_t* perm_out) {
  std::vector<u32> p(n);
  for (u32 i = 0; i < n; ++i) p[i] = i;
  std::stable_sort(p.begin(), p.end(), [&](u32 a, u32 b) { return created_at[b] < created_at[a]; });
  for (u32 i = 0; i < n; ++i) perm_out[i] = p[i];
}

// ng/mod.rs:424-434 over NodeGroup.nodes: BTreeSet<String> (mod.rs:63-69)
int64_t orc_idx_in_group(const char* const* member_addrs, uint32_t n, const char* addr) {
  std::set<std::string> nodes;
  for (u32 i = 0; i < n; ++i) nodes.insert(member_addrs[i]);
  int64_t pos = 0;
  for (const auto& s : nodes) {
    if (s == addr) return pos;
    ++pos;
  }
  return -1;
}

// ------------------------------------------------------------------ SoA side
// The same predicate (ng/mod.rs:206-215 -> node.rs:377-541) on the engine's
// plain-data tables; the model clause is the interned bit test.
int orc_soa_compatible(const pm_worker_a* a, const pm_worker_b* b, const pm_ask* ask,
                       const pm_gpu_opt* opts, const uint32_t* model_bits, uint32_t words) {
  const u32 wf = a->flags;
  if (!(ask->flags & PM_A_HAS_REQ)) return 1;   // (None, _) => true
  if (!(wf & PM_W_HAS_SPECS)) return 0;         // (Some, None) => false
  if (ask->flags & PM_A_REQ_CPU) {              // node.rs:381-393
    if (!(wf & PM_W_HAS_CPU)) return 0;
    if (ask->flags & PM_A_REQ_CPU_CORES) {
      if (!(wf & PM_W_HAS_CPU_CORES) || b->cpu_cores < ask->cpu_cores) return 0;
    }
  }
  if (ask->flags & PM_A_REQ_RAM) {
    if (!(wf & PM_W_HAS_RAM) || b->ram_mb < ask->ram_mb) return 0;
  }
  if (ask->flags & PM_A_REQ_STORAGE) {
    if (!(wf & PM_W_HAS_STORAGE) || b->storage_gb < ask->storage_gb) return 0;
  }
  if (ask->n_opts == 0) return 1;
  if (!(wf & PM_W_HAS_GPU)) return 0;
  for (u32 o = 0; o < ask->n_opts; ++o) {
    const pm_gpu_opt& q = opts[ask->opt_off + o];
    if (q.present & PM_O_COUNT) {
      if (!(wf & PM_W_HAS_GPU_COUNT)) {
        if (q.count > 0) continue;
      } else if (a->gpu_count != q.count) {
        continue;
      }
    }
    if (q.present & PM_O_MODEL) {
      if (!(wf & PM_W_HAS_GPU_MODEL)) continue;
      u32 m = a->model_id;
      if (!((model_bits[size_t(q.pattern_id) * words + (m >> 5)] >> (m & 31)) & 1u)) continue;
    }
    const bool has_mem = (wf & PM_W_HAS_GPU_MEM) != 0;
    if ((q.present & PM_O_MEM) && (!has_mem || a->gpu_mem_mb < q.memory_mb)) continue;
    if ((q.present & PM_O_MEM_MIN) && (!has_mem || a->gpu_mem_mb < q.memory_mb_min)) continue;
    if ((q.present & PM_O_MEM_MAX) && (!has_mem || a->gpu_mem_mb > q.memory_mb_max)) continue;
    if (has_mem && (wf & PM_W_HAS_GPU_COUNT)) {
      u32 total = a->gpu_count * a->gpu_mem_mb;  // wraps
      if ((q.present & PM_O_TOT_MIN) && total < q.total_memory_min) continue;
      if ((q.present & PM_O_TOT_MAX) && total > q.total_memory_max) continue;
    }
    return 1;
  }
  return 0;
}

static inline bool soa_candidate(u32 flags) {
  return (flags & (PM_W_HEALTHY | PM_W_P2P | PM_W_ASSIGNED)) == (PM_W_HEALTHY | PM_W_P2P);
}

static double soa_distance(const double* lat, const double* lon, u32 a, u32 b) {
  return calculate_distance(Location{lat[a], lon[a]}, Location{lat[b], lon[b]});
}

// Same allocator as orc_form_groups on SoA tables.  One compat filter per
// configuration: the reference's per-group re-filter of the remaining nodes
// yields exactly this list minus the members already taken (both modes only
// ever remove members of the list they were drawn from).
orc_groups* orc_soa_form_groups(const pm_worker_a* a, const pm_worker_b* b, uint32_t n_workers,
                                const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts,
                                const uint32_t* model_bits, uint32_t words,
                                const uint32_t* addr_rank, const double* lat, const double* lon,
                                int proximity) {
  auto* out = new orc_groups;
  out->off.push_back(0);
  std::vector<u32> remaining;
  for (u32 w = 0; w < n_workers; ++w)
    if (soa_candidate(a[w].flags)) remaining.push_back(w);
  std::vector<char> taken(n_workers, 0);

  auto emit = [&](u32 ci, std::vector<u32>& mem) {
    std::sort(mem.begin(), mem.end(), [&](u32 x, u32 y) {
      u32 rx = addr_rank ? addr_rank[x] : x, ry = addr_rank ? addr_rank[y] : y;
      return rx < ry;
    });
    out->cfg.push_back(ci);
    for (u32 w : mem) out->members.push_back(w);
    out->off.push_back(u32(out->members.size()));
  };

  for (u32 ci = 0; ci < n_asks; ++ci) {
    const pm_ask& ask = asks[ci];
    const u64 mn = ask.min_group_size, mx = ask.max_group_size;
    if (remaining.size() < mn) continue;  // while total_available >= min (:507)
    std::vector<u32> compat;
    for (u32 w : remaining) {
      ++out->evals;
      if (orc_soa_compatible(&a[w], &b[w], &ask, opts, model_bits, words)) compat.push_back(w);
    }
    size_t n_taken_here = 0;
    if (!proximity) {
      size_t pos = 0;
      for (;;) {
        size_t left = compat.size() - pos;
        if (remaining.size() - n_taken_here < mn) break;  // :507
        if (left < mn) break;                               // :517
        size_t take = std::min<u64>(left, mx);
        if (take < mn) break;  // :564
        std::vector<u32> mem(compat.begin() + pos, compat.begin() + pos + take);
        for (u32 w : mem) taken[w] = 1;
        emit(ci, mem);
        pos += take;
        n_taken_here += take;
        if (take == 0) break;  // :606 no progress
      }
    } else if (proximity == 2 && std::all_of(compat.begin(), compat.end(), [&](u32 w) {
                 return !(a[w].flags & PM_W_HAS_LOC) || std::fabs(lat[w]) <= 90.0;   // the bound needs real latitudes
               })) {
      // Same groups as the branch below (tested against it), without re-sorting every remaining worker for every
      // group: haversine distance >= R * |delta latitude| (a >= sin^2(dlat/2) in calculate_distance), so the located
      // workers are kept in latitude order and a group looks outward from its seed only while that lower bound can
      // still beat its current k-th nearest.  Plan for the device-side sweep (DESIGN.md 6d); here it makes the
      // checker usable at swarm scale.
      const size_t K = compat.size();
      std::vector<char> alive(K, 1);
      std::vector<u32> by_lat;                      // compat indices of located workers, by (latitude, canonical position)
      for (u32 i = 0; i < K; ++i)
        if (a[compat[i]].flags & PM_W_HAS_LOC) by_lat.push_back(i);
      std::sort(by_lat.begin(), by_lat.end(), [&](u32 x, u32 y) {
        const double lx = lat[compat[x]], ly = lat[compat[y]];
        return lx < ly || (lx == ly && x < y);
      });
      const u32 NONE = 0xFFFFFFFFu;
      std::vector<u32> lat_pos(K, NONE), prv(by_lat.size()), nxt(by_lat.size());
      for (u32 r = 0; r < by_lat.size(); ++r) {
        lat_pos[by_lat[r]] = r;
        prv[r] = r ? r - 1 : NONE;
        nxt[r] = r + 1 < by_lat.size() ? r + 1 : NONE;
      }
      auto unlink = [&](u32 i) {                    // compat index i leaves the alive sets
        alive[i] = 0;
        const u32 r = lat_pos[i];
        if (r == NONE) return;
        if (prv[r] != NONE) nxt[prv[r]] = nxt[r];
        if (nxt[r] != NONE) prv[nxt[r]] = prv[r];
      };
      size_t n_alive = K, n_alive_loc = by_lat.size(), ploc = 0, pany = 0;
      const double kRadsPerDeg = 3.14159265358979323846264338327950288 / 180.0;
      for (;;) {
        if (remaining.size() - n_taken_here < mn) break;
        if (n_alive < mn) break;
        std::vector<u32> mem;                       // compat indices
        if (n_alive) {
          u32 seed;
          if (n_alive_loc) {
            while (!(alive[ploc] && lat_pos[ploc] != NONE)) ++ploc;
            seed = u32(ploc);
          } else {
            while (!alive[pany]) ++pany;
            seed = u32(pany);
          }
          const size_t want = std::min<u64>(mx ? mx - 1 : 0, n_alive - 1);
          if (1 + want < mn) break;                 // mem.size() < min: nothing is taken
          mem.push_back(seed);
          if (want && lat_pos[seed] != NONE) {
            typedef std::pair<double, u32> DI;      // (distance, canonical position): max-heap keeps the `want` smallest
            std::priority_queue<DI> heap;
            const double slat = lat[compat[seed]];
            u32 lo = prv[lat_pos[seed]], hi = nxt[lat_pos[seed]];
            auto consider = [&](u32 r) -> bool {    // false: this side cannot improve the result any more
              const u32 i = by_lat[r];
              const double dl = std::fabs(lat[compat[i]] - slat) * kRadsPerDeg;
              const double lb = 6371.0 * dl * (1.0 - 1e-9) - 1e-9;
              if (heap.size() == want && lb > heap.top().first) return false;
              const DI cand(soa_distance(lat, lon, compat[seed], compat[i]), i);
              if (heap.size() < want) heap.push(cand);
              else if (cand < heap.top()) { heap.pop(); heap.push(cand); }
              return true;
            };
            while (lo != NONE || hi != NONE) {
              bool take_lo;
              if (lo == NONE) take_lo = false;
              else if (hi == NONE) take_lo = true;
              else take_lo = (slat - lat[compat[by_lat[lo]]]) <= (lat[compat[by_lat[hi]]] - slat);
              if (take_lo) { if (consider(lo)) lo = prv[lo]; else lo = NONE; }
              else { if (consider(hi)) hi = nxt[hi]; else hi = NONE; }
            }
            std::vector<DI> picked;
            while (!heap.empty()) { picked.push_back(heap.top()); heap.pop(); }
            for (size_t q = picked.size(); q-- > 0;) mem.push_back(picked[q].second);
          }
          // distance f64::MAX (no location), or a seed without location: the next ones in canonical order
          for (size_t q = pany; mem.size() < 1 + want && q < K; ++q) {
            if (!alive[q] || q == seed) continue;
            if (lat_pos[seed] != NONE && lat_pos[q] != NONE) continue;   // located ones were ranked by distance above
            mem.push_back(u32(q));
          }
        }
        if (mem.size() < mn) break;
        std::vector<u32> workers;
        for (u32 i : mem) {
          if (lat_pos[i] != NONE) --n_alive_loc;
          --n_alive;
          unlink(i);
          taken[compat[i]] = 1;
          workers.push_back(compat[i]);
        }
        const size_t took = workers.size();
        emit(ci, workers);
        n_taken_here += took;
        if (took == 0) break;
      }
    } else {
      std::vector<u32> list = compat;  // still-available compatible, canonical order
      for (;;) {
        if (remaining.size() - n_taken_here < mn) break;
        if (list.size() < mn) break;
        std::vector<u32> mem;
        int seed_pos = -1;
        for (size_t i = 0; i < list.size(); ++i)
          if (a[list[i]].flags & PM_W_HAS_LOC) {
            seed_pos = int(i);
            break;
          }
        if (seed_pos < 0 && !list.empty()) seed_pos = 0;
        if (seed_pos >= 0) {
          u32 seed = list[size_t(seed_pos)];
          mem.push_back(seed);
          std::vector<u32> rest;
          for (size_t i = 0; i < list.size(); ++i)
            if (int(i) != seed_pos) rest.push_back(list[i]);
          if (a[seed].flags & PM_W_HAS_LOC) {
            std::vector<double> d(rest.size());
            for (size_t i = 0; i < rest.size(); ++i)
              d[i] = (a[rest[i]].flags & PM_W_HAS_LOC) ? soa_distance(lat, lon, seed, rest[i])
                                                        : 1.7976931348623157e308;
            std::vector<u32> ord(rest.size());
            for (size_t i = 0; i < ord.size(); ++i) ord[i] = u32(i);
            std::stable_sort(ord.begin(), ord.end(), [&](u32 x, u32 y) { return d[x] < d[y]; });
            std::vector<u32> sorted(rest.size());
            for (size_t i = 0; i < ord.size(); ++i) sorted[i] = rest[ord[i]];
            rest.swap(sorted);
          }
          for (u32 w : rest) {
            if (mem.size() >= mx) break;
            mem.push_back(w);
          }
        }
        if (mem.size() < mn) break;
        for (u32 w : mem) taken[w] = 1;
        size_t took = mem.size();
        emit(ci, mem);
        std::vector<u32> next;
        for (u32 w : list)
          if (!taken[w]) next.push_back(w);
        list.swap(next);
        n_taken_here += took;
        if (took == 0) break;
      }
    }
    if (n_taken_here) {
      std::vector<u32> next;
      next.reserve(remaining.size() - n_taken_here);
      for (u32 w : remaining)
        if (!taken[w]) next.push_back(w);
      remaining.swap(next);
    }
  }
  return out;
}

uint64_t orc_soa_eval_matrix(const pm_worker_a* a, const pm_worker_b* b, const pm_ask* asks,
                             const pm_gpu_opt* opts, const uint32_t* model_bits, uint32_t words,
                             uint32_t t0, uint32_t t1, uint32_t w0, uint32_t w1, uint32_t threads,
                             int64_t* cost_out, int64_t* row_best_out, uint32_t* row_count_out,
                             uint32_t* col_first_out) {
  const u32 nt = t1 - t0, nw = w1 - w0;
  if (threads == 0) threads = 1;
  if (col_first_out)
    for (u32 i = 0; i < nw; ++i) col_first_out[i] = PM_NONE;
  // rows are split across threads; col_first needs a min-merge afterwards
  std::vector<std::vector<u32>> col_parts(col_first_out ? threads : 0);
  auto work = [&](u32 tid) {
    std::vector<u32>* cf = nullptr;
    if (col_first_out) {
      col_parts[tid].assign(nw, PM_NONE);
      cf = &col_parts[tid];
    }
    u32 r0 = u32(u64(nt) * tid / threads), r1 = u32(u64(nt) * (tid + 1) / threads);
    for (u32 r = r0; r < r1; ++r) {
      const pm_ask& ask = asks[t0 + r];
      int64_t best = PM_COST_INF;
      u32 count = 0;
      for (u32 c = 0; c < nw; ++c) {
        const u32 w = w0 + c;
        int64_t cost = PM_COST_INF;
        // a first-fit configuration with max_group_size == 0 can never take a worker
        // (ng/mod.rs:555-556): its row of the cost matrix is masked
        if (ask.max_group_size != 0 && soa_candidate(a[w].flags) &&
            orc_soa_compatible(&a[w], &b[w], &ask, opts, model_bits, words)) {
          // packed cost = price << 32 | worker; the price is the extension column (0 in the reference's own modes)
          cost = (int64_t(b[w].ext_ask_price) << 32) | int64_t(w);
          ++count;
          if (cf && (*cf)[c] == PM_NONE) (*cf)[c] = t0 + r;
        }
        if (cost < best) best = cost;
        if (cost_out) cost_out[size_t(r) * nw + c] = cost;
      }
      if (row_best_out) row_best_out[r] = best;
      if (row_count_out) row_count_out[r] = count;
    }
  };
  std::vector<std::thread> pool;
  for (u32 t = 1; t < threads; ++t) pool.emplace_back(work, t);
  work(0);
  for (auto& th : pool) th.join();
  if (col_first_out)
    for (u32 t = 0; t < threads; ++t)
      for (u32 c = 0; c < nw; ++c)
        if (col_parts[t][c] < col_first_out[c]) col_first_out[c] = col_parts[t][c];
  return u64(nt) * nw;
}


// The acceptance table the engine is handed, computed here from the strings with the reference's own clause
// (model_matches = node.rs:463-484), so tests do not have to trust the product's interner for it.
void orc_model_table(const char* const* models, uint32_t n_models, const char* const* patterns,
                     uint32_t n_patterns, uint32_t words, uint32_t threads, uint32_t* bits_out) {
  if (threads == 0) threads = 1;
  for (size_t i = 0; i < size_t(n_patterns) * words; ++i) bits_out[i] = 0;
  auto work = [&](u32 tid) {
    for (u32 p = tid; p < n_patterns; p += threads)
      for (u32 m = 0; m < n_models; ++m)
        if (model_matches(models[m], patterns[p])) bits_out[size_t(p) * words + (m >> 5)] |= 1u << (m & 31);
  };
  std::vector<std::thread> pool;
  for (u32 t = 1; t < threads; ++t) pool.emplace_back(work, t);
  work(0);
  for (auto& th : pool) th.join();
}

// First configuration (priority order) a worker is a compatible candidate of, PM_NONE if none — per worker, with
// early exit, workers split over threads.  With only solo configurations (min == max == 1) try_form_new_groups
// gives every remaining compatible node its own group at the first configuration that accepts it (mod.rs:505-609),
// so this IS the allocation there; it lets tests reach ask counts where the per-configuration loop is too slow.
void orc_soa_first_feasible(const pm_worker_a* a, const pm_worker_b* b, uint32_t n_workers,
                            const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts,
                            const uint32_t* model_bits, uint32_t words, uint32_t threads, uint32_t* first_out) {
  if (threads == 0) threads = 1;
  auto work = [&](u32 tid) {
    for (u32 w = tid; w < n_workers; w += threads) {
      u32 f = PM_NONE;
      if (soa_candidate(a[w].flags))
        for (u32 t = 0; t < n_asks; ++t)
          if (asks[t].max_group_size != 0 && orc_soa_compatible(&a[w], &b[w], &asks[t], opts, model_bits, words)) { f = t; break; }
      first_out[w] = f;
    }
  };
  std::vector<std::thread> pool;
  for (u32 t = 1; t < threads; ++t) pool.emplace_back(work, t);
  work(0);
  for (auto& th : pool) th.join();
}

// EXTENSION, self-oracle (see pm_oracle.h): synchronous forward auction, sequentially.
uint32_t orc_soa_auction(const pm_worker_a* a, const pm_worker_b* b, uint32_t n_workers,
                         const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts,
                         const uint32_t* model_bits, uint32_t words, const uint32_t* price_cap,
                         uint64_t cost_scale, uint64_t eps_start, uint32_t eps_div,
                         uint32_t* ask_worker_out, int64_t* worker_price_out) {
  return orc_soa_auction_rep(a, b, n_workers, asks, n_asks, opts, model_bits, words, price_cap, nullptr, nullptr, cost_scale,
                             eps_start, eps_div, ask_worker_out, worker_price_out);
}

// ... with the `reputation` worker column (north-star extension): a pair is feasible only when
// reputation[w] >= min_reputation[t]; either pointer may be null (column of zeros).
uint32_t orc_soa_auction_rep(const pm_worker_a* a, const pm_worker_b* b, uint32_t n_workers,
                             const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts,
                             const uint32_t* model_bits, uint32_t words, const uint32_t* price_cap,
                             const uint32_t* reputation, const uint32_t* min_reputation,
                             uint64_t cost_scale, uint64_t eps_start, uint32_t eps_div,
                             uint32_t* ask_worker_out, int64_t* worker_price_out) {
  if (cost_scale == 0) cost_scale = 1;
  if (eps_start == 0) eps_start = 1;
  {  // the engine's integer domain: (max ask_price + max cap + 2) * S + eps_start < 2^61, in 128 bits
    uint32_t P = 0, K = 0;
    for (u32 w = 0; w < n_workers; ++w) P = std::max(P, b[w].ext_ask_price);
    for (u32 t = 0; t < n_asks; ++t) K = std::max(K, price_cap[t]);
    if (((unsigned __int128)P + K + 2u) * cost_scale + eps_start >= ((unsigned __int128)1 << 61)) return ORC_AUCTION_REFUSED;
  }
  const int64_t S = int64_t(cost_scale);
  const int64_t NEG = INT64_MIN / 4;
  std::vector<int64_t> price(n_workers, 0);
  std::vector<u32> owner(n_workers, PM_NONE), assigned(n_asks, PM_NONE);
  std::vector<char> withdrawn(n_asks, 0);
  // feasibility lists (so every round costs only the feasible pairs)
  std::vector<std::vector<u32>> feas(n_asks);
  for (u32 t = 0; t < n_asks; ++t)
    for (u32 w = 0; w < n_workers; ++w)
      if (soa_candidate(a[w].flags) && b[w].ext_ask_price <= price_cap[t] &&
          (reputation ? reputation[w] : 0u) >= (min_reputation ? min_reputation[t] : 0u) &&
          orc_soa_compatible(&a[w], &b[w], &asks[t], opts, model_bits, words))
        feas[t].push_back(w);
  u32 rounds = 0;
  if (eps_div < 2) eps_div = 2;
  for (uint64_t eps = eps_start;; eps = std::max<uint64_t>(1, eps / eps_div)) {
    std::fill(owner.begin(), owner.end(), PM_NONE);
    std::fill(assigned.begin(), assigned.end(), PM_NONE);
    std::fill(withdrawn.begin(), withdrawn.end(), 0);
    for (;;) {
      std::vector<u32> bid_w(n_asks, PM_NONE);
      std::vector<int64_t> bid_p(n_asks, 0);
      u32 n_active = 0;
      for (u32 t = 0; t < n_asks; ++t)
        if (assigned[t] == PM_NONE && !withdrawn[t]) ++n_active;
      if (n_active == 0) break;
      ++rounds;  // a round = one bidding pass over the unassigned, not-withdrawn asks
      for (u32 t = 0; t < n_asks; ++t) {
        if (assigned[t] != PM_NONE || withdrawn[t]) continue;
        const int64_t outside = -((int64_t(price_cap[t]) + 1) * S);
        int64_t b1 = NEG, b2 = NEG;
        u32 w1 = PM_NONE;
        for (u32 w : feas[t]) {
          const int64_t v = -(int64_t(b[w].ext_ask_price) * S) - price[w];
          if (v > b1) { b2 = b1; b1 = v; w1 = w; }
          else if (v > b2) b2 = v;
        }
        if (w1 == PM_NONE || b1 < outside) { withdrawn[t] = 1; continue; }
        if (b2 < outside) b2 = outside;
        bid_w[t] = w1;
        bid_p[t] = price[w1] + (b1 - b2) + int64_t(eps);
      }
      // a worker takes the highest bid; ties go to the lowest task index
      std::vector<u32> winner(n_workers, PM_NONE);
      for (u32 t = 0; t < n_asks; ++t) {
        const u32 w = bid_w[t];
        if (w == PM_NONE) continue;
        if (winner[w] == PM_NONE || bid_p[t] > bid_p[winner[w]]) winner[w] = t;
      }
      for (u32 w = 0; w < n_workers; ++w) {
        const u32 t = winner[w];
        if (t == PM_NONE) continue;
        if (owner[w] != PM_NONE) assigned[owner[w]] = PM_NONE;
        owner[w] = t;
        assigned[t] = w;
        price[w] = bid_p[t];
      }
    }
    if (eps == 1) break;
  }
  for (u32 t = 0; t < n_asks; ++t) ask_worker_out[t] = assigned[t];
  if (worker_price_out)
    for (u32 w = 0; w < n_workers; ++w) worker_price_out[w] = price[w];
  return rounds;
}

}  // extern "C"
