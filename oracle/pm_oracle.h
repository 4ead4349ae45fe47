/*
 * pm_oracle.h — CPU ORACLE.  TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * A CPU restatement of the reference orchestrator's matching/allocation path
 * (PrimeIntellect-ai/protocol @ 1bb7f87c).  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load this library.
 * Nothing under protocol_b200/ links, imports or calls it.
 *
 * The reference is Rust and cannot be compiled in this environment (no
 * rustc/cargo, no redis-server), so there is no oracle/_ref build.  Parity is
 * pinned instead by porting the reference's own known-answer tests:
 *   - all 33 tests of crates/shared/src/models/node.rs:659-1241 (parser+meets)
 *   - crates/orchestrator/src/plugins/newest_task/mod.rs:29-54
 *   - crates/orchestrator/src/store/domains/node_store.rs:419-465
 *   - the allocator properties of crates/orchestrator/src/plugins/node_groups/tests.rs
 * (see tests/test_oracle_kat.py, tests/test_oracle_groups.py).
 *
 * Determinisation rules adopted where the reference is non-deterministic
 * (SURVEY.md 8c): canonical worker order = input row order; group id = running
 * counter in creation order; task choice = NewestTask rule; u32 multiply wraps.
 */
#ifndef PM_ORACLE_H
#define PM_ORACLE_H

#include <stddef.h>
#include <stdint.h>
#include "../include/prime_match.h" /* shares only the plain-data table structs */

#ifdef __cplusplus
extern "C" {
#endif

/* ---- reference-shaped (AoS, heap strings) model ------------------------- */
enum orc_has {
  ORC_HAS_SPECS = 1u << 0,
  ORC_HAS_GPU = 1u << 1,
  ORC_HAS_GPU_COUNT = 1u << 2,
  ORC_HAS_GPU_MODEL = 1u << 3,
  ORC_HAS_GPU_MEM = 1u << 4,
  ORC_HAS_CPU = 1u << 5,
  ORC_HAS_CPU_CORES = 1u << 6,
  ORC_HAS_RAM = 1u << 7,
  ORC_HAS_STORAGE = 1u << 8,
  ORC_HAS_P2P = 1u << 9,
  ORC_HAS_LOC = 1u << 10,
  ORC_ASSIGNED = 1u << 11
};

/* NodeStatus ordinals, crates/orchestrator/src/models/node.rs:74-85 */
enum orc_status {
  ORC_DISCOVERED = 0, ORC_WAITING = 1, ORC_HEALTHY = 2, ORC_UNHEALTHY = 3,
  ORC_DEAD = 4, ORC_EJECTED = 5, ORC_BANNED = 6, ORC_LOWBALANCE = 7
};

typedef struct orc_node {
  uint32_t has;          /* orc_has bits */
  uint32_t status;       /* orc_status   */
  uint32_t gpu_count, gpu_mem_mb, cpu_cores, ram_mb, storage_gb;
  uint32_t pad;
  const char* gpu_model; /* valid iff ORC_HAS_GPU_MODEL */
  const char* address;   /* Address::to_string(), taken as given (EIP-55 cased) */
  double lat, lon;       /* valid iff ORC_HAS_LOC */
} orc_node;

typedef struct orc_req orc_req; /* parsed ComputeRequirements */

/* ComputeRequirements::from_str, node.rs:180-374.  NULL + message on Err.  */
orc_req* orc_req_parse(const char* s, char* err, size_t err_len);
void     orc_req_free(orc_req*);
/* inspection (for the ported parser tests) */
uint32_t orc_req_n_gpu(const orc_req*);
/* field: 0 count,1 memory_mb,2 memory_mb_min,3 memory_mb_max,4 total_min,5 total_max.
 * returns 1 and *val if Some, 0 if None */
int orc_req_gpu_u32(const orc_req*, uint32_t opt, int field, uint32_t* val);
/* returns NULL if None */
const char* orc_req_gpu_model(const orc_req*, uint32_t opt);
/* field: 0 cpu.cores, 1 ram_mb, 2 storage_gb; returns 1/0 like above; for
 * field 0, returns -1 when requirements.cpu itself is None */
int orc_req_scalar(const orc_req*, int field, uint32_t* val);

/* ComputeSpecs::meets, node.rs:377-441 (node must have ORC_HAS_SPECS) */
int orc_meets(const orc_node* node, const orc_req* req);
/* NodeGroupsPlugin::is_node_compatible_with_config, mod.rs:206-215; req may be NULL */
int orc_node_compatible(const orc_node* node, const orc_req* req);
/* GpuSpecs::meets model clause only, node.rs:463-484 */
int orc_model_matches(const char* spec_model, const char* req_model);

/* NodeGroupsPlugin::calculate_distance, mod.rs:218-231 */
double orc_haversine_km(double lat1, double lon1, double lat2, double lon2);

typedef struct orc_config {
  const char* name;
  uint64_t min_group_size, max_group_size;
  const orc_req* req; /* NULL == compute_requirements: None */
} orc_config;

/* ctor sort, mod.rs:150-164 (stable).  perm_out[i] = input index at priority i */
void orc_sort_configs(const orc_config* cfgs, uint32_t n, uint32_t* perm_out);
/* get_available_configurations, mod.rs:399-418: keep enabled[i]!=0 then stable
 * sort by min desc.  Input is the ctor-sorted template list.  Returns count. */
uint32_t orc_available_configs(const orc_config* sorted_templates, const uint8_t* enabled,
                               uint32_t n, uint32_t* idx_out);
/* NodeStore::get_nodes ordering, node_store.rs:195-206 (stable by status class) */
void orc_sort_nodes_by_status(const uint32_t* status, uint32_t n, uint32_t* perm_out);

typedef struct orc_groups orc_groups;
/* try_form_new_groups, mod.rs:478-628, faithful loop structure (re-filters all
 * remaining healthy nodes for every group formed, string retain, comparator
 * recomputes haversine).  cfgs = available configurations in priority order. */
orc_groups* orc_form_groups(const orc_node* nodes, uint32_t n_nodes,
                            const orc_config* cfgs, uint32_t n_cfgs, int proximity);
void            orc_groups_free(orc_groups*);
uint32_t        orc_groups_count(const orc_groups*);
uint32_t        orc_groups_members_total(const orc_groups*);
const uint32_t* orc_groups_cfg(const orc_groups*);      /* [G] index into cfgs            */
const uint32_t* orc_groups_off(const orc_groups*);      /* [G+1]                          */
const uint32_t* orc_groups_members(const orc_groups*);  /* node idx, BTreeSet address order */
uint64_t        orc_groups_evals(const orc_groups*);    /* compat predicate executions     */

/* try_merge_solo_groups + helpers, mod.rs:631-971 (faithful).  solos = the groups with exactly
 * one node (get_all_groups order is re-established here: sorted by id string, mod.rs:1040);
 * has_task = get_current_group_task(id).is_some() (only read when !prefer_larger_groups).
 * Returns the merged groups in creation order: cfg index, members = node indices in BTreeSet
 * address order.  A solo group is dissolved iff its node appears in a merged group.          */
typedef struct orc_solo {
  const char* id;
  uint32_t node;      /* index into nodes */
  uint32_t has_task;
} orc_solo;
orc_groups* orc_merge_solo_groups(const orc_node* nodes, uint32_t n_nodes, const orc_solo* solos,
                                  uint32_t n_solos, const orc_config* cfgs, uint32_t n_cfgs,
                                  int proximity, int task_switching_enabled, int prefer_larger_groups);

/* NewestTaskPlugin::filter_tasks, newest_task/mod.rs:8-19: index of the task
 * max_by_key(created_at) returns (LAST maximum), or PM_NONE if n == 0.        */
uint32_t orc_newest_task(const int64_t* created_at, uint32_t n);
/* TaskStore::get_all_tasks ordering, task_store.rs:79: stable sort created_at desc */
void orc_sort_tasks(const int64_t* created_at, uint32_t n, uint32_t* perm_out);
/* get_idx_in_group, mod.rs:424-434: position of addr in BTreeSet order, -1 if absent */
int64_t orc_idx_in_group(const char* const* member_addrs, uint32_t n, const char* addr);

/* ---- SoA / interned restatement (same predicate on the engine's tables) --- */
int orc_soa_compatible(const pm_worker_a* a, const pm_worker_b* b, const pm_ask* ask,
                       const pm_gpu_opt* opts, const uint32_t* model_bits, uint32_t words);

/* Same allocator on SoA tables, one compat filter per configuration (equal
 * output to the faithful loop; checked in tests/test_oracle_groups.py).
 * addr_rank may be NULL (identity).  lat/lon may be NULL when !proximity.     */
orc_groups* orc_soa_form_groups(const pm_worker_a* a, const pm_worker_b* b, uint32_t n_workers,
                                const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts,
                                const uint32_t* model_bits, uint32_t words,
                                const uint32_t* addr_rank, const double* lat, const double* lon,
                                int proximity /* 0 first fit, 1 the reference's proximity loop, 2 same result with latitude pruning */);

/* Full evaluation of the sub-matrix asks[t0,t1) x workers[w0,w1) over `threads`
 * host threads: cost[t][w] = compat && candidate ? (price<<32 | w) : INF with
 * price = pm_worker_b.ext_ask_price (0 in the reference's own modes); rows of asks with max_group_size == 0 are all INF
 * (such a configuration never takes a worker).  Any out pointer may be NULL.
 *   cost_out      [(t1-t0) * (w1-w0)] row-major
 *   row_best_out  [t1-t0] min over w      row_count_out [t1-t0] #feasible
 *   col_first_out [w1-w0] first feasible ask index (global) or PM_NONE
 * Returns the number of predicate evaluations executed ((t1-t0)*(w1-w0)).     */
uint64_t orc_soa_eval_matrix(const pm_worker_a* a, const pm_worker_b* b,
                             const pm_ask* asks, const pm_gpu_opt* opts,
                             const uint32_t* model_bits, uint32_t words,
                             uint32_t t0, uint32_t t1, uint32_t w0, uint32_t w1,
                             uint32_t threads, int64_t* cost_out, int64_t* row_best_out,
                             uint32_t* row_count_out, uint32_t* col_first_out);

/* The (pattern x model) acceptance bit table from the strings, with the reference's model clause
 * (GpuSpecs::meets, node.rs:463-484): bits_out[p * words + (m >> 5)] bit (m & 31).               */
void orc_model_table(const char* const* models, uint32_t n_models, const char* const* patterns,
                     uint32_t n_patterns, uint32_t words, uint32_t threads, uint32_t* bits_out);
/* First configuration (priority order) whose compat filter + candidate filter accept the worker, or
 * PM_NONE.  For solo configurations this is the worker's group (mod.rs:505-609).                 */
void orc_soa_first_feasible(const pm_worker_a* a, const pm_worker_b* b, uint32_t n_workers,
                            const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts,
                            const uint32_t* model_bits, uint32_t words, uint32_t threads, uint32_t* first_out);

/* ---- north-star EXTENSION: price-capped auction.  SELF-ORACLE: the reference has no
 * prices, caps or auction (SURVEY 0); parity for this mode is UNPINNED BY THE REFERENCE.
 * Sequential restatement of the synchronous (Jacobi) forward auction the engine runs:
 *   feasible(t,w) = candidate(w) && compatible(t,w) && ask_price[w] <= price_cap[t]
 *   value(t,w)    = -(ask_price[w] * S) - price[w];  outside option = -((price_cap[t]+1) * S)
 *   (S = cost_scale: 1 gives an assignment within T*eps of the optimum; T+1 with eps = 1 the optimum)
 *   each round every unassigned task bids price[w1] + (best - second) + eps on its best worker
 *   (ties: lowest worker index); a worker takes the highest bid (ties: lowest task index) and
 *   releases its previous owner; a task whose best value drops below its outside option withdraws.
 * eps runs eps_start, eps_start/eps_div, ..., 1 (assignment cleared between phases, prices kept).
 * ask_worker_out[T]: assigned worker or PM_NONE.  Returns the number of bidding rounds, or
 * ORC_AUCTION_REFUSED (nothing written) outside the engine's integer domain (prime_match.h,
 * pm_set_auction_params): (max ext_ask_price + max price_cap + 2) * cost_scale + eps_start >= 2^61. */
#define ORC_AUCTION_REFUSED 0xFFFFFFFFu

uint32_t orc_soa_auction(const pm_worker_a* a, const pm_worker_b* b, uint32_t n_workers,
                         const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts,
                         const uint32_t* model_bits, uint32_t words, const uint32_t* price_cap,
                         uint64_t cost_scale, uint64_t eps_start, uint32_t eps_div,
                         uint32_t* ask_worker_out, int64_t* worker_price_out);
/* ... plus the north-star `reputation` worker column: feasible(t,w) also needs
 * reputation[w] >= min_reputation[t]; either pointer may be null (all zeros).              */
uint32_t orc_soa_auction_rep(const pm_worker_a* a, const pm_worker_b* b, uint32_t n_workers,
                             const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts,
                             const uint32_t* model_bits, uint32_t words, const uint32_t* price_cap,
                             const uint32_t* reputation, const uint32_t* min_reputation,
                             uint64_t cost_scale, uint64_t eps_start, uint32_t eps_div,
                             uint32_t* ask_worker_out, int64_t* worker_price_out);

#ifdef __cplusplus
}
#endif
#endif
