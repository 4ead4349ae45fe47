/*
 * prime_match.h — C ABI of the H100-native task<->worker matching engine.
 *
 * Drop-in boundary for the Prime Protocol orchestrator's scheduling hot path.
 * Every entry point below names the reference interface (file:line under the
 * reference checkout, crates/...) that it replaces or feeds.  Plain pointers
 * and sizes only; no C++/torch types cross this boundary.  All functions
 * return 0 (PM_OK) or a negative pm_status, never unwind, never abort
 * (reference error convention: failures are swallowed to an empty answer and
 * retried next tick — crates/orchestrator/src/plugins/node_groups/
 * scheduler_impl.rs:24-30,86-104 and mod.rs:188-194).
 *
 * Vocabulary follows the reference: worker == OrchestratorNode
 * (crates/orchestrator/src/models/node.rs:10-37), ask == one
 * NodeGroupConfiguration row {min,max,ComputeRequirements}
 * (crates/orchestrator/src/plugins/node_groups/mod.rs:30-37), evaluation ==
 * one is_node_compatible_with_config call (mod.rs:206-215).
 */
#ifndef PRIME_MATCH_H
#define PRIME_MATCH_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PM_ABI_VERSION 1u
#define PM_NONE 0xFFFFFFFFu
#define PM_COST_INF INT64_MAX

typedef enum pm_status {
  PM_OK = 0,
  PM_E_INVALID = -1,     /* bad argument / table shape                        */
  PM_E_CUDA = -2,        /* CUDA runtime error; text in pm_last_error         */
  PM_E_NO_DEVICE = -3,   /* no sm_90 device visible: the engine never falls   */
                         /* back to a CPU path                                */
  PM_E_STATE = -4,       /* call order violated (e.g. match before tables)    */
  PM_E_NOMEM = -5,
  PM_E_UNSUPPORTED = -6,
  PM_E_PARSE = -7        /* requirement string rejected (node.rs:180-374)     */
} pm_status;

/* ------------------------------------------------------------------------ */
/* Worker table: SoA mirror of OrchestratorNode + ComputeSpecs               */
/* (crates/shared/src/models/node.rs:25-35,72-78,153-157).  Two 16-byte      */
/* planes so that one worker is exactly two coalesced 128-bit loads.         */
/* ------------------------------------------------------------------------ */
enum pm_worker_flag {
  PM_W_HEALTHY        = 1u << 0,  /* status == NodeStatus::Healthy  (mod.rs:494) */
  PM_W_P2P            = 1u << 1,  /* p2p_id.is_some()               (mod.rs:495) */
  PM_W_ASSIGNED       = 1u << 2,  /* present in node_to_group       (mod.rs:496) */
  PM_W_HAS_SPECS      = 1u << 3,  /* compute_specs.is_some()                     */
  PM_W_HAS_GPU        = 1u << 4,  /* specs.gpu.is_some()                         */
  PM_W_HAS_GPU_COUNT  = 1u << 5,
  PM_W_HAS_GPU_MEM    = 1u << 6,
  PM_W_HAS_GPU_MODEL  = 1u << 7,
  PM_W_HAS_CPU        = 1u << 8,  /* specs.cpu.is_some()                         */
  PM_W_HAS_CPU_CORES  = 1u << 9,
  PM_W_HAS_RAM        = 1u << 10,
  PM_W_HAS_STORAGE    = 1u << 11,
  PM_W_HAS_LOC        = 1u << 12  /* location.is_some()                          */
};

typedef struct pm_worker_a {   /* plane A, 16 B */
  uint32_t gpu_count;          /* GpuSpecs.count      */
  uint32_t gpu_mem_mb;         /* GpuSpecs.memory_mb  */
  uint32_t model_id;           /* interned GpuSpecs.model (pm_intern_model); must be < n_models of the model table in */
                               /* force when PM_W_HAS_GPU_MODEL is set (a precondition: the kernels index the table by it) */
  uint32_t flags;              /* pm_worker_flag bits */
} pm_worker_a;

typedef struct pm_worker_b {   /* plane B, 16 B */
  uint32_t cpu_cores;          /* CpuSpecs.cores */
  uint32_t ram_mb;
  uint32_t storage_gb;
  uint32_t ext_ask_price;      /* north-star extension column; 0 when unused */
} pm_worker_b;

/* ------------------------------------------------------------------------ */
/* Ask table: one row per enabled NodeGroupConfiguration in PRIORITY ORDER   */
/* (mod.rs:150-164 then :399-418; pm_sort_configs reproduces it), plus a     */
/* CSR list of GpuRequirements OR-options (node.rs:58-70).                   */
/* ------------------------------------------------------------------------ */
enum pm_ask_flag {
  PM_A_HAS_REQ        = 1u << 0,  /* compute_requirements.is_some()  (mod.rs:210-214) */
  PM_A_REQ_CPU        = 1u << 1,  /* requirements.cpu.is_some()      (node.rs:381)    */
  PM_A_REQ_CPU_CORES  = 1u << 2,  /* requirements.cpu.cores.is_some  (node.rs:533)    */
  PM_A_REQ_RAM        = 1u << 3,
  PM_A_REQ_STORAGE    = 1u << 4
};

typedef struct pm_ask {        /* 32 B */
  uint32_t flags;              /* pm_ask_flag bits */
  uint32_t n_opts;             /* requirements.gpu.len() */
  uint32_t opt_off;            /* first pm_gpu_opt of this ask */
  uint32_t cpu_cores;
  uint32_t ram_mb;
  uint32_t storage_gb;
  uint32_t min_group_size;
  uint32_t max_group_size;
} pm_ask;

enum pm_opt_present {
  PM_O_COUNT   = 1u << 0,
  PM_O_MODEL   = 1u << 1,
  PM_O_MEM     = 1u << 2,   /* memory_mb        */
  PM_O_MEM_MIN = 1u << 3,   /* memory_mb_min    */
  PM_O_MEM_MAX = 1u << 4,   /* memory_mb_max    */
  PM_O_TOT_MIN = 1u << 5,   /* total_memory_min */
  PM_O_TOT_MAX = 1u << 6    /* total_memory_max */
};

typedef struct pm_gpu_opt {    /* 32 B; field-for-field GpuRequirements */
  uint32_t present;            /* pm_opt_present bits */
  uint32_t count;
  uint32_t memory_mb;
  uint32_t memory_mb_min;
  uint32_t memory_mb_max;
  uint32_t total_memory_min;
  uint32_t total_memory_max;
  uint32_t pattern_id;         /* interned requirement model list (pm_intern_pattern) */
} pm_gpu_opt;

/* ------------------------------------------------------------------------ */
/* Host-side model-string interning.  The substring predicate of            */
/* GpuSpecs::meets (node.rs:463-484) is evaluated once per distinct          */
/* (requirement pattern, worker model) pair on the host and shipped to the   */
/* device as a bit table; per (ask, worker) pair the device does one bit     */
/* test.  No GPU needed for these calls.                                     */
/* ------------------------------------------------------------------------ */
typedef struct pm_interner pm_interner;
pm_interner* pm_interner_create(void);
void         pm_interner_destroy(pm_interner*);
uint32_t     pm_intern_model(pm_interner*, const char* spec_model);      /* worker side */
uint32_t     pm_intern_pattern(pm_interner*, const char* req_model);     /* ask side    */
/* bits[p * words + (m >> 5)] >> (m & 31) & 1  <=>  pattern p accepts model m;  */
/* words = ceil(n_models / 32).  Pointer is valid until the next intern call.   */
int pm_interner_table(pm_interner*, const uint32_t** bits, uint32_t* n_patterns,
                      uint32_t* n_models, uint32_t* words_per_pattern);

/* ComputeRequirements::from_str (node.rs:180-374).  Fills *ask (flags, n_opts,
 * cpu/ram/storage; opt_off/min/max untouched) and up to max_opts options.   */
int pm_parse_requirements(const char* s, pm_interner* interner, pm_ask* ask,
                          pm_gpu_opt* opts, uint32_t max_opts, uint32_t* n_opts,
                          char* err, size_t err_len);

/* NodeGroupsPlugin::new_with_policy sort (mod.rs:150-164): stable, by
 * min_group_size desc, then with-requirements before without.  perm_out[i] =
 * index of the config that lands at priority i.                             */
int pm_sort_configs(const uint32_t* min_group_size, const uint8_t* has_requirements,
                    uint32_t n, uint32_t* perm_out);

/* Node ids.  The reference parses every wire id (`node.id.parse::<Address>()`, discovery/monitor.rs:240) and uses
 * `Address::to_string()` — "0x" + 40 hex digits in EIP-55 checksum case (alloy-primitives 1.1.0, Cargo.lock) — as the
 * key of every store, of node_to_group and of the BTreeSet that decides GROUP_INDEX (mod.rs:63-69,424-434).
 * pm_address_canonical does the same for a C string: accepts 40 hex digits with or without "0x", any case (no
 * checksum validation, like Address::from_str), writes the 42-character checksummed form + NUL.  PM_E_INVALID otherwise. */
int pm_address_canonical(const char* address, char out[43]);

/* ------------------------------------------------------------------------ */
/* Engine                                                                     */
/* ------------------------------------------------------------------------ */
typedef struct pm_engine pm_engine;

enum pm_cfg_flag {
  PM_CFG_TIMING = 1u << 0     /* record CUDA events per kernel class (pm_stats.ms_*) */
};

typedef struct pm_cfg {
  uint32_t abi_version;        /* PM_ABI_VERSION */
  int32_t  device;             /* CUDA ordinal */
  uint32_t flags;              /* pm_cfg_flag */
  uint32_t reserved0;
  uint64_t cost_tile_bytes;    /* HBM budget for one materialised cost tile; 0 = 8 GiB.  Tile rows are sized at
                                  8 B per element; the 32-bit tile covers the same rows in half of it */
  /* Worker sharding across GPUs (SURVEY 8e): this engine evaluates the        */
  /* contiguous canonical-order range [shard_first, shard_first+shard_count)   */
  /* of the global worker table; shard_count == 0 means "all".                 */
  uint32_t shard_first;
  uint32_t shard_count;
  void*    stream;             /* cudaStream_t to launch on (e.g. the caller's torch     */
                               /* stream, so its CUDA events bracket the kernels);        */
                               /* NULL = the engine creates a private non-blocking stream */
} pm_cfg;

int         pm_create(const pm_cfg* cfg, pm_engine** out);
void        pm_destroy(pm_engine*);
const char* pm_last_error(const pm_engine*);   /* NULL engine -> last create error */

/* Pinned host memory for the caller-owned tables (SURVEY 8b "ownership").   */
void* pm_alloc_pinned(size_t bytes);
void  pm_free_pinned(void*);

/* replaces the per-pass TaskStore/config reads (mod.rs:399-418)             */
/* [opt_off, opt_off + n_opts) ranges may overlap or be shared between asks.  */
int pm_set_asks(pm_engine*, const pm_ask* asks, uint32_t n_asks,
                const pm_gpu_opt* opts, uint32_t n_opts);
/* Enabled configurations (get_available_configurations, mod.rs:399-418; enable_configuration, mod.rs:1328-1346).
 * After pm_set_asks every ask is enabled.  A disabled ask behaves as if it were absent from the table: no worker's
 * first feasible ask is a disabled one, no under-filled tail is handed down to one, it forms no group (not the empty
 * group of min_group_size == 0 either), its ask_best reads PM_COST_INF and its ask_count 0, its pm_build_cost_tile
 * rows are all infeasible, and per-table facts are taken over the enabled asks (a disabled max_group_size == 0 ask does
 * not make PM_MODE_PROXIMITY refuse).  Result indices (worker_ask, group_ask, ask_best / ask_count positions) stay
 * indices of the full table.  enabled[i] != 0 enables ask idx[i]; the last entry for an ask decides.  An index
 * >= n_asks is PM_E_INVALID and changes nothing; PM_E_STATE without an ask table.  PM_MODE_AUCTION returns
 * PM_E_UNSUPPORTED while any ask is disabled.  The stored evaluation of PM_INCREMENTAL is kept: see "Incremental
 * passes".                                                                                                          */
int pm_set_ask_enabled(pm_engine*, const uint32_t* idx, const uint8_t* enabled, uint32_t n);
/* Ask-table deltas: a resident ask table changed in place (a new task with a price cap is an appended row, a finished
 * one a removed row).  After any sequence of pm_set_asks, pm_update_asks, pm_resize_asks, pm_remove_asks, pm_insert_asks
 * and pm_set_ask_enabled calls the engine is the engine pm_set_asks would give for the current rows with the same
 * enabled mask, caps, floors and demands: every array
 * pm_fetch_result returns, pm_build_cost_tile and a cold auction pass are bit-identical to a fresh engine's, with or
 * without PM_INCREMENTAL, on every path and in every mode.  Ask index stays priority.
 *   pm_update_asks   replace rows idx[i] (each < n_asks) by asks[i]; asks[i].opt_off / n_opts index `opts`, as in
 *                    pm_set_asks.  A replaced row keeps its enabled flag, its price cap and its reputation floor.  For
 *                    repeated indices the last entry decides.
 *   pm_resize_asks   shrink: drop asks [n_asks, old); grow: append `n_asks - old` rows from `added` (options in `opts`)
 *                    at the lowest priorities, enabled, with cap 0 and floor 0 until pm_set_ask_price_caps /
 *                    pm_set_ask_min_reputation set them (both still take exactly n_asks entries).
 *   pm_remove_asks   remove rows idx[0..n) (any order; a repeated index removes its row once); the rows after them move
 *                    up, order kept.  Removing the tail is pm_resize_asks shrinking, bit for bit.
 *   pm_insert_asks   insert rows asks[0..n) (options in `opts`, as pm_set_asks) before the current rows before[i];
 *                    before[] non-decreasing, before[i] <= n_asks (n_asks = append); rows with equal before[] keep their
 *                    order.  Inserting every row at n_asks is pm_resize_asks growing, bit for bit.
 * A removed row takes its enabled flag, price cap, reputation floor and demand with it.  An inserted (or appended) row is
 * enabled, with cap 0, floor 0 and demand 1 until pm_set_ask_price_caps / pm_set_ask_min_reputation /
 * pm_set_ask_demand set them (each still takes exactly n_asks entries).  A kept row keeps its flag, cap, floor and
 * demand under its new index.
 * Refusals, none of which changes anything (no table, no stored evaluation, no auction state, no demands, no
 * pm_table_version): PM_E_INVALID for a null pointer with a count > 0, an index >= n_asks, a before[] that decreases or
 * exceeds n_asks, max_group_size < min_group_size, an option range outside `opts`, growth without `added`, n_asks >= 2^30,
 * more than 2^31 converted option rows, or added rows that take the demands' total D to 2^30; PM_E_STATE without an
 * ask table.  Every row is checked on the host before anything on the device is touched.  A row that
 * references a pattern beyond the model table is accepted; the next pass returns PM_E_STATE, as after pm_set_asks.
 * Unlike pm_set_asks, all four keep the stored evaluation of PM_INCREMENTAL and the stored auction state: see "Incremental
 * passes", "Auction warm start", "Auction warm repair" and "Auction certificate".  Each call converts the whole table
 * again on the device (O(T + the option rows)).  Only the option ranges the new rows reference are copied from `opts`
 * (a caller may pass its whole option table); the option rows replaced or removed rows leave behind are compacted
 * away once they outnumber the live ones.                                                                                    */
int pm_update_asks(pm_engine*, const uint32_t* idx, const pm_ask* asks, uint32_t n,
                   const pm_gpu_opt* opts, uint32_t n_opts);
int pm_resize_asks(pm_engine*, uint32_t n_asks, const pm_ask* added, const pm_gpu_opt* opts, uint32_t n_opts);
int pm_remove_asks(pm_engine*, const uint32_t* idx, uint32_t n);
int pm_insert_asks(pm_engine*, const uint32_t* before, const pm_ask* asks, uint32_t n, const pm_gpu_opt* opts,
                   uint32_t n_opts);
int pm_set_model_table(pm_engine*, const uint32_t* bits, uint32_t n_patterns,
                       uint32_t n_models, uint32_t words_per_pattern);
/* replaces NodeStore::get_nodes per pass (store/domains/node_store.rs:163-209);
 * row index == canonical order (SURVEY 8c determinisation rule 1).          */
int pm_set_worker_count(pm_engine*, uint32_t n_workers);
int pm_upsert_workers(pm_engine*, const pm_worker_a* a, const pm_worker_b* b,
                      uint32_t first, uint32_t n);
/* NodeLocation.latitude/longitude (node.rs:543-550); only read in proximity mode.
 * A row flagged PM_W_HAS_LOC needs finite coordinates (any finite value is accepted). */
int pm_set_worker_locations(pm_engine*, const double* lat, const double* lon,
                            uint32_t first, uint32_t n);
/* rank of the worker's address string in BTreeSet<String> order
 * (mod.rs:63-69,424-434); decides member order inside a group               */
int pm_set_worker_addr_rank(pm_engine*, const uint32_t* rank, uint32_t first, uint32_t n);
/* status / assigned deltas (status_update_impl.rs:8-39, mod.rs:1423-1487)   */
int pm_set_flags(pm_engine*, const uint32_t* idx, const uint32_t* flags, uint32_t n);

/* Resident tables with deltas: a long-running host keeps the worker table on the device between management passes and
 * sends only the rows that changed (status / assigned / specs / location), instead of NodeStore::get_nodes' full
 * read per pass (store/domains/node_store.rs:163-209).
 *   pm_resize_workers   grow (or shrink) the table, keeping the rows it holds; new rows are empty (no candidate)
 *   pm_update_workers   scatter n rows by index; lat/lon both NULL or both given
 *   pm_table_version    changes whenever any table call ran: lets a caller detect that someone else used the engine
 *   pm_create_sibling   a second engine on the same device with the same configuration (own stream and tables)   */
int      pm_resize_workers(pm_engine*, uint32_t n_workers);
int      pm_update_workers(pm_engine*, const uint32_t* idx, const pm_worker_a* a, const pm_worker_b* b,
                           const double* lat, const double* lon, uint32_t n);
/* Worker-table splices: a worker leaves (deregistered, banned, out of the auction's market) or joins at any position.
 *   pm_remove_workers  remove rows idx[0..n) (any order; a repeated index removes its row once); the rows after them
 *                      move up, order kept.  Removing the tail is pm_resize_workers shrinking.
 *   pm_insert_workers  insert rows a[i], b[i] before the current rows before[i]; before[] non-decreasing, before[i] <=
 *                      n_workers (n_workers = append); rows with equal before[] keep their order.  lat / lon both NULL
 *                      (the new rows at (0, 0), as rows added by pm_resize_workers) or both given.  Inserting every row
 *                      at n_workers is pm_resize_workers growing followed by pm_update_workers of the new rows.
 * Every per-row column moves with its row: planes A and B, location, address rank and reputation.  An inserted row has
 * address rank 0 and reputation 0 until pm_set_worker_addr_rank / pm_set_worker_reputation set them.
 * THE DEFINING RULE: after any sequence of worker- and ask-table calls the engine equals a fresh engine loaded with the
 * current rows (pm_set_worker_count + pm_upsert_workers + locations + ranks + reputation, the same asks, enabled mask,
 * caps, floors and demands): every pm_fetch_result array, pm_build_cost_tile and a cold auction pass are bit-identical,
 * in every mode, on every path, with and without PM_INCREMENTAL.  The tail cases equal pm_resize_workers (+
 * pm_update_workers) in the tables, the stored evaluation, and the next pass's results, auction state and pm_stats.
 * The exports between the call and that pass differ: after a splice they report the current rows (n_workers prices,
 * PM_NONE for a removed holder), while after a shrink pm_auction_state still returns the stored pass's W prices and
 * pm_auction_assignment the cut-off row's old index.
 * Both calls keep the stored evaluation of PM_INCREMENTAL: each row's stored first ask moves with it on the device,
 * removed rows vanish and inserted rows are written.  A communicator's share and an open-ended pm_set_shard range move
 * with W as under pm_resize_workers (rows that enter a rank's range count as written there, rows that leave it return
 * to PM_NONE); a fixed pm_set_shard range stays where it is and the rows that shift into it count as written.  The
 * next incremental pass walks the inserted rows and the rows that crossed a range boundary only.
 * Both keep the stored auction state: prices and owners move with their rows and the per-slot assignment is renamed to
 * the new indices.  The holder of a removed row is released in step 1 of the next PM_AUCTION_WARM (or repair) pass and
 * counts in n_released, exactly as the holder of a row a shrink cut off; the warm cutoff counts the removed rows as it
 * counts the rows a shrink cut off.  Inserted rows are changed rows (R0): price 0, unowned.  pm_auction_state,
 * pm_auction_assignment and pm_auction_slot_assignment report the renamed state over the current rows (a removed
 * holder reads PM_NONE); pm_auction_certificate returns PM_E_STATE until the next auction pass.
 * Refusals, none of which changes anything (no table, no stored evaluation, no auction state, no pm_table_version):
 * PM_E_STATE without a worker table; PM_E_INVALID for a NULL pointer with n > 0, an index >= n_workers, a before[] that
 * decreases or exceeds n_workers, lat without lon or the reverse, or a table that would reach PM_NONE rows.  Every
 * check runs on the host before anything on the device is touched.  A call is one O(W) device pass.  The first
 * splice allocates a second copy of every per-row column in use (up to 76 bytes per row: 76 MB at 1M workers), kept
 * for the splices that follow and released by pm_set_worker_count. */
int      pm_remove_workers(pm_engine*, const uint32_t* idx, uint32_t n);
int      pm_insert_workers(pm_engine*, const uint32_t* before, const pm_worker_a* a, const pm_worker_b* b,
                           const double* lat, const double* lon, uint32_t n);
uint64_t pm_table_version(const pm_engine*);
int      pm_create_sibling(const pm_engine*, pm_engine** out);

/* NORTH-STAR EXTENSION columns (no reference counterpart; only PM_MODE_AUCTION reads them):
 * per-ask price cap against pm_worker_b.ext_ask_price, and the auction's parameters
 * (value = -(ask_price * cost_scale) - price; eps runs eps_start, /eps_div, ..., 1).
 * PM_MODE_AUCTION has no group sizes: an ask with max_group_size == 0, which no reference mode fills, takes a worker
 * like any other there (and in pm_auction_certificate).  An ask takes one worker, or up to its demand with
 * pm_set_ask_demand ("Auction demands" below); min_group_size is never enforced.
 * Integer domain of PM_MODE_AUCTION: with P = the largest ext_ask_price over every row of the worker table (feasible or
 * not), K = the largest price cap, S = cost_scale and E = eps_start (0 counts as 1 for both),
 *     (P + K + 2) * S + E < 2^61          (evaluated without overflow).
 * Inside it every value, outside option, bid, price, profit and sort key the auction computes in int64 lies strictly
 * between -2^61 and 2^61 (DESIGN 4).  pm_set_auction_params refuses cost_scale or eps_start >= 2^61 (PM_E_INVALID,
 * nothing changes: the stored auction state is kept).  pm_match(PM_MODE_AUCTION ...) refuses a pass whose tables and
 * parameters are outside the domain with PM_E_INVALID before it changes anything: the stored warm state,
 * pm_auction_state and pm_auction_reverse_stats stay as they were.  Round counts grow with S (an eps = 1 price war
 * between equal workers takes O(S) rounds): large scales want eps-scaling with PM_AUCTION_REVERSE.                   */
int pm_set_ask_price_caps(pm_engine*, const uint32_t* price_cap, uint32_t n_asks);
int pm_set_auction_params(pm_engine*, uint64_t cost_scale, uint64_t eps_start, uint32_t eps_div);
/* `reputation` (north_star worker column; SURVEY 8 A21 side column ext_reputation:u32) and the per-ask floor on it:
 *   feasible(t,w) additionally requires reputation[w] >= min_reputation[t]   (PM_MODE_AUCTION only).
 * Both default to 0 (no clause).  The worker column follows the worker table: pm_resize_workers keeps it,
 * pm_set_worker_count drops it.  min_reputation is per ask, after pm_set_asks, like the price caps.      */
int pm_set_worker_reputation(pm_engine*, const uint32_t* reputation, uint32_t first, uint32_t n);
int pm_set_ask_min_reputation(pm_engine*, const uint32_t* min_reputation, uint32_t n_asks);
/* Auction demands (north-star extension column; PM_MODE_AUCTION only, the reference modes never read it).
 * demand[t] >= 1 is the number of workers ask t may take; each of them is priced and capped separately: value(t, w),
 * feasible(t, w) and the outside option -(cap[t] + 1) * S do not change.  Fills may be partial: an ask with demand 4
 * may end holding 0 to 4 workers.  min_group_size is NOT enforced: an all-or-nothing gang is not an assignment
 * problem (its LP relaxation loses integrality, and the eps-CS argument with it; DESIGN 4).
 * THE DEFINING RULE: an engine with demands d behaves as the engine whose ask table repeats row t d[t] times at
 * consecutive priorities, with its cap and floor repeated.  Each copy is a SLOT; there are D = sum d[t] of them, in ask
 * order (slot s of ask t is sum_{u<t} d[u] + k, k < d[t]).  Every auction pass kind (cold, eps-scaled with
 * PM_AUCTION_REVERSE, PM_AUCTION_WARM, PM_AUCTION_WARM | PM_AUCTION_REPAIR) gives that twin's assignment, prices,
 * rounds, warm / n_released and reverse stats, bit for bit; the results are folded per ask; the guarantee is the twin's:
 * a total cost within D * eps of the optimum, exact with cost_scale = D + 1.
 * pm_set_ask_demand takes exactly n_asks entries, as pm_set_ask_price_caps does.  Without the call, or with every demand
 * 1, behaviour is today's byte for byte (the same kernels, no extra launch).  After pm_set_asks every demand is 1;
 * pm_update_asks keeps a replaced row's demand (as it keeps its cap); pm_resize_asks and pm_insert_asks add rows with
 * demand 1; a shrink and pm_remove_asks drop the removed rows' demands; a kept row's demand moves with it.
 * Refusals change nothing (not the demands, not the stored auction state, not pm_table_version): PM_E_INVALID for a
 * NULL pointer with n_asks > 0, n_asks other than the table's, a demand of 0, or D >= 2^30 (the ask-count limit; a
 * pm_resize_asks growth or pm_insert_asks that would take D there is refused the same way); PM_E_STATE without an ask
 * table.
 * A demand change under a stored auction state: each ask's first min(old, new) slots keep their holds; a removed slot's
 * worker becomes unowned at its stored price and counts against the warm cutoff, like a removed ask's holder; the added
 * slots hold nothing and are in A0.  The warm start and the repair then run unchanged on the remapped state (DESIGN 4).
 * Result form with demands (pm_fetch_result): one group per ask holding at least one worker, in ask order, its members
 * in increasing worker index; worker_ask[w] is the ask and worker_group[w] the group; ask_count[t] the workers held;
 * ask_best[t] the smallest ask_price << 32 | w over them (PM_COST_INF for none); n_groups the asks holding a worker,
 * n_members the workers held.  With every demand 1 this is exactly the one-worker-per-ask form.
 * pm_stats keeps its meanings, counted over slots.  pm_auction_certificate is over slots: n_held, n_slack_over and
 * max_slack count or range over slots, bound = sum_t d[t] * row(t) - sum_w price[w], ask_bound stays per ask (every
 * slot of an ask has the same row term), evals stays T x W.  pm_auction_assignment and pm_auction_restore return
 * PM_E_UNSUPPORTED while any demand exceeds 1 (their format is one worker per ask); pm_auction_slot_assignment and
 * pm_auction_restore_slots export and restore the state per slot ("Auction state restore per slot" below).  The
 * auction stays single-GPU: there
 * is no pm_multi_ form. */
int pm_set_ask_demand(pm_engine*, const uint32_t* demand, uint32_t n_asks);

enum pm_mode {
  PM_MODE_FIRST_FIT = 0,   /* try_form_new_groups, ProximityOptimizationPolicy{enabled:false} */
  PM_MODE_PROXIMITY = 1,   /* ... {enabled:true}  (mod.rs:524-552), the reference default     */
  PM_MODE_PROXIMITY_MERGE = 3, /* try_merge_solo_groups' batch selection (mod.rs:752-848) over a table that  */
                           /* holds only the nodes of solo groups, in get_all_groups() order               */
  PM_MODE_AUCTION   = 2    /* north-star extension: price-capped forward auction, one worker  */
                           /* per ask or per slot of its demand (pm_set_ask_demand;           */
                           /* pm_auction.cuh); no reference counterpart, self-oracle          */
};
enum pm_path {
  PM_PATH_MATERIALIZED = 0,      /* build a cost tile in HBM (the 32-bit cost word when every price is
                                    below 0x7FFFFFFF, else the int64 packed cost), then argmin over it */
  PM_PATH_FUSED        = 1u << 8,/* evaluate + reduce on chip, matrix never written   */
  PM_NO_ASK_STATS      = 1u << 9,/* with PM_PATH_FUSED: skip ask_best / ask_count (the reference modes only
                                    need the per-worker first feasible ask); they read INF / 0 then      */
  PM_INCREMENTAL       = 1u << 10,/* reuse the engine's stored per-worker first feasible ask: re-evaluate only the worker
                                    rows written since the last evaluation on this engine, or everything when there is no
                                    valid stored evaluation or more rows changed than the cutoff (PM_TUNE_INCR at
                                    pm_create).  Every array pm_fetch_result returns equals the same call's without the
                                    flag (ask_best = PM_COST_INF, ask_count = 0).  Valid with PM_PATH_FUSED |
                                    PM_NO_ASK_STATS and a reference mode only (else PM_E_INVALID).  Works on a sharded
                                    engine through pm_match_local and with a communicator attached (pm_comm, pm_multi);
                                    PM_E_UNSUPPORTED from pm_match on a shard engine without a communicator.  See
                                    "Incremental passes" below */
  PM_AUCTION_WARM      = 1u << 11,/* PM_MODE_AUCTION only (else PM_E_INVALID): start from the last auction pass's prices and
                                    assignment, releasing only the asks the changes since disturb; a cold pass when there is
                                    no stored state or the changes exceed the cutoff.  See "Auction warm start" below */
  PM_AUCTION_REVERSE   = 1u << 12,/* PM_MODE_AUCTION only, not with PM_AUCTION_WARM (else PM_E_INVALID): every eps phase
                                    ends with reverse rounds that return every unowned worker to price 0, which makes
                                    eps_start > 1 keep the eps = 1 bound.  See "Auction reverse rounds" below */
  PM_AUCTION_REPAIR    = 1u << 13 /* only as PM_MODE_AUCTION | PM_AUCTION_WARM | PM_AUCTION_REPAIR (else PM_E_INVALID; not
                                    with PM_AUCTION_REVERSE): a warm pass that keeps every stored price, raises the changed
                                    rows instead of releasing what they disturb, and ends with reverse rounds.  See
                                    "Auction warm repair" below */
};

/* Incremental passes (PM_INCREMENTAL).  Every full evaluation, with the flag or without, keeps a copy of its
 * per-worker result over the engine's range: the whole table, the pm_cfg / pm_set_shard range, or with a communicator
 * the rank's equal share; PM_NONE outside it (a communicator engine takes the copy before the exchange).  A row becomes
 * "written" through pm_upsert_workers (the range), pm_update_workers and pm_set_flags (the in-range indices, each once)
 * and pm_resize_workers (the rows past the old end).  An incremental pass re-evaluates the written rows inside the
 * engine's range only; the others still count for the O(W) checks of the replicated table.  A communicator's share
 * (ceil(W / N) per rank) moves when pm_resize_workers changes W: rows that enter a rank's range count as written there,
 * rows that leave it return to PM_NONE.  A fixed pm_set_shard range does not move; a shrink that cuts into it fails at
 * the next pass (PM_E_INVALID), as without the flag.
 * pm_set_worker_locations, pm_set_worker_addr_rank and pm_set_worker_reputation write nothing the predicate reads.
 * pm_set_asks, pm_set_model_table, pm_set_worker_count, pm_set_shard, pm_attach_comm and a pass that fails discard the
 * stored evaluation.  "A pass that fails" is a reference-mode pass that returns an error once its mode bits are
 * accepted (PM_E_UNSUPPORTED in proximity mode with an enabled max_group_size == 0 ask, say).  Two refusals are not:
 * a call that pm_match or pm_match_local refuses in its mode check, before any pass runs (PM_E_INVALID for a flag
 * combination, PM_E_UNSUPPORTED for PM_INCREMENTAL from pm_match on a shard engine without a communicator), and an
 * auction-mode pass, refused (disabled asks, shard engines, outside the integer domain) or not, neither of which reads
 * or writes the stored evaluation: both keep it and the rows written since.  Without the flag pm_match evaluates every
 * pair as before.
 * pm_match on a shard engine without a communicator refuses the flag (PM_E_UNSUPPORTED): that call resolves one range
 * as if it were the table, so it has no whole-table result to keep incremental.  pm_match_local takes it on any engine.
 * pm_set_ask_enabled keeps the stored evaluation: the next incremental pass also walks the workers whose stored first
 * ask was disabled since ("orphans", from the ask after it) and evaluates every worker against the asks enabled since
 * (only those whose stored first ask lies beyond the first of them; an ask switched off and on again counts as
 * neither).  With many asks enabled the pass evaluates everything instead: the pairs of that walk, |E| x nw, count as
 * |E| x nw / T written rows against the PM_TUNE_INCR cutoff, next to the range's written rows.
 * pm_update_asks, pm_resize_asks, pm_remove_asks and pm_insert_asks keep it too.  A replaced row counts as disabled
 * and enabled again: it is in E when it is enabled now and in D when it was enabled at the stored evaluation, and its orphans are walked from the ask
 * itself, not the one after it (the new row may still accept them); workers whose stored first ask lies beyond it
 * meet it in the E-pass.  Appended and inserted rows are in E.  pm_remove_asks and pm_insert_asks (and a shrink, their
 * tail case) move every stored first ask f with its row, on the device: f - (removed rows below f) + (rows inserted
 * before a position <= f).  A worker whose stored first ask was removed lands on the next kept row and is walked again
 * from that row itself (an orphan); with no kept row after it, its stored first ask is PM_NONE (it had no feasible ask
 * before the removed one).  Replaced, appended and inserted asks count against the cutoff as E does.  Each
 * engine decides
 * against the cutoff by its own range's counts, so in one sharded pass some ranks may evaluate their range in full
 * while others run incrementally; every rank still makes the one exchange.  pm_stats under the flag (nw = the range's
 * workers, W on an unsharded engine):
 *   evals    pair evaluations executed: T x nw on a full evaluation; on an incremental one the kernels' own count over
 *            the three walks (written rows, orphans, newly enabled asks) in the range; 0 when no row and no mask changed;
 *   n_tiles  worker rows walked in full: nw on a full evaluation, else the range's written rows + orphans.         */

/* Auction warm start (PM_AUCTION_WARM).  Every successful auction pass, cold or warm, keeps its state on the device:
 * the worker prices, the assignment, and the caps and reputation floors it ran with.  A warm pass (DESIGN 4):
 *   1. changed rows R0: rows written through pm_upsert_workers, pm_update_workers, pm_set_flags or
 *      pm_set_worker_reputation, and rows added by pm_resize_workers; changed asks A0: asks whose cap or floor differs
 *      from the stored one, and asks toggled by pm_set_ask_enabled since;
 *   2. releases every ask of A0, every owner of a row of R0 and every owner of a row a shrink removed: a released ask
 *      gives up its worker, whose price becomes 0; every other unowned worker with a positive price (only an eps-scaled
 *      pass leaves one) goes to 0 too.  Every changed row and every reset worker joins R;
 *   3. releases, until nothing changes, every ask still holding w_t for which some w in R is feasible with
 *      value(w) - 1 > value(w_t); its worker goes to price 0 and joins R;
 *   4. runs the rounds at eps = 1 (whatever eps_start is) from that state, every unassigned ask active.
 * The result is within T of the optimum of the current instance (the optimum with cost_scale = T + 1), as a cold
 * pass's is; it need not equal the cold pass's result.  The warm pass runs when a stored state exists and
 * |R0| + |A0| <= the PM_TUNE_INCR cutoff, else the pass is cold.  pm_set_asks, pm_set_model_table,
 * pm_set_worker_count, pm_set_auction_params, pm_set_shard, pm_attach_comm and a failed auction pass discard the
 * stored state; reference-mode passes leave it alone.  An auction pass refused before it runs keeps it: disabled asks
 * (PM_E_UNSUPPORTED), tables outside the integer domain (PM_E_INVALID), and an ask, enabled or not, referencing a
 * model pattern missing from the model table (PM_E_STATE; any pattern_id >= n_patterns, 0xFFFFFFFF included); so does
 * a certificate refused for any reason.  pm_update_asks, pm_resize_asks, pm_remove_asks and pm_insert_asks keep it:
 * kept asks keep their holds (slot by slot, under their new indices), A0 also holds every replaced ask and every
 * appended or inserted ask (which has no stored cap or floor, and holds nothing), and step 1 also releases the holder of
 * every removed ask (a shrink of pm_resize_asks, or pm_remove_asks): that worker becomes unowned at its stored price as the shrink runs, joins
 * R at price 0 here when its price was positive, and is not counted in n_released (its ask no longer exists).  The
 * cutoff test counts |R0| + |A0| + the rows past a worker shrink + the removed asks that held a worker.  pm_stats of a
 * warm pass: evals = the release's pair evaluations
 * (classes x raised workers per iteration) + the rounds'; n_rounds = the warm rounds.
 * pm_auction_state reports on the last auction pass: price [its n_workers] (or NULL), warm = 1 if it started warm,
 * n_released = the asks its warm start released; PM_E_STATE when no auction pass ran since the state was discarded. */
int pm_auction_state(pm_engine*, int64_t* price, uint32_t* warm, uint32_t* n_released);

/* Auction reverse rounds (PM_AUCTION_REVERSE).  Each eps phase (eps_start, eps_start / eps_div, ..., 1) runs the
 * forward rounds as without the bit (assignment cleared, prices kept, until every ask holds a worker or withdrew), then
 * reverse rounds until no unowned worker has a positive price.  With S = cost_scale, a(w) = -(ask_price[w] * S), an
 * ask's profit pi(t) = a(w_t) - price[w_t] when it holds w_t, else -(cap[t] + 1) * S.  One reverse round, every bid
 * reading the state at the round's start:
 *   - the bidders are the unowned workers with price > 0;
 *   - a bidder w takes g(t) = a(w) - pi(t) over the asks it is feasible for (candidate, compatible, ask_price <= cap,
 *     reputation >= floor): beta the largest, t* the lowest ask reaching it, omega the second value of the multiset;
 *   - no feasible ask, or beta <= eps: price[w] = 0 and w stays unowned;
 *   - else w offers itself to t* at p' = max(0, omega - eps);
 *   - each ask takes the offer with the highest a(w) - p' (ties: the lowest worker): the worker's price becomes p', the
 *     ask holds it (withdrawn or not before), and the ask's previous worker becomes unowned at its price.
 * The reverse rounds keep eps-complementary slackness and end with every unowned worker at price 0, so the final
 * eps = 1 phase gives a total cost within T of the optimum (the optimum with cost_scale = T + 1), whatever eps_start
 * is (DESIGN 4).  With eps_start = 1 there is nothing to do: the pass equals the pass without the bit.  The pass
 * stores its state like any auction pass; a later PM_AUCTION_WARM pass may start from it.  pm_stats: n_rounds counts
 * the forward rounds; evals adds the reverse rounds' predicate evaluations (classes x bids); with PM_CFG_TIMING,
 * ms_build is the time of the reverse rounds (part of ms_fused).
 * pm_auction_reverse_stats reports on the last auction pass: its eps phases, reverse rounds and bids (each NULL-able),
 * all 0 for a pass without the bit; PM_E_STATE where pm_auction_state returns it. */
int pm_auction_reverse_stats(pm_engine*, uint32_t* n_phases, uint32_t* n_reverse_rounds, uint64_t* n_reverse_bids);

/* Auction warm repair (PM_MODE_AUCTION | PM_AUCTION_WARM | PM_AUCTION_REPAIR).  The same stored state, changed rows R0,
 * changed asks A0 and PM_TUNE_INCR cutoff as a warm pass; without a stored state or above the cutoff it is the cold pass
 * PM_AUCTION_WARM falls back to (warm = 0).  Otherwise, with eps = 1 and a(w), pi(t) as for the reverse rounds:
 *   1. release: every ask of A0, every owner of a row of R0 and every holder of a row a shrink cut off gives up its
 *      worker, which becomes unowned AT ITS STORED PRICE; every other price stays as stored (an eps-scaled pass's
 *      positive prices on unowned workers too);
 *   2. raise: every row of R0 and every row added since (rows >= the stored pass's row count after any shrink) gets
 *      price[w] = max(0, beta(w) - eps), beta(w) = the largest a(w) - pi(t) over the asks t that still hold a worker
 *      after step 1 and are feasible for w (candidate, compatible, ask_price <= cap, reputation >= floor), or 0 when
 *      there is none.  Every beta is read from the state after step 1; a raised row holds no ask, so the order of the
 *      rows does not matter.  Asks that hold no worker do not count: they bid in step 3;
 *   3. the forward rounds at eps = 1 from that state, every unassigned ask active (withdrawn ones too);
 *   4. one reverse stage at eps = 1 (the rounds of PM_AUCTION_REVERSE), until no unowned worker has a positive price.
 * eps-complementary slackness holds after every step, so the result is within T of the optimum of the current instance
 * (the optimum with cost_scale = T + 1), as a cold pass's is (DESIGN 4); it need not equal the cold or the warm pass's
 * result.  Nothing is released beyond step 1.  After pm_update_asks / pm_resize_asks / pm_remove_asks / pm_insert_asks, A0 and the release are those
 * of the warm start: a removed ask's worker is unowned at its stored price.  pm_auction_state: warm = 1, n_released =
 * the asks of step 1.
 * pm_auction_reverse_stats: 1 phase, the reverse rounds and bids of step 4.  pm_stats: n_rounds = the forward rounds;
 * evals = classes x raised rows + the rounds' evaluations + classes x reverse bids; with PM_CFG_TIMING, ms_build = the
 * reverse rounds.  The pass stores its state like any auction pass.  Refusals are those of PM_AUCTION_WARM (disabled
 * asks, shard engines: PM_E_UNSUPPORTED; outside the integer domain: PM_E_INVALID), and none changes the stored state. */

/* Auction certificate.  pm_auction_certificate checks the stored prices and assignment of the last auction pass
 * against the tables, caps, floors and cost_scale as they stand now (so it also audits a stored state after table
 * changes, before the next warm pass), with one sweep over every (ask, worker) pair.  With S = cost_scale,
 * feasible(t,w) as for the reverse rounds and key(w) = ask_price[w] * S + price[w]:
 *   row(t)  = min((cap[t] + 1) * S, the least key(w) over the workers feasible for t)     (ask_bound[t])
 *   bound   = sum_t row(t) - sum_w price[w]: for any prices >= 0 a lower bound on the optimal total cost (weak duality)
 *   cost    = sum over held asks of ask_price[w_t] * S + sum over unheld asks of (cap[t] + 1) * S
 *   gap     = cost - bound >= cost - optimum
 *   slack(t) = key(w_t) - row(t) when t holds w_t, else (cap[t] + 1) * S - row(t)
 * Without shared holds gap = sum_t slack(t) + the sum of the prices of unowned workers; so every slack <= eps with every
 * unowned worker at price 0 gives gap <= T * eps, and with S = T + 1 (every cost a multiple of S) gap < S proves the
 * assignment optimal (DESIGN 4).  After a cold pass at eps_start = 1, a PM_AUCTION_REVERSE pass, a warm pass or a warm
 * repair, on unchanged tables: no bad, shared or priced unowned hold, n_slack_over = 0 and gap <= T; an eps-scaled pass
 * without reverse rounds can leave priced unowned workers, and the gap shows it.  Ownership is recounted from the
 * assignment.  cost, bound, gap and the
 * priced-unowned sum are exact 128-bit integers (hi: the signed high 64 bits, lo: the low 64 bits).  evals = T x W.
 * ask_bound (NULL-able): row(t) per ask.  Refusals, none of which changes anything: NULL engine or out: PM_E_INVALID;
 * no stored state (where pm_auction_state returns PM_E_STATE), a worker count other than the stored pass's, an ask table
 * resized by pm_resize_asks, pm_remove_asks or pm_insert_asks since the last auction pass (pm_update_asks is audited:
 * n_bad_holds shows the holds the new rows reject), or an ask
 * referencing a model pattern missing from the model table: PM_E_STATE; disabled asks: PM_E_UNSUPPORTED; tables and
 * parameters outside the auction's integer domain: PM_E_INVALID.  The call changes nothing pm_fetch_result,
 * pm_get_stats, pm_table_version, pm_auction_state or pm_auction_reverse_stats report, nor what the next warm or repair
 * pass starts from. */
typedef struct pm_auction_cert {
  int64_t  cost_hi;   uint64_t cost_lo;    /* the stored assignment's total cost                           */
  int64_t  bound_hi;  uint64_t bound_lo;   /* a lower bound on the optimum of the current tables           */
  int64_t  gap_hi;    uint64_t gap_lo;     /* cost - bound                                                 */
  uint32_t n_held;                         /* asks holding a worker                                        */
  uint32_t n_bad_holds;                    /* held pairs infeasible under the current tables               */
  uint32_t n_shared;                       /* workers held by more than one ask                            */
  uint32_t n_priced_unowned;               /* unowned workers with price > 0                               */
  uint32_t n_slack_over;                   /* asks whose slack exceeds 1 (the eps of every pass's last phase) */
  uint32_t reserved;
  int64_t  max_slack;                      /* over the asks; 0 without asks                                */
  uint64_t priced_unowned_lo, priced_unowned_hi;   /* the sum of their prices                              */
  uint64_t evals;                          /* (ask, worker) pairs evaluated                                */
} pm_auction_cert;
int pm_auction_certificate(pm_engine*, pm_auction_cert* out, int64_t* ask_bound);

/* Auction state restore.  The stored state lives only in the engine that made it: pm_set_asks, pm_set_worker_count,
 * pm_set_model_table, pm_set_shard, pm_attach_comm, a failed auction pass, a restart and a move to another engine all
 * lose it, and the next pass is cold.  pm_auction_state (the prices) and pm_auction_assignment export it;
 * pm_auction_restore takes it back, into this engine or another one with the same tables.
 * pm_auction_assignment: the stored state's assignment, assigned[t] = the worker ask t holds, or PM_NONE, over the
 * current n_asks (after the remaps of pm_update_asks / pm_resize_asks / pm_remove_asks / pm_insert_asks; worker
 * indices are the stored pass's rows).
 * PM_E_STATE where pm_auction_state returns it; a NULL assigned with n_asks > 0: PM_E_INVALID.
 * pm_auction_restore audits the caller's state against the tables as they stand now, then makes it the stored state.
 * With S = cost_scale, feasible(t,w) as for the reverse rounds (candidate, compatible, ask_price <= cap, reputation >=
 * floor), and key(w), row(t) and slack(t) = key(w_t) - row(t) as for the certificate, under the current tables, caps,
 * floors and S, every hold assigned[t] = w_t is checked in this order and dropped (the ask holds nothing) when
 *   1. bad:     feasible(t, w_t) is false;
 *   2. shared:  w_t is named by more than one ask (every such hold, feasible or not, counts as naming it);
 *   3. slack:   slack(t) > 1.
 * Every other hold is kept.  No price changes: a dropped hold's worker is unowned at its given price.  Dropping holds
 * changes no kept ask's slack, so one pass is enough; the kept holds are feasible, unshared and eps-complementary slack
 * at eps = 1, the state a warm start needs (DESIGN 4).
 * On success the audited state replaces the stored state, if there is one: the stored caps and floors become the
 * current ones, no row or ask counts as changed since it, pm_auction_state reports the restored prices with warm = 0
 * and n_released = 0, pm_auction_reverse_stats reports zeros, and the next PM_AUCTION_WARM pass, with or without
 * PM_AUCTION_REPAIR, starts warm from it.  The certificate of the restored state shows no bad, shared or over-slack
 * hold, and the next warm or repair pass is within T of the optimum of the current instance (the optimum with
 * cost_scale = T + 1), as a cold pass is.  pm_fetch_result, pm_get_stats, pm_table_version and the reference modes'
 * stored evaluation (PM_INCREMENTAL) are untouched.  report (NULL-able) gets the counts; evals = T x W.
 * Refusals, none of which changes anything (neither the stored state nor anything reported on it):
 *   PM_E_INVALID      a NULL pointer with a count > 0; n_workers or n_asks other than the current tables'; an assigned
 *                     entry neither PM_NONE nor < n_workers; a price < 0 or > (K + 1) * S + max(E, 1), K the largest
 *                     current cap and E = eps_start (the bound the warm pass's and the repair's packed-key decisions
 *                     assume); tables and parameters outside the auction's integer domain;
 *   PM_E_STATE        no worker or ask table, no price caps, or an ask referencing a missing model pattern;
 *   PM_E_UNSUPPORTED  disabled asks, a shard range or a communicator (the auction's own refusals).           */
int pm_auction_assignment(pm_engine*, uint32_t* assigned);
typedef struct pm_auction_restore_report {
  uint32_t n_held;            /* holds kept                                                          */
  uint32_t n_dropped_bad;     /* holds infeasible under the current tables                           */
  uint32_t n_dropped_shared;  /* feasible holds of a worker named by more than one ask (all of them)   */
  uint32_t n_dropped_slack;   /* feasible, unshared holds with slack > 1                             */
  uint64_t evals;             /* (ask, worker) pairs evaluated: T x W                                */
} pm_auction_restore_report;
int pm_auction_restore(pm_engine*, const int64_t* price, uint32_t n_workers, const uint32_t* assigned, uint32_t n_asks,
                       pm_auction_restore_report* report);

/* Auction state restore per slot: the export and restore of an engine with demands ("Auction demands").  A slot is one
 * copy of an ask row: slot s of ask t is sum_{u<t} d[u] + k, k < d[t]; there are D = sum d[t] of them (D = n_asks
 * without demands or with every demand 1).
 * pm_auction_slot_assignment: the stored state's assignment per slot, assigned[s] = a worker or PM_NONE, over the
 * current slot table (after the remaps of pm_update_asks, pm_resize_asks, pm_remove_asks, pm_insert_asks and
 * pm_set_ask_demand).  *n_slots is in/out:
 * with assigned NULL the call writes D and returns PM_OK; otherwise *n_slots must equal D.  Refusals: PM_E_INVALID for
 * a NULL n_slots, or *n_slots other than D (D is written back); PM_E_STATE where pm_auction_state returns it (before
 * the size query: nothing is written).  Without demands the output is pm_auction_assignment's, byte for byte.
 * pm_auction_restore_slots: THE RULE: on an engine with demands d it does what pm_auction_restore does on the twin
 * engine (row t repeated d[t] times, its cap and floor repeated), with assigned as the twin's per-ask assignment.  So
 * the same holds are kept, checked in the same order: bad (the pair is infeasible), shared (the worker is named by
 * more than one slot, two slots of one ask included, every naming counts), slack (key(w) - row(t) > 1, t the slot's
 * ask); the same counts are reported, except evals = T x W (the sweep stays per ask; the twin reports D x W, as the
 * certificate does); no price changes.  After a success the audited state is the stored state, every slot may carry a
 * hold, no row or ask counts as changed, pm_auction_state reports the restored prices with warm = 0 and 0 released,
 * pm_auction_reverse_stats reports zeros; pm_fetch_result, pm_get_stats, pm_table_version and the stored evaluation of
 * PM_INCREMENTAL are untouched; the next PM_AUCTION_WARM pass, with or without PM_AUCTION_REPAIR, equals the twin's
 * next pass after its own restore, bit for bit.  Refusals are pm_auction_restore's, with n_slots in place of n_asks
 * (PM_E_INVALID for n_slots other than D, which includes an array exported before a demand change), and none changes
 * anything: not the stored state, the demands, the version or any report.  Without demands the call is
 * pm_auction_restore in every respect. */
int pm_auction_slot_assignment(pm_engine*, uint32_t* assigned, uint32_t* n_slots);
int pm_auction_restore_slots(pm_engine*, const int64_t* price, uint32_t n_workers, const uint32_t* assigned, uint32_t n_slots,
                             pm_auction_restore_report* report);

typedef struct pm_stats {
  uint64_t evals;            /* predicate evaluations executed on the device        */
  uint64_t cost_bytes_written;
  uint64_t cost_bytes_read;
  uint32_t n_tiles;          /* cost tiles; auction mode: class (re)scans           */
  uint32_t n_launches;       /* kernels of this library launched by the last match  */
  uint32_t n_bumped;         /* workers displaced by an under-filled tail group     */
  uint32_t n_rounds;         /* auction rounds (extension mode)                     */
  float ms_build;            /* sum over launches, CUDA events on the engine stream */
  float ms_argmin;
  float ms_fused;
  float ms_resolve;
  float ms_total;
  uint32_t n_build_launches; /* auction mode: class pool refills                    */
  uint32_t n_argmin_launches;
  uint32_t n_fused_launches; /* auction mode: per-ask fallback scans                */
  float    ms_exchange;      /* sharded pass: pack + all-gather + fold, on the engine stream */
  uint64_t exchange_bytes;   /* bytes this rank received in the exchange            */
} pm_stats;

typedef struct pm_result {
  uint32_t n_workers;
  uint32_t n_asks;
  uint32_t n_groups;
  uint32_t n_members;
  /* all arrays are engine-owned pinned host memory, valid until the next
   * pm_fetch_result / pm_destroy on this engine                             */
  const uint32_t* worker_group;   /* [n_workers] group index or PM_NONE                 */
  const uint32_t* worker_ask;     /* [n_workers] ask (config) index or PM_NONE          */
  const uint32_t* group_ask;      /* [n_groups]  configuration of the group             */
  const uint32_t* group_off;      /* [n_groups+1] CSR offsets into group_members        */
  const uint32_t* group_members;  /* worker indices, BTreeSet (addr_rank) order         */
  const int64_t*  ask_best;       /* [n_asks] row argmin: cost<<32 | worker, PM_COST_INF */
  const uint32_t* ask_count;      /* [n_asks] feasible candidate workers of the ask      */
  pm_stats stats;
} pm_result;

/* The management pass (replaces try_form_new_groups, mod.rs:478-628).
 * mode = pm_mode | pm_path.  Device compute only: tables must be resident.  */
int pm_match(pm_engine*, uint32_t mode);
/* D2H of the last match into engine-owned pinned buffers.                   */
int pm_fetch_result(pm_engine*, pm_result* out);
int pm_get_stats(const pm_engine*, pm_stats* out);
/* Build the cost rows of asks [t0, t0+nt) against this engine's worker range and
 * copy them to host_out[nt * n_cols] (row-major, n_cols = shard width): the
 * materialised matrix itself, for external solvers and for bit-exact checks.  */
int pm_build_cost_tile(pm_engine*, uint32_t t0, uint32_t nt, int64_t* host_out);

/* Multi-GPU plumbing (SURVEY 8e): between pm_match_local and pm_match_finish
 * the host all-reduces/all-gathers these device buffers with NCCL.          */
enum pm_buffer {
  PM_BUF_WORKER_FIRST_ASK = 0,  /* uint32[n_workers] global; only the shard range is written */
  PM_BUF_ASK_BEST         = 1,  /* int64 [n_asks] packed row argmin (allreduce MIN)          */
  PM_BUF_ASK_COUNT        = 2,  /* uint32[n_asks] (allreduce SUM)                            */
  PM_BUF_COST_TILE        = 3   /* the cost tile the last materialised pass left, read-only:  */
                                /* bytes = what its tiles spanned (rows per tile x ld x 4 or 8) */
};
/* Re-target the engine at the range [first, first+count) of the worker table (count 0 = to the end). */
int pm_set_shard(pm_engine*, uint32_t first, uint32_t count);
int pm_match_local(pm_engine*, uint32_t mode);    /* evaluation over this shard only */
int pm_match_finish(pm_engine*, uint32_t mode);   /* resolution sweep over the global arrays */
int pm_device_buffer(pm_engine*, uint32_t which, void** dev_ptr, size_t* bytes);
int pm_stream_sync(pm_engine*);

/* ------------------------------------------------------------------------ */
/* Multi-GPU inside the engine (SURVEY 8b "multi-GPU is inside the engine", 8e).  */
/* The path shards by workers: every GPU evaluates all asks against an equal     */
/* contiguous share of the canonical worker order; ONE packed all-gather per     */
/* pass (NCCL over NVLink, resolved at run time) carries {per-ask (min cost,     */
/* argmin) + feasible count, per-worker first feasible ask}; every GPU then runs */
/* the same O(W+T) resolution sweep on identical arrays.  With a communicator    */
/* attached pm_match does all of it; the shard is the rank's share.              */
/* ------------------------------------------------------------------------ */
typedef struct pm_comm pm_comm;
#define PM_COMM_ID_BYTES 128
/* one process per GPU: rank 0 makes the id, the host hands it to every rank (any transport) */
int  pm_comm_unique_id(uint8_t id_out[PM_COMM_ID_BYTES]);
int  pm_comm_create(const uint8_t unique_id[PM_COMM_ID_BYTES], uint32_t n_ranks, uint32_t rank, int32_t device,
                    pm_comm** out);
void pm_comm_destroy(pm_comm*);
int  pm_attach_comm(pm_engine*, pm_comm*);   /* NULL detaches; the communicator must outlive the engine's use of it */

/* One process, several GPUs — the form the orchestrator's single management loop                          */
/* (crates/orchestrator/src/main.rs:283-289, mod.rs:180-203) calls: table calls go to every device,        */
/* pm_multi_match is one sharded pass, the result is read from device 0.  cfg->device/shard/stream ignored. */
typedef struct pm_multi pm_multi;
int         pm_multi_create(const pm_cfg* cfg, const int32_t* devices, uint32_t n_devices, pm_multi** out);
void        pm_multi_destroy(pm_multi*);
uint32_t    pm_multi_size(const pm_multi*);
pm_engine*  pm_multi_engine(pm_multi*, uint32_t i);   /* per-device access (stats, auction params, ...) */
const char* pm_multi_last_error(const pm_multi*);
int pm_multi_set_asks(pm_multi*, const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts, uint32_t n_opts);
int pm_multi_set_ask_enabled(pm_multi*, const uint32_t* idx, const uint8_t* enabled, uint32_t n);
/* pm_update_asks / pm_resize_asks / pm_remove_asks / pm_insert_asks on every device; a refused call changes no device */
int pm_multi_update_asks(pm_multi*, const uint32_t* idx, const pm_ask* asks, uint32_t n,
                         const pm_gpu_opt* opts, uint32_t n_opts);
int pm_multi_resize_asks(pm_multi*, uint32_t n_asks, const pm_ask* added, const pm_gpu_opt* opts, uint32_t n_opts);
int pm_multi_remove_asks(pm_multi*, const uint32_t* idx, uint32_t n);
int pm_multi_insert_asks(pm_multi*, const uint32_t* before, const pm_ask* asks, uint32_t n, const pm_gpu_opt* opts,
                         uint32_t n_opts);
int pm_multi_set_model_table(pm_multi*, const uint32_t* bits, uint32_t n_patterns, uint32_t n_models,
                             uint32_t words_per_pattern);
int pm_multi_set_worker_count(pm_multi*, uint32_t n_workers);
int pm_multi_upsert_workers(pm_multi*, const pm_worker_a* a, const pm_worker_b* b, uint32_t first, uint32_t n);
int pm_multi_set_worker_locations(pm_multi*, const double* lat, const double* lon, uint32_t first, uint32_t n);
int pm_multi_set_worker_addr_rank(pm_multi*, const uint32_t* rank, uint32_t first, uint32_t n);
int pm_multi_set_flags(pm_multi*, const uint32_t* idx, const uint32_t* flags, uint32_t n);
/* the resident-table deltas (pm_resize_workers, pm_update_workers) on every device: with them the management loop
 * runs PM_INCREMENTAL through pm_multi_match, each device re-evaluating only its share's written rows */
int pm_multi_resize_workers(pm_multi*, uint32_t n_workers);
int pm_multi_update_workers(pm_multi*, const uint32_t* idx, const pm_worker_a* a, const pm_worker_b* b, const double* lat,
                            const double* lon, uint32_t n);
/* pm_remove_workers / pm_insert_workers on every device's replicated table, each device keeping its own share's stored
 * evaluation (as pm_multi_resize_workers does); a refused call changes no device */
int pm_multi_remove_workers(pm_multi*, const uint32_t* idx, uint32_t n);
int pm_multi_insert_workers(pm_multi*, const uint32_t* before, const pm_worker_a* a, const pm_worker_b* b, const double* lat,
                            const double* lon, uint32_t n);
int pm_multi_sync(pm_multi*);
/* changes whenever any table call changed a table on any device, including calls made directly on
 * pm_multi_engine(m, i) (the sum of the engines' pm_table_version); 0 for NULL                                      */
uint64_t pm_multi_table_version(const pm_multi*);
/* With more than one device, a pass that fails on any device aborts every communicator, so that no device is left
 * waiting in the exchange.  The next pm_multi_match re-creates them over the same devices (ncclCommInitAll), attaches
 * them again and discards every device's stored evaluation (as pm_attach_comm does): that pass runs in full on every
 * device.  A refused pass (PM_E_UNSUPPORTED in proximity mode with an enabled max_group_size == 0 ask, say) is
 * therefore retried like any other once its cause is gone.                                                            */
int pm_multi_match(pm_multi*, uint32_t mode);
int pm_multi_fetch_result(pm_multi*, pm_result* out);

uint32_t pm_abi_version(void);

/* ------------------------------------------------------------------------ */
/* Host mirror of the reference's plugin interface for this path              */
/* (protocol_b200/csrc/pm_plugin.cpp).  In-process tables replace Redis; group */
/* formation always runs on the engine (no CPU evaluation path).              */
/* ------------------------------------------------------------------------ */
typedef struct pm_plugin pm_plugin;

typedef struct pm_plugin_policy {     /* mod.rs:71-98 */
  uint8_t task_switching_enabled;     /* TaskSwitchingPolicy.enabled               */
  uint8_t prefer_larger_groups;       /* TaskSwitchingPolicy.prefer_larger_groups  */
  uint8_t proximity_enabled;          /* ProximityOptimizationPolicy.enabled       */
  uint8_t canonical_addresses;        /* 1: every address that enters the mirror goes through pm_address_canonical (what the  */
                                      /* reference's Address parse + to_string does); an id that is not an address is rejected */
                                      /* (discovery entries: skipped, monitor.rs:240,425-429).  0: strings are opaque.        */
} pm_plugin_policy;

typedef struct pm_kv { const char* key; const char* value; } pm_kv;

typedef struct pm_task_desc {         /* shared/src/models/task.rs:162-184 (fields on the path) */
  const char* id;                     /* Uuid as string */
  const char* name;
  const char* image;
  int64_t created_at;
  const pm_kv* env_vars;      uint32_t n_env_vars;      int32_t has_env_vars;      /* Option<HashMap> */
  const char* const* cmd;     uint32_t n_cmd;           int32_t has_cmd;           /* Option<Vec>     */
  const pm_kv* volume_mounts; uint32_t n_volume_mounts; int32_t has_volume_mounts; /* {host_path, container_path} */
  /* scheduling_config (task.rs:58-61): 0 = None; 1 = Some, no "node_groups" plugin entry;
   * 2 = "node_groups" entry without "allowed_topologies"; 3 = allowed_topologies list below */
  int32_t scheduling;
  const char* const* allowed_topologies; uint32_t n_allowed_topologies;
} pm_task_desc;

typedef struct pm_node_desc {         /* orchestrator/src/models/node.rs:10-37 (fields on the path) */
  const char* address;                /* Address::to_string(), opaque, EIP-55 cased by the caller */
  uint32_t status;                    /* NodeStatus ordinal: Discovered=0, WaitingForHeartbeat, Healthy=2,
                                         Unhealthy, Dead=4, Ejected, Banned, LowBalance=7 (node.rs:74-85) */
  const char* p2p_id;                 /* NULL == None */
  uint32_t spec_flags;                /* PM_W_HAS_* presence bits of compute_specs */
  uint32_t gpu_count, gpu_mem_mb;
  const char* gpu_model;
  uint32_t cpu_cores, ram_mb, storage_gb;
  int32_t has_location;
  double lat, lon;
  const char* ip_address;             /* NULL keeps the stored value */
  uint16_t port;
  uint16_t reserved;
  int64_t last_status_change_ms;      /* 0 keeps the stored value (Option<DateTime<Utc>>) */
} pm_node_desc;

typedef struct pm_discovery_node {    /* shared/src/models/node.rs:552-570 (fields the monitor reads) */
  pm_node_desc node;                  /* id (as address), compute_specs, location; status/p2p ignored */
  const char* ip_address;
  uint16_t port;
  uint8_t is_validated, is_active, is_provider_whitelisted, is_blacklisted;
  uint8_t has_latest_balance, latest_balance_is_zero;
  int64_t last_updated_ms;            /* < 0 == None */
} pm_discovery_node;

/* NodeGroupsPlugin::new_with_policy (mod.rs:129-175).  engine may be NULL (then
 * pm_plugin_try_form_new_groups fails with PM_E_NO_DEVICE); policy NULL = defaults. */
int  pm_plugin_create(pm_engine* engine, const pm_plugin_policy* policy, pm_plugin** out);
/* Same, with the formation pass on several GPUs: every table call of pm_plugin_try_form_new_groups goes through
 * pm_multi_* and the pass is pm_multi_match (each device evaluates its share of the workers, incrementally on resident
 * tables).  Solo-group merging runs on a sibling engine of pm_multi_engine(multi, 0), on device 0 only.  multi NULL is
 * PM_E_INVALID.  The plugin does not own the pm_multi (nor an engine): destroy the plugin first.                      */
int  pm_plugin_create_multi(pm_multi* multi, const pm_plugin_policy* policy, pm_plugin** out);
void pm_plugin_destroy(pm_plugin*);
const char* pm_plugin_last_error(const pm_plugin*);
/* duplicate name / max < min are PM_E_INVALID (the reference panics, mod.rs:141-147);
 * requirements NULL == compute_requirements: None, else ComputeRequirements::from_str */
int pm_plugin_add_config(pm_plugin*, const char* name, uint32_t min_group_size, uint32_t max_group_size,
                         const char* requirements);
int pm_plugin_seal_configs(pm_plugin*);                                   /* the ctor's sort, mod.rs:150-164 */
int pm_plugin_enable_configuration(pm_plugin*, const char* name, int enable);   /* mod.rs:1328-1346 */
int pm_plugin_upsert_node(pm_plugin*, const pm_node_desc*);                /* NodeStore::add_node / update */
int pm_plugin_set_node_status(pm_plugin*, const char* address, uint32_t status); /* + handle_status_change */
/* DiscoveryMonitor: reconcile validated discovery nodes into the table
 * (discovery/monitor.rs:195-435); the Theta(N^2) same-endpoint scan is a hash lookup here. */
int pm_plugin_sync_discovery(pm_plugin*, const pm_discovery_node* nodes, uint32_t n, int64_t now_ms,
                             uint32_t max_healthy_nodes_with_same_endpoint, uint32_t* n_new);
/* same, from the discovery service's wire format: {"success":true,"data":[DiscoveryNode,...]} */
int pm_plugin_sync_discovery_json(pm_plugin*, const char* json, size_t len, int64_t now_ms,
                                  uint32_t max_healthy_nodes_with_same_endpoint, uint32_t* n_new);
int pm_plugin_get_node(pm_plugin*, const char* address, char* buf, size_t len);   /* JSON or null */
int pm_plugin_add_task(pm_plugin*, const pm_task_desc*);                   /* TaskStore::add_task + on_task_created */
int pm_plugin_delete_task(pm_plugin*, const char* id);                     /* delete_task + on_task_deleted */
int pm_plugin_try_form_new_groups(pm_plugin*, uint32_t* n_formed);         /* mod.rs:478-628 via pm_match */
int pm_plugin_try_merge_solo_groups(pm_plugin*, uint32_t* n_merged);       /* mod.rs:631-971 via pm_match */
/* the "upload:<node>:<group>:<file>" key the storage route records; feeds ${TOTAL_UPLOAD_COUNT} */
int pm_plugin_record_upload(pm_plugin*, const char* address, const char* group_id, const char* file_name);
/* JSON out (NUL-terminated into buf): NodeGroup {"id","nodes","configuration_name","task_id"} or null */
int pm_plugin_get_node_group(pm_plugin*, const char* address, char* buf, size_t len);
int pm_plugin_get_all_groups(pm_plugin*, char* buf, size_t len);           /* sorted by id, mod.rs:1040 */
/* get_group_by_id (mod.rs:1046-1055); validate_group_exists (:1067-1070) is `result != null`      */
int pm_plugin_get_group_by_id(pm_plugin*, const char* group_id, char* buf, size_t len);
/* handle_group_not_found (mod.rs:1073-1119): the task of a group that was dissolved under the scheduler goes
 * to the first idle group in get_all_groups() order (SET NX); *reassigned = 1 when one took it      */
int pm_plugin_handle_group_not_found(pm_plugin*, const char* group_id, const char* task_id, uint32_t* reassigned);
/* The node table as the engine's SoA tables (SURVEY 8 A21 / 8f-1), exactly what a management pass uploads: rows in
 * node_store.get_nodes() order (stable status-class sort, node_store.rs:195-206), candidate flags (PM_W_HEALTHY / P2P /
 * ASSIGNED, mod.rs:492-497), locations, BTreeSet<String> address ranks.  Any array may be NULL; capacity in rows.    */
int pm_plugin_export_tables(pm_plugin*, pm_worker_a* a, pm_worker_b* b, double* lat, double* lon, uint32_t* addr_rank,
                            uint32_t capacity, uint32_t* n_rows);
/* The inverse of pm_plugin_redis_writeback, for start-up: a group read back from the reference's keys
 * (`node_group:<id>` JSON + `group_task:<id>`) is put into the tables as it is.  nodes come in the stored
 * (BTreeSet) order; task_id NULL = no claim; created_at_ms < 0 = now.  PM_E_STATE when the id exists or a node is
 * already in a group.  The group id counter moves past ids of the engine's own form (lower-case hex).        */
int pm_plugin_restore_group(pm_plugin*, const char* id, const char* configuration_name, const char* const* nodes,
                            uint32_t n_nodes, const char* task_id, int64_t created_at_ms);
/* Redis write-back in the reference's key formats (mod.rs:25-28,299-322,471-476), as a JSON array of
 * commands, so /groups, /nodes, storage routes and the metrics sync keep working unchanged.        */
int pm_plugin_redis_writeback(pm_plugin*, char* buf, size_t len);
/* Scheduler::get_task_for_node (scheduler/mod.rs:26-74) with the plugin chain
 * [NodeGroupsPlugin] when configurations exist, else [NewestTaskPlugin]:
 * writes {"current_task": Task|null} (shared/src/models/heartbeat.rs:7-22). */
int pm_scheduler_get_task_for_node(pm_plugin*, const char* address, char* buf, size_t len);

#ifdef __cplusplus
}
#endif
#endif /* PRIME_MATCH_H */
