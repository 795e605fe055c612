// engine.cu -- libgrove_place.so: host side of the placement engine and the C ABI of
// include/grove_place.h.  Everything that computes a placement runs in the kernels of kernels.cuh;
// the host sorts the topology once per label change, validates and uploads tables, and drives the
// relaxation rounds (relax.cuh).  There is no CPU fallback: without a CUDA device the engine cannot be created.
#include <omp.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdio>
#include <array>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <new>
#include <numeric>
#include <string>
#include <vector>

#include <cub/device/device_merge_sort.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "kernels.cuh"

using namespace grove;

namespace {

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;  // elements
  ~DevBuf() { release(); }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  // grows geometrically: a pending set that creeps up tick after tick (churn) must not pay a cudaFree + cudaMalloc
  // of every table per cycle; falls back to the exact size when the padded one does not fit
  cudaError_t ensure(size_t n) {
    if (n <= cap) return cudaSuccess;
    const size_t want = std::max<size_t>(std::max<size_t>(n, (64u << 10) / sizeof(T)), cap + cap / 2);
    release();
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(T));
    if (e == cudaSuccess) { cap = want; return e; }
    (void)cudaGetLastError();
    e = cudaMalloc(reinterpret_cast<void**>(&p), std::max<size_t>(n, 1) * sizeof(T));
    if (e == cudaSuccess) cap = std::max<size_t>(n, 1); else p = nullptr;
    return e;
  }
};

template <typename T>
struct PinBuf {
  T* p = nullptr;
  size_t cap = 0;
  ~PinBuf() { if (p) cudaFreeHost(p); }
  cudaError_t ensure(size_t n) {
    if (n <= cap) return cudaSuccess;
    // pinned allocations cost milliseconds: start at 256 KB and double, so a growing pending set re-allocates rarely
    const size_t want = std::max<size_t>(std::max<size_t>(n, (256u << 10) / sizeof(T)), cap * 2);
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    cudaError_t e = cudaMallocHost(reinterpret_cast<void**>(&p), want * sizeof(T));
    if (e == cudaSuccess) cap = want; else p = nullptr;
    return e;
  }
};

// Size of the engine's host thread team (table validation, signature interning, staging copies).  One size for every
// parallel region: libgomp re-creates its team whenever the size changes.  Not taken from OMP_NUM_THREADS: launchers
// such as torchrun export OMP_NUM_THREADS=1 for every rank, which would serialise the per-cycle host work; the knob is
// GROVE_HOST_THREADS (default 8), capped by the processors this process may run on.
int host_threads() {
  static const int t = [] {
    int want = 8;
    if (const char* v = std::getenv("GROVE_HOST_THREADS")) want = std::atoi(v);
    return std::max(1, std::min(want, omp_get_num_procs()));
  }();
  return t;
}

// a host table the engine owns, in pinned memory: the caller's array is copied in once (by a few threads when it is
// large) and the upload from it is a plain asynchronous DMA
template <typename T>
struct PinVec {
  PinBuf<T> b;
  size_t n = 0;
  T& operator[](size_t i) { return b.p[i]; }
  const T& operator[](size_t i) const { return b.p[i]; }
  T* data() { return b.p; }
  cudaError_t assign(const T* src, size_t cnt) {
    cudaError_t e = b.ensure(cnt);
    if (e != cudaSuccess) return e;
    n = cnt;
    const size_t bytes = cnt * sizeof(T);
    // one team size for every parallel region of the engine: libgomp re-creates its thread team whenever the size changes
    const int T_ = bytes >= (256u << 10) ? host_threads() : 1;
#pragma omp parallel for num_threads(T_) schedule(static)
    for (int t = 0; t < T_; ++t) {
      const size_t a = bytes * t / T_, z = bytes * (t + 1) / T_;
      std::memcpy(reinterpret_cast<char*>(b.p) + a, reinterpret_cast<const char*>(src) + a, z - a);
    }
    return cudaSuccess;
  }
};

uint32_t fmix32(uint32_t x) {
  x = x * 0x9E3779B1u + 0x7F4A7C15u;
  x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
  return x;
}

}  // namespace

struct grove_engine {
  grove_config_t cfg{};
  std::string err;
  cudaStream_t stream = nullptr;
  cudaStream_t stream_score = nullptr;  // K2 runs beside the relaxation (they only share the fit data)
  cudaEvent_t ev_fit = nullptr, ev_score = nullptr, ev_s0 = nullptr, ev_s1 = nullptr;
  cudaEvent_t ev_nodes_up = nullptr, ev_tables_up = nullptr;  // the last upload out of the pinned node staging buffer / gang tables
  cudaEvent_t ev[10]{};

  // ---- topology (static until labels change) ----
  uint32_t N = 0, Npad = 0, L = 0, words = 0;
  std::vector<uint32_t> raw_dom;      // caller order, N * MAX_LEVELS: cache key
  std::vector<uint32_t> perm, inv;    // sorted <-> caller
  std::vector<uint32_t> tdom;         // sorted order, N * MAX_LEVELS tree-ified ids
  std::vector<uint8_t> vdepth;
  std::vector<uint32_t> dom_lo[GROVE_MAX_LEVELS], dom_hi[GROVE_MAX_LEVELS];
  uint32_t n_dom[GROVE_MAX_LEVELS]{}, unit[GROVE_MAX_LEVELS]{};
  DevBuf<grove_node_t> d_nodes_in;    // caller order, as loaded
  DevBuf<uint4> d_nres, d_ndom;
  DevBuf<uint32_t> d_perm, d_inv;
  DevBuf<uint8_t> d_vdepth;
  DevBuf<uint32_t> d_dom_lo[GROVE_MAX_LEVELS], d_dom_hi[GROVE_MAX_LEVELS], d_next_dom[GROVE_MAX_LEVELS];
  bool nodes_loaded = false;

  // ---- gang tables ----
  uint32_t G = 0, Q = 0, S = 0, P = 0;
  PinVec<grove_gang_t> gangs;
  PinVec<grove_clique_t> cliques;
  PinVec<grove_scope_t> scopes;
  PinVec<uint32_t> ccount;         // [Q] min_replicas | replicas << 16: what the engine reads, whichever entry submitted
  bool wide = false;               // some gang has more than GROVE_MAX_GANG_PODS pods or some clique more than 255 replicas
  PinBuf<uint8_t> h_state0;        // initial gang states of a cycle
  PinBuf<GangInfo> ginfo_pin;      // derived tables are built straight into pinned memory: their upload is a plain DMA
  PinBuf<CliqueInfo> cinfo_pin;
  PinBuf<uint32_t> by_rank_pin;
  PinBuf<uint32_t> shape_rep_pin;
  GangInfo* ginfo = nullptr;
  CliqueInfo* cinfo = nullptr;
  std::vector<uint4> sigs;
  uint32_t n_sigs = 0;
  bool gangs_loaded = false, ginfo_dirty = true;
  DevBuf<grove_gang_t> d_gangs;
  DevBuf<grove_clique_t> d_cliques;
  DevBuf<grove_scope_t> d_scopes;
  DevBuf<uint32_t> d_ccount;           // uploaded for wide submissions (the kernels of an ordinary cycle read the clique records)
  DevBuf<uint32_t> d_wide_node;        // wide cycles: one entry stack per k_eval warp (relax.cuh Relax::wide_node)
  DevBuf<uint16_t> d_wide_meta;
  DevBuf<GangInfo> d_ginfo;
  DevBuf<CliqueInfo> d_cinfo;
  DevBuf<uint4> d_sigs;
  DevBuf<uint32_t> d_by_rank;
  std::vector<uint32_t> shape_rep;     // one representative gang per distinct gang shape
  uint32_t n_shapes = 0, pl_words = 0, pl_off[GROVE_MAX_LEVELS]{};
  bool shape_tables = false;
  DevBuf<uint32_t> d_shape_rep, d_shape_bits;

  // ---- relaxation state (relax.cuh) ----
  DevBuf<uint32_t> d_ctl, d_chg_round, d_eval_list, d_ent_node, d_cur_info, d_cur_glo, d_extent, d_sc_lo;
  DevBuf<uint32_t> d_nxt_node, d_nxt_info, d_nxt_glo, d_nxt_extent, d_nxt_sc_lo;
  DevBuf<uint32_t> d_rem_round, d_last_eval, d_fail_upto, d_nlive, d_ovf_head, d_ovf_next, d_add_stamp, d_rem_stamp, d_F, d_capsum, d_capmax, d_fin, d_totals;
  DevBuf<uint16_t> d_ent_meta, d_cur_n, d_nxt_meta, d_nxt_n;
  DevBuf<uint8_t> d_last_att, d_state, d_tstate, d_dirty, d_sc_lvl, d_nxt_tstate, d_nxt_sc_lvl, d_cap8, d_T;
  DevBuf<uint4> d_claims, d_ovf_claim;
  DevBuf<int4> d_ctot;
  DevBuf<uint32_t> d_cmaxr;
  DevBuf<grove_gang_status_t> d_status;
  DevBuf<grove_scope_status_t> d_scope_status;
  DevBuf<grove_placement_t> d_out;
  bool any_preferred = false;  // some gang / scope / clique carries a Preferred level
  uint32_t max_gang_pods = 0;
  uint32_t n_sm = 132;  // H100 SXM; replaced by the device's own count at creation
  uint32_t cap_off[GROVE_MAX_LEVELS]{}, cap_stride = 0;
  bool dbg_on = false;
  DevBuf<uint32_t> d_dbg;
  uint32_t tune_window = 0;        // gangs beyond the settled prefix that relax concurrently (0: all)
  uint32_t tune_entry = 1024;      // gangs that may join the window per round (0: no limit)
  uint32_t tune_refresh = 1536;    // rebuild the capacity tables once the settled prefix has advanced this many gangs
  uint32_t tune_warp_ctas = 4;     // CTAs per SM of the warp-per-gang bookkeeping kernels (apply / detect / settle)
  uint32_t tune_batch = 3;         // rounds enqueued between two looks at the control words (GROVE_TUNE_AHEAD=0 / GROVE_DEBUG_ADMIT)
  uint32_t tune_ahead = 3;         // rounds kept in the queue while the host follows the relaxation through host-mapped progress words
  uint32_t tune_eval_ctas = 0;     // k_eval CTAs in all (0: tune_heavy_ctas per SM)
  uint32_t tune_heavy_att = 4;     // a gang whose last evaluation made this many attempts is heavy: a whole k_eval CTA next time
  uint32_t tune_max_att = 3;       // a light (one-warp) evaluation gives up after this many attempts and comes back heavy
  uint32_t tune_heavy_ctas = 2;    // k_eval CTAs per SM: 2 fill the register file (8 warps x 128 registers each)
  bool tune_overlap = true;        // K2 on a second stream beside the relaxation (GROVE_TUNE_OVERLAP=0 serialises them, e.g. to time K2 alone)
  bool tune_score = false;         // K2 score matrix: false = materialised on request (grove_build_score_matrix / the row getters),
                                   // true = every cycle, on the second stream beside the relaxation
  bool score_valid = false;        // d_T holds the matrix of the last cycle's start snapshot
  DevBuf<uint32_t> d_F0;           // K1 output over the cycle-start snapshot (the engine's own F follows the committed state)
  PinBuf<uint32_t> h_upd_idx;
  PinBuf<grove_node_t> h_upd_recs;
  cudaEvent_t ev_upd = nullptr;
  DevBuf<uint32_t> d_upd_idx;
  DevBuf<grove_node_t> d_upd_recs;
  DevBuf<grove_node_t> d_nodes_out;  // grove_get_nodes scratch
  PinBuf<uint32_t> h_ctl;
  uint32_t* h_live = nullptr;      // host-mapped words the last CTA of k_detect writes every round (round, front, done, refresh, ...):
  uint32_t* d_live = nullptr;      // the host follows the relaxation by reading memory, without a blocking call (grove_run_cycle)
  PinBuf<grove_gang_status_t> h_status;
  PinBuf<grove_scope_status_t> h_scope_status;
  PinBuf<grove_placement_t> h_out;
  PinBuf<grove_node_t> h_stage_nodes;
  uint32_t n_out = 0;
  bool have_results = false, have_scopes = false;
  grove_cycle_stats_t last{};

  bool in_cycle = false;
  uint64_t launches = 0;
  std::vector<grove_victim_t> victims;   // of the last grove_run_cycle_preempt
  // node-range shard of this handle (cfg.rank of cfg.world; the whole table when world <= 1): sorted node indices, cut at
  // top-level domain boundaries
  uint32_t shard_lo = 0, shard_hi = 0;
  bool score_pass_valid = false;   // the capacity tables + T describe the loaded snapshot (grove_run_score_pass)
  uint32_t t_c0 = 0, t_cpr = 0;    // ... and T holds the 16-node chunks [t_c0, t_c0 + t_cpr) of every row
  DevBuf<uint32_t> d_sig_sum;
  // holds of the replacement gangs of a grove_run_cycle_reuse (relax.cuh "holds"); holds_on only while such a cycle runs
  DevBuf<uint32_t> d_hold_off;
  DevBuf<uint4> d_hold;
  uint32_t n_hold = 0;
  bool holds_on = false;
  // reclaim views of a grove_run_cycle_reuse_preempt (reclaim.cuh): the running gangs' holdings by sorted node, their
  // priorities, the gone mask, the class's free table, the free table after the ordinary pass (restored on an error), and
  // the row gather / patch buffers
  DevBuf<uint32_t> d_rc_off, d_rc_idx, d_rc_bad;
  DevBuf<uint4> d_rc_ent, d_rc_real, d_rc_base, d_rc_rows, d_rc_patch;
  DevBuf<int32_t> d_rc_prio;
  DevBuf<uint8_t> d_rc_gone, d_rc_evict;
  // the donor sets of grove_run_cycle_reclaim_queues (donor.cuh): per scanned queue its pairs in victim order, the quotas, the
  // running gangs' usage, queues and chains, the per-class loads and the per-(running gang, depth) verdicts
  DevBuf<uint32_t> d_dn_off, d_dn_qid, d_dn_parent, d_dn_rq;
  DevBuf<uint2> d_dn_pr;
  DevBuf<unsigned long long> d_dn_quota;
  DevBuf<long long> d_dn_load, d_dn_use;
  DevBuf<uint8_t> d_dn_fin, d_dn_bits;
  // grove_diagnose (diagnose.cuh): whether the outputs on the device describe an ordinary cycle over the current inputs, the
  // per-node usage lists, the batch descriptors, the per-domain capacity sums and the records
  enum Diag : uint8_t { kDiagNoCycle, kDiagReady, kDiagRunning, kDiagChanged, kDiagSpread, kDiagFence, kDiagImex, kDiagFairShare } diag = kDiagNoCycle;
  DevBuf<uint32_t> d_dg_cnt, d_dg_off, d_dg_cur, d_dg_minr;
  DevBuf<uint4> d_dg_rec;
  DevBuf<DiagGang> d_dg_gang;
  DevBuf<unsigned long long> d_dg_col;
  DevBuf<grove_gang_diag_t> d_dg_gout;
  DevBuf<grove_clique_diag_t> d_dg_qout;
  // topology spread (grove_set_spread; spread.cuh): the set of the current submission; the spread kernels run only while it has
  // members (sp_members > 0)
  uint32_t sp_groups = 0, sp_members = 0, sp_cnt_words = 0, sp_dcls_words = 0, sp_dcls_off[GROVE_MAX_LEVELS]{};
  DevBuf<uint32_t> d_sp_group, d_sp_row, d_sp_info, d_sp_mem_off, d_sp_mem, d_sp_cls, d_sp_cnt_off, d_sp_seed, d_sp_cnt, d_sp_dcls;
  DevBuf<uint32_t> d_sp_allowed, d_sp_stamp;
  DevBuf<uint8_t> d_sp_skewed;
  PinBuf<uint8_t> h_sp_skewed;
  // fences (grove_set_fences; fence.cuh): the fencing gangs of the current submission in rank order; the fence kernels run only
  // while there are some
  std::vector<uint32_t> fc_gangs, fc_off;   // (fc_off: first word of each gang's per-clique, per-domain sums; fc_words in all.  The
  size_t fc_words = 0;                      // labels, hence the domains, cannot change while the set is kept)
  DevBuf<uint32_t> d_fc_gang, d_fc_off, d_fc_have, d_fc_slot;
  DevBuf<uint4> d_fc_list;
  // grove_run_cycle_consolidate (consolidate.cuh): the moves of the last such cycle, a target's view W, its per-domain capacity sums
  // over F and W, the ranked try ranges and the (gang, offset) words k_fence_have reads
  std::vector<grove_move_t> moves;
  DevBuf<uint4> d_cs_view;
  DevBuf<uint32_t> d_cs_have, d_cs_rank, d_cs_zero;
  // queue limits (grove_set_queues; queue.cuh): the tables of the current submission's members; the queue kernels run only while
  // there are some (qu_members > 0)
  uint32_t qu_members = 0, qu_scanned = 0;
  bool qu_given = false;                   // a set was given for the current submission, members or not
  std::vector<grove_queue_t> qu_queues;    // ... and what it was (grove_run_cycle_preempt_queues)
  std::vector<uint32_t> qu_gang_queue;
  DevBuf<uint32_t> d_qu_slot, d_qu_mem, d_qu_mem_fin, d_qu_q_off;
  DevBuf<uint4> d_qu_mem_pair, d_qu_pr;
  DevBuf<long long> d_qu_rmin, d_qu_q_base, d_qu_head;
  DevBuf<unsigned long long> d_qu_use;
  DevBuf<uint8_t> d_qu_gate, d_qu_cap;
  // bin-packing (grove_set_binpack; binpack.cuh): the pack level of every gang of the current submission (GROVE_LEVEL_NONE = not a
  // member); the pick kernels run only while there are members (bp_members > 0)
  std::vector<uint8_t> bp_level;
  uint32_t bp_members = 0;
  bool bp_given = false;                   // a set was given for the current submission, members or not
  bool bp_anchors = false;                 // d_ginfo holds picked anchors (the host's ginfo keeps the defaults)
  std::vector<uint32_t> bp_picks;          // caller index of each gang's pick in the last cycle that ran with a set
  bool bp_have_picks = false;
  PinBuf<uint4> h_bp_mem;
  PinBuf<uint32_t> h_bp_pick;
  DevBuf<uint4> d_bp_mem;
  DevBuf<BpSum> d_bp_sum;
  DevBuf<BpKey> d_bp_key;
  DevBuf<uint32_t> d_bp_idx, d_bp_rank, d_bp_pick;
  DevBuf<uint8_t> d_bp_tmp;
  // ComputeDomain exclusivity (grove_set_compute_domains; imex.cuh): the CD of every clique and gang of the current submission and
  // owner0 in caller order; the kImex kernels run only while some clique is enrolled (im_enrolled > 0)
  std::vector<uint32_t> im_cd, im_gang_cd, im_owner0, im_owners;
  uint32_t im_enrolled = 0;
  bool im_given = false;                   // a set was given for the current submission, enrolled cliques or not
  bool im_have_owners = false;             // im_owners holds the owners after the last cycle that ran with a set
  std::vector<uint32_t> h_im_rank_cd, h_im_owner;
  DevBuf<uint32_t> d_im_cd, d_im_rank_cd, d_im_owner, d_im_nenr;
  // fair-share order (grove_set_fair_share; fairshare.cuh): the quotas of the queue set, kept with it; the turn order and the
  // fixed-point counts of the last fair-share cycle; the tree and per-gang tables of O(R) and its sort / scan buffers
  bool fs_given = false, fs_have_order = false;
  std::vector<grove_queue_quota_t> fs_quotas;
  std::vector<uint32_t> fs_order;
  grove_fair_share_stats_t fs_stats{};
  DevBuf<uint32_t> d_fs_parent, d_fs_leaf, d_fs_rank, d_fs_owner, d_fs_vals, d_fs_prev, d_fs_first;
  DevBuf<uint8_t> d_fs_depth, d_fs_tmp;
  DevBuf<long long> d_fs_load0;
  DevBuf<unsigned long long> d_fs_quota;
  DevBuf<FsKey> d_fs_keys, d_fs_keys2;
  DevBuf<FsUse> d_fs_use, d_fs_useq, d_fs_before;
  PinBuf<uint32_t> h_fs_order;
};


#define CU_TRY(e, expr)                                                                       \
  do {                                                                                        \
    cudaError_t _c = (expr);                                                                  \
    if (_c != cudaSuccess) {                                                                  \
      (e)->err = std::string(#expr) + ": " + cudaGetErrorString(_c);                          \
      return _c == cudaErrorMemoryAllocation ? GROVE_ERR_OOM : GROVE_ERR_CUDA;                \
    }                                                                                         \
  } while (0)

static int32_t fail(grove_engine* e, int32_t code, const char* msg) { e->err = msg; return code; }
static int32_t refuse_spread(grove_engine* e, const char* entry) {
  e->err = std::string(entry) + ": not supported while a topology spread set with members is in place (grove_set_spread)";
  return GROVE_ERR_STATE;
}
static int32_t refuse_fences(grove_engine* e, const char* entry) {
  e->err = std::string(entry) + ": not supported while a fence set is in place (grove_set_fences)";
  return GROVE_ERR_STATE;
}
static int32_t refuse_queues(grove_engine* e, const char* entry) {
  e->err = std::string(entry) + ": not supported while a queue set with members is in place (grove_set_queues)";
  return GROVE_ERR_STATE;
}
static int32_t refuse_binpack(grove_engine* e, const char* entry) {
  e->err = std::string(entry) + ": not supported while a bin-packing set with members is in place (grove_set_binpack)";
  return GROVE_ERR_STATE;
}
static int32_t refuse_imex(grove_engine* e, const char* entry) {
  e->err = std::string(entry) + ": not supported while a ComputeDomain set with an enrolled clique is in place (grove_set_compute_domains)";
  return GROVE_ERR_STATE;
}
static int32_t refuse_wide(grove_engine* e, const char* entry) {
  e->err = std::string(entry) + ": not supported for a wide submission (a gang of more than " + std::to_string(GROVE_MAX_GANG_PODS) +
           " pods or a clique of more than 255 replicas)";
  return GROVE_ERR_LIMIT;
}

// A kernel of the relaxation chain, launched as a programmatic dependent of the kernel before it on the stream: its CTAs are
// launched and become resident while that kernel drains, and wait in cudaGridDependencySynchronize() -- the first statement of
// every kernel launched this way -- until it has completed and its writes are visible.  Behind anything else on the stream
// (a copy, a memset, an event) the launch is ordered as usual.
template <typename... P, typename... A>
static cudaError_t launch_chained(void (*k)(P...), dim3 grid, uint32_t block, cudaStream_t s, A&&... args) {
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t c{};
  c.gridDim = grid; c.blockDim = dim3(block); c.dynamicSmemBytes = 0; c.stream = s; c.attrs = at; c.numAttrs = 1;
  return cudaLaunchKernelEx(&c, k, std::forward<A>(args)...);
}

// ---------------------------------------------------------------------------------------------
// topology: sort by label path, tree-ify ids, domain ranges.  Host side; runs only when labels change.
// Restates what the reference hands a scheduler as the ordered level list
// (operator/internal/scheduler/kai/topology.go:103-135) plus the per-node label values.
// ---------------------------------------------------------------------------------------------
static int32_t build_topology(grove_engine* e, const grove_node_t* nodes, uint32_t n) {
  const uint32_t L = e->L;
  e->N = n;
  e->Npad = (n + 1023u) & ~1023u;
  e->words = e->Npad / 32;
  e->raw_dom.resize(size_t(n) * GROVE_MAX_LEVELS);
  for (uint32_t i = 0; i < n; ++i) std::memcpy(&e->raw_dom[size_t(i) * GROVE_MAX_LEVELS], nodes[i].dom, sizeof(uint32_t) * GROVE_MAX_LEVELS);
  e->perm.resize(n); e->inv.resize(n);
  std::iota(e->perm.begin(), e->perm.end(), 0u);
  const uint32_t* rd = e->raw_dom.data();
  std::sort(e->perm.begin(), e->perm.end(), [rd, L](uint32_t a, uint32_t b) {
    const uint32_t* x = rd + size_t(a) * GROVE_MAX_LEVELS; const uint32_t* y = rd + size_t(b) * GROVE_MAX_LEVELS;
    for (uint32_t l = 0; l < L; ++l) if (x[l] != y[l]) return x[l] < y[l];
    return a < b;
  });
  for (uint32_t i = 0; i < n; ++i) e->inv[e->perm[i]] = i;
  e->tdom.assign(size_t(e->Npad) * GROVE_MAX_LEVELS, GROVE_DOM_ABSENT);
  e->vdepth.assign(e->Npad, 0);
  for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) { e->dom_lo[l].clear(); e->dom_hi[l].clear(); e->n_dom[l] = 0; e->unit[l] = 0; }
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t* cur = rd + size_t(e->perm[i]) * GROVE_MAX_LEVELS;
    const uint32_t* prv = i ? rd + size_t(e->perm[i - 1]) * GROVE_MAX_LEVELS : nullptr;
    bool same_path = prv != nullptr;  // do cur and prv agree (and exist) on every level above l?
    uint32_t depth = 0;
    for (uint32_t l = 0; l < L; ++l) {
      if (cur[l] == GROVE_DOM_ABSENT) break;  // deeper labels are ignored once one is missing
      bool same = same_path && e->vdepth[i - 1] > l && prv[l] == cur[l];
      if (same) {
        uint32_t id = e->tdom[size_t(i - 1) * GROVE_MAX_LEVELS + l];
        e->tdom[size_t(i) * GROVE_MAX_LEVELS + l] = id;
        e->dom_hi[l][id] = i + 1;
      } else {
        e->tdom[size_t(i) * GROVE_MAX_LEVELS + l] = uint32_t(e->dom_lo[l].size());
        e->dom_lo[l].push_back(i); e->dom_hi[l].push_back(i + 1);
      }
      same_path = same;
      depth = l + 1;
    }
    e->vdepth[i] = uint8_t(depth);
  }
  for (uint32_t l = 0; l < L; ++l) {
    e->n_dom[l] = uint32_t(e->dom_lo[l].size());
    bool u = e->n_dom[l] > 0;
    for (uint32_t d = 0; d < e->n_dom[l] && u; ++d) u = (e->dom_hi[l][d] - e->dom_lo[l][d]) == 1;
    e->unit[l] = u ? 1u : 0u;
  }
  e->cap_stride = 0;
  for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) {
    e->cap_off[l] = e->cap_stride;
    if (l < L && !e->unit[l]) e->cap_stride += e->n_dom[l];
  }
  // upload static tables
  CU_TRY(e, e->d_perm.ensure(n)); CU_TRY(e, e->d_inv.ensure(n));
  CU_TRY(e, e->d_ndom.ensure(e->Npad)); CU_TRY(e, e->d_nres.ensure(e->Npad)); CU_TRY(e, e->d_vdepth.ensure(e->Npad));
  CU_TRY(e, cudaMemcpyAsync(e->d_perm.p, e->perm.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_inv.p, e->inv.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_ndom.p, e->tdom.data(), sizeof(uint4) * e->Npad, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_vdepth.p, e->vdepth.data(), e->Npad, cudaMemcpyHostToDevice, e->stream));
  std::vector<uint32_t> nxt(size_t(n) + 1);
  for (uint32_t l = 0; l < L; ++l) {
    const uint32_t nd = e->n_dom[l];
    CU_TRY(e, e->d_dom_lo[l].ensure(nd)); CU_TRY(e, e->d_dom_hi[l].ensure(nd)); CU_TRY(e, e->d_next_dom[l].ensure(size_t(n) + 1));
    if (nd) {
      CU_TRY(e, cudaMemcpyAsync(e->d_dom_lo[l].p, e->dom_lo[l].data(), sizeof(uint32_t) * nd, cudaMemcpyHostToDevice, e->stream));
      CU_TRY(e, cudaMemcpyAsync(e->d_dom_hi[l].p, e->dom_hi[l].data(), sizeof(uint32_t) * nd, cudaMemcpyHostToDevice, e->stream));
    }
    uint32_t d = 0;
    for (uint32_t i = 0; i <= n; ++i) {  // first domain whose lo >= i
      while (d < nd && e->dom_lo[l][d] < i) ++d;
      nxt[i] = d;
    }
    CU_TRY(e, cudaMemcpyAsync(e->d_next_dom[l].p, nxt.data(), sizeof(uint32_t) * (size_t(n) + 1), cudaMemcpyHostToDevice, e->stream));
    CU_TRY(e, cudaStreamSynchronize(e->stream));  // nxt is reused
  }
  e->ginfo_dirty = true;
  // this handle's node-range shard: the top-level domains dealt out in order, as evenly as their sizes allow; nodes that lack
  // the top-level label (sorted last) go to the last rank
  {
    const uint32_t W = std::max<uint32_t>(e->cfg.world, 1u), R = e->cfg.world > 1 ? e->cfg.rank : 0u;
    auto cut = [&](uint32_t r) -> uint32_t {   // first node of rank r's shard
      if (r == 0) return 0u;
      if (r >= W) return n;
      const uint64_t target = uint64_t(n) * r / W;
      for (uint32_t d = 0; d < e->n_dom[0]; ++d) if (e->dom_lo[0][d] >= target) return e->dom_lo[0][d];
      return n;
    };
    e->shard_lo = cut(R); e->shard_hi = cut(R + 1);
  }
  return GROVE_OK;
}

// Gangs that relax concurrently: the knob, else all of them -- except in a cycle with bin-packing members, whose picks send many
// gangs to the same fullest domains: every gang of the window then claims the same first nodes, and each such node's overflow
// chain grows as long as the window (DESIGN.md section 1 "Bin-packing").  kBinpackWindow bounds it; cycle_begin sizes the pool.
static constexpr uint32_t kBinpackWindow = 128;
static uint32_t window_of(const grove_engine* e) {
  if (e->tune_window) return e->tune_window;
  return e->bp_members ? std::max(std::min(e->G, kBinpackWindow), 1u) : std::max(e->G, 1u);
}

static Topo make_topo(grove_engine* e) {
  Topo t{};
  t.nres = e->d_nres.p; t.ndom = e->d_ndom.p;
  for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) {
    t.dom_lo[l] = e->d_dom_lo[l].p; t.dom_hi[l] = e->d_dom_hi[l].p; t.next_dom[l] = e->d_next_dom[l].p;
    t.n_dom[l] = e->n_dom[l]; t.unit[l] = e->unit[l];
  }
  t.n = e->N; t.npad = e->Npad; t.L = e->L; t.words = e->words;
  for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) t.cap_off[l] = e->cap_off[l];
  t.cap_stride = e->cap_stride;
  return t;
}


static Tables make_tables(grove_engine* e) {
  Tables t{};
  t.gangs = e->d_gangs.p; t.cliques = e->d_cliques.p; t.scopes = e->d_scopes.p;
  t.ginfo = e->d_ginfo.p; t.cinfo = e->d_cinfo.p; t.sigs = e->d_sigs.p; t.by_rank = e->d_by_rank.p;
  t.G = e->G; t.Q = e->Q; t.S = e->n_sigs; t.NS = e->S;
  return t;
}

static Relax make_relax(grove_engine* e) {
  Relax r{};
  r.ctl = e->d_ctl.p; r.state = e->d_state.p; r.tstate = e->d_tstate.p; r.dirty = e->d_dirty.p; r.chg_round = e->d_chg_round.p;
  r.eval_list = e->d_eval_list.p; r.last_att = e->d_last_att.p;
  r.ent_node = e->d_ent_node.p; r.ent_meta = e->d_ent_meta.p; r.cur_n = e->d_cur_n.p; r.cur_info = e->d_cur_info.p; r.cur_glo = e->d_cur_glo.p;
  r.extent = e->d_extent.p; r.sc_lvl = e->d_sc_lvl.p; r.sc_lo = e->d_sc_lo.p;
  r.nxt_node = e->d_nxt_node.p; r.nxt_meta = e->d_nxt_meta.p; r.nxt_n = e->d_nxt_n.p; r.nxt_tstate = e->d_nxt_tstate.p;
  r.nxt_info = e->d_nxt_info.p; r.nxt_glo = e->d_nxt_glo.p; r.nxt_extent = e->d_nxt_extent.p; r.nxt_sc_lvl = e->d_nxt_sc_lvl.p; r.nxt_sc_lo = e->d_nxt_sc_lo.p;
  r.claims = e->d_claims.p; r.nlive = e->d_nlive.p; r.ovf_head = e->d_ovf_head.p; r.ovf_next = e->d_ovf_next.p; r.ovf_claim = e->d_ovf_claim.p;
  r.ovf_cap = uint32_t(std::min<size_t>(e->d_ovf_claim.cap, 0xFFFFFFF0u));
  r.ctot = e->d_ctot.p; r.cmaxr = e->d_cmaxr.p;
  r.add_stamp = e->d_add_stamp.p; r.rem_stamp = e->d_rem_stamp.p; r.rem_round = e->d_rem_round.p; r.last_eval = e->d_last_eval.p; r.fail_upto = e->d_fail_upto.p;
  r.F = e->d_F.p; r.cap8 = e->d_cap8.p; r.capsum = e->d_capsum.p; r.capmax = e->d_capmax.p; r.T = e->d_T.p;
  r.shape_bits = e->shape_tables ? e->d_shape_bits.p : nullptr; r.pl_words = e->pl_words;
  for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) r.pl_off[l] = e->pl_off[l];
  r.P = e->P; r.window = window_of(e); r.entry = e->tune_entry ? e->tune_entry : r.window; r.heavy_att = e->tune_heavy_att;
  r.hold_off = e->holds_on ? e->d_hold_off.p : nullptr; r.hold = e->d_hold.p;
  r.dbg = e->dbg_on ? e->d_dbg.p : nullptr;
  r.live = e->d_live;
  r.ccount = e->wide ? e->d_ccount.p : nullptr; r.wide_node = e->d_wide_node.p; r.wide_meta = e->d_wide_meta.p; r.wide_cap = e->max_gang_pods;
  if (e->sp_members) {
    Spread& sp = r.sp;
    sp.group = e->d_sp_group.p; sp.row = e->d_sp_row.p; sp.info = e->d_sp_info.p; sp.mem_off = e->d_sp_mem_off.p; sp.mem = e->d_sp_mem.p;
    sp.cls = e->d_sp_cls.p; sp.cnt_off = e->d_sp_cnt_off.p; sp.seed = e->d_sp_seed.p; sp.cnt = e->d_sp_cnt.p; sp.dcls = e->d_sp_dcls.p;
    for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) sp.dcls_off[l] = e->sp_dcls_off[l];
    sp.allowed = e->d_sp_allowed.p; sp.stamp = e->d_sp_stamp.p; sp.skewed = e->d_sp_skewed.p; sp.n_groups = e->sp_groups;
  }
  if (!e->fc_gangs.empty()) { r.fc.list = e->d_fc_list.p; r.fc.slot = e->d_fc_slot.p; r.fc.n = uint32_t(e->fc_gangs.size()); }
  if (e->qu_members) {
    Queue& qu = r.qu;
    qu.slot = e->d_qu_slot.p; qu.mem = e->d_qu_mem.p; qu.mem_pair = e->d_qu_mem_pair.p; qu.mem_fin = e->d_qu_mem_fin.p; qu.rmin = e->d_qu_rmin.p;
    qu.q_off = e->d_qu_q_off.p; qu.q_base = e->d_qu_q_base.p; qu.pr = e->d_qu_pr.p; qu.head = e->d_qu_head.p; qu.use = e->d_qu_use.p;
    qu.gate = e->d_qu_gate.p; qu.cap = e->d_qu_cap.p; qu.n_mem = e->qu_members;
  }
  if (e->im_enrolled) { r.im.cd = e->d_im_cd.p; r.im.rank_cd = e->d_im_rank_cd.p; r.im.owner = e->d_im_owner.p; r.im.nenr = e->d_im_nenr.p; }
  return r;
}

// ---------------------------------------------------------------------------------------------
extern "C" {

uint32_t grove_abi_version(void) { return GROVE_ABI_VERSION; }

const char* grove_last_error(grove_engine_t* e) { return e ? e->err.c_str() : "null engine"; }

int32_t grove_engine_create(const grove_config_t* cfg, grove_engine_t** out) {
  if (!cfg || !out) return GROVE_ERR_INVALID_ARG;
  *out = nullptr;
  if (cfg->abi_version != GROVE_ABI_VERSION) return GROVE_ERR_INVALID_ARG;
  if (cfg->n_levels < 1 || cfg->n_levels > GROVE_MAX_LEVELS) return GROVE_ERR_INVALID_ARG;
  if (cfg->world > 1 && cfg->rank >= cfg->world) return GROVE_ERR_INVALID_ARG;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return GROVE_ERR_NO_DEVICE;  // no CPU fallback
  if (cfg->device < 0 || cfg->device >= ndev) return GROVE_ERR_NO_DEVICE;
  if (cudaSetDevice(cfg->device) != cudaSuccess) return GROVE_ERR_NO_DEVICE;
  grove_engine* e = new (std::nothrow) grove_engine();
  if (!e) return GROVE_ERR_OOM;
  e->cfg = *cfg; e->L = cfg->n_levels;
  { int sm = 0; if (cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, cfg->device) == cudaSuccess && sm > 0) e->n_sm = uint32_t(sm); }
  e->tune_window = cfg->window;
  if (const char* v = std::getenv("GROVE_TUNE_WINDOW")) if (!cfg->window) e->tune_window = uint32_t(std::max(0, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_ENTRY")) e->tune_entry = uint32_t(std::max(0, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_REFRESH")) e->tune_refresh = uint32_t(std::max(1, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_EVAL_CTAS")) e->tune_eval_ctas = uint32_t(std::max(1, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_WARP_CTAS")) e->tune_warp_ctas = uint32_t(std::max(1, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_BATCH")) e->tune_batch = uint32_t(std::max(1, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_AHEAD")) e->tune_ahead = uint32_t(std::max(0, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_HEAVY_ATT")) e->tune_heavy_att = uint32_t(std::max(1, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_MAX_ATT")) e->tune_max_att = uint32_t(std::max(0, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_HEAVY_CTAS")) e->tune_heavy_ctas = uint32_t(std::max(1, std::atoi(v)));
  if (const char* v = std::getenv("GROVE_TUNE_OVERLAP")) e->tune_overlap = std::atoi(v) != 0;
  if (const char* v = std::getenv("GROVE_TUNE_SCORE")) e->tune_score = std::atoi(v) != 0;
  if (std::getenv("GROVE_DEBUG_ADMIT")) e->dbg_on = true;
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);  // the latency-bound relaxation gets the SMs first
  if (cudaStreamCreateWithPriority(&e->stream, cudaStreamNonBlocking, prio_hi) != cudaSuccess) { delete e; return GROVE_ERR_CUDA; }
  if (cudaStreamCreateWithPriority(&e->stream_score, cudaStreamNonBlocking, prio_lo) != cudaSuccess) { delete e; return GROVE_ERR_CUDA; }
  if (cudaEventCreateWithFlags(&e->ev_fit, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&e->ev_score, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_nodes_up, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&e->ev_tables_up, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_upd, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreate(&e->ev_s0) != cudaSuccess || cudaEventCreate(&e->ev_s1) != cudaSuccess) { delete e; return GROVE_ERR_CUDA; }
  for (auto& ev : e->ev) if (cudaEventCreate(&ev) != cudaSuccess) { delete e; return GROVE_ERR_CUDA; }
  if (e->h_ctl.ensure(kCtlWords) != cudaSuccess) { delete e; return GROVE_ERR_OOM; }
  if (cudaHostAlloc(reinterpret_cast<void**>(&e->h_live), sizeof(uint32_t) * kLiveWords, cudaHostAllocMapped) != cudaSuccess ||
      cudaHostGetDevicePointer(reinterpret_cast<void**>(&e->d_live), e->h_live, 0) != cudaSuccess) { (void)cudaGetLastError(); e->h_live = nullptr; e->d_live = nullptr; }
  *out = e;
  return GROVE_OK;
}

void grove_engine_destroy(grove_engine_t* e) {
  if (!e) return;
  cudaSetDevice(e->cfg.device);
  cudaStreamSynchronize(e->stream);
  cudaStreamSynchronize(e->stream_score);
  for (auto& ev : e->ev) if (ev) cudaEventDestroy(ev);
  if (e->ev_s0) cudaEventDestroy(e->ev_s0);
  if (e->ev_s1) cudaEventDestroy(e->ev_s1);
  if (e->ev_fit) cudaEventDestroy(e->ev_fit);
  if (e->ev_nodes_up) cudaEventDestroy(e->ev_nodes_up);
  if (e->ev_tables_up) cudaEventDestroy(e->ev_tables_up);
  if (e->ev_upd) cudaEventDestroy(e->ev_upd);
  if (e->ev_score) cudaEventDestroy(e->ev_score);
  if (e->h_live) cudaFreeHost(e->h_live);
  if (e->stream_score) cudaStreamDestroy(e->stream_score);
  if (e->stream) cudaStreamDestroy(e->stream);
  delete e;
}


static int32_t load_nodes_common(grove_engine* e, const grove_node_t* host_nodes, const void* dev_nodes, uint32_t n) {
  if (n == 0 || n > GROVE_MAX_NODES) return fail(e, GROVE_ERR_INVALID_ARG, "node count out of range");
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  if (e->diag == grove_engine::kDiagReady || e->diag == grove_engine::kDiagSpread || e->diag == grove_engine::kDiagFence ||
      e->diag == grove_engine::kDiagImex) e->diag = grove_engine::kDiagChanged;
  e->sp_groups = e->sp_members = 0;   // a spread set belongs to the nodes and gangs it was validated against
  e->fc_gangs.clear();                // (a fence set too)
  e->qu_members = 0; e->qu_given = false;   // (and a queue set, with its fair-share set)
  e->fs_given = false; e->fs_have_order = false;
  e->bp_members = 0; e->bp_given = false;   // (and a bin-packing set)
  e->im_enrolled = 0; e->im_given = false;  // (and a ComputeDomain set)
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  if (host_nodes) {
    CU_TRY(e, cudaEventSynchronize(e->ev_nodes_up));  // an earlier upload may still be reading the staging buffer
    CU_TRY(e, e->d_nodes_in.ensure(n));
    CU_TRY(e, e->h_stage_nodes.ensure(n));
    // one pass over the caller's snapshot by a few threads: copy to the pinned staging buffer (the caller's array is
    // not retained) and compare the labels with the cached topology's
    const bool cached = e->nodes_loaded && n == e->N;
    const int T = n >= 8192 ? host_threads() : 1;
    int differs = 0;
#pragma omp parallel for num_threads(T) schedule(static) reduction(| : differs)
    for (int t = 0; t < T; ++t) {
      const uint32_t a = uint32_t(uint64_t(n) * t / T), z = uint32_t(uint64_t(n) * (t + 1) / T);
      std::memcpy(e->h_stage_nodes.p + a, host_nodes + a, sizeof(grove_node_t) * (z - a));
      if (cached) {
        const uint32_t* rd = e->raw_dom.data();
        int d = 0;
        for (uint32_t i = a; i < z; ++i)
          d |= std::memcmp(rd + size_t(i) * GROVE_MAX_LEVELS, host_nodes[i].dom, sizeof(uint32_t) * GROVE_MAX_LEVELS) != 0;
        differs |= d;
      }
    }
    if (!cached || differs) { int32_t rc = build_topology(e, host_nodes, n); if (rc) return rc; }
    CU_TRY(e, cudaMemcpyAsync(e->d_nodes_in.p, e->h_stage_nodes.p, sizeof(grove_node_t) * n, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(e, cudaEventRecord(e->ev_nodes_up, e->stream));
  } else {
    if (!e->nodes_loaded || n != e->N) return fail(e, GROVE_ERR_STATE, "device load needs a prior host load with the same labels");
    CU_TRY(e, cudaMemcpyAsync(e->d_nodes_in.p, dev_nodes, sizeof(grove_node_t) * n, cudaMemcpyDeviceToDevice, e->stream));
  }
  k_gather<<<(e->Npad + 255) / 256, 256, 0, e->stream>>>(e->d_nodes_in.p, e->d_perm.p, e->d_vdepth.p, e->d_nres.p, e->N, e->Npad);
  CU_TRY(e, cudaGetLastError());
  // (device source: read asynchronously on the engine's stream -- the header asks the caller to leave it alone until the next
  // blocking call on the handle returns; a synchronize here would cost every device-resident cycle a host round trip)
  e->nodes_loaded = true; e->score_pass_valid = false;
  return GROVE_OK;
}

int32_t grove_load_nodes(grove_engine_t* e, const grove_node_t* nodes, uint32_t n) {
  if (!e || !nodes) return GROVE_ERR_INVALID_ARG;
  return load_nodes_common(e, nodes, nullptr, n);
}

int32_t grove_load_nodes_device(grove_engine_t* e, const void* d_nodes, uint32_t n) {
  if (!e || !d_nodes) return GROVE_ERR_INVALID_ARG;
  return load_nodes_common(e, nullptr, d_nodes, n);
}

int32_t grove_update_nodes(grove_engine_t* e, const uint32_t* idx, const grove_node_t* recs, uint32_t n) {
  if (!e || (n && (!idx || !recs))) return GROVE_ERR_INVALID_ARG;
  if (!e->nodes_loaded) return fail(e, GROVE_ERR_STATE, "no node snapshot loaded");
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  if (e->diag == grove_engine::kDiagReady || e->diag == grove_engine::kDiagSpread || e->diag == grove_engine::kDiagFence ||
      e->diag == grove_engine::kDiagImex) e->diag = grove_engine::kDiagChanged;
  if (n == 0) return GROVE_OK;
  e->score_pass_valid = false;
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  CU_TRY(e, cudaEventSynchronize(e->ev_upd));  // an earlier update may still be reading the pinned staging buffers
  CU_TRY(e, e->h_upd_idx.ensure(n)); CU_TRY(e, e->h_upd_recs.ensure(n));
  for (uint32_t i = 0; i < n; ++i) {
    if (idx[i] >= e->N) return fail(e, GROVE_ERR_INVALID_ARG, "node index out of range");
    if (std::memcmp(&e->raw_dom[size_t(idx[i]) * GROVE_MAX_LEVELS], recs[i].dom, sizeof(uint32_t) * GROVE_MAX_LEVELS) != 0)
      return fail(e, GROVE_ERR_INVALID_ARG, "grove_update_nodes cannot change labels; reload the snapshot");
    e->h_upd_idx.p[i] = e->inv[idx[i]];
  }
  std::memcpy(e->h_upd_recs.p, recs, sizeof(grove_node_t) * n);   // nothing of the caller's is referenced after return
  CU_TRY(e, e->d_upd_idx.ensure(n)); CU_TRY(e, e->d_upd_recs.ensure(n));
  CU_TRY(e, cudaMemcpyAsync(e->d_upd_idx.p, e->h_upd_idx.p, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_upd_recs.p, e->h_upd_recs.p, sizeof(grove_node_t) * n, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaEventRecord(e->ev_upd, e->stream));
  k_update<<<(n + 255) / 256, 256, 0, e->stream>>>(e->d_upd_idx.p, e->d_upd_recs.p, e->d_vdepth.p, e->d_perm.p, e->d_nres.p, e->d_nodes_in.p, n);
  CU_TRY(e, cudaGetLastError());
  return GROVE_OK;   // stream-ordered: the next call on this handle sees the update
}


int32_t grove_get_nodes(grove_engine_t* e, grove_node_t* out, uint32_t cap) {
  if (!e || !out) return GROVE_ERR_INVALID_ARG;
  if (!e->nodes_loaded) return fail(e, GROVE_ERR_STATE, "no node snapshot loaded");
  if (cap < e->N) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  CU_TRY(e, e->d_nodes_out.ensure(e->N));
  k_scatter<<<(e->N + 255) / 256, 256, 0, e->stream>>>(e->d_nodes_out.p, e->d_nodes_in.p, e->d_perm.p, e->d_nres.p, e->N);
  CU_TRY(e, cudaGetLastError());
  CU_TRY(e, cudaMemcpyAsync(out, e->d_nodes_out.p, sizeof(grove_node_t) * e->N, cudaMemcpyDeviceToHost, e->stream));
  CU_TRY(e, cudaStreamSynchronize(e->stream));
  return GROVE_OK;
}

// one gang; returns nullptr when it is well formed, else the reason (code through *code)
static const char* validate_gang(const grove_engine* e, const grove_gang_t* gangs, uint32_t G, const grove_clique_t* cliques,
                                 const uint32_t* ccount, uint32_t Q, const grove_scope_t* scopes, uint32_t S, uint32_t gi,
                                 uint32_t max_pods, int32_t* code) {
  const uint32_t L = e->L;
  const grove_gang_t& g = gangs[gi];
  *code = GROVE_ERR_LIMIT;
  if (g.n_cliques == 0 || g.n_cliques > GROVE_MAX_GANG_CLIQUES) return "gang clique count out of range";
  if (g.n_scopes == 0 || g.n_scopes > GROVE_MAX_GANG_SCOPES) return "gang scope count out of range";
  *code = GROVE_ERR_INVALID_ARG;
  if (uint64_t(g.clique_off) + g.n_cliques > Q || uint64_t(g.scope_off) + g.n_scopes > S) return "gang table offsets out of range";
  if (g.level != GROVE_LEVEL_NONE && g.level >= L) return "gang level out of range";
  if (g.preferred != GROVE_LEVEL_NONE && (g.preferred >= L || (g.level != GROVE_LEVEL_NONE && g.preferred <= g.level)))
    return "gang preferred level must be a level deeper than the required one";
  if (g.anchor_node != GROVE_NONE_U32 && e->nodes_loaded && g.anchor_node >= e->N) return "anchor node out of range";
  if (g.base_gang != GROVE_NONE_U32 && (g.base_gang >= G || g.base_gang == gi)) return "base gang out of range";
  uint32_t pods = 0, next = 0;
  for (uint32_t si = 0; si < g.n_scopes; ++si) {
    const grove_scope_t& s = scopes[g.scope_off + si];
    if (s.first_clique != next || s.n_cliques == 0) return "scopes must tile the gang's cliques in order";
    if (s.level != GROVE_LEVEL_NONE && s.level >= L) return "scope level out of range";
    if (s.preferred1 && (s.preferred1 > L || (s.level != GROVE_LEVEL_NONE && uint32_t(s.preferred1) - 1u <= s.level)))
      return "scope preferred level must be a level deeper than the required one";
    if (next + s.n_cliques > g.n_cliques) return "scope exceeds gang";
    for (uint32_t i = 0; i < s.n_cliques; ++i) {
      const grove_clique_t& q = cliques[g.clique_off + next + i];
      if (GROVE_CLIQUE_SCOPE(q.scope) != si) return "clique.scope does not match its scope";
      if (q.level != GROVE_LEVEL_NONE && q.level >= L) return "clique level out of range";
      const uint32_t qp = GROVE_CLIQUE_PREFERRED(q.scope);
      if (qp != GROVE_LEVEL_NONE && (qp >= L || (q.level != GROVE_LEVEL_NONE && qp <= q.level)))
        return "clique preferred level must be a level deeper than the required one";
      const uint32_t c = ccount[g.clique_off + next + i];
      if ((c >> 16) < (c & 0xFFFFu)) return "replicas < min_replicas";
      pods += c >> 16;
    }
    next += s.n_cliques;
  }
  if (next != g.n_cliques) return "scopes do not cover the gang";
  if (pods > max_pods) {
    *code = GROVE_ERR_LIMIT;
    return max_pods == GROVE_MAX_GANG_PODS ? "gang exceeds GROVE_MAX_GANG_PODS" : "gang exceeds GROVE_MAX_WIDE_GANG_PODS";
  }
  return nullptr;
}

// same structural rules as the PodGang admission webhook guarantees
// (operator/internal/webhook/admission/pcs/validation/topologyconstraints.go:195-280); the first offending gang
// (lowest index) is reported whatever the thread count
static int32_t validate(grove_engine* e, const grove_gang_t* gangs, uint32_t G, const grove_clique_t* cliques, const uint32_t* ccount,
                        uint32_t Q, const grove_scope_t* scopes, uint32_t S, uint32_t max_pods) {
  uint32_t first_bad = GROVE_NONE_U32;
  const int T = G >= 2048 ? host_threads() : 1;
#pragma omp parallel for num_threads(T) schedule(static) reduction(min : first_bad)
  for (uint32_t gi = 0; gi < G; ++gi) {
    int32_t code;
    if (gi < first_bad && validate_gang(e, gangs, G, cliques, ccount, Q, scopes, S, gi, max_pods, &code)) first_bad = gi;
  }
  if (first_bad == GROVE_NONE_U32) return GROVE_OK;
  int32_t code = GROVE_ERR_INVALID_ARG;
  const char* why = validate_gang(e, gangs, G, cliques, ccount, Q, scopes, S, first_bad, max_pods, &code);
  return fail(e, code, why ? why : "malformed gang tables");
}

// both submit entries: ccount[q] = min_replicas | replicas << 16 of clique q, at most max_pods pods per gang
static int32_t submit(grove_engine* e, const grove_gang_t* gangs, uint32_t n_gangs, const grove_clique_t* cliques,
                      const std::vector<uint32_t>& ccount, uint32_t n_cliques, const grove_scope_t* scopes, uint32_t n_scopes, uint32_t max_pods) {
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  if (e->diag == grove_engine::kDiagReady || e->diag == grove_engine::kDiagSpread || e->diag == grove_engine::kDiagFence ||
      e->diag == grove_engine::kDiagImex) e->diag = grove_engine::kDiagChanged;
  if (n_gangs >= (1u << 24)) return fail(e, GROVE_ERR_LIMIT, "too many gangs");  // order rank + round tag share a stamp word
  e->sp_groups = e->sp_members = 0;
  e->fc_gangs.clear();
  e->qu_members = 0; e->qu_given = false;
  e->fs_given = false; e->fs_have_order = false;
  e->bp_members = 0; e->bp_given = false;
  e->im_enrolled = 0; e->im_given = false;
  int32_t rc = validate(e, gangs, n_gangs, cliques, ccount.data(), n_cliques, scopes, n_scopes, max_pods);
  if (rc) return rc;
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  CU_TRY(e, cudaEventSynchronize(e->ev_tables_up));  // an earlier upload may still be reading the pinned tables
  e->G = n_gangs; e->Q = n_cliques; e->S = n_scopes;
  CU_TRY(e, e->gangs.assign(gangs, n_gangs));
  CU_TRY(e, e->cliques.assign(cliques, n_cliques));
  CU_TRY(e, e->scopes.assign(scopes, n_scopes));
  CU_TRY(e, e->ccount.assign(ccount.data(), n_cliques));
  bool wide = false;
  for (uint32_t i = 0; i < n_cliques && !wide; ++i) wide |= (ccount[i] >> 16) > 255u;
  for (uint32_t g = 0; g < n_gangs && !wide; ++g)
    for (uint32_t c = 0, pods = 0; c < gangs[g].n_cliques && !wide; ++c) wide |= (pods += ccount[gangs[g].clique_off + c] >> 16) > GROVE_MAX_GANG_PODS;
  e->wide = wide;
  if (!wide)   // the ordinary kernels read the clique records' own counts: a wide-entry submission within the old limits brings them in
    for (uint32_t i = 0; i < n_cliques; ++i) { e->cliques[i].min_replicas = uint8_t(ccount[i]); e->cliques[i].replicas = uint8_t(ccount[i] >> 16); }
  if (wide) {
    CU_TRY(e, e->d_ccount.ensure(n_cliques));
    CU_TRY(e, cudaMemcpyAsync(e->d_ccount.p, e->ccount.data(), sizeof(uint32_t) * n_cliques, cudaMemcpyHostToDevice, e->stream));
  }
  e->gangs_loaded = true; e->ginfo_dirty = true; e->have_results = false; e->score_pass_valid = false;
  bool pref = false;
  for (uint32_t g = 0; g < n_gangs && !pref; ++g) pref |= gangs[g].preferred != GROVE_LEVEL_NONE;
  for (uint32_t i = 0; i < n_scopes && !pref; ++i) pref |= scopes[i].preferred1 != 0;
  for (uint32_t i = 0; i < n_cliques && !pref; ++i) pref |= (cliques[i].scope >> 5) != 0;
  e->any_preferred = pref;
  CU_TRY(e, e->d_gangs.ensure(n_gangs)); CU_TRY(e, e->d_cliques.ensure(n_cliques)); CU_TRY(e, e->d_scopes.ensure(n_scopes));
  if (n_gangs) CU_TRY(e, cudaMemcpyAsync(e->d_gangs.p, e->gangs.data(), sizeof(grove_gang_t) * n_gangs, cudaMemcpyHostToDevice, e->stream));
  if (n_cliques) CU_TRY(e, cudaMemcpyAsync(e->d_cliques.p, e->cliques.data(), sizeof(grove_clique_t) * n_cliques, cudaMemcpyHostToDevice, e->stream));
  if (n_scopes) CU_TRY(e, cudaMemcpyAsync(e->d_scopes.p, e->scopes.data(), sizeof(grove_scope_t) * n_scopes, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaEventRecord(e->ev_tables_up, e->stream));
  return GROVE_OK;  // the uploads read engine-owned pinned memory: nothing of the caller's is referenced any more
}

int32_t grove_submit_gangs(grove_engine_t* e, const grove_gang_t* gangs, uint32_t n_gangs, const grove_clique_t* cliques,
                           uint32_t n_cliques, const grove_scope_t* scopes, uint32_t n_scopes) {
  if (!e || (n_gangs && (!gangs || !cliques || !scopes))) return GROVE_ERR_INVALID_ARG;
  std::vector<uint32_t> ccount(n_cliques);
  for (uint32_t i = 0; i < n_cliques; ++i) ccount[i] = uint32_t(cliques[i].min_replicas) | uint32_t(cliques[i].replicas) << 16;
  return submit(e, gangs, n_gangs, cliques, ccount, n_cliques, scopes, n_scopes, GROVE_MAX_GANG_PODS);
}

int32_t grove_submit_gangs_wide(grove_engine_t* e, const grove_gang_t* gangs, uint32_t n_gangs, const grove_clique_t* cliques,
                                const grove_clique_count_t* counts, uint32_t n_cliques, const grove_scope_t* scopes, uint32_t n_scopes) {
  if (!e || (n_gangs && (!gangs || !cliques || !counts || !scopes))) return GROVE_ERR_INVALID_ARG;
  std::vector<uint32_t> ccount(n_cliques);
  for (uint32_t i = 0; i < n_cliques; ++i) ccount[i] = uint32_t(counts[i].min_replicas) | uint32_t(counts[i].replicas) << 16;
  return submit(e, gangs, n_gangs, cliques, ccount, n_cliques, scopes, n_scopes, GROVE_MAX_WIDE_GANG_PODS);
}


// derived per-gang / per-clique tables: order rank, anchor (sorted index + ancestor ranges), entry slots
static int32_t build_ginfo(grove_engine* e) {
  const uint32_t G = e->G, Q = e->Q;
  const auto t_b0 = std::chrono::steady_clock::now();
  CU_TRY(e, e->ginfo_pin.ensure(G)); CU_TRY(e, e->cinfo_pin.ensure(Q)); CU_TRY(e, e->by_rank_pin.ensure(std::max<uint32_t>(G, 1)));
  e->ginfo = e->ginfo_pin.p; e->cinfo = e->cinfo_pin.p;
  {  // ginfo zeroed, cinfo all-ones (gang == NONE marks a row no gang owns yet), by the engine's thread team
    const int T0 = G >= 2048 ? host_threads() : 1;
#pragma omp parallel for num_threads(T0) schedule(static)
    for (int t = 0; t < T0; ++t) {
      const size_t g0 = size_t(G) * t / T0, g1 = size_t(G) * (t + 1) / T0, q0 = size_t(Q) * t / T0, q1 = size_t(Q) * (t + 1) / T0;
      std::memset(e->ginfo + g0, 0, sizeof(GangInfo) * (g1 - g0));
      std::memset(e->cinfo + q0, 0xFF, sizeof(CliqueInfo) * (q1 - q0));
    }
  }
  e->sigs.clear();
  const auto t_m0 = std::chrono::steady_clock::now();
  // order rank = position by (priority desc, index asc), and the anchors.  PriorityClasses are few: every thread counts
  // the distinct priorities of its gang range, one thread turns the counts into start offsets per (priority, thread),
  // and every thread numbers its own range -- a stable counting sort without the sorted array.
  bool bad_anchor = false;
  {
    constexpr size_t kMaxPrio = 64;
    const int T1 = G >= 2048 ? host_threads() : 1;
    std::vector<std::vector<std::pair<int32_t, uint32_t>>> seen(T1);   // per thread: (priority, count) in first-seen order
    std::vector<int32_t> prios;                                         // distinct, descending
    std::vector<uint32_t> start;                                        // [thread][priority index] first rank
    bool many = false;
#pragma omp parallel num_threads(T1)
    {
      const int t = omp_get_thread_num();
      const uint32_t g0 = uint32_t(uint64_t(G) * t / T1), g1 = uint32_t(uint64_t(G) * (t + 1) / T1);
      auto& mine = seen[t];
      bool over = false;
      for (uint32_t g = g0; g < g1 && !over; ++g) {
        const int32_t p = e->gangs[g].priority;
        size_t i = 0;
        while (i < mine.size() && mine[i].first != p) ++i;
        if (i == mine.size()) { if (mine.size() == kMaxPrio) { over = true; break; } mine.push_back({p, 0u}); }
        mine[i].second++;
      }
      if (over) {
#pragma omp atomic write
        many = true;
      }
#pragma omp barrier
#pragma omp single
      {
        for (const auto& v : seen) for (const auto& pc : v) prios.push_back(pc.first);
        std::sort(prios.begin(), prios.end(), std::greater<int32_t>());
        prios.erase(std::unique(prios.begin(), prios.end()), prios.end());
        if (prios.size() > kMaxPrio) many = true;
        if (!many) {
          start.assign(size_t(T1) * prios.size(), 0u);
          uint32_t run = 0;
          for (size_t k = 0; k < prios.size(); ++k)
            for (int tt = 0; tt < T1; ++tt) {
              start[size_t(tt) * prios.size() + k] = run;
              for (const auto& pc : seen[tt]) if (pc.first == prios[k]) run += pc.second;
            }
        }
      }  // implicit barrier
      bool bad = false;
      uint32_t next[kMaxPrio];
      if (!many) for (size_t k = 0; k < prios.size(); ++k) next[k] = start[size_t(t) * prios.size() + k];
      for (uint32_t gi = g0; gi < g1; ++gi) {
        const grove_gang_t& g = e->gangs[gi];
        if (!many) {
          size_t k = 0;
          while (prios[k] != g.priority) ++k;
          e->ginfo[gi].order = next[k]++;
        }
        if (g.anchor_node != GROVE_NONE_U32 && g.anchor_node >= e->N) { bad = true; continue; }
        e->ginfo[gi].anchor = g.anchor_node != GROVE_NONE_U32 ? e->inv[g.anchor_node] : fmix32(gi) % e->N;
      }
      if (bad) {
#pragma omp atomic write
        bad_anchor = true;
      }
    }
    if (many) {  // more distinct priorities than a scheduler has PriorityClasses: plain stable sort
      std::vector<uint32_t> ord(G);
      std::iota(ord.begin(), ord.end(), 0u);
      std::stable_sort(ord.begin(), ord.end(), [e](uint32_t a, uint32_t b) { return e->gangs[a].priority > e->gangs[b].priority; });
      for (uint32_t r = 0; r < G; ++r) e->ginfo[ord[r]].order = r;
    }
  }
  if (bad_anchor) return fail(e, GROVE_ERR_INVALID_ARG, "anchor node out of range");
  {  // the inverse: which gang has its turn at each rank
    const int T2 = G >= 2048 ? host_threads() : 1;
#pragma omp parallel for num_threads(T2) schedule(static)
    for (uint32_t gi = 0; gi < G; ++gi) e->by_rank_pin.p[e->ginfo[gi].order] = gi;
  }
  const auto t_m1 = std::chrono::steady_clock::now();
  // per-clique derived data + signature interning.  PodCliques stamped from one template (PCS / PCSG
  // replicas) share requests, selector class and binding depth: they share one fit-bitmap row.  Gang
  // ranges are processed by a few host threads with thread-local signature tables, merged afterwards.
  const auto t_m2 = std::chrono::steady_clock::now();
  struct SigTab {
    std::vector<std::array<uint32_t, 6>> tab = std::vector<std::array<uint32_t, 6>>(256, std::array<uint32_t, 6>{0, 0, 0, 0, 0, GROVE_NONE_U32});
    std::vector<std::array<uint32_t, 5>> keys;
    static uint32_t hash5(const std::array<uint32_t, 5>& k) { uint32_t h = k[0] * 0x9E3779B1u ^ k[1] * 0x85EBCA6Bu ^ (k[2] << 20) ^ (k[3] << 4) ^ k[4]; return h ^ (h >> 15); }
    uint32_t intern(const std::array<uint32_t, 5>& key) {
      if (keys.size() * 2 >= tab.size()) {
        std::vector<std::array<uint32_t, 6>> nt(tab.size() * 4, std::array<uint32_t, 6>{0, 0, 0, 0, 0, GROVE_NONE_U32});
        for (const auto& r : tab) if (r[5] != GROVE_NONE_U32) {
          size_t h = hash5({r[0], r[1], r[2], r[3], r[4]}) & (nt.size() - 1);
          while (nt[h][5] != GROVE_NONE_U32) h = (h + 1) & (nt.size() - 1);
          nt[h] = r;
        }
        tab.swap(nt);
      }
      size_t h = hash5(key) & (tab.size() - 1);
      while (tab[h][5] != GROVE_NONE_U32 && !(tab[h][0] == key[0] && tab[h][1] == key[1] && tab[h][2] == key[2] && tab[h][3] == key[3] && tab[h][4] == key[4]))
        h = (h + 1) & (tab.size() - 1);
      if (tab[h][5] == GROVE_NONE_U32) { tab[h] = {key[0], key[1], key[2], key[3], key[4], uint32_t(keys.size())}; keys.push_back(key); }
      return tab[h][5];
    }
  };
  const int T = G >= 2048 ? host_threads() : 1;
  std::vector<SigTab> local(T);
  std::vector<uint32_t> gang_pods(G, 0);
  int shared_rows = 0;
#pragma omp parallel num_threads(T) reduction(+ : shared_rows)
  {
    const int t = omp_get_thread_num();
    const uint32_t g0 = uint32_t(uint64_t(G) * t / T), g1 = uint32_t(uint64_t(G) * (t + 1) / T);
    SigTab& st = local[t];
    for (uint32_t gi = g0; gi < g1; ++gi) {
      const grove_gang_t& g = e->gangs[gi];
      uint32_t pods = 0;
      for (uint32_t si = 0; si < g.n_scopes; ++si) {
        const grove_scope_t& s = e->scopes[g.scope_off + si];
        for (uint32_t i = 0; i < s.n_cliques; ++i) {
          const uint32_t qi = g.clique_off + s.first_clique + i;
          const grove_clique_t& q = e->cliques[qi];
          uint32_t nd = 0;
          if (g.level != GROVE_LEVEL_NONE) nd = std::max(nd, uint32_t(g.level) + 1);
          if (s.level != GROVE_LEVEL_NONE) nd = std::max(nd, uint32_t(s.level) + 1);
          if (q.level != GROVE_LEVEL_NONE) nd = std::max(nd, uint32_t(q.level) + 1);
          if (e->cinfo[qi].gang != GROVE_NONE_U32) shared_rows++;  // rows of different threads never overlap unless the tables are malformed
          e->cinfo[qi] = CliqueInfo{gi, nd, st.intern({q.req_cpu_milli, q.req_mem_mib, q.req_gpu, q.class_mask, nd}), uint32_t(t)};
          pods += e->ccount[qi] >> 16;
        }
      }
      gang_pods[gi] = pods;
    }
  }
  const auto t_m3 = std::chrono::steady_clock::now();
  if (shared_rows) return fail(e, GROVE_ERR_INVALID_ARG, "clique rows shared between gangs");
  SigTab global;
  std::vector<std::vector<uint32_t>> remap(T);
  for (int t = 0; t < T; ++t) { remap[t].resize(local[t].keys.size()); for (size_t k = 0; k < local[t].keys.size(); ++k) remap[t][k] = global.intern(local[t].keys[k]); }
  e->sigs.resize(global.keys.size());
  for (size_t k = 0; k < global.keys.size(); ++k) { const auto& key = global.keys[k]; e->sigs[k] = make_uint4(key[0], key[1], key[2], key[3] | (key[4] << 16)); }
  // thread-local signature ids -> global ids (pad carried the id of the thread that interned the row)
#pragma omp parallel for num_threads(T) schedule(static)
  for (uint32_t qi = 0; qi < Q; ++qi)
    if (e->cinfo[qi].gang != GROVE_NONE_U32) { e->cinfo[qi].sig = remap[e->cinfo[qi].pad][e->cinfo[qi].sig]; e->cinfo[qi].pad = 0; }
  // Gang SHAPES: what the candidate pre-filter of a gang depends on is its structure (levels, scopes, per-clique
  // signature / MinReplicas / level), not its anchor or rank.  PodGangs stamped from one template share a shape, so the
  // pre-filter is evaluated once per (shape, candidate domain) per capacity-table build (k_shape_plaus) instead of once
  // per (gang evaluation, candidate).  Interned like the signatures: thread-local tables over gang ranges, merged.
  {
    auto shape_hash = [e](uint32_t gi) {
      const grove_gang_t& g = e->gangs[gi];
      uint64_t h = 0x9E3779B97F4A7C15ull ^ (uint64_t(g.n_cliques) << 32 | uint64_t(g.n_scopes) << 16 | uint64_t(g.level) << 8 | g.preferred);
      auto mix = [&h](uint64_t v) { h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); };
      for (uint32_t si = 0; si < g.n_scopes; ++si) { const grove_scope_t& s = e->scopes[g.scope_off + si]; mix(uint64_t(s.first_clique) | uint64_t(s.n_cliques) << 16 | uint64_t(s.level) << 32 | uint64_t(s.preferred1) << 40); }
      for (uint32_t c = 0; c < g.n_cliques; ++c) { const grove_clique_t& q = e->cliques[g.clique_off + c]; mix(uint64_t(e->cinfo[g.clique_off + c].sig) | uint64_t(e->ccount[g.clique_off + c] & 0xFFFFu) << 32 | uint64_t(q.level) << 40 | uint64_t(q.scope) << 48); }
      return h;
    };
    auto shape_equal = [e](uint32_t a, uint32_t b) {
      const grove_gang_t& x = e->gangs[a]; const grove_gang_t& y = e->gangs[b];
      if (x.n_cliques != y.n_cliques || x.n_scopes != y.n_scopes || x.level != y.level || x.preferred != y.preferred) return false;
      for (uint32_t si = 0; si < x.n_scopes; ++si) {
        const grove_scope_t& s = e->scopes[x.scope_off + si]; const grove_scope_t& t = e->scopes[y.scope_off + si];
        if (s.first_clique != t.first_clique || s.n_cliques != t.n_cliques || s.level != t.level || s.preferred1 != t.preferred1) return false;
      }
      for (uint32_t c = 0; c < x.n_cliques; ++c) {
        const grove_clique_t& q = e->cliques[x.clique_off + c]; const grove_clique_t& r = e->cliques[y.clique_off + c];
        if (e->cinfo[x.clique_off + c].sig != e->cinfo[y.clique_off + c].sig || ((e->ccount[x.clique_off + c] ^ e->ccount[y.clique_off + c]) & 0xFFFFu) ||
            q.level != r.level || q.scope != r.scope) return false;
      }
      return true;
    };
    struct ShapeTab {   // open addressing on the hash; value = representative gang
      std::vector<std::pair<uint64_t, uint32_t>> tab = std::vector<std::pair<uint64_t, uint32_t>>(256, {0, GROVE_NONE_U32});
      std::vector<uint32_t> reps;
      size_t used = 0;
    };
    auto intern = [&](ShapeTab& st, uint32_t gi, uint64_t h) -> uint32_t {   // -> index into st.reps
      if (st.used * 2 >= st.tab.size()) {
        std::vector<std::pair<uint64_t, uint32_t>> nt(st.tab.size() * 4, {0, GROVE_NONE_U32});
        for (const auto& r : st.tab) if (r.second != GROVE_NONE_U32) { size_t k = r.first & (nt.size() - 1); while (nt[k].second != GROVE_NONE_U32) k = (k + 1) & (nt.size() - 1); nt[k] = r; }
        st.tab.swap(nt);
      }
      size_t k = h & (st.tab.size() - 1);
      while (st.tab[k].second != GROVE_NONE_U32 && !(st.tab[k].first == h && shape_equal(st.reps[st.tab[k].second], gi))) k = (k + 1) & (st.tab.size() - 1);
      if (st.tab[k].second == GROVE_NONE_U32) { st.tab[k] = {h, uint32_t(st.reps.size())}; st.reps.push_back(gi); st.used++; }
      return st.tab[k].second;
    };
    std::vector<ShapeTab> lsh(T);
    std::vector<uint32_t> lid(G);
#pragma omp parallel num_threads(T)
    {
      const int t = omp_get_thread_num();
      const uint32_t g0 = uint32_t(uint64_t(G) * t / T), g1 = uint32_t(uint64_t(G) * (t + 1) / T);
      for (uint32_t gi = g0; gi < g1; ++gi) lid[gi] = intern(lsh[t], gi, shape_hash(gi));
    }
    ShapeTab gsh;
    std::vector<std::vector<uint32_t>> smap(T);
    for (int t = 0; t < T; ++t) { smap[t].resize(lsh[t].reps.size()); for (size_t k = 0; k < lsh[t].reps.size(); ++k) smap[t][k] = intern(gsh, lsh[t].reps[k], shape_hash(lsh[t].reps[k])); }
    e->shape_rep = gsh.reps;
    e->n_shapes = uint32_t(gsh.reps.size());
#pragma omp parallel num_threads(T)
    {
      const int t = omp_get_thread_num();
      const uint32_t g0 = uint32_t(uint64_t(G) * t / T), g1 = uint32_t(uint64_t(G) * (t + 1) / T);
      for (uint32_t gi = g0; gi < g1; ++gi) e->ginfo[gi].pad = smap[t][lid[gi]];
    }
    // bit layout of one shape's row: every level's domains, each level padded to a word
    uint32_t bits = 0;
    for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) { e->pl_off[l] = bits; if (l < e->L) bits += (e->n_dom[l] + 31u) & ~31u; }
    e->pl_words = bits / 32;
    // worth it while the rows stay small next to the work they save; otherwise every evaluation runs the pre-filter itself
    e->shape_tables = e->n_shapes && uint64_t(e->n_shapes) * e->pl_words * 4 <= (256ull << 20) && e->n_shapes <= G / 2 + 16;
  }
  uint32_t pod_off = 0;
  e->max_gang_pods = 0;
  for (uint32_t gi = 0; gi < G; ++gi) { e->ginfo[gi].pod_off = pod_off; pod_off += gang_pods[gi]; e->max_gang_pods = std::max(e->max_gang_pods, gang_pods[gi]); }
  e->P = pod_off;
  const auto t_b1 = std::chrono::steady_clock::now();
  for (uint32_t qi = 0; qi < Q; ++qi)
    if (e->cinfo[qi].gang == GROVE_NONE_U32) return fail(e, GROVE_ERR_INVALID_ARG, "clique row owned by no gang");
  e->n_sigs = uint32_t(e->sigs.size());
  CU_TRY(e, e->d_ginfo.ensure(G)); CU_TRY(e, e->d_cinfo.ensure(Q)); CU_TRY(e, e->d_sigs.ensure(e->n_sigs));
  CU_TRY(e, e->d_by_rank.ensure(std::max<uint32_t>(G, 1)));
  if (e->n_sigs) CU_TRY(e, cudaMemcpyAsync(e->d_sigs.p, e->sigs.data(), sizeof(uint4) * e->n_sigs, cudaMemcpyHostToDevice, e->stream));
  if (G) {
    CU_TRY(e, cudaMemcpyAsync(e->d_ginfo.p, e->ginfo, sizeof(GangInfo) * G, cudaMemcpyHostToDevice, e->stream));
    k_anchor<<<(G + 255) / 256, 256, 0, e->stream>>>(make_topo(e), e->d_ginfo.p, G);  // ancestor ranges from the device-resident tree
    CU_TRY(e, cudaGetLastError());
  }
  if (Q) CU_TRY(e, cudaMemcpyAsync(e->d_cinfo.p, e->cinfo, sizeof(CliqueInfo) * Q, cudaMemcpyHostToDevice, e->stream));
  if (G) CU_TRY(e, cudaMemcpyAsync(e->d_by_rank.p, e->by_rank_pin.p, sizeof(uint32_t) * G, cudaMemcpyHostToDevice, e->stream));
  if (e->shape_tables) {
    CU_TRY(e, e->d_shape_rep.ensure(e->n_shapes)); CU_TRY(e, e->d_shape_bits.ensure(size_t(e->n_shapes) * e->pl_words));
    CU_TRY(e, e->shape_rep_pin.ensure(e->n_shapes));   // (pinned: the upload is a plain DMA the host does not wait for; the buffer is
    std::memcpy(e->shape_rep_pin.p, e->shape_rep.data(), sizeof(uint32_t) * e->n_shapes);   //  rewritten only after the cycle that reads it)
    CU_TRY(e, cudaMemcpyAsync(e->d_shape_rep.p, e->shape_rep_pin.p, sizeof(uint32_t) * e->n_shapes, cudaMemcpyHostToDevice, e->stream));
  }
  e->ginfo_dirty = false; e->bp_anchors = false;
  if (std::getenv("GROVE_DEBUG_HOST")) {
    const auto t_b2 = std::chrono::steady_clock::now();
    auto us = [](auto a, auto b) { return (long)std::chrono::duration_cast<std::chrono::microseconds>(b - a).count(); };
    std::fprintf(stderr, "build_ginfo: tables %ld us (init %ld, order %ld, anchors %ld, cliques %ld, merge %ld), upload %ld us\n", us(t_b0, t_b1), us(t_b0, t_m0), us(t_m0, t_m1), us(t_m1, t_m2), us(t_m2, t_m3), us(t_m3, t_b1), us(t_b1, t_b2));
  }
  return GROVE_OK;
}

// capacity tables over the committed state: K1 fit bitmap for every signature, per-node capacities, per-domain sum / max
static int32_t build_cap_tables(grove_engine* e, const Topo& tp, const Tables& tb, const Relax& rx) {
  if (!e->n_sigs) return GROVE_OK;
  dim3 gfit(e->Npad / 1024, std::min<uint32_t>((e->n_sigs + kFitTile - 1) / kFitTile, 65535u));
  if (e->cap_stride) {   // k_fit accumulates the per-domain sums / maxima with atomics
    CU_TRY(e, cudaMemsetAsync(e->d_capsum.p, 0, sizeof(uint32_t) * size_t(e->n_sigs) * e->cap_stride, e->stream));
    CU_TRY(e, cudaMemsetAsync(e->d_capmax.p, 0, sizeof(uint32_t) * size_t(e->n_sigs) * e->cap_stride, e->stream));
  }
  k_fit<<<gfit, 1024, 0, e->stream>>>(tp, tb, e->d_F.p, e->d_cap8.p, e->cap_stride ? e->d_capsum.p : nullptr, e->cap_stride ? e->d_capmax.p : nullptr);
  CU_TRY(e, launch_chained(k_clear_stale, (e->Npad / 4 + 255) / 256, 256, e->stream, rx, e->Npad / 4));
  if (e->shape_tables) {   // the candidate pre-filter of every gang shape over every domain of its candidate levels
    // only the levels some shape takes its candidates from (Preferred down to Required): a CTA that has nothing to do still
    // costs its launch, and the unit level alone would be tens of thousands of them
    uint32_t mx = 0;
    for (uint32_t i = 0; i < e->n_shapes; ++i) {
      const grove_gang_t& g = e->gangs[e->shape_rep[i]];
      const int base = g.level != GROVE_LEVEL_NONE ? int(g.level) : -1;
      const int first = g.preferred != GROVE_LEVEL_NONE && int(g.preferred) > base ? int(g.preferred) : base;
      for (int l = std::max(base, 0); l <= first && l < int(e->L); ++l) mx = std::max(mx, e->n_dom[l]);
    }
    if (mx) CU_TRY(e, launch_chained(e->wide ? k_shape_plaus<true> : k_shape_plaus<false>, dim3((mx + 31) / 32, e->n_shapes, e->L), 128, e->stream, tp, tb, rx, e->d_shape_rep.p));
    e->launches += 1;
  }
  CU_TRY(e, cudaGetLastError());
  e->launches += 3;
  return GROVE_OK;
}

// K3 CTAs: they take work items from a queue; by default as many as are resident at once (heavy gangs take whole CTAs)
static uint32_t eval_ctas(const grove_engine* e) {
  const uint32_t W = window_of(e);
  return std::max(1u, e->tune_eval_ctas ? e->tune_eval_ctas : std::min(W, e->n_sm * e->tune_heavy_ctas));
}

// a node snapshot loaded, gangs submitted, no cycle in flight
static int32_t check_ready(grove_engine* e) {
  if (!e->nodes_loaded) return fail(e, GROVE_ERR_STATE, "no node snapshot loaded");
  if (!e->gangs_loaded) return fail(e, GROVE_ERR_STATE, "no gangs submitted");
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  return GROVE_OK;
}

static int32_t cycle_begin(grove_engine* e) {
  if (int32_t rc = check_ready(e)) return rc;
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  if (e->ginfo_dirty) { int32_t rc = build_ginfo(e); if (rc) return rc; }
  const uint32_t G = e->G, Q = e->Q, S = e->S, P = e->P, N = e->Npad;
  const size_t g1 = std::max<uint32_t>(G, 1), p1 = std::max<uint32_t>(P, 1), s1 = std::max<uint32_t>(S, 1);
  CU_TRY(e, e->d_ctl.ensure(kCtlWords));
  CU_TRY(e, e->d_state.ensure(g1)); CU_TRY(e, e->d_tstate.ensure(g1)); CU_TRY(e, e->d_dirty.ensure(g1)); CU_TRY(e, e->d_chg_round.ensure(g1));
  CU_TRY(e, e->d_eval_list.ensure(g1)); CU_TRY(e, e->d_last_att.ensure(g1));
  CU_TRY(e, e->d_ent_node.ensure(p1)); CU_TRY(e, e->d_ent_meta.ensure(p1)); CU_TRY(e, e->d_cur_n.ensure(g1)); CU_TRY(e, e->d_cur_info.ensure(g1));
  CU_TRY(e, e->d_cur_glo.ensure(g1)); CU_TRY(e, e->d_extent.ensure(g1)); CU_TRY(e, e->d_sc_lvl.ensure(s1)); CU_TRY(e, e->d_sc_lo.ensure(s1));
  CU_TRY(e, e->d_nxt_node.ensure(p1)); CU_TRY(e, e->d_nxt_meta.ensure(p1)); CU_TRY(e, e->d_nxt_n.ensure(g1)); CU_TRY(e, e->d_nxt_tstate.ensure(g1));
  CU_TRY(e, e->d_nxt_info.ensure(g1)); CU_TRY(e, e->d_nxt_glo.ensure(g1)); CU_TRY(e, e->d_nxt_extent.ensure(g1));
  CU_TRY(e, e->d_nxt_sc_lvl.ensure(s1)); CU_TRY(e, e->d_nxt_sc_lo.ensure(s1));
  CU_TRY(e, e->d_claims.ensure(size_t(N) * kClaimSlots)); CU_TRY(e, e->d_nlive.ensure(N / 4)); CU_TRY(e, e->d_ovf_head.ensure(N));
  // (the overflow pool takes the holds as well as the claims: a node's line may be full of both)
  // (and in a cycle with bin-packing members, room on every node for a chain as long as the window -- the tentative claims of a
  // pile-up -- plus 110, the Kubernetes default pod limit, for the settled ones; at most 2^26 entries)
  size_t ovf = 4 * p1 + 1024 + (e->holds_on ? e->n_hold : 0u);
  if (e->bp_members) ovf += std::min<size_t>(size_t(N) * (window_of(e) + 110u), size_t(1) << 26);
  CU_TRY(e, e->d_ovf_next.ensure(ovf)); CU_TRY(e, e->d_ovf_claim.ensure(ovf));
  CU_TRY(e, e->d_ctot.ensure(N)); CU_TRY(e, e->d_cmaxr.ensure(N));
  CU_TRY(e, e->d_add_stamp.ensure(N)); CU_TRY(e, e->d_rem_stamp.ensure(e->words)); CU_TRY(e, e->d_rem_round.ensure(e->words));
  CU_TRY(e, e->d_last_eval.ensure(g1)); CU_TRY(e, e->d_fail_upto.ensure(g1));
  CU_TRY(e, e->d_status.ensure(g1)); CU_TRY(e, e->d_scope_status.ensure(s1)); CU_TRY(e, e->d_out.ensure(p1));
  if (e->wide) {   // the entry stacks of a wide cycle's evaluations: one per k_eval warp, as deep as the largest gang
    const size_t ws = size_t(eval_ctas(e)) * kEvalWarps * e->max_gang_pods;
    CU_TRY(e, e->d_wide_node.ensure(ws)); CU_TRY(e, e->d_wide_meta.ensure(ws));
  }
  CU_TRY(e, e->h_status.ensure(g1)); CU_TRY(e, e->h_scope_status.ensure(s1)); CU_TRY(e, e->h_out.ensure(p1));
  CU_TRY(e, e->d_fin.ensure((G + kFinThreads - 1) / kFinThreads + 4)); CU_TRY(e, e->d_totals.ensure(4));
  // the S x N tables and the Q x N score matrix
  {
    const size_t fw = size_t(e->n_sigs) * e->words, cb = size_t(e->n_sigs) * N, tw = size_t(e->n_sigs) * std::max<uint32_t>(e->cap_stride, 1);
    if (e->d_F.ensure(std::max<size_t>(fw, 1)) != cudaSuccess || e->d_cap8.ensure(std::max<size_t>(cb, 1)) != cudaSuccess ||
        e->d_capsum.ensure(tw) != cudaSuccess || e->d_capmax.ensure(tw) != cudaSuccess ||
        (e->tune_score && e->d_T.ensure(std::max<size_t>(size_t(Q) * N, 1)) != cudaSuccess)) {
      (void)cudaGetLastError();
      return fail(e, GROVE_ERR_OOM, "fit / capacity / score matrices do not fit in device memory");
    }
  }
  if (e->sp_members) {   // the spread set's per-cycle scratch: counts per domain, classes per domain, stamps per group, flags
    CU_TRY(e, e->d_sp_cnt.ensure(std::max<uint32_t>(e->sp_cnt_words, 1))); CU_TRY(e, e->d_sp_dcls.ensure(std::max<uint32_t>(e->sp_dcls_words, 1)));
    CU_TRY(e, e->d_sp_stamp.ensure(std::max<uint32_t>(e->sp_groups, 1))); CU_TRY(e, e->d_sp_skewed.ensure(g1)); CU_TRY(e, e->h_sp_skewed.ensure(g1));
  }
  if (!e->fc_gangs.empty()) {   // the fence set's buffers (make_relax hands their pointers to every kernel of the cycle)
    const size_t nf = e->fc_gangs.size();
    CU_TRY(e, e->d_fc_gang.ensure(nf)); CU_TRY(e, e->d_fc_off.ensure(nf)); CU_TRY(e, e->d_fc_list.ensure(nf)); CU_TRY(e, e->d_fc_slot.ensure(g1));
  }
  if (e->im_enrolled) {   // the ComputeDomain set's buffers (make_relax hands their pointers to every kernel of the cycle)
    CU_TRY(e, e->d_im_cd.ensure(std::max<size_t>(Q, 1))); CU_TRY(e, e->d_im_rank_cd.ensure(g1));
    CU_TRY(e, e->d_im_owner.ensure(N)); CU_TRY(e, e->d_im_nenr.ensure(N));
  }
  if (e->dbg_on) { CU_TRY(e, e->d_dbg.ensure(g1 * 8 + 8)); CU_TRY(e, cudaMemsetAsync(e->d_dbg.p, 0, g1 * 32 + 32, e->stream)); }
  {
    const uint32_t W = window_of(e);
    const uint32_t E = e->tune_entry ? e->tune_entry : W;
    if (e->h_live) { std::memset(e->h_live, 0, sizeof(uint32_t) * kLiveWords); e->h_live[kLiveRound] = 1; }
    k_reset<<<e->n_sm * 4, 256, 0, e->stream>>>(make_relax(e), G, S, N, e->words, std::min(G, std::min(W, E)));
    CU_TRY(e, cudaGetLastError());
  }
  e->launches = 0; e->in_cycle = true; e->have_results = false; e->have_scopes = false; e->diag = grove_engine::kDiagNoCycle;
  e->victims.clear(); e->moves.clear(); e->score_pass_valid = false;
  std::memset(&e->last, 0, sizeof(e->last));
  return GROVE_OK;
}

static int32_t finish_cycle(grove_engine* e) {
  const Topo tp = make_topo(e); const Tables tb = make_tables(e); const Relax rx = make_relax(e);
  const uint32_t G = e->G;
  e->n_out = 0;
  if (G) {
    const uint32_t ncta = (G + kFinThreads - 1) / kFinThreads;
    CU_TRY(e, cudaMemsetAsync(e->d_fin.p + ncta, 0, sizeof(uint32_t) * 4, e->stream));
    k_fin_count<<<ncta, kFinThreads, 0, e->stream>>>(tb, rx, e->d_fin.p);
    k_fin_scan<<<1, 1024, 0, e->stream>>>(e->d_fin.p, ncta, e->d_totals.p);
    k_fin_status<<<ncta, kFinThreads, 0, e->stream>>>(tb, rx, e->d_fin.p, e->d_perm.p, e->d_status.p);
    k_emit<<<(G * 32 + 255) / 256, 256, 0, e->stream>>>(tb, rx, e->d_perm.p, e->d_status.p, e->d_out.p, e->d_scope_status.p);
    CU_TRY(e, cudaGetLastError());
    e->launches += 4;
    if (!e->fc_gangs.empty()) {   // the flag, level and domain of the rejected gangs whose fence held
      k_fence_status<<<1, GROVE_MAX_FENCES, 0, e->stream>>>(tb, rx, e->d_perm.p, e->d_status.p);
      CU_TRY(e, cudaGetLastError());
      e->launches += 1;
    }
    if (e->qu_members) {   // the members' flags, from the headroom over the final states
      k_queue_scan<<<e->qu_scanned, 256, 0, e->stream>>>(tb, rx, 1u);
      k_queue_gate<<<(e->qu_members + 255) / 256, 256, 0, e->stream>>>(tb, rx, 2u, e->d_status.p);
      CU_TRY(e, cudaGetLastError());
      e->launches += 2;
    }
    CU_TRY(e, cudaMemcpyAsync(e->h_ctl.p, e->d_totals.p, sizeof(uint32_t) * 4, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(e, cudaMemcpyAsync(e->h_status.p, e->d_status.p, sizeof(grove_gang_status_t) * G, cudaMemcpyDeviceToHost, e->stream));
    // the placement count is only known on the device: copy the upper bound's worth in the same breath when it is small,
    // else wait for the count
    const bool eager = size_t(e->P) * sizeof(grove_placement_t) <= (8u << 20);   // a few hundred KB at C4: cheaper than a second round trip
    if (eager && e->P) CU_TRY(e, cudaMemcpyAsync(e->h_out.p, e->d_out.p, sizeof(grove_placement_t) * e->P, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(e, cudaStreamSynchronize(e->stream));
    e->n_out = e->h_ctl.p[0];
    if (!eager) {
      if (e->n_out) CU_TRY(e, cudaMemcpyAsync(e->h_out.p, e->d_out.p, sizeof(grove_placement_t) * e->n_out, cudaMemcpyDeviceToHost, e->stream));
      CU_TRY(e, cudaStreamSynchronize(e->stream));
    }
    e->last.gangs_admitted = e->h_ctl.p[1]; e->last.gangs_rejected = e->h_ctl.p[2];
  }
  (void)tp;
  e->last.pods_bound = e->n_out; e->last.kernel_launches = e->launches;
  e->have_results = true; e->in_cycle = false;
  return GROVE_OK;
}

// Bin-packing picks (binpack.cuh), after the first capacity-table build of a cycle with members: the per-domain sums of the levels
// the members pack at, each level's domains ranked by (free GPUs, CPU, memory, first node), then a warp per member rewrites its
// anchor.  The picks come back with the cycle's outputs (finish_cycle waits for the copy).
static int32_t binpack_picks(grove_engine* e, const Topo& tp, const Tables& tb, const Relax& rx) {
  const uint32_t G = e->G, M = e->bp_members;
  CU_TRY(e, e->h_bp_mem.ensure(M)); CU_TRY(e, e->d_bp_mem.ensure(M));
  uint32_t levels = 0;
  for (uint32_t g = 0, k = 0; g < G; ++g) {
    const uint8_t b = e->bp_level[g];
    if (b == GROVE_LEVEL_NONE) continue;
    e->h_bp_mem.p[k++] = make_uint4(g, b, e->ginfo[g].anchor, 0u);   // (the default anchor: the host's ginfo is never rewritten)
    levels |= 1u << b;
  }
  BpOff off{};
  uint32_t total = 0;
  for (uint32_t l = 0; l < e->L; ++l) if ((levels >> l) & 1u) { off.o[l] = total; total += e->n_dom[l]; }
  size_t tmp = 0;
  for (uint32_t l = 0; l < e->L; ++l) {
    if (!((levels >> l) & 1u)) continue;
    size_t t = 0;
    CU_TRY(e, cub::DeviceRadixSort::SortPairs(nullptr, t, e->d_bp_key.p, e->d_bp_key.p, e->d_bp_idx.p, e->d_bp_rank.p, e->n_dom[l], BpKeyDecomposer{}, e->stream));
    tmp = std::max(tmp, t);
  }
  CU_TRY(e, e->d_bp_sum.ensure(std::max(total, 1u))); CU_TRY(e, e->d_bp_key.ensure(2 * size_t(std::max(total, 1u))));
  CU_TRY(e, e->d_bp_idx.ensure(std::max(total, 1u))); CU_TRY(e, e->d_bp_rank.ensure(std::max(total, 1u)));
  CU_TRY(e, e->d_bp_tmp.ensure(std::max<size_t>(tmp, 1))); CU_TRY(e, e->d_bp_pick.ensure(G)); CU_TRY(e, e->h_bp_pick.ensure(G));
  CU_TRY(e, cudaMemcpyAsync(e->d_bp_mem.p, e->h_bp_mem.p, sizeof(uint4) * M, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemsetAsync(e->d_bp_sum.p, 0, sizeof(BpSum) * total, e->stream));
  CU_TRY(e, cudaMemsetAsync(e->d_bp_pick.p, 0xFF, sizeof(uint32_t) * G, e->stream));
  k_binpack_sum<<<e->Npad / 256, 256, 0, e->stream>>>(tp, levels, off, e->d_bp_sum.p);
  e->launches += 1;
  BpKey* keys_out = e->d_bp_key.p + total;
  for (uint32_t l = 0; l < e->L; ++l) {
    if (!((levels >> l) & 1u)) continue;
    const uint32_t o = off.o[l], nd = e->n_dom[l];
    if (!nd) continue;   // (no node carries the level's label: no domain to rank)
    k_binpack_keys<<<(nd + 255) / 256, 256, 0, e->stream>>>(e->d_bp_sum.p + o, nd, e->d_bp_key.p + o, e->d_bp_idx.p + o);
    size_t t = e->d_bp_tmp.cap;
    CU_TRY(e, cub::DeviceRadixSort::SortPairs(e->d_bp_tmp.p, t, e->d_bp_key.p + o, keys_out + o, e->d_bp_idx.p + o, e->d_bp_rank.p + o, nd,
                                              BpKeyDecomposer{}, e->stream));
    e->launches += 2;
  }
  k_binpack_pick<<<(M * 32 + 255) / 256, 256, 0, e->stream>>>(tp, tb, rx, e->d_bp_mem.p, M, e->d_bp_sum.p, e->d_bp_rank.p, off, e->d_ginfo.p, e->d_bp_pick.p);
  CU_TRY(e, cudaGetLastError());
  CU_TRY(e, cudaMemcpyAsync(e->h_bp_pick.p, e->d_bp_pick.p, sizeof(uint32_t) * G, cudaMemcpyDeviceToHost, e->stream));
  e->launches += 1;
  e->bp_anchors = true;
  return GROVE_OK;
}

struct CycleGuard {   // every error exit of a cycle leaves the handle usable (ADVICE round 1: in_cycle stayed set)
  grove_engine* e; bool armed = true;
  ~CycleGuard() { if (armed) { e->in_cycle = false; cudaStreamSynchronize(e->stream); cudaStreamSynchronize(e->stream_score); } }
};

static int32_t run_cycle(grove_engine* e, grove_cycle_stats_t* stats) {
  int32_t rc = cycle_begin(e);
  if (rc) return rc;
  CycleGuard guard{e};
  const Topo tp = make_topo(e); const Tables tb = make_tables(e); const Relax rx = make_relax(e);
  const uint32_t G = e->G;
  CU_TRY(e, cudaEventRecord(e->ev[8], e->stream));
  uint32_t rounds = 0;
  if (G && e->bp_anchors) {   // an earlier cycle's picks: back to the default anchors (this cycle's members are picked again)
    CU_TRY(e, cudaMemcpyAsync(e->d_ginfo.p, e->ginfo, sizeof(GangInfo) * G, cudaMemcpyHostToDevice, e->stream));
    k_anchor<<<(G + 255) / 256, 256, 0, e->stream>>>(tp, e->d_ginfo.p, G);
    CU_TRY(e, cudaGetLastError());
    e->launches += 1;
    e->bp_anchors = false;
  }
  if (G && e->holds_on) {   // the holds join the committed state (so every table built from it bounds every gang's view) as claims
    k_hold_publish<<<(G * 32 + 255) / 256, 256, 0, e->stream>>>(tb, rx, e->d_nres.p);
    CU_TRY(e, cudaGetLastError());
    e->launches += 1;
  }
  const bool spread = e->sp_members > 0;   // (the running-gang entries refuse a spread set: no holds here)
  if (G && spread) {   // the classes of every domain's schedulable nodes, over the cycle-start table; no member's stamp
    CU_TRY(e, cudaMemsetAsync(e->d_sp_dcls.p, 0, sizeof(uint32_t) * e->sp_dcls_words, e->stream));
    CU_TRY(e, cudaMemsetAsync(e->d_sp_stamp.p, 0xFF, sizeof(uint32_t) * e->sp_groups, e->stream));
    k_spread_classes<<<(e->N + 255) / 256, 256, 0, e->stream>>>(tp, rx);
    CU_TRY(e, cudaGetLastError());
    e->launches += 1;
  }
  const bool fences = !e->fc_gangs.empty();   // (the running-gang entries and spread cycles refuse a fence set)
  const bool queues = e->qu_members > 0;   // (the running-gang entries, spread and fenced cycles refuse a queue set)
  const bool imex = e->im_enrolled > 0;    // (the running-gang entries and the other sets' cycles refuse an enrolled clique)
  if (G && imex) {   // the CD of every clique and of every rank's gang, owner0 in sorted order (padding: no owner), no enrolled claim
    e->h_im_rank_cd.resize(G); e->h_im_owner.resize(e->Npad);
    for (uint32_t g = 0; g < G; ++g) e->h_im_rank_cd[e->ginfo[g].order] = e->im_gang_cd[g];
    for (uint32_t i = 0; i < e->Npad; ++i) e->h_im_owner[i] = i < e->N ? e->im_owner0[e->perm[i]] : GROVE_CD_NONE;
    CU_TRY(e, cudaMemcpyAsync(e->d_im_cd.p, e->im_cd.data(), sizeof(uint32_t) * e->Q, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(e, cudaMemcpyAsync(e->d_im_rank_cd.p, e->h_im_rank_cd.data(), sizeof(uint32_t) * G, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(e, cudaMemcpyAsync(e->d_im_owner.p, e->h_im_owner.data(), sizeof(uint32_t) * e->Npad, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(e, cudaMemsetAsync(e->d_im_nenr.p, 0, sizeof(uint32_t) * e->Npad, e->stream));
  }
  if (G && queues) {   // the members' gates and caps before round 1: no member holds anything yet, H_Q = limit - load
    k_queue_scan<<<e->qu_scanned, 256, 0, e->stream>>>(tb, rx, 0u);
    k_queue_gate<<<(e->qu_members + 255) / 256, 256, 0, e->stream>>>(tb, rx, 0u, nullptr);
    CU_TRY(e, cudaGetLastError());
    e->launches += 2;
  }
  if (G && fences) {   // the picks, over the cycle-start table
    const uint32_t nf = uint32_t(e->fc_gangs.size());
    CU_TRY(e, e->d_fc_have.ensure(std::max<size_t>(e->fc_words, 1)));
    CU_TRY(e, cudaMemcpyAsync(e->d_fc_gang.p, e->fc_gangs.data(), sizeof(uint32_t) * nf, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(e, cudaMemcpyAsync(e->d_fc_off.p, e->fc_off.data(), sizeof(uint32_t) * nf, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(e, cudaMemsetAsync(e->d_fc_have.p, 0, sizeof(uint32_t) * e->fc_words, e->stream));
    CU_TRY(e, cudaMemsetAsync(e->d_fc_slot.p, 0xFF, sizeof(uint32_t) * G, e->stream));
    k_fence_have<<<dim3(e->Npad / 256, nf), 256, 0, e->stream>>>(tp, tb, e->d_fc_gang.p, e->d_fc_off.p, e->d_fc_have.p);
    k_fence_pick<<<1, 1024, 0, e->stream>>>(tp, tb, e->d_fc_gang.p, e->d_fc_off.p, e->d_fc_have.p, nf, e->d_fc_list.p, e->d_fc_slot.p);
    CU_TRY(e, cudaGetLastError());
    e->launches += 2;
  }
  if (G) {
    // K1 + capacity tables over the cycle-start snapshot; K2 (score matrix) forks to the second stream
    CU_TRY(e, cudaEventRecord(e->ev[0], e->stream));
    rc = build_cap_tables(e, tp, tb, rx);
    if (rc) return rc;
    CU_TRY(e, cudaEventRecord(e->ev[1], e->stream));
    if (e->bp_members) { rc = binpack_picks(e, tp, tb, rx); if (rc) return rc; }   // (before K2: it scores against the picks)
    CU_TRY(e, e->d_F0.ensure(std::max<size_t>(size_t(e->n_sigs) * e->words, 1)));
    CU_TRY(e, cudaMemcpyAsync(e->d_F0.p, e->d_F.p, sizeof(uint32_t) * size_t(e->n_sigs) * e->words, cudaMemcpyDeviceToDevice, e->stream));
    e->score_valid = false;
    if (e->tune_score && e->Q) {
      cudaStream_t ss = e->tune_overlap ? e->stream_score : e->stream;
      if (e->tune_overlap) CU_TRY(e, cudaEventRecord(e->ev_fit, e->stream));
      if (e->tune_overlap) CU_TRY(e, cudaStreamWaitEvent(ss, e->ev_fit, 0));
      CU_TRY(e, cudaEventRecord(e->ev_s0, ss));
      k_score<<<dim3(1, std::min<uint32_t>(e->Q, 65535u)), 256, 0, ss>>>(tp, tb, e->d_F0.p, e->d_T.p, e->Q, 0u, e->Npad >> 4, size_t(e->Npad));  // one CTA per row
      e->score_valid = true;
      CU_TRY(e, cudaEventRecord(e->ev_s1, ss));
      if (e->tune_overlap) CU_TRY(e, cudaEventRecord(e->ev_score, e->stream_score));
      e->launches += 1;
    }
    CU_TRY(e, cudaEventRecord(e->ev[2], e->stream));
    const uint32_t W = rx.window;
    const uint32_t n_eval_ctas = eval_ctas(e);
    const uint32_t warp_ctas = std::max(1u, std::min((W * 32 + 255) / 256, e->n_sm * e->tune_warp_ctas));
    // Rounds are enqueued `batch` at a time without waiting: every kernel returns at once when the cycle is over, so the
    // host only looks at the control words between batches (to rebuild the capacity tables when the settled prefix has
    // moved on, and to know when to stop).  GROVE_DEBUG_ADMIT looks after every round.
    const uint32_t batch = e->dbg_on ? 1u : std::max(1u, e->tune_batch);
    uint32_t next_round = 1;   // number of the next round to be enqueued (rounds advance one by one until the cycle is over)
    auto enqueue_round = [&]() -> int32_t {
      if (next_round > 1 && next_round % kTagRounds == 0) {   // the stamp tags wrap: forget the stamps of the epoch that ends
        CU_TRY(e, cudaMemsetAsync(e->d_add_stamp.p, 0xFF, sizeof(uint32_t) * e->Npad, e->stream));
        CU_TRY(e, cudaMemsetAsync(e->d_rem_stamp.p, 0xFF, sizeof(uint32_t) * e->words, e->stream));
        if (spread) CU_TRY(e, cudaMemsetAsync(e->d_sp_stamp.p, 0xFF, sizeof(uint32_t) * e->sp_groups, e->stream));
      }
      if (spread) {   // a spread cycle: the members' allowed domains first, then its own instantiations of the round's kernels
        CU_TRY(e, launch_chained(k_spread, e->sp_groups, 256, e->stream, tp, tb, rx, 0u));
        CU_TRY(e, launch_chained(e->any_preferred ? k_eval<true, false, false, true> : k_eval<false, false, false, true>, n_eval_ctas,
                                 kEvalWarps * 32, e->stream, tp, tb, rx, e->tune_max_att));
        CU_TRY(e, launch_chained(k_apply<false, true>, warp_ctas, 256, e->stream, tb, rx));
        CU_TRY(e, launch_chained(k_detect<true>, warp_ctas, 256, e->stream, tp, tb, rx, e->tune_refresh));
        e->launches += 4;
        ++next_round;
        return GROVE_OK;
      }
      if (fences) {   // a fenced cycle: its own instantiations of K3 and k_apply
        CU_TRY(e, launch_chained(e->any_preferred ? k_eval<true, false, false, false, true> : k_eval<false, false, false, false, true>,
                                 n_eval_ctas, kEvalWarps * 32, e->stream, tp, tb, rx, e->tune_max_att));
        CU_TRY(e, launch_chained(k_apply<false, false, true>, warp_ctas, 256, e->stream, tb, rx));
        CU_TRY(e, launch_chained(k_detect<false>, warp_ctas, 256, e->stream, tp, tb, rx, e->tune_refresh));
        e->launches += 3;
        ++next_round;
        return GROVE_OK;
      }
      if (imex) {   // a cycle with enrolled cliques: its own instantiations of K3 and k_apply
        CU_TRY(e, launch_chained(e->any_preferred ? k_eval<true, false, false, false, false, false, true> : k_eval<false, false, false, false, false, false, true>,
                                 n_eval_ctas, kEvalWarps * 32, e->stream, tp, tb, rx, e->tune_max_att));
        CU_TRY(e, launch_chained(k_apply<false, false, false, false, true>, warp_ctas, 256, e->stream, tb, rx));
        CU_TRY(e, launch_chained(k_detect<false>, warp_ctas, 256, e->stream, tp, tb, rx, e->tune_refresh));
        e->launches += 3;
        ++next_round;
        return GROVE_OK;
      }
      if (queues) {   // a queue cycle: its own instantiations of K3 and k_apply, then the headroom and the gates before k_detect
        CU_TRY(e, launch_chained(e->any_preferred ? k_eval<true, false, false, false, false, true> : k_eval<false, false, false, false, false, true>,
                                 n_eval_ctas, kEvalWarps * 32, e->stream, tp, tb, rx, e->tune_max_att));
        CU_TRY(e, launch_chained(k_apply<false, false, false, true>, warp_ctas, 256, e->stream, tb, rx));
        CU_TRY(e, launch_chained(k_queue_scan, e->qu_scanned, 256, e->stream, tb, rx, 0u));
        CU_TRY(e, launch_chained(k_queue_gate, (e->qu_members + 255) / 256, 256, e->stream, tb, rx, 1u, (grove_gang_status_t*)nullptr));
        CU_TRY(e, launch_chained(k_detect<false>, warp_ctas, 256, e->stream, tp, tb, rx, e->tune_refresh));
        e->launches += 5;
        ++next_round;
        return GROVE_OK;
      }
      // one stream-ordered chain: evaluate -> publish -> detect, each launched while the one before drains
      // (a wide cycle never has holds: grove_run_cycle_reuse refuses wide submissions)
      auto* k3 = e->wide ? (e->any_preferred ? k_eval<true, false, true> : k_eval<false, false, true>)
                 : e->holds_on ? (e->any_preferred ? k_eval<true, true, false> : k_eval<false, true, false>)
                               : (e->any_preferred ? k_eval<true, false, false> : k_eval<false, false, false>);
      CU_TRY(e, launch_chained(k3, n_eval_ctas, kEvalWarps * 32, e->stream, tp, tb, rx, e->tune_max_att));
      CU_TRY(e, launch_chained(e->holds_on ? k_apply<true> : k_apply<false>, warp_ctas, 256, e->stream, tb, rx));
      CU_TRY(e, launch_chained(k_detect<false>, warp_ctas, 256, e->stream, tp, tb, rx, e->tune_refresh));
      e->launches += 3;
      ++next_round;
      return GROVE_OK;
    };
    auto fold = [&]() -> int32_t {   // the final gangs' claims -> committed state (relax.cuh k_fold)
      CU_TRY(e, launch_chained(imex ? k_fold<false, true> : e->holds_on ? k_fold<true> : k_fold<false>, warp_ctas, 256, e->stream, tb, rx, e->d_nres.p));
      CU_TRY(e, launch_chained(k_fold_mark, 1, 1, e->stream, rx));
      e->launches += 2;
      CU_TRY(e, cudaGetLastError());
      return GROVE_OK;
    };
    auto fold_and_rebuild = [&]() -> int32_t { int32_t r = fold(); return r ? r : build_cap_tables(e, tp, tb, rx); };
    // Following the relaxation WITHOUT blocking calls: the last CTA of k_detect leaves (round, done, refresh, ...) in host-mapped
    // memory; the host keeps `ahead` rounds enqueued beyond the one that runs and adds one more each time it sees a round end
    // (or a table rebuild first, when the device asked for one).  The GPU never waits for the host; the only waste is the
    // <= ahead rounds in the queue when the cycle ends, which return at once.
    const bool polled = e->h_live && e->tune_ahead > 0 && !e->dbg_on;
    bool use_batch = !polled;   // the batch protocol below: also the way out should the progress words ever stop moving
    if (polled) {
      volatile uint32_t* lv = e->h_live;
      uint32_t enq = 0, rebuild_at = 0;   // rounds enqueued; the last rebuild enqueued runs before round rebuild_at + 1
      for (; enq < e->tune_ahead; ++enq) { rc = enqueue_round(); if (rc) return rc; }
      CU_TRY(e, cudaGetLastError());
      uint64_t spins = 0;
      for (;;) {
        const uint32_t completed = lv[kLiveRound] - 1u;
        if (lv[kLiveDone] && completed >= 1u) break;
        if (completed + e->tune_ahead > enq) {   // fewer than `ahead` rounds in flight: top the queue up
          if (lv[kLiveRefresh] && completed > rebuild_at) { rc = fold_and_rebuild(); if (rc) return rc; rebuild_at = enq; }   // (the flag is fresh again once round rebuild_at + 1 has ended)
          rc = enqueue_round(); if (rc) return rc;
          ++enq; spins = 0;
          continue;
        }
#if defined(__x86_64__) || defined(__i386__)
        __builtin_ia32_pause();   // (a polite spin: the sibling hyper-thread may be another rank's)
#endif
        if ((++spins & 0xFFFFu) == 0) {   // a failed launch / a sticky error must not leave the host spinning
          const cudaError_t q = cudaStreamQuery(e->stream);
          if (q != cudaSuccess && q != cudaErrorNotReady) { e->err = std::string("relaxation: ") + cudaGetErrorString(q); return GROVE_ERR_CUDA; }
          // nothing left in flight on the engine's stream, yet the words say rounds are outstanding: do not trust them any
          // further -- the control words themselves are read from here on
          if (q == cudaSuccess && lv[kLiveRound] - 1u == completed && !lv[kLiveDone]) { use_batch = true; break; }
        }
      }
    }
    for (; use_batch;) {   // (the batch protocol: look at the control words between batches of rounds)
      for (uint32_t b = 0; b < batch; ++b) { rc = enqueue_round(); if (rc) return rc; }
      CU_TRY(e, cudaGetLastError());
      CU_TRY(e, cudaMemcpyAsync(e->h_ctl.p, e->d_ctl.p, sizeof(uint32_t) * kCtlWords, cudaMemcpyDeviceToHost, e->stream));
      CU_TRY(e, cudaStreamSynchronize(e->stream));
      const uint32_t* c = e->h_ctl.p;
      rounds = c[kRound] - 1;
      if (e->dbg_on) {
        std::fprintf(stderr, "round %u: front %u hi %u evals so far %u ovf %u\n", rounds, c[kFront], c[kHi], c[kEvals], c[kOvfCount]);
        std::vector<uint32_t> h(size_t(G) * 8); std::vector<uint8_t> ts(G);
        cudaMemcpy(h.data(), e->d_dbg.p, h.size() * 4, cudaMemcpyDeviceToHost);
        cudaMemcpy(ts.data(), e->d_tstate.p, G, cudaMemcpyDeviceToHost);
        std::vector<uint32_t> idx;
        for (uint32_t g = 0; g < G; ++g) if (h[size_t(g) * 8 + 7] == rounds) idx.push_back(g);
        std::sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return h[size_t(a) * 8 + 4] > h[size_t(b) * 8 + 4]; });
        uint64_t cyc = 0; for (uint32_t g : idx) cyc += h[size_t(g) * 8 + 4];
        std::fprintf(stderr, "  %zu packed evals, mean %.0f cyc, median %u; slowest:", idx.size(), idx.empty() ? 0.0 : double(cyc) / idx.size(), idx.empty() ? 0u : h[size_t(idx[idx.size() / 2]) * 8 + 4]);
        for (size_t i = 0; i < std::min<size_t>(idx.size(), 6); ++i) {
          const uint32_t g = idx[i]; const uint32_t* d = &h[size_t(g) * 8];
          std::fprintf(stderr, " [g%u rank%u st%u scopes%u: %u cyc, %u plaus, %u att]", g, e->ginfo[g].order, unsigned(ts[g]), unsigned(e->gangs[g].n_scopes), d[4], d[6], d[5]);
        }
        std::fprintf(stderr, "\n");
      }
      if (c[kOvfCount] > rx.ovf_cap) return fail(e, GROVE_ERR_LIMIT, "claim overflow pool exhausted");
      if (c[kDone]) break;
      if (c[kRefresh]) { rc = fold_and_rebuild(); if (rc) return rc; }
    }
    if (polled && !use_batch) {   // the cycle is over (the queue holds at most a few rounds that return at once): the final control words
      CU_TRY(e, cudaMemcpyAsync(e->h_ctl.p, e->d_ctl.p, sizeof(uint32_t) * kCtlWords, cudaMemcpyDeviceToHost, e->stream));
      CU_TRY(e, cudaStreamSynchronize(e->stream));
      if (e->h_ctl.p[kOvfCount] > rx.ovf_cap) return fail(e, GROVE_ERR_LIMIT, "claim overflow pool exhausted");
      rounds = e->h_ctl.p[kRound] - 1;
    }
    rc = fold(); if (rc) return rc;   // everything is final now: the committed state and the final states of the outputs
    if (imex)   // the owners after the last fold (read back with the statuses: finish_cycle waits for the copy)
      CU_TRY(e, cudaMemcpyAsync(e->h_im_owner.data(), e->d_im_owner.p, sizeof(uint32_t) * e->N, cudaMemcpyDeviceToHost, e->stream));
    if (e->holds_on) {   // the admitted owners' leftovers: the running gangs they replace are gone
      k_hold_release<<<(G * 32 + 255) / 256, 256, 0, e->stream>>>(tb, rx, e->d_nres.p);
      CU_TRY(e, cudaGetLastError());
      e->launches += 1;
    }
    if (spread) {   // which SOFT members landed outside their allowed domains (read back with the statuses); k_spread writes the
                    // members' bytes only, so every other gang reads 0
      CU_TRY(e, cudaMemsetAsync(e->d_sp_skewed.p, 0, G, e->stream));
      k_spread<<<e->sp_groups, 256, 0, e->stream>>>(tp, tb, rx, 1u);
      CU_TRY(e, cudaGetLastError());
      CU_TRY(e, cudaMemcpyAsync(e->h_sp_skewed.p, e->d_sp_skewed.p, G, cudaMemcpyDeviceToHost, e->stream));
      e->launches += 1;
    }
    e->last.evaluations = e->h_ctl.p[kEvals];
  }
  CU_TRY(e, cudaEventRecord(e->ev[3], e->stream));
  if (e->tune_score && e->tune_overlap && G && e->Q) CU_TRY(e, cudaStreamWaitEvent(e->stream, e->ev_score, 0));  // the cycle ends when K2 has too
  rc = finish_cycle(e);
  if (rc) return rc;
  if (spread)   // (finish_cycle waited for the copy)
    for (uint32_t g = 0; g < G; ++g) if (e->h_sp_skewed.p[g]) e->h_status.p[g].reserved0 |= GROVE_STATUS_SPREAD_SKEWED;
  if (e->bp_given) {   // (so did it for the picks')
    e->bp_picks.assign(G, GROVE_NONE_U32);
    if (e->bp_members)
      for (uint32_t g = 0; g < G; ++g) if (e->h_bp_pick.p[g] != kFull) e->bp_picks[g] = e->perm[e->h_bp_pick.p[g]];
    e->bp_have_picks = true;
  }
  if (e->im_given) {   // owner0, plus the CD of every admitted gang's enrolled pods
    e->im_owners = e->im_owner0;
    if (imex && G) for (uint32_t i = 0; i < e->N; ++i) e->im_owners[e->perm[i]] = e->h_im_owner[i];
    e->im_have_owners = true;
  }
  CU_TRY(e, cudaEventRecord(e->ev[9], e->stream));
  CU_TRY(e, cudaEventSynchronize(e->ev[9]));
  guard.armed = false;
  float t = 0;
  if (G) {
    cudaEventElapsedTime(&t, e->ev[0], e->ev[1]); e->last.ms_fit = t;
    if (e->tune_score && e->Q) { cudaEventElapsedTime(&t, e->ev_s0, e->ev_s1); e->last.ms_score = t; }
    cudaEventElapsedTime(&t, e->ev[2], e->ev[3]); e->last.ms_admit = t;
  }
  cudaEventElapsedTime(&t, e->ev[3], e->ev[9]); e->last.ms_commit = t;
  cudaEventElapsedTime(&t, e->ev[8], e->ev[9]); e->last.ms_total = t;
  e->last.rounds = rounds;
  e->last.pairs_evaluated = uint64_t(e->tune_score ? e->Q : e->n_sigs) * e->N;   // K1 works per signature, K2 per clique
  if (e->dbg_on && G) {
    std::vector<uint32_t> h(size_t(G) * 8 + 8);
    cudaMemcpy(h.data(), e->d_dbg.p, h.size() * 4, cudaMemcpyDeviceToHost);
    { const uint32_t* w = &h[size_t(G) * 8];
      std::fprintf(stderr, "warp 0 of every evaluation: %u evals, %.0f cyc each; %u staged attempts: staging %.0f cyc, sub-domain pre-filter %.0f, packing %.0f per attempt\n",
                   w[5], w[5] ? double(w[4]) / w[5] : 0.0, w[3], w[3] ? double(w[0]) / w[3] : 0.0, w[3] ? double(w[1]) / w[3] : 0.0, w[3] ? double(w[2]) / w[3] : 0.0);
      std::fprintf(stderr, "  of the staging: claim lines %.0f cyc, overflow chains %.0f per attempt\n", w[3] ? double(w[6]) / w[3] : 0.0, w[3] ? double(w[7]) / w[3] : 0.0); }
    uint64_t ev = 0, pl = 0, at = 0, mx = 0;
    for (uint32_t g = 0; g < G; ++g) { ev += h[g * 8]; pl += h[g * 8 + 1]; at += h[g * 8 + 2]; mx = std::max<uint64_t>(mx, h[g * 8]); }
    std::fprintf(stderr, "cycle: %u rounds, %llu evaluations (max %llu per gang), plausible/eval %.1f, attempts/eval %.2f\n", rounds,
                 (unsigned long long)ev, (unsigned long long)mx, ev ? double(pl) / ev : 0.0, ev ? double(at) / ev : 0.0);
  }
  if (stats) *stats = e->last;
  return GROVE_OK;
}

static int32_t fair_share_cycle(grove_engine* e, grove_cycle_stats_t* stats);

int32_t grove_run_cycle(grove_engine_t* e, grove_cycle_stats_t* stats) {
  if (!e) return GROVE_ERR_INVALID_ARG;
  if (e->fs_given) return fair_share_cycle(e, stats);
  const bool spread = e->sp_members > 0, fences = !e->fc_gangs.empty();
  if (spread && fences) return fail(e, GROVE_ERR_STATE, "grove_run_cycle: a spread set with members and a fence set together are not supported");
  if (e->qu_members && (spread || fences))
    return fail(e, GROVE_ERR_STATE, "grove_run_cycle: a queue set with members together with a spread set with members or a fence set is not supported");
  if (e->bp_members && (spread || fences))
    return fail(e, GROVE_ERR_STATE, "grove_run_cycle: a bin-packing set with members together with a spread set with members or a fence set is not supported");
  if (e->im_enrolled && (spread || fences || e->qu_members || e->bp_members))
    return fail(e, GROVE_ERR_STATE, "grove_run_cycle: a ComputeDomain set with an enrolled clique together with a spread set with members, a fence set, "
                                    "a queue set with members or a bin-packing set with members is not supported");
  const int32_t rc = run_cycle(e, stats);
  if (rc == GROVE_OK)
    e->diag = spread ? grove_engine::kDiagSpread : fences ? grove_engine::kDiagFence : e->im_enrolled ? grove_engine::kDiagImex : grove_engine::kDiagReady;
  return rc;
}

// the entries with running gangs judge their gangs against other views: grove_diagnose refuses their outputs
struct NoDiagnosis {
  grove_engine* e;
  ~NoDiagnosis() { if (e) e->diag = grove_engine::kDiagRunning; }
};

int32_t grove_get_placements(grove_engine_t* e, grove_placement_t* out, uint32_t cap, uint32_t* n_out) {
  if (!e || !n_out) return GROVE_ERR_INVALID_ARG;
  if (!e->have_results) return fail(e, GROVE_ERR_STATE, "no completed cycle");
  *n_out = e->n_out;
  if (!out) return GROVE_OK;
  if (cap < e->n_out) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  std::memcpy(out, e->h_out.p, sizeof(grove_placement_t) * e->n_out);
  return GROVE_OK;
}

int32_t grove_get_gang_status(grove_engine_t* e, grove_gang_status_t* out, uint32_t cap) {
  if (!e || !out) return GROVE_ERR_INVALID_ARG;
  if (!e->have_results) return fail(e, GROVE_ERR_STATE, "no completed cycle");
  if (cap < e->G) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  std::memcpy(out, e->h_status.p, sizeof(grove_gang_status_t) * e->G);
  return GROVE_OK;
}

int32_t grove_get_scope_domains(grove_engine_t* e, grove_scope_status_t* out, uint32_t cap) {
  if (!e || !out) return GROVE_ERR_INVALID_ARG;
  if (!e->have_results) return fail(e, GROVE_ERR_STATE, "no completed cycle");
  if (cap < e->S) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  if (!e->have_scopes && e->S) {   // fetched on demand: most callers only bind pods
    CU_TRY(e, cudaSetDevice(e->cfg.device));
    CU_TRY(e, cudaMemcpyAsync(e->h_scope_status.p, e->d_scope_status.p, sizeof(grove_scope_status_t) * e->S, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(e, cudaStreamSynchronize(e->stream));
    e->have_scopes = true;
  }
  std::memcpy(out, e->h_scope_status.p, sizeof(grove_scope_status_t) * e->S);
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// Topology spread (include/grove_place.h "topology spread"; DESIGN.md section 1; kernels in spread.cuh).  Validated against the
// loaded nodes and the submission and uploaded here; the cycle only builds the per-domain classes and runs k_spread.
// ---------------------------------------------------------------------------------------------
int32_t grove_set_spread(grove_engine_t* e, const grove_spread_t* groups, uint32_t n_groups, const uint32_t* gang_group, uint32_t n_gangs,
                         const grove_spread_seed_t* seeds, uint32_t n_seeds) {
  if (!e) return GROVE_ERR_INVALID_ARG;
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  if (!e->nodes_loaded || !e->gangs_loaded) return fail(e, GROVE_ERR_STATE, "grove_set_spread: load nodes and submit gangs first");
  if ((n_groups && !groups) || (n_gangs && !gang_group) || (n_seeds && !seeds)) return GROVE_ERR_INVALID_ARG;
  if (n_gangs != e->G) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_spread: n_gangs is not the number of submitted gangs");
  if (e->wide) return refuse_wide(e, "grove_set_spread");
  for (uint32_t s = 0; s < n_groups; ++s) {
    if (groups[s].level >= e->L) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_spread: spread level out of range");
    if (groups[s].mode != GROVE_SPREAD_HARD && groups[s].mode != GROVE_SPREAD_SOFT)
      return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_spread: mode must be GROVE_SPREAD_HARD or GROVE_SPREAD_SOFT");
    if (groups[s].max_skew == 0) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_spread: max_skew must be at least 1");
  }
  uint32_t members = 0;
  for (uint32_t g = 0; g < n_gangs; ++g) {
    const uint32_t s = gang_group[g];
    if (s == GROVE_NONE_U32) continue;
    if (s >= n_groups) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_spread: spread group out of range");
    const grove_gang_t& gg = e->gangs[g];
    if (gg.level == GROVE_LEVEL_NONE || gg.level < groups[s].level)
      return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_spread: a member needs a gang Required level at or below its group's level");
    bool need = false;
    for (uint32_t c = 0; c < gg.n_cliques; ++c) need |= (e->ccount[gg.clique_off + c] & 0xFFFFu) > 0;
    if (!need) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_spread: a member needs a clique with MinReplicas > 0");
    ++members;
  }
  for (uint32_t i = 0; i < n_seeds; ++i) {
    if (seeds[i].group >= n_groups) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_spread: seed group out of range");
    if (seeds[i].node >= e->N) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_spread: seed node out of range");
  }
  e->sp_groups = e->sp_members = 0;
  if (!members) return GROVE_OK;   // nothing to spread: the ordinary cycle
  // members by group in rank order (priority desc, index asc); an allowed row and a count row per group's level
  const uint32_t G = n_gangs;
  std::vector<uint32_t> order(G);
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), [e](uint32_t a, uint32_t b) { return e->gangs[a].priority > e->gangs[b].priority; });
  std::vector<uint32_t> mem_off(n_groups + 1, 0), cnt_off(n_groups, 0), info(n_groups), row(G, GROVE_NONE_U32), group(gang_group, gang_group + G);
  for (uint32_t g = 0; g < G; ++g) if (group[g] != GROVE_NONE_U32) ++mem_off[group[g] + 1];
  for (uint32_t s = 0; s < n_groups; ++s) mem_off[s + 1] += mem_off[s];
  std::vector<uint32_t> mem(members), cls(members), fill(mem_off.begin(), mem_off.end() - 1);
  for (uint32_t g : order) {
    const uint32_t s = group[g];
    if (s == GROVE_NONE_U32) continue;
    const grove_gang_t& gg = e->gangs[g];
    uint32_t m = 0;
    for (uint32_t c = 0; c < gg.n_cliques; ++c) m |= e->cliques[gg.clique_off + c].class_mask;
    mem[fill[s]] = g; cls[fill[s]] = m; ++fill[s];
  }
  uint64_t cnt_words = 0, row_words = 0;
  for (uint32_t s = 0; s < n_groups; ++s) {
    const uint32_t nd = e->n_dom[groups[s].level];
    info[s] = uint32_t(groups[s].level) | uint32_t(groups[s].mode) << 8 | uint32_t(groups[s].max_skew) << 16;
    cnt_off[s] = uint32_t(cnt_words); cnt_words += nd;
    for (uint32_t j = mem_off[s]; j < mem_off[s + 1]; ++j) { row[mem[j]] = uint32_t(row_words); row_words += (nd + 31u) / 32u; }
  }
  // members x domains of their level, one bit each (DESIGN.md section 2): refused beyond 1 GB
  if (row_words > (uint64_t(1) << 28) || cnt_words > (uint64_t(1) << 28))
    return fail(e, GROVE_ERR_LIMIT, "grove_set_spread: the allowed-domain rows (members x domains of their level) exceed 1 GB");
  std::vector<uint32_t> seed(std::max<uint64_t>(cnt_words, 1), 0u);
  for (uint32_t i = 0; i < n_seeds; ++i) {
    const uint32_t s = seeds[i].group, d = e->tdom[size_t(e->inv[seeds[i].node]) * GROVE_MAX_LEVELS + groups[s].level];
    if (d != GROVE_DOM_ABSENT) seed[cnt_off[s] + d] += 1u;   // a node without the level's label is in no domain of it
  }
  uint32_t dw = 0;
  for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) { e->sp_dcls_off[l] = dw; if (l < e->L) dw += e->n_dom[l]; }
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  auto up = [e](DevBuf<uint32_t>& d, const std::vector<uint32_t>& h) -> cudaError_t {
    cudaError_t c = d.ensure(std::max<size_t>(h.size(), 1));
    if (c == cudaSuccess && !h.empty()) c = cudaMemcpyAsync(d.p, h.data(), sizeof(uint32_t) * h.size(), cudaMemcpyHostToDevice, e->stream);
    return c;
  };
  CU_TRY(e, up(e->d_sp_group, group)); CU_TRY(e, up(e->d_sp_row, row)); CU_TRY(e, up(e->d_sp_info, info)); CU_TRY(e, up(e->d_sp_mem_off, mem_off));
  CU_TRY(e, up(e->d_sp_mem, mem)); CU_TRY(e, up(e->d_sp_cls, cls)); CU_TRY(e, up(e->d_sp_cnt_off, cnt_off)); CU_TRY(e, up(e->d_sp_seed, seed));
  CU_TRY(e, e->d_sp_allowed.ensure(std::max<uint64_t>(row_words, 1)));
  CU_TRY(e, cudaStreamSynchronize(e->stream));   // (the host vectors go out of scope)
  e->sp_groups = n_groups; e->sp_members = members; e->sp_cnt_words = uint32_t(cnt_words); e->sp_dcls_words = dw;
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// Fences (include/grove_place.h "fences"; DESIGN.md section 1; kernels in fence.cuh).  Validated against the submission; the
// cycle makes the picks and runs the kFence instantiations.
// ---------------------------------------------------------------------------------------------
int32_t grove_set_fences(grove_engine_t* e, const uint32_t* gangs, uint32_t n) {
  if (!e) return GROVE_ERR_INVALID_ARG;
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  if (!e->nodes_loaded || !e->gangs_loaded) return fail(e, GROVE_ERR_STATE, "grove_set_fences: load nodes and submit gangs first");
  if (n && !gangs) return GROVE_ERR_INVALID_ARG;
  if (n > GROVE_MAX_FENCES) return fail(e, GROVE_ERR_LIMIT, "grove_set_fences: more than GROVE_MAX_FENCES fencing gangs");
  if (e->wide) return refuse_wide(e, "grove_set_fences");
  std::vector<uint32_t> v(gangs, gangs + n);
  for (uint32_t k = 0; k < n; ++k) {
    if (v[k] >= e->G) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_fences: gang index out of range");
    if (e->gangs[v[k]].level == GROVE_LEVEL_NONE) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_fences: a fencing gang needs a gang Required level");
  }
  std::vector<uint32_t> sorted(v);
  std::sort(sorted.begin(), sorted.end());
  if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_fences: a gang is named twice");
  std::stable_sort(v.begin(), v.end(), [e](uint32_t a, uint32_t b) {   // rank order: priority desc, index asc
    return e->gangs[a].priority != e->gangs[b].priority ? e->gangs[a].priority > e->gangs[b].priority : a < b;
  });
  std::vector<uint32_t> off(n);
  size_t words = 0;
  for (uint32_t k = 0; k < n; ++k) {
    const grove_gang_t& gg = e->gangs[v[k]];
    off[k] = uint32_t(words); words += size_t(gg.n_cliques) * e->n_dom[gg.level];
  }
  if (words > (size_t(1) << 28))
    return fail(e, GROVE_ERR_LIMIT, "grove_set_fences: the per-domain sums (fencing gangs x cliques x domains of their level) exceed 1 GB");
  e->fc_gangs = std::move(v); e->fc_off = std::move(off); e->fc_words = words;
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// Bin-packing (include/grove_place.h "bin-packing"; DESIGN.md section 1; kernels in binpack.cuh).  Validated against the
// submission; the cycle makes the picks over its own F0.
// ---------------------------------------------------------------------------------------------
int32_t grove_set_binpack(grove_engine_t* e, const uint8_t* level_of, uint32_t n_gangs) {
  if (!e) return GROVE_ERR_INVALID_ARG;
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  if (!e->nodes_loaded || !e->gangs_loaded) return fail(e, GROVE_ERR_STATE, "grove_set_binpack: load nodes and submit gangs first");
  if (n_gangs != e->G) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_binpack: n_gangs is not the number of gangs submitted");
  if (n_gangs && !level_of) return GROVE_ERR_INVALID_ARG;
  if (e->wide) return refuse_wide(e, "grove_set_binpack");
  uint32_t members = 0;
  for (uint32_t g = 0; g < n_gangs; ++g) {
    const uint8_t b = level_of[g];
    if (b == GROVE_LEVEL_NONE) continue;
    if (b >= e->L) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_binpack: pack level out of range");
    if (e->gangs[g].level != GROVE_LEVEL_NONE && b < e->gangs[g].level)
      return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_binpack: a pack level above the gang's Required level");
    ++members;
  }
  e->bp_level.assign(level_of, level_of + n_gangs);
  e->bp_members = members; e->bp_given = true;
  return GROVE_OK;
}

int32_t grove_get_binpack_picks(grove_engine_t* e, uint32_t* out, uint32_t cap) {
  if (!e || !out) return GROVE_ERR_INVALID_ARG;
  if (!e->bp_have_picks) return fail(e, GROVE_ERR_STATE, "grove_get_binpack_picks: no cycle has run with a bin-packing set");
  if (cap < e->bp_picks.size()) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  std::copy(e->bp_picks.begin(), e->bp_picks.end(), out);
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// ComputeDomain exclusivity (include/grove_place.h "ComputeDomain exclusivity"; DESIGN.md section 1; imex.cuh).  Validated against
// the submission and the node table; the cycle uploads the set and runs the kImex instantiations.
// ---------------------------------------------------------------------------------------------
int32_t grove_set_compute_domains(grove_engine_t* e, const uint32_t* cd, uint32_t n_cliques, const uint32_t* owner0, uint32_t n_nodes) {
  if (!e) return GROVE_ERR_INVALID_ARG;
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  if (!e->nodes_loaded || !e->gangs_loaded) return fail(e, GROVE_ERR_STATE, "grove_set_compute_domains: load nodes and submit gangs first");
  if (n_cliques != e->Q) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_compute_domains: n_cliques is not the number of cliques submitted");
  if (n_nodes != e->N) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_compute_domains: n_nodes is not the number of nodes loaded");
  if ((n_cliques && !cd) || !owner0) return GROVE_ERR_INVALID_ARG;
  if (e->wide) return refuse_wide(e, "grove_set_compute_domains");
  std::vector<uint32_t> gang_cd(e->G, GROVE_CD_NONE);
  uint32_t enrolled = 0;
  for (uint32_t g = 0; g < e->G; ++g) {
    const grove_gang_t& gg = e->gangs[g];
    for (uint32_t c = 0; c < gg.n_cliques; ++c) {
      const uint32_t q = gg.clique_off + c, v = cd[q];
      if (v == GROVE_CD_NONE) continue;
      if (v == GROVE_CD_NO_IMEX) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_compute_domains: GROVE_CD_NO_IMEX is not a clique's CD");
      if (e->cliques[q].req_gpu == 0) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_compute_domains: an enrolled clique requests no GPU");
      if (gang_cd[g] != GROVE_CD_NONE && gang_cd[g] != v)
        return fail(e, GROVE_ERR_LIMIT, "grove_set_compute_domains: the enrolled cliques of one gang name two CDs");
      gang_cd[g] = v;
      ++enrolled;
    }
  }
  e->im_cd.assign(cd, cd + n_cliques); e->im_gang_cd = std::move(gang_cd); e->im_owner0.assign(owner0, owner0 + n_nodes);
  e->im_enrolled = enrolled; e->im_given = true;
  return GROVE_OK;
}

int32_t grove_get_compute_domain_owners(grove_engine_t* e, uint32_t* out, uint32_t cap) {
  if (!e || !out) return GROVE_ERR_INVALID_ARG;
  if (!e->im_have_owners) return fail(e, GROVE_ERR_STATE, "grove_get_compute_domain_owners: no cycle has run with a ComputeDomain set");
  if (cap < e->im_owners.size()) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  std::copy(e->im_owners.begin(), e->im_owners.end(), out);
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// Queue limits (include/grove_place.h "queue limits"; DESIGN.md section 1; kernels in queue.cuh).  Validated against the submission;
// the tables the kernels read are built here once: the members in rank order with their chains and R_min, the queues with a
// finite limit with limit - load, and the (queue, member) pairs sorted by (queue, rank).
// ---------------------------------------------------------------------------------------------
static int32_t install_queues(grove_engine* e, const grove_queue_t* queues, uint32_t n_queues, const uint32_t* gang_queue);

int32_t grove_set_queues(grove_engine_t* e, const grove_queue_t* queues, uint32_t n_queues, const uint32_t* gang_queue, uint32_t n_gangs) {
  if (!e) return GROVE_ERR_INVALID_ARG;
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  if (!e->nodes_loaded || !e->gangs_loaded) return fail(e, GROVE_ERR_STATE, "grove_set_queues: load nodes and submit gangs first");
  if ((n_queues && !queues) || (n_gangs && !gang_queue)) return GROVE_ERR_INVALID_ARG;
  if (n_gangs != e->G) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_queues: n_gangs is not the number of submitted gangs");
  if (n_queues > GROVE_MAX_QUEUES) return fail(e, GROVE_ERR_LIMIT, "grove_set_queues: more than GROVE_MAX_QUEUES queues");
  if (e->wide) return refuse_wide(e, "grove_set_queues");
  std::vector<uint32_t> depth(n_queues, 1);
  for (uint32_t q = 0; q < n_queues; ++q) {
    const uint32_t p = queues[q].parent;
    if (p == GROVE_NONE_U32) continue;
    if (p >= q) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_queues: a parent must come before its queue");
    depth[q] = depth[p] + 1;
    if (depth[q] > GROVE_MAX_QUEUE_DEPTH) return fail(e, GROVE_ERR_LIMIT, "grove_set_queues: a chain deeper than GROVE_MAX_QUEUE_DEPTH");
  }
  for (uint32_t g = 0; g < n_gangs; ++g)
    if (gang_queue[g] != GROVE_NONE_U32 && gang_queue[g] >= n_queues) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_queues: queue index out of range");
  e->qu_given = false; e->fs_given = false; e->fs_have_order = false;
  const int32_t rc = install_queues(e, queues, n_queues, gang_queue);
  if (rc) return rc;
  e->qu_queues.assign(queues, queues + n_queues);
  e->qu_gang_queue.assign(gang_queue, gang_queue + n_gangs);
  e->qu_given = true;
  return GROVE_OK;
}

// The tables of a queue set (checked by grove_set_queues) over the current submission; also the per-class sets of
// grove_run_cycle_preempt_queues, whose `used` make the loads equal load'.
static int32_t install_queues(grove_engine* e, const grove_queue_t* queues, uint32_t n_queues, const uint32_t* gang_queue) {
  e->qu_members = e->qu_scanned = 0;
  // load = own used + the descendants' (parents come first: one pass from the back), saturating; limit - load in signed 64 bits,
  // both clamped to 2^62 (no gang asks for that much, so no decision changes)
  constexpr uint64_t kClamp = uint64_t(1) << 62;
  std::vector<uint64_t> load(size_t(n_queues) * 3);
  for (uint32_t q = 0; q < n_queues; ++q) for (int r = 0; r < 3; ++r) load[q * 3 + r] = std::min(queues[q].used[r], kClamp);
  for (uint32_t q = n_queues; q-- > 0;)
    if (queues[q].parent != GROVE_NONE_U32)
      for (int r = 0; r < 3; ++r) load[queues[q].parent * 3 + r] = std::min(load[queues[q].parent * 3 + r] + load[q * 3 + r], kClamp);
  std::vector<uint32_t> scan_id(n_queues, GROVE_NONE_U32);   // the queues with a finite limit, renumbered
  std::vector<long long> q_base;
  uint32_t scanned = 0;
  for (uint32_t q = 0; q < n_queues; ++q) {
    bool fin = false;
    for (int r = 0; r < 3; ++r) fin |= queues[q].limit[r] != GROVE_QUEUE_UNLIMITED;
    if (!fin) continue;
    scan_id[q] = scanned++;
    for (int r = 0; r < 3; ++r)
      q_base.push_back(queues[q].limit[r] == GROVE_QUEUE_UNLIMITED ? 0ll : (long long)std::min(queues[q].limit[r], kClamp) - (long long)load[q * 3 + r]);
  }
  // members in rank order; a gang whose chain has no finite limit is not one (it would behave as a non-member anyway)
  const uint32_t G = e->G;
  std::vector<uint32_t> order(G);
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), [e](uint32_t a, uint32_t b) { return e->gangs[a].priority > e->gangs[b].priority; });
  std::vector<uint32_t> slot(G, GROVE_NONE_U32), mem, mem_fin, chains, q_off(scanned + 1, 0);
  std::vector<long long> rmin;
  for (uint32_t g : order) {
    if (gang_queue[g] == GROVE_NONE_U32) continue;
    uint32_t chain[GROVE_MAX_QUEUE_DEPTH] = {GROVE_NONE_U32, GROVE_NONE_U32, GROVE_NONE_U32, GROVE_NONE_U32}, n = 0, fin = 0;
    for (uint32_t q = gang_queue[g]; q != GROVE_NONE_U32; q = queues[q].parent) {
      if (scan_id[q] == GROVE_NONE_U32) continue;
      for (int r = 0; r < 3; ++r) if (queues[q].limit[r] != GROVE_QUEUE_UNLIMITED) fin |= 1u << (3 * n + r);
      ++q_off[scan_id[q] + 1];
      chain[n++] = scan_id[q];
    }
    if (!n) continue;
    slot[g] = uint32_t(mem.size()); mem.push_back(g); mem_fin.push_back(fin);
    chains.insert(chains.end(), chain, chain + GROVE_MAX_QUEUE_DEPTH);
    const grove_gang_t& gg = e->gangs[g];
    long long R[3] = {0, 0, 0};
    for (uint32_t c = 0; c < gg.n_cliques; ++c) {
      const grove_clique_t& q = e->cliques[gg.clique_off + c];
      R[0] += (long long)q.min_replicas * q.req_cpu_milli; R[1] += (long long)q.min_replicas * q.req_mem_mib; R[2] += (long long)q.min_replicas * q.req_gpu;
    }
    rmin.insert(rmin.end(), R, R + 3);
  }
  if (mem.empty()) return GROVE_OK;   // nothing to limit: the ordinary cycle
  for (uint32_t q = 0; q < scanned; ++q) q_off[q + 1] += q_off[q];
  // the pairs: members are taken in rank order, so each queue's pairs come out in rank order
  std::vector<uint32_t> fill(q_off.begin(), q_off.end() - 1);
  // the rank of every gang.  GangInfo::order is only built when the cycle starts (build_ginfo); it is the same order --
  // priority desc, then submission index asc, which this stable sort over the submission gives -- and k_queue_scan's bound test
  // (pr.z) and k_queue_gate's (GangInfo::order) rely on the two being equal
  std::vector<uint32_t> rank_of(G);
  for (uint32_t k = 0; k < G; ++k) rank_of[order[k]] = k;
  std::vector<uint4> pr_list(q_off[scanned]);
  std::vector<uint4> mem_pair(mem.size());
  for (size_t j = 0; j < mem.size(); ++j) {
    uint32_t pr[GROVE_MAX_QUEUE_DEPTH];
    for (uint32_t k = 0; k < GROVE_MAX_QUEUE_DEPTH; ++k) {
      const uint32_t q = chains[j * GROVE_MAX_QUEUE_DEPTH + k];
      pr[k] = q == GROVE_NONE_U32 ? GROVE_NONE_U32 : fill[q]++;
      if (q != GROVE_NONE_U32) pr_list[pr[k]] = make_uint4(mem[j], uint32_t(j), rank_of[mem[j]], 0u);
    }
    mem_pair[j] = make_uint4(pr[0], pr[1], pr[2], pr[3]);
  }
  const uint32_t M = uint32_t(mem.size()), P = q_off[scanned];
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  auto up = [e](auto& d, const auto& h) -> cudaError_t {
    cudaError_t c = d.ensure(std::max<size_t>(h.size(), 1));
    if (c == cudaSuccess && !h.empty()) c = cudaMemcpyAsync(d.p, h.data(), sizeof(h[0]) * h.size(), cudaMemcpyHostToDevice, e->stream);
    return c;
  };
  CU_TRY(e, up(e->d_qu_slot, slot)); CU_TRY(e, up(e->d_qu_mem, mem)); CU_TRY(e, up(e->d_qu_mem_pair, mem_pair)); CU_TRY(e, up(e->d_qu_mem_fin, mem_fin));
  CU_TRY(e, up(e->d_qu_rmin, rmin)); CU_TRY(e, up(e->d_qu_q_off, q_off)); CU_TRY(e, up(e->d_qu_q_base, q_base)); CU_TRY(e, up(e->d_qu_pr, pr_list));
  CU_TRY(e, e->d_qu_head.ensure(size_t(P) * 3)); CU_TRY(e, e->d_qu_use.ensure(size_t(M) * 3));
  CU_TRY(e, e->d_qu_gate.ensure(M)); CU_TRY(e, e->d_qu_cap.ensure(std::max<uint32_t>(e->Q, 1)));
  CU_TRY(e, cudaStreamSynchronize(e->stream));   // (the host vectors go out of scope)
  e->qu_members = M; e->qu_scanned = scanned;
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// Diagnosis (include/grove_place.h "diagnosis of rejected gangs"; DESIGN.md section 1; kernels in diagnose.cuh).  Reads the
// outputs of the last ordinary cycle on the device (committed table, placements, ranks) and writes only its own buffers.
// ---------------------------------------------------------------------------------------------
// Rejected gangs go through the kernels in batches whose per-(gang, clique, domain) capacity sums take at most this many
// 8-byte columns (64 MB); a gang that needs more on its own (32 cliques x 262 144 domains) is a batch of its own.
static constexpr size_t kDiagScratchCols = size_t(1) << 23;

int32_t grove_diagnose(grove_engine_t* e, grove_gang_diag_t* gangs, uint32_t cap_g, grove_clique_diag_t* cliques, uint32_t cap_q) {
  if (!e) return GROVE_ERR_INVALID_ARG;
  switch (e->diag) {
    case grove_engine::kDiagReady: break;
    case grove_engine::kDiagNoCycle: return fail(e, GROVE_ERR_STATE, "grove_diagnose: no completed cycle");
    case grove_engine::kDiagRunning:
      return fail(e, GROVE_ERR_STATE, "grove_diagnose: the last cycle ran with running gangs (preempt / reuse); only grove_run_cycle is diagnosed");
    case grove_engine::kDiagSpread:
      return fail(e, GROVE_ERR_STATE, "grove_diagnose: the last cycle had topology spread members, which the diagnosis does not model");
    case grove_engine::kDiagFence:
      return fail(e, GROVE_ERR_STATE, "grove_diagnose: the last cycle had fences, which the diagnosis does not model");
    case grove_engine::kDiagImex:
      return fail(e, GROVE_ERR_STATE, "grove_diagnose: the last cycle had enrolled cliques (ComputeDomains), which the diagnosis does not model");
    case grove_engine::kDiagFairShare:
      return fail(e, GROVE_ERR_STATE, "grove_diagnose: the last cycle ran in fair-share order, which the diagnosis does not model");
    default: return fail(e, GROVE_ERR_STATE, "grove_diagnose: nodes or gangs were loaded, updated or submitted since the last cycle");
  }
  const uint32_t G = e->G, Q = e->Q;
  if ((G && !gangs) || (Q && !cliques)) return GROVE_ERR_INVALID_ARG;
  if (cap_g < G || cap_q < Q) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  if (G) std::memset(gangs, 0, sizeof(grove_gang_diag_t) * G);
  if (Q) std::memset(cliques, 0, sizeof(grove_clique_diag_t) * Q);
  // the rejected gangs, in batches
  std::vector<DiagGang> dg;
  std::vector<uint32_t> batch_at{0};
  std::vector<size_t> batch_cols{0};
  for (uint32_t g = 0; g < G; ++g) {
    if (e->h_status.p[g].state != GROVE_GANG_REJECTED || (e->h_status.p[g].reserved0 & GROVE_STATUS_OVER_LIMIT)) continue;
    const grove_gang_t& x = e->gangs[g];
    DiagGang d{};
    d.gang = g; d.rank = e->ginfo[g].order; d.n_cliques = x.n_cliques; d.level = x.level;
    d.ncol = x.level == GROVE_LEVEL_NONE ? 1u : e->n_dom[x.level];
    const size_t need = size_t(x.n_cliques) * d.ncol;
    const uint32_t in_batch = uint32_t(dg.size()) - batch_at.back();
    if (in_batch && (batch_cols.back() + need > kDiagScratchCols || in_batch == 65535u)) { batch_at.push_back(uint32_t(dg.size())); batch_cols.push_back(0); }
    d.col_off = uint32_t(batch_cols.back());
    batch_cols.back() += need;
    dg.push_back(d);
  }
  batch_at.push_back(uint32_t(dg.size()));
  if (dg.empty()) return GROVE_OK;
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  const uint32_t Np = e->Npad, n_out = e->n_out;
  CU_TRY(e, e->d_dg_gout.ensure(G)); CU_TRY(e, e->d_dg_qout.ensure(Q)); CU_TRY(e, e->d_dg_minr.ensure(Q));
  CU_TRY(e, e->d_dg_cnt.ensure(Np)); CU_TRY(e, e->d_dg_off.ensure(size_t(Np) + 1)); CU_TRY(e, e->d_dg_cur.ensure(Np));
  CU_TRY(e, e->d_dg_rec.ensure(std::max<uint32_t>(n_out, 1))); CU_TRY(e, e->d_dg_gang.ensure(dg.size()));
  CU_TRY(e, e->d_dg_col.ensure(std::max<size_t>(*std::max_element(batch_cols.begin(), batch_cols.end()), 1)));
  CU_TRY(e, cudaMemsetAsync(e->d_dg_gout.p, 0, sizeof(grove_gang_diag_t) * G, e->stream));
  CU_TRY(e, cudaMemsetAsync(e->d_dg_qout.p, 0, sizeof(grove_clique_diag_t) * Q, e->stream));
  CU_TRY(e, cudaMemsetAsync(e->d_dg_cnt.p, 0, sizeof(uint32_t) * Np, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_dg_minr.p, e->ccount.data(), sizeof(uint32_t) * Q, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_dg_gang.p, dg.data(), sizeof(DiagGang) * dg.size(), cudaMemcpyHostToDevice, e->stream));
  const Topo tp = make_topo(e); const Tables tb = make_tables(e);
  // the admitted gangs' usage per node, in rank order with suffix sums
  if (n_out) k_diag_count<<<(n_out + 255) / 256, 256, 0, e->stream>>>(e->d_out.p, n_out, e->d_inv.p, e->d_dg_cnt.p);
  k_diag_scan<<<1, 1024, 0, e->stream>>>(e->d_dg_cnt.p, e->d_dg_off.p, e->d_dg_cur.p, Np);
  if (n_out) k_diag_fill<<<(n_out + 255) / 256, 256, 0, e->stream>>>(e->d_out.p, n_out, e->d_inv.p, tb, e->d_dg_off.p, e->d_dg_cur.p, e->d_dg_rec.p);
  k_diag_suffix<<<(e->N + 255) / 256, 256, 0, e->stream>>>(e->d_dg_off.p, e->d_dg_rec.p, e->N);
  CU_TRY(e, cudaGetLastError());
  const DiagUse use{e->d_dg_off.p, e->d_dg_rec.p};
  for (size_t b = 0; b + 1 < batch_at.size(); ++b) {
    const uint32_t a = batch_at[b], nb = batch_at[b + 1] - a;
    if (batch_cols[b]) CU_TRY(e, cudaMemsetAsync(e->d_dg_col.p, 0, sizeof(unsigned long long) * batch_cols[b], e->stream));
    k_diag_fit<<<dim3(Np / 256, nb), 256, 0, e->stream>>>(tp, tb, use, e->d_dg_gang.p + a, e->d_dg_minr.p, e->d_dg_col.p, e->d_dg_qout.p);
    k_diag_verdict<<<nb, 256, 0, e->stream>>>(tb, e->d_dg_gang.p + a, e->d_dg_minr.p, e->d_dg_col.p, e->d_dg_qout.p, e->d_dg_gout.p);
    CU_TRY(e, cudaGetLastError());
  }
  CU_TRY(e, cudaMemcpyAsync(gangs, e->d_dg_gout.p, sizeof(grove_gang_diag_t) * G, cudaMemcpyDeviceToHost, e->stream));
  CU_TRY(e, cudaMemcpyAsync(cliques, e->d_dg_qout.p, sizeof(grove_clique_diag_t) * Q, cudaMemcpyDeviceToHost, e->stream));
  CU_TRY(e, cudaStreamSynchronize(e->stream));
  return GROVE_OK;
}

// K2 over the snapshot the last cycle started from: T[q][n] = fit ? 1 + closeness(n, anchor of q's gang) : 0.  The admission
// derives its visiting order from the anchor's ancestor ranges and never reads this matrix, so it is materialised on
// request (a scheduler that wants per-node scores -- the Score extension point -- asks for it); GROVE_TUNE_SCORE=1 builds
// it every cycle instead, on a second stream beside the relaxation.  *ms (nullable) = device time of the kernel.
int32_t grove_build_score_matrix(grove_engine_t* e, float* ms) {
  if (!e) return GROVE_ERR_INVALID_ARG;
  if (!e->have_results) return fail(e, GROVE_ERR_STATE, "no completed cycle");
  if (ms) *ms = 0.f;
  if (e->Q == 0) return GROVE_OK;
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  if (e->score_valid && !ms) return GROVE_OK;
  if (e->d_T.ensure(size_t(e->Q) * e->Npad) != cudaSuccess) { (void)cudaGetLastError(); return fail(e, GROVE_ERR_OOM, "score matrix does not fit in device memory"); }
  const Topo tp = make_topo(e); const Tables tb = make_tables(e);
  CU_TRY(e, cudaEventRecord(e->ev_s0, e->stream));
  k_score<<<dim3(1, std::min<uint32_t>(e->Q, 65535u)), 256, 0, e->stream>>>(tp, tb, e->d_F0.p, e->d_T.p, e->Q, 0u, e->Npad >> 4, size_t(e->Npad));  // one CTA per row
  CU_TRY(e, cudaGetLastError());
  CU_TRY(e, cudaEventRecord(e->ev_s1, e->stream));
  CU_TRY(e, cudaEventSynchronize(e->ev_s1));
  float t = 0; cudaEventElapsedTime(&t, e->ev_s0, e->ev_s1);
  e->last.ms_score = t; e->score_valid = true;
  if (ms) *ms = t;
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// Reclaim pass (include/grove_place.h "preemption / reclaim"; DESIGN.md section 1).  Host orchestration around the same
// device path: the gangs the ordinary pass rejected are re-submitted priority class by priority class (descending) against
// the reclaim view of that class -- the evaluation of a gang does not depend on WHICH running gangs end up evicted, only on
// what is free plus what is evictable, so a whole class is one ordinary cycle on the augmented node table; the victims
// are then chosen gang by gang in order, exactly as the sequential statement says.  reclaim_cycle (below) runs that loop for
// the three reclaim entries; consolidation runs its own over the same pieces, which come first.
// ---------------------------------------------------------------------------------------------
namespace {
struct Res {   // resources on one node: a free-table row, a usage or a change
  int64_t cpu = 0, mem = 0, gpu = 0, pods = 0;
  bool covers(const Res& r) const { return cpu >= r.cpu && mem >= r.mem && gpu >= r.gpu && pods >= r.pods; }
  void add(const Res& r, int64_t k = 1) { cpu += k * r.cpu; mem += k * r.mem; gpu += k * r.gpu; pods += k * r.pods; }
};
inline Res held(const grove_holding_t& h) { return Res{h.cpu_milli, h.mem_mib, h.gpu, h.pods}; }

// the caller's submission and the outputs of the ordinary pass (the handle is re-used for the sub-cycles)
struct Snapshot {
  std::vector<grove_gang_t> gangs; std::vector<grove_clique_t> cliques; std::vector<grove_scope_t> scopes;
  std::vector<grove_gang_status_t> status; std::vector<grove_placement_t> place; std::vector<grove_scope_status_t> sstat;
};

// Whatever goes wrong while armed, the handle goes back to the caller's submission, and queue set when one was given (queues
// non-null), on the free table the ordinary pass left, kept in d_rc_base; the error of the failing call is what the caller sees.
// put_back() alone is the normal end: the device table is then the free table as it is.
struct Restore {
  grove_engine* e; const Snapshot* s; const std::vector<grove_queue_t>* queues; const std::vector<uint32_t>* gang_queue;
  bool armed = true;
  int32_t put_back() const {
    int32_t rc = grove_submit_gangs(e, s->gangs.data(), uint32_t(s->gangs.size()), s->cliques.data(), uint32_t(s->cliques.size()),
                                    s->scopes.data(), uint32_t(s->scopes.size()));
    if (rc || !queues) return rc;
    // (after the submission, which clears the queue set)
    rc = install_queues(e, queues->data(), uint32_t(queues->size()), gang_queue->data());
    if (rc) return rc;
    e->qu_queues = *queues; e->qu_gang_queue = *gang_queue; e->qu_given = true;
    return GROVE_OK;
  }
  ~Restore() {
    if (!armed) return;
    const std::string keep = e->err;
    cudaMemcpyAsync(e->d_nres.p, e->d_rc_base.p, sizeof(uint4) * e->Npad, cudaMemcpyDeviceToDevice, e->stream);
    cudaStreamSynchronize(e->stream);
    put_back();
    e->err = keep;
  }
};

// a sub-submission of some of the caller's gangs: its gang k is the caller's ids[k]
struct Sub {
  std::vector<uint32_t> ids;
  std::vector<grove_gang_t> gangs; std::vector<grove_clique_t> cliques; std::vector<grove_scope_t> scopes;
};

// the running gangs on each node (caller order) as a CSR: run[off[n] .. off[n + 1]), running gangs ascending
struct RunningByNode { std::vector<uint32_t> off, run; };
}  // namespace

// the running gangs' inputs: every holding range inside `holdings`, every holding on a node of the snapshot
static int32_t check_running(grove_engine* e, const grove_running_gang_t* running, uint32_t n_running, const grove_holding_t* holdings,
                             uint32_t n_holdings) {
  for (uint32_t r = 0; r < n_running; ++r)
    if (uint64_t(running[r].holding_off) + running[r].n_holdings > n_holdings) return fail(e, GROVE_ERR_INVALID_ARG, "running gang holdings out of range");
  for (uint32_t h = 0; h < n_holdings; ++h)
    if (holdings[h].node >= e->N) return fail(e, GROVE_ERR_INVALID_ARG, "holding on a node out of range");
  return GROVE_OK;
}

// cpu, mem, gpu summed over a running gang's holdings
static std::array<int64_t, 3> usage_of(const grove_running_gang_t& r, const grove_holding_t* holdings) {
  std::array<int64_t, 3> u{0, 0, 0};
  for (uint32_t h = 0; h < r.n_holdings; ++h) {
    const grove_holding_t& x = holdings[r.holding_off + h];
    u[0] += x.cpu_milli; u[1] += x.mem_mib; u[2] += x.gpu;
  }
  return u;
}

static int32_t snapshot(grove_engine* e, Snapshot* s) {
  const uint32_t G = e->G, Q = e->Q, S = e->S;
  s->gangs.assign(e->gangs.data(), e->gangs.data() + G);
  s->cliques.assign(e->cliques.data(), e->cliques.data() + Q);
  s->scopes.assign(e->scopes.data(), e->scopes.data() + S);
  s->status.assign(e->h_status.p, e->h_status.p + G);
  s->place.assign(e->h_out.p, e->h_out.p + e->n_out);
  s->sstat.assign(std::max<uint32_t>(S, 1), grove_scope_status_t{});
  return S ? grove_get_scope_domains(e, s->sstat.data(), S) : GROVE_OK;
}

static RunningByNode running_by_node(uint32_t N, const grove_running_gang_t* running, uint32_t n_running, const grove_holding_t* holdings) {
  RunningByNode at;
  size_t n_held = 0;   // (ranges of running gangs may overlap: size by what the fill below writes)
  for (uint32_t r = 0; r < n_running; ++r) n_held += running[r].n_holdings;
  at.off.assign(size_t(N) + 1, 0); at.run.resize(n_held);
  for (uint32_t r = 0; r < n_running; ++r) for (uint32_t h = 0; h < running[r].n_holdings; ++h) ++at.off[holdings[running[r].holding_off + h].node + 1];
  for (uint32_t n = 0; n < N; ++n) at.off[n + 1] += at.off[n];
  std::vector<uint32_t> cur(at.off.begin(), at.off.end() - 1);
  for (uint32_t r = 0; r < n_running; ++r) for (uint32_t h = 0; h < running[r].n_holdings; ++h) at.run[cur[holdings[running[r].holding_off + h].node]++] = r;
  return at;
}

// the victim rule: lowest priority first, then the highest running index.  Does running gang x go before v (GROVE_NONE_U32: none)?
static bool evicted_before(const grove_running_gang_t* running, uint32_t x, uint32_t v) {
  return v == GROVE_NONE_U32 || running[x].priority < running[v].priority || (running[x].priority == running[v].priority && x > v);
}

// the victim among the running gangs on node n that `eligible` admits, GROVE_NONE_U32 when there is none
static uint32_t choose_victim(const RunningByNode& at, uint32_t n, const grove_running_gang_t* running,
                              const std::function<bool(uint32_t)>& eligible) {
  uint32_t v = GROVE_NONE_U32;
  for (uint32_t a = at.off[n]; a < at.off[n + 1]; ++a)
    if (eligible(at.run[a]) && evicted_before(running, at.run[a], v)) v = at.run[a];
  return v;
}

// gang g of the caller's submission appended to a sub-submission: anchor pinned to the one the ordinary pass derived, no gating (a
// rejected gang's base gang, if any, was admitted before it), cliques and scopes rebased -> the appended record
static grove_gang_t& add_gang(grove_engine* e, const Snapshot& s, uint32_t g, Sub& sub) {
  const grove_gang_t& o = s.gangs[g];
  grove_gang_t x = o;
  if (x.anchor_node == GROVE_NONE_U32) x.anchor_node = e->perm[fmix32(g) % e->N];
  x.base_gang = GROVE_NONE_U32;
  x.clique_off = uint32_t(sub.cliques.size()); x.scope_off = uint32_t(sub.scopes.size());
  sub.cliques.insert(sub.cliques.end(), s.cliques.begin() + o.clique_off, s.cliques.begin() + o.clique_off + o.n_cliques);
  sub.scopes.insert(sub.scopes.end(), s.scopes.begin() + o.scope_off, s.scopes.begin() + o.scope_off + o.n_scopes);
  sub.ids.push_back(g); sub.gangs.push_back(x);
  return sub.gangs.back();
}

static int32_t submit_sub(grove_engine* e, const Sub& sub) {
  return grove_submit_gangs(e, sub.gangs.data(), uint32_t(sub.gangs.size()), sub.cliques.data(), uint32_t(sub.cliques.size()),
                            sub.scopes.data(), uint32_t(sub.scopes.size()));
}

// the scope domains of the sub-cycle just run
static int32_t sub_scope_domains(grove_engine* e, const Sub& sub, std::vector<grove_scope_status_t>& out) {
  out.assign(std::max<size_t>(sub.scopes.size(), 1), grove_scope_status_t{});
  return sub.scopes.empty() ? GROVE_OK : grove_get_scope_domains(e, out.data(), uint32_t(sub.scopes.size()));
}

// a sub-cycle's stats added to the call's
static void accumulate(grove_cycle_stats_t& st0, const grove_cycle_stats_t& s) {
  st0.rounds += s.rounds; st0.evaluations += s.evaluations; st0.kernel_launches += s.kernel_launches;
  st0.ms_fit += s.ms_fit; st0.ms_admit += s.ms_admit; st0.ms_commit += s.ms_commit; st0.ms_total += s.ms_total;
}

// the rows of the free table kept aside in d_rc_real at these nodes (caller order)
static int32_t read_rows(grove_engine* e, const std::vector<uint32_t>& nodes, std::vector<Res>& rows, grove_cycle_stats_t& st) {
  rows.assign(nodes.size(), Res{});
  if (nodes.empty()) return GROVE_OK;
  std::vector<uint32_t> idx(nodes.size());
  for (size_t i = 0; i < nodes.size(); ++i) idx[i] = e->inv[nodes[i]];
  std::vector<uint4> got(idx.size());
  CU_TRY(e, e->d_rc_idx.ensure(idx.size())); CU_TRY(e, e->d_rc_rows.ensure(idx.size()));
  CU_TRY(e, cudaMemcpyAsync(e->d_rc_idx.p, idx.data(), sizeof(uint32_t) * idx.size(), cudaMemcpyHostToDevice, e->stream));
  k_reclaim_rows<<<uint32_t((idx.size() + 255) / 256), 256, 0, e->stream>>>(e->d_rc_real.p, e->d_rc_idx.p, e->d_rc_rows.p, uint32_t(idx.size()));
  CU_TRY(e, cudaGetLastError());
  CU_TRY(e, cudaMemcpyAsync(got.data(), e->d_rc_rows.p, sizeof(uint4) * got.size(), cudaMemcpyDeviceToHost, e->stream));
  CU_TRY(e, cudaStreamSynchronize(e->stream));
  for (size_t i = 0; i < got.size(); ++i) rows[i] = Res{got[i].x, got[i].y, got[i].z & 0xFFFFu, got[i].z >> 16};
  st.kernel_launches += 1;
  return GROVE_OK;
}

// What the sub-cycle just run gave gang k of its sub-submission: its usage per node, nodes in the order its placement first names
// them, and its placements with the cliques numbered as in the caller's submission (appended to pl).
static void placed(grove_engine* e, const Snapshot& s, const Sub& sub, uint32_t k, std::vector<uint32_t>& nodes, std::vector<Res>& use,
                   std::vector<grove_placement_t>& pl) {
  const grove_gang_status_t& sp = e->h_status.p[k];
  const uint32_t off = s.gangs[sub.ids[k]].clique_off;
  for (uint32_t i = 0; i < sp.n_pods; ++i) {
    const grove_placement_t x = e->h_out.p[sp.placement_off + i];
    const grove_clique_t& q = sub.cliques[x.clique];
    const size_t j = size_t(std::find(nodes.begin(), nodes.end(), x.node) - nodes.begin());
    if (j == nodes.size()) { nodes.push_back(x.node); use.emplace_back(); }
    use[j].add(Res{q.req_cpu_milli, q.req_mem_mib, q.req_gpu, 1});
    pl.push_back(grove_placement_t{off + (x.clique - sub.gangs[k].clique_off), x.node});
  }
}

// gang k of a sub-submission, admitted, into the outputs of the caller's gang sub.ids[k]: status o (placement_off is assigned when
// the outputs are merged) and the scope domains ssp of the sub-cycle
static void merge_gang(Snapshot& s, const Sub& sub, uint32_t k, const grove_gang_status_t& o, const std::vector<grove_scope_status_t>& ssp) {
  const uint32_t g = sub.ids[k];
  s.status[g] = o;
  for (uint32_t si = 0; si < s.gangs[g].n_scopes; ++si) s.sstat[s.gangs[g].scope_off + si] = ssp[sub.gangs[k].scope_off + si];
}

// d = (sorted node, change) -> one record per node, added to the device's node table (reclaim.cuh k_reclaim_patch); nothing to do
// for an empty d
static int32_t patch_nodes(grove_engine* e, std::vector<std::pair<uint32_t, Res>>& d, grove_cycle_stats_t& st) {
  if (d.empty()) return GROVE_OK;
  std::sort(d.begin(), d.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  std::vector<uint4> patch;
  for (size_t i = 0; i < d.size();) {
    const uint32_t n = d[i].first;
    Res v;
    for (; i < d.size() && d[i].first == n; ++i) v.add(d[i].second);
    patch.push_back(make_uint4(n, uint32_t(v.cpu), uint32_t(v.mem), uint32_t(v.gpu + v.pods * 65536)));
  }
  CU_TRY(e, e->d_rc_patch.ensure(patch.size()));
  CU_TRY(e, cudaMemcpyAsync(e->d_rc_patch.p, patch.data(), sizeof(uint4) * patch.size(), cudaMemcpyHostToDevice, e->stream));
  k_reclaim_patch<<<uint32_t((patch.size() + 255) / 256), 256, 0, e->stream>>>(e->d_nres.p, e->d_rc_patch.p, uint32_t(patch.size()));
  CU_TRY(e, cudaGetLastError());
  st.kernel_launches += 1;
  return GROVE_OK;
}

// the outputs of a cycle with a reclaim or consolidation pass, merged: placements grouped by gang in submission order (those of a
// preemptor, a reclaimer, a consolidated target or a moved spec row from `extra`)
static int32_t publish_reclaim(grove_engine* e, std::vector<grove_gang_status_t>& status, const std::vector<grove_placement_t>& place,
                               const std::vector<std::vector<grove_placement_t>>& extra, const std::vector<grove_scope_status_t>& sstat,
                               grove_cycle_stats_t st0, std::vector<grove_victim_t> victims, grove_cycle_stats_t* stats) {
  const uint32_t G = e->G, S = e->S;
  CU_TRY(e, e->h_status.ensure(std::max<uint32_t>(G, 1))); CU_TRY(e, e->h_scope_status.ensure(std::max<uint32_t>(S, 1)));
  size_t total = 0;
  for (uint32_t g = 0; g < G; ++g) total += status[g].state == GROVE_GANG_ADMITTED ? status[g].n_pods : 0u;
  CU_TRY(e, e->h_out.ensure(std::max<size_t>(total, 1)));
  std::vector<grove_placement_t> merged; merged.reserve(total);
  for (uint32_t g = 0; g < G; ++g) {
    if (status[g].state != GROVE_GANG_ADMITTED) continue;
    const uint32_t off = uint32_t(merged.size());
    if (status[g].reserved0 & (GROVE_STATUS_PREEMPTOR | GROVE_STATUS_RECLAIMER | GROVE_STATUS_CONSOLIDATED | GROVE_STATUS_MOVED))
      merged.insert(merged.end(), extra[g].begin(), extra[g].end());
    else merged.insert(merged.end(), place.begin() + status[g].placement_off, place.begin() + status[g].placement_off + status[g].n_pods);
    status[g].placement_off = off;
  }
  std::memcpy(e->h_out.p, merged.data(), sizeof(grove_placement_t) * merged.size());
  std::memcpy(e->h_status.p, status.data(), sizeof(grove_gang_status_t) * G);
  if (S) std::memcpy(e->h_scope_status.p, sstat.data(), sizeof(grove_scope_status_t) * S);
  e->n_out = uint32_t(merged.size());
  st0.pods_bound = e->n_out;
  e->last = st0;
  e->victims = std::move(victims);
  e->have_results = true; e->have_scopes = true; e->score_valid = false;
  if (stats) *stats = st0;
  return GROVE_OK;
}

int32_t grove_get_victims(grove_engine_t* e, grove_victim_t* out, uint32_t cap, uint32_t* n_out) {
  if (!e || !n_out) return GROVE_ERR_INVALID_ARG;
  if (!e->have_results) return fail(e, GROVE_ERR_STATE, "no completed cycle");
  *n_out = uint32_t(e->victims.size());
  if (!out) return GROVE_OK;
  if (cap < e->victims.size()) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  std::memcpy(out, e->victims.data(), sizeof(grove_victim_t) * e->victims.size());
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// Reservation reuse (include/grove_place.h "reservation reuse"; DESIGN.md section 1).  The host validates the inputs and turns the
// predecessors' holdings into one hold record per (replacement gang, node), in sorted node order; the ordinary cycle then runs with
// the holds (relax.cuh k_hold_publish / k_fold / k_hold_release).
// ---------------------------------------------------------------------------------------------
// the inputs of a cycle with replacements (grove_run_cycle_reuse, grove_run_cycle_reuse_preempt)
static int32_t check_reuse_inputs(grove_engine* e, const uint32_t* replaces, uint32_t n_gangs, const grove_running_gang_t* running,
                                  uint32_t n_running, const grove_holding_t* holdings, uint32_t n_holdings) {
  int32_t rc = check_ready(e);
  if (rc) return rc;
  if (n_gangs != e->G) return fail(e, GROVE_ERR_INVALID_ARG, "replaces must have one entry per submitted gang");
  rc = check_running(e, running, n_running, holdings, n_holdings);
  if (rc) return rc;
  std::vector<uint8_t> taken(n_running, 0);
  for (uint32_t g = 0; g < n_gangs; ++g) {
    const uint32_t r = replaces[g];
    if (r == GROVE_NONE_U32) continue;
    if (r >= n_running) return fail(e, GROVE_ERR_INVALID_ARG, "replaces names a running gang out of range");
    if (taken[r]) return fail(e, GROVE_ERR_INVALID_ARG, "a running gang is replaced by more than one gang");
    taken[r] = 1;
  }
  return GROVE_OK;
}

// The cycle over the submitted gangs in which gang g with replaces[g] != GROVE_NONE_U32 holds what that running gang holds
// (inputs checked by check_reuse_inputs); with no hold at all, the ordinary cycle.  check_fit: first make sure that free plus every
// hold fits the node record's fields.
static int32_t run_cycle_holds(grove_engine* e, const uint32_t* replaces, const grove_running_gang_t* running, const grove_holding_t* holdings,
                               bool check_fit, grove_cycle_stats_t* stats) {
  const uint32_t n_gangs = e->G;
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  // one record per (gang, node): x = sorted node, then cpu, mem, gpu, pods summed over the predecessor's holdings there
  struct Rec { uint32_t node; uint64_t v[4]; };
  std::vector<uint32_t> off(size_t(n_gangs) + 1, 0);
  std::vector<Rec> recs;
  for (uint32_t g = 0; g < n_gangs; ++g) {
    off[g] = uint32_t(recs.size());
    const uint32_t r = replaces[g];
    if (r == GROVE_NONE_U32) continue;
    const size_t first = recs.size();
    for (uint32_t k = 0; k < running[r].n_holdings; ++k) {
      const grove_holding_t& h = holdings[running[r].holding_off + k];
      recs.push_back(Rec{e->inv[h.node], {h.cpu_milli, h.mem_mib, h.gpu, h.pods}});
    }
    std::sort(recs.begin() + first, recs.end(), [](const Rec& a, const Rec& b) { return a.node < b.node; });
    size_t w = first;
    for (size_t i = first; i < recs.size(); ++i) {
      if (w > first && recs[w - 1].node == recs[i].node) { for (int k = 0; k < 4; ++k) recs[w - 1].v[k] += recs[i].v[k]; }
      else recs[w++] = recs[i];
    }
    recs.resize(w);
  }
  if (recs.empty()) return run_cycle(e, stats);
  off[n_gangs] = uint32_t(recs.size());
  // the free table plus every hold must fit the node record's fields
  if (check_fit) {
    std::vector<uint4> nres(e->Npad);
    CU_TRY(e, cudaMemcpyAsync(nres.data(), e->d_nres.p, sizeof(uint4) * e->Npad, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(e, cudaStreamSynchronize(e->stream));
    std::vector<Rec> tot(recs);
    std::sort(tot.begin(), tot.end(), [](const Rec& a, const Rec& b) { return a.node < b.node; });
    for (size_t i = 0; i < tot.size();) {
      const uint32_t n = tot[i].node;
      uint64_t v[4] = {nres[n].x, nres[n].y, nres[n].z & 0xFFFFu, nres[n].z >> 16};
      for (; i < tot.size() && tot[i].node == n; ++i) for (int k = 0; k < 4; ++k) v[k] += tot[i].v[k];
      if (v[0] > UINT32_MAX || v[1] > UINT32_MAX || v[2] > UINT16_MAX || v[3] > UINT16_MAX)
        return fail(e, GROVE_ERR_INVALID_ARG, "free resources plus holdings overflow a field of a node record");
    }
  }
  std::vector<uint4> hold(recs.size());
  for (size_t i = 0; i < recs.size(); ++i)
    hold[i] = make_uint4(recs[i].node, uint32_t(recs[i].v[0]), uint32_t(recs[i].v[1]), uint32_t(recs[i].v[2]) | (uint32_t(recs[i].v[3]) << 16));
  CU_TRY(e, e->d_hold_off.ensure(off.size())); CU_TRY(e, e->d_hold.ensure(hold.size()));
  CU_TRY(e, cudaMemcpyAsync(e->d_hold_off.p, off.data(), sizeof(uint32_t) * off.size(), cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_hold.p, hold.data(), sizeof(uint4) * hold.size(), cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaStreamSynchronize(e->stream));   // (pageable sources)
  struct HoldsOn { grove_engine* e; ~HoldsOn() { e->holds_on = false; e->n_hold = 0; } } holds_guard{e};
  e->holds_on = true; e->n_hold = uint32_t(recs.size());
  return run_cycle(e, stats);
}

int32_t grove_run_cycle_reuse(grove_engine_t* e, const uint32_t* replaces, uint32_t n_gangs, const grove_running_gang_t* running,
                              uint32_t n_running, const grove_holding_t* holdings, uint32_t n_holdings, grove_cycle_stats_t* stats) {
  if (!e || (n_gangs && !replaces) || (n_running && !running) || (n_holdings && !holdings)) return GROVE_ERR_INVALID_ARG;
  if (e->sp_members) return refuse_spread(e, "grove_run_cycle_reuse");
  if (e->qu_members) return refuse_queues(e, "grove_run_cycle_reuse");
  if (!e->fc_gangs.empty()) return refuse_fences(e, "grove_run_cycle_reuse");
  if (e->bp_members) return refuse_binpack(e, "grove_run_cycle_reuse");
  if (e->im_enrolled) return refuse_imex(e, "grove_run_cycle_reuse");
  NoDiagnosis no_diag{e};
  if (e->wide) return refuse_wide(e, "grove_run_cycle_reuse");
  const int32_t rc = check_reuse_inputs(e, replaces, n_gangs, running, n_running, holdings, n_holdings);
  if (rc) return rc;
  return run_cycle_holds(e, replaces, running, holdings, true, stats);
}

// ---------------------------------------------------------------------------------------------
// The reclaim loop of grove_run_cycle_preempt, grove_run_cycle_reuse_preempt and grove_run_cycle_preempt_queues (include/grove_place.h
// "preemption / reclaim", "reuse with reclaim", "reclaim within queue limits"; DESIGN.md section 1).  The ordinary pass is the cycle
// with holds.  Then every priority class of the gangs it rejected is ONE cycle with holds (the members whose predecessor ranks at
// or above the class hold what it holds) over the class view, which reclaim.cuh builds on the device from the running gangs'
// holdings: the free table plus whatever the standing running gangs of a lower priority hold.  Under a queue set the class cycle
// is a queue cycle with a set of its own, whose `used` leave out what the gangs of E(p) hold: its loads are load'; queue loads are
// followed here, between classes.  Victims are chosen on the host, gang by gang in rank order, over the rows of the nodes the
// class's preemptors use: the node step, then for a queue member the queue step.  Then the device takes the holdings of the
// running gangs still standing off the table again, which leaves the free table.
// ---------------------------------------------------------------------------------------------
// The running gangs of the reclaim loop and grove_run_cycle_consolidate on the device (reclaim.cuh): their holdings by
// sorted node, running gangs ascending within a row, and their priorities, uploaded once; the gone mask (one byte per running gang)
// is the caller's to upload.  Then the check that free plus every running gang's holdings fits the node record's fields: then so
// does every view built from them.
static int32_t upload_running(grove_engine* e, const grove_running_gang_t* running, uint32_t n_running, const grove_holding_t* holdings,
                              ReclaimCsr* csr) {
  const uint32_t N = e->N, nblk = (N + 255) / 256;
  std::vector<uint32_t> off(size_t(N) + 1, 0);
  for (uint32_t r = 0; r < n_running; ++r)
    for (uint32_t k = 0; k < running[r].n_holdings; ++k) ++off[e->inv[holdings[running[r].holding_off + k].node] + 1];
  for (uint32_t n = 0; n < N; ++n) off[n + 1] += off[n];
  std::vector<uint4> ent(std::max<uint32_t>(off[N], 1));
  {
    std::vector<uint32_t> cur(off.begin(), off.end() - 1);
    for (uint32_t r = 0; r < n_running; ++r)
      for (uint32_t k = 0; k < running[r].n_holdings; ++k) {
        const grove_holding_t& h = holdings[running[r].holding_off + k];
        ent[cur[e->inv[h.node]]++] = make_uint4(r, h.cpu_milli, h.mem_mib, uint32_t(h.gpu) | (uint32_t(h.pods) << 16));
      }
  }
  std::vector<int32_t> prio(std::max<uint32_t>(n_running, 1), 0);
  for (uint32_t r = 0; r < n_running; ++r) prio[r] = running[r].priority;
  CU_TRY(e, e->d_rc_off.ensure(off.size())); CU_TRY(e, e->d_rc_ent.ensure(ent.size())); CU_TRY(e, e->d_rc_bad.ensure(1));
  CU_TRY(e, e->d_rc_prio.ensure(prio.size())); CU_TRY(e, e->d_rc_gone.ensure(prio.size()));
  CU_TRY(e, e->d_rc_real.ensure(e->Npad)); CU_TRY(e, e->d_rc_base.ensure(e->Npad));
  CU_TRY(e, cudaMemcpyAsync(e->d_rc_off.p, off.data(), sizeof(uint32_t) * off.size(), cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_rc_ent.p, ent.data(), sizeof(uint4) * ent.size(), cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_rc_prio.p, prio.data(), sizeof(int32_t) * prio.size(), cudaMemcpyHostToDevice, e->stream));
  CU_TRY(e, cudaMemsetAsync(e->d_rc_bad.p, 0, sizeof(uint32_t), e->stream));
  *csr = ReclaimCsr{e->d_rc_off.p, e->d_rc_ent.p, e->d_rc_prio.p, e->d_rc_gone.p};
  k_reclaim_check<<<nblk, 256, 0, e->stream>>>(e->d_nres.p, *csr, N, e->d_rc_bad.p);
  CU_TRY(e, cudaGetLastError());
  uint32_t bad = 0;
  CU_TRY(e, cudaMemcpyAsync(&bad, e->d_rc_bad.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
  CU_TRY(e, cudaStreamSynchronize(e->stream));   // (pageable sources)
  if (bad) return fail(e, GROVE_ERR_INVALID_ARG, "free resources plus holdings overflow a field of a node record");
  return GROVE_OK;
}

// The donor sets of grove_run_cycle_reclaim_queues on the device (donor.cuh): the (scanned queue, running gang) pairs in victim
// order with the depth of the queue in the running gang's chain, and what k_donor_scan / k_donor_mark read besides, uploaded
// once per call.  -> the number of scanned queues (those with a finite quota on some resource); 0: every E(Q) is empty.
static int32_t upload_donors(grove_engine* e, const grove_running_gang_t* running, uint32_t n_running, const uint32_t* run_queue,
                             const std::vector<grove_queue_t>& queues, const grove_queue_quota_t* quotas,
                             const std::vector<std::array<int64_t, 3>>& usage, uint32_t* scanned, DonorSet* d) {
  const uint32_t NQ = uint32_t(queues.size());
  std::vector<uint32_t> scan_id(NQ, GROVE_NONE_U32), q_id, parent(std::max<uint32_t>(NQ, 1), GROVE_NONE_U32);
  std::vector<uint8_t> fin(std::max<uint32_t>(NQ, 1), 0);
  std::vector<unsigned long long> quota(std::max<size_t>(size_t(NQ) * 3, 1), GROVE_QUEUE_UNLIMITED);
  for (uint32_t q = 0; q < NQ; ++q) {
    parent[q] = queues[q].parent;
    for (int k = 0; k < 3; ++k) { quota[q * 3 + k] = quotas[q].deserved[k]; fin[q] |= quotas[q].deserved[k] != GROVE_QUEUE_UNLIMITED; }
    if (fin[q]) { scan_id[q] = uint32_t(q_id.size()); q_id.push_back(q); }
  }
  *scanned = uint32_t(q_id.size());
  if (!*scanned || !n_running) { *scanned = 0; return GROVE_OK; }
  // the running gangs in victim order (evicted_before), each appended to the pairs of every scanned queue of its chain
  std::vector<uint32_t> order(n_running);
  std::iota(order.begin(), order.end(), 0u);
  std::sort(order.begin(), order.end(), [running](uint32_t a, uint32_t b) { return a != b && evicted_before(running, a, b); });
  std::vector<std::vector<uint2>> per(q_id.size());
  for (uint32_t r : order) {
    uint32_t k = 0;
    for (uint32_t X = run_queue[r]; X != GROVE_NONE_U32; X = queues[X].parent, ++k)
      if (scan_id[X] != GROVE_NONE_U32) per[scan_id[X]].push_back(make_uint2(r, k));
  }
  std::vector<uint32_t> off(q_id.size() + 1, 0);
  std::vector<uint2> pr;
  for (size_t i = 0; i < per.size(); ++i) { pr.insert(pr.end(), per[i].begin(), per[i].end()); off[i + 1] = uint32_t(pr.size()); }
  if (pr.empty()) pr.push_back(make_uint2(0u, 0u));
  std::vector<long long> use(size_t(n_running) * 3);
  for (uint32_t r = 0; r < n_running; ++r) for (int k = 0; k < 3; ++k) use[r * 3 + k] = usage[r][k];
  auto up = [e](auto& dv, const auto& h) -> cudaError_t {
    cudaError_t c = dv.ensure(h.size());
    if (c == cudaSuccess) c = cudaMemcpyAsync(dv.p, h.data(), sizeof(h[0]) * h.size(), cudaMemcpyHostToDevice, e->stream);
    return c;
  };
  const std::vector<uint32_t> rq(run_queue, run_queue + n_running);
  CU_TRY(e, up(e->d_dn_off, off)); CU_TRY(e, up(e->d_dn_qid, q_id)); CU_TRY(e, up(e->d_dn_pr, pr)); CU_TRY(e, up(e->d_dn_quota, quota));
  CU_TRY(e, up(e->d_dn_use, use)); CU_TRY(e, up(e->d_dn_parent, parent)); CU_TRY(e, up(e->d_dn_rq, rq)); CU_TRY(e, up(e->d_dn_fin, fin));
  CU_TRY(e, e->d_dn_load.ensure(std::max<size_t>(size_t(NQ) * 3, 1))); CU_TRY(e, e->d_dn_bits.ensure(size_t(n_running) * GROVE_MAX_QUEUE_DEPTH));
  CU_TRY(e, e->d_rc_evict.ensure(n_running));
  CU_TRY(e, cudaStreamSynchronize(e->stream));   // (pageable sources)
  *d = DonorSet{e->d_dn_off.p, e->d_dn_qid.p, e->d_dn_pr.p, e->d_dn_quota.p, e->d_dn_load.p, e->d_dn_use.p, e->d_dn_parent.p,
                e->d_dn_rq.p, e->d_dn_fin.p, e->d_rc_gone.p, e->d_dn_bits.p};
  return GROVE_OK;
}

// share_Q = max over the resources x with a finite deserved_Q[x] of load_Q[x] / deserved_Q[x] as (num, den), den 0 = +inf; 0/0 and
// no finite quota = 0.  less() compares two exactly (128-bit cross products).
namespace {
struct Share {
  uint64_t num = 0, den = 1;
  static bool less(const Share& a, const Share& b) {
    if (b.den == 0) return a.den != 0;
    if (a.den == 0) return false;
    return (unsigned __int128)a.num * b.den < (unsigned __int128)b.num * a.den;
  }
};
}  // namespace
static Share share_of(const grove_queue_quota_t& q, const std::array<int64_t, 3>& load) {
  Share s;
  for (int k = 0; k < 3; ++k) {
    if (q.deserved[k] == GROVE_QUEUE_UNLIMITED) continue;
    const uint64_t l = uint64_t(std::max<int64_t>(load[k], 0));
    const Share x = q.deserved[k] ? Share{l, q.deserved[k]} : (l ? Share{1, 0} : Share{0, 1});
    if (Share::less(s, x)) s = x;
  }
  return s;
}

// replaces (null: no gang replaces a running gang) as for grove_run_cycle_reuse; running_queue (null: no queue set) the queue of each
// running gang in the queue set of the current submission; quotas (null: no queue classes) one row per queue of that set, and then
// the queue classes run first (grove_run_cycle_reclaim_queues); priority: the priority classes run (after the queue classes, from
// the state they leave: grove_run_cycle_reclaim_preempt_queues).  Inputs checked by the entry.
static int32_t reclaim_cycle(grove_engine* e, const uint32_t* replaces, const grove_running_gang_t* running, uint32_t n_running,
                             const grove_holding_t* holdings, const uint32_t* running_queue, const grove_queue_quota_t* quotas,
                             bool priority, grove_cycle_stats_t* stats) {
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  const uint32_t G = e->G, N = e->N, nblk = (N + 255) / 256;
  ReclaimCsr csr{};
  int32_t rc = upload_running(e, running, n_running, holdings, &csr);
  if (rc) return rc;
  CU_TRY(e, e->d_rc_evict.ensure(std::max<uint32_t>(n_running, 1)));
  // without replacements nothing holds; without a queue set no gang and no running gang is in a queue, and the queue step never runs
  std::vector<uint32_t> rep(G, GROVE_NONE_U32), run_queue(n_running, GROVE_NONE_U32);
  if (replaces) std::copy(replaces, replaces + G, rep.begin());
  if (running_queue) std::copy(running_queue, running_queue + n_running, run_queue.begin());
  // the queue set of the current submission (the class cycles re-use the handle) and what each running gang holds
  const std::vector<grove_queue_t> queues = running_queue ? e->qu_queues : std::vector<grove_queue_t>{};
  const std::vector<uint32_t> gang_queue = running_queue ? e->qu_gang_queue : std::vector<uint32_t>(G, GROVE_NONE_U32);
  const uint32_t NQ = uint32_t(queues.size());
  std::vector<std::array<int64_t, 3>> usage(n_running);
  for (uint32_t r = 0; r < n_running; ++r) usage[r] = usage_of(running[r], holdings);
  std::vector<std::array<int64_t, 3>> own(NQ, {0, 0, 0});   // own used, then followed through the cycle
  for (uint32_t q = 0; q < NQ; ++q) for (int k = 0; k < 3; ++k) own[q][k] = int64_t(std::min<uint64_t>(queues[q].used[k], uint64_t(1) << 62));
  std::vector<uint8_t> gone(std::max<uint32_t>(n_running, 1), 0);   // released or evicted
  // the caps of a class: the limits for a priority class, min(limit, deserved) for a queue class
  std::vector<std::array<uint64_t, 3>> limit(NQ), cap(NQ);
  for (uint32_t q = 0; q < NQ; ++q)
    for (int k = 0; k < 3; ++k) {
      limit[q][k] = queues[q].limit[k];
      cap[q][k] = quotas ? std::min(queues[q].limit[k], quotas[q].deserved[k]) : queues[q].limit[k];
    }

  // 1. the ordinary pass: the cycle with holds (the reuse cycle; without replacements the ordinary cycle, under a queue set the
  // queue cycle).  An admitted new version's predecessor is released.
  grove_cycle_stats_t st0{};
  rc = run_cycle_holds(e, rep.data(), running, holdings, false, &st0);
  if (rc) return rc;
  Snapshot snap;
  rc = snapshot(e, &snap);
  if (rc) return rc;
  for (uint32_t g = 0; g < G; ++g)
    if (snap.status[g].state == GROVE_GANG_ADMITTED && rep[g] != GROVE_NONE_U32) gone[rep[g]] = 1;
  // the loads: own used + the admitted members' usage, then every queue's own plus its descendants'
  for (uint32_t g = 0; g < G; ++g) {
    if (snap.status[g].state != GROVE_GANG_ADMITTED || gang_queue[g] == GROVE_NONE_U32) continue;
    for (uint32_t i = 0; i < snap.status[g].n_pods; ++i) {
      const grove_clique_t& q = snap.cliques[snap.place[snap.status[g].placement_off + i].clique];
      own[gang_queue[g]][0] += q.req_cpu_milli; own[gang_queue[g]][1] += q.req_mem_mib; own[gang_queue[g]][2] += q.req_gpu;
    }
  }
  std::vector<std::array<int64_t, 3>> load(own);
  for (uint32_t q = NQ; q-- > 0;)
    if (queues[q].parent != GROVE_NONE_U32) for (int k = 0; k < 3; ++k) load[queues[q].parent][k] += load[q][k];
  auto account = [&](uint32_t q, const int64_t* u, int64_t sign) {   // usage u joins (+1) or leaves (-1) queue q
    for (int k = 0; k < 3; ++k) own[q][k] += sign * u[k];
    for (; q != GROVE_NONE_U32; q = queues[q].parent) for (int k = 0; k < 3; ++k) load[q][k] += sign * u[k];
  };
  auto in_subtree = [&](uint32_t q, uint32_t Qx) {   // is Qx in chain(q)?
    for (; q != GROVE_NONE_U32; q = queues[q].parent) if (q == Qx) return true;
    return false;
  };
  // evict[r]: running gang r may be evicted by the current class (fixed when the class starts: it stood then)
  std::vector<uint8_t> evict(std::max<uint32_t>(n_running, 1), 0);
  auto standing = [&]() {   // does a running gang the class may evict still stand?
    for (uint32_t r = 0; r < n_running; ++r) if (evict[r] && !gone[r]) return true;
    return false;
  };
  std::vector<grove_victim_t> victims;
  std::vector<std::vector<grove_placement_t>> extra(G);   // placements of the preemptors and reclaimers, by gang
  RunningByNode at;
  std::vector<int32_t> slot;   // node (caller order) -> its row in `rows` while a class chooses its victims

  // One class: its members (gangs still rejected, in rank order) against the running gangs `evict` marks, under the queue caps
  // `caps`.  Its admitted members carry `flag`; give_back: a member admitted by the class cycle once none of them stands any more
  // gives its room back (the priority classes' rule).
  auto run_class = [&](const std::vector<uint32_t>& members, const std::vector<std::array<uint64_t, 3>>& caps, uint16_t flag,
                       bool give_back) -> int32_t {
    // 2. the class's members as a submission of their own.  A member holds its predecessor's holdings when that one still stands
    // and is not evictable; when it is, it is released instead.
    Sub sub;
    std::vector<uint32_t> sub_rep, sub_queue;
    for (uint32_t g : members) {
      add_gang(e, snap, g, sub);
      const uint32_t r = rep[g];
      sub_rep.push_back(r != GROVE_NONE_U32 && !gone[r] && !evict[r] ? r : GROVE_NONE_U32);
      sub_queue.push_back(gang_queue[g]);
    }
    // the class view, on the device: free + the standing holdings the class may evict; the free table itself is kept for the
    // victim choice
    CU_TRY(e, cudaMemcpyAsync(e->d_rc_evict.p, evict.data(), n_running, cudaMemcpyHostToDevice, e->stream));
    k_reclaim_view<<<nblk, 256, 0, e->stream>>>(e->d_nres.p, e->d_rc_real.p, csr.off, csr.ent, e->d_rc_evict.p, N, 1u);
    CU_TRY(e, cudaGetLastError());
    int32_t rc = submit_sub(e, sub); if (rc) return rc;
    if (running_queue) {   // the class's queue set: own used without what the evictable gangs hold, so that its loads are load';
                           // the caps in place of the limits
      std::vector<grove_queue_t> cq(queues);
      std::vector<std::array<int64_t, 3>> o(own);
      for (uint32_t r = 0; r < n_running; ++r)
        if (evict[r] && run_queue[r] != GROVE_NONE_U32) for (int k = 0; k < 3; ++k) o[run_queue[r]][k] -= usage[r][k];
      for (uint32_t q = 0; q < NQ; ++q) for (int k = 0; k < 3; ++k) { cq[q].used[k] = uint64_t(o[q][k]); cq[q].limit[k] = caps[q][k]; }
      rc = install_queues(e, cq.data(), NQ, sub_queue.data()); if (rc) return rc;
    }
    grove_cycle_stats_t stp{};
    rc = run_cycle_holds(e, sub_rep.data(), running, holdings, false, &stp); if (rc) return rc;
    accumulate(st0, stp); st0.kernel_launches += 2;   // (+ the two k_reclaim_view)
    std::vector<grove_scope_status_t> ssp;
    rc = sub_scope_domains(e, sub, ssp); if (rc) return rc;
    // the free-table rows of the nodes the class's admitted members use
    std::vector<uint32_t> used;
    for (uint32_t k = 0; k < sub.ids.size(); ++k) {
      const grove_gang_status_t& sp = e->h_status.p[k];
      if (sp.state != GROVE_GANG_ADMITTED) continue;
      for (uint32_t i = 0; i < sp.n_pods; ++i) used.push_back(e->h_out.p[sp.placement_off + i].node);
    }
    std::sort(used.begin(), used.end());
    used.erase(std::unique(used.begin(), used.end()), used.end());
    std::vector<Res> rows;
    rc = read_rows(e, used, rows, st0); if (rc) return rc;
    for (size_t i = 0; i < used.size(); ++i) slot[used[i]] = int32_t(i);
    auto release = [&](uint32_t v) {   // everything v held returns to the free table (only the tracked rows matter here)
      gone[v] = 1;
      for (uint32_t h = 0; h < running[v].n_holdings; ++h) {
        const grove_holding_t& x = holdings[running[v].holding_off + h];
        if (slot[x.node] >= 0) rows[slot[x.node]].add(held(x));
      }
    };
    auto evict_one = [&](uint32_t v, uint32_t g) {   // released, and its usage leaves its queues
      release(v);
      if (run_queue[v] != GROVE_NONE_U32) account(run_queue[v], usage[v].data(), -1);
      victims.push_back(grove_victim_t{v, g});
    };
    // 3. victims, gang by gang in rank order (sub-submission order == order rank)
    std::vector<std::pair<uint32_t, Res>> back;   // (sorted node, change)
    for (uint32_t k = 0; k < sub.ids.size(); ++k) {
      const grove_gang_status_t& sp = e->h_status.p[k];
      if (sp.state != GROVE_GANG_ADMITTED) continue;
      std::vector<uint32_t> nodes; std::vector<Res> use; std::vector<grove_placement_t> pl;
      placed(e, snap, sub, k, nodes, use, pl);
      if (give_back && !standing()) {   // admitted by the class cycle after E(p) ran out: it stays as the ordinary pass left it.
                                        // What the class cycle committed for it goes back: +U, and -H for a member with a hold (a
                                        // queue charge was never taken here)
        for (size_t j = 0; j < nodes.size(); ++j) back.push_back({e->inv[nodes[j]], use[j]});
        if (sub_rep[k] != GROVE_NONE_U32)
          for (uint32_t h = 0; h < running[sub_rep[k]].n_holdings; ++h) {
            const grove_holding_t& x = holdings[running[sub_rep[k]].holding_off + h];
            Res c; c.add(held(x), -1);
            back.push_back({e->inv[x.node], c});
          }
        continue;
      }
      const uint32_t g = sub.ids[k], r = rep[g];
      const bool holds = sub_rep[k] != GROVE_NONE_U32;
      if (r != GROVE_NONE_U32 && !holds && !gone[r]) release(r);   // its predecessor is evictable: released first, not a victim
      std::vector<Res> mine(nodes.size());
      if (holds)   // what its predecessor holds on each of those nodes: used first
        for (uint32_t h = 0; h < running[r].n_holdings; ++h) {
          const grove_holding_t& x = holdings[running[r].holding_off + h];
          for (size_t j = 0; j < nodes.size(); ++j) if (nodes[j] == x.node) mine[j].add(held(x));
        }
      // (a) the node step: the reclaim pass's rule
      for (size_t j = 0; j < nodes.size(); ++j) {
        const uint32_t n = nodes[j];
        const Res need{std::max<int64_t>(use[j].cpu - mine[j].cpu, 0), std::max<int64_t>(use[j].mem - mine[j].mem, 0),
                       std::max<int64_t>(use[j].gpu - mine[j].gpu, 0), std::max<int64_t>(use[j].pods - mine[j].pods, 0)};
        Res& have = rows[slot[n]];
        while (!have.covers(need)) {
          const uint32_t v = choose_victim(at, n, running, [&](uint32_t x) { return evict[x] && !gone[x]; });
          if (v == GROVE_NONE_U32) return fail(e, GROVE_ERR_STATE, "reclaim pass: a preemptor's node cannot be freed");
          evict_one(v, g);
        }
        have.add(need, -1);
      }
      if (holds) gone[r] = 1;   // released; its leftover came back when the class cycle ended (k_hold_release)
      // (b) the queue step: g's chain, leaf first, back within its caps on the resources g uses
      const uint32_t gq = gang_queue[g];
      if (gq != GROVE_NONE_U32) {
        int64_t U[3] = {0, 0, 0};
        for (const Res& u : use) { U[0] += u.cpu; U[1] += u.mem; U[2] += u.gpu; }
        account(gq, U, 1);
        for (uint32_t Qx = gq; Qx != GROVE_NONE_U32; Qx = queues[Qx].parent) {
          for (;;) {
            uint32_t over = 0;   // the resources g uses on which Qx is over its finite cap
            for (int t = 0; t < 3; ++t)
              if (U[t] > 0 && caps[Qx][t] != GROVE_QUEUE_UNLIMITED && load[Qx][t] > 0 && uint64_t(load[Qx][t]) > caps[Qx][t]) over |= 1u << t;
            if (!over) break;
            uint32_t v = GROVE_NONE_U32;   // by the victim rule, among the evictable gangs in Qx's subtree that hold some of it
            for (uint32_t x = 0; x < n_running; ++x) {
              if (!evict[x] || gone[x] || run_queue[x] == GROVE_NONE_U32 || !in_subtree(run_queue[x], Qx)) continue;
              bool holds_some = false;
              for (int t = 0; t < 3; ++t) holds_some |= ((over >> t) & 1u) && usage[x][t] > 0;
              if (holds_some && evicted_before(running, x, v)) v = x;
            }
            if (v == GROVE_NONE_U32) return fail(e, GROVE_ERR_STATE, "reclaim pass: a preemptor's queue cannot be brought within its limit");
            evict_one(v, g);
          }
        }
      }
      grove_gang_status_t o = sp;
      o.reserved0 = uint16_t(flag | (sp.reserved0 & GROVE_STATUS_SURPLUS_CAPPED));
      merge_gang(snap, sub, k, o, ssp);
      extra[g] = std::move(pl);
      st0.gangs_admitted += 1; st0.gangs_rejected -= 1;
    }
    for (uint32_t n : used) slot[n] = -1;
    rc = patch_nodes(e, back, st0); if (rc) return rc;
    // back to the free table: take off what the evictable running gangs that still stand hold
    for (uint32_t r = 0; r < n_running; ++r) evict[r] = evict[r] && !gone[r];
    CU_TRY(e, cudaMemcpyAsync(e->d_rc_evict.p, evict.data(), n_running, cudaMemcpyHostToDevice, e->stream));
    k_reclaim_view<<<nblk, 256, 0, e->stream>>>(e->d_nres.p, e->d_rc_real.p, csr.off, csr.ent, e->d_rc_evict.p, N, 0u);
    CU_TRY(e, cudaGetLastError());
    return GROVE_OK;
  };
  auto arm = [&]() -> cudaError_t {   // before the first class: the free table after the ordinary pass is kept aside
    at = running_by_node(N, running, n_running, holdings);
    slot.assign(N, -1);
    return cudaMemcpyAsync(e->d_rc_base.p, e->d_nres.p, sizeof(uint4) * e->Npad, cudaMemcpyDeviceToDevice, e->stream);
  };
  // armed once, before the first class of either loop; the handle goes back to the caller's submission (and queue set) after the
  // last, and the device table is then the free table
  Restore restore{e, &snap, running_queue ? &queues : nullptr, &gang_queue, false};
  auto ensure_armed = [&]() -> int32_t {
    if (restore.armed) return GROVE_OK;
    CU_TRY(e, arm());
    restore.armed = true;
    return GROVE_OK;
  };

  if (quotas) {
    // queue classes: the queues of the rejected gangs, by ascending share at the start of the pass, ties by queue index; each
    // against its donor set E(Q) under the caps
    std::vector<uint32_t> classes;
    for (uint32_t g = 0; g < G; ++g)
      if (snap.status[g].state == GROVE_GANG_REJECTED && gang_queue[g] != GROVE_NONE_U32) classes.push_back(gang_queue[g]);
    std::sort(classes.begin(), classes.end());
    classes.erase(std::unique(classes.begin(), classes.end()), classes.end());
    std::vector<Share> share(NQ);
    for (uint32_t q : classes) share[q] = share_of(quotas[q], load[q]);
    std::stable_sort(classes.begin(), classes.end(), [&](uint32_t a, uint32_t b) { return Share::less(share[a], share[b]); });
    uint32_t scanned = 0;
    DonorSet dn{};
    if (!classes.empty()) { rc = upload_donors(e, running, n_running, run_queue.data(), queues, quotas, usage, &scanned, &dn); if (rc) return rc; }
    if (scanned) {
      rc = ensure_armed(); if (rc) return rc;
      std::vector<long long> ld(size_t(NQ) * 3);
      for (uint32_t Q : classes) {
        // E(Q) on the device, from the current loads and the standing set
        for (uint32_t q = 0; q < NQ; ++q) for (int k = 0; k < 3; ++k) ld[q * 3 + k] = load[q][k];
        CU_TRY(e, cudaMemcpyAsync(e->d_dn_load.p, ld.data(), sizeof(long long) * ld.size(), cudaMemcpyHostToDevice, e->stream));
        CU_TRY(e, cudaMemcpyAsync(e->d_rc_gone.p, gone.data(), n_running, cudaMemcpyHostToDevice, e->stream));
        k_donor_scan<<<scanned, 256, 0, e->stream>>>(dn);
        CU_TRY(e, cudaGetLastError());
        k_donor_mark<<<(n_running + 255) / 256, 256, 0, e->stream>>>(dn, Q, n_running, e->d_rc_evict.p);
        CU_TRY(e, cudaGetLastError());
        CU_TRY(e, cudaMemcpyAsync(evict.data(), e->d_rc_evict.p, n_running, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(e, cudaStreamSynchronize(e->stream));
        st0.kernel_launches += 2;
        if (!standing()) continue;   // an empty donor set: the members keep their ordinary-pass outcome
        std::vector<uint32_t> members;
        for (uint32_t g = 0; g < G; ++g)
          if (snap.status[g].state == GROVE_GANG_REJECTED && gang_queue[g] == Q) members.push_back(g);
        std::stable_sort(members.begin(), members.end(), [&](uint32_t a, uint32_t b) { return snap.gangs[a].priority > snap.gangs[b].priority; });
        rc = run_class(members, cap, GROVE_STATUS_RECLAIMER, false); if (rc) return rc;
      }
    }
  }
  if (priority) {
    // priority classes: every priority of a gang still rejected, descending, while E(p) -- the standing running gangs of a priority
    // below p -- is non-empty (it only shrinks from one class to the next); each under the limits
    std::vector<int32_t> classes;
    for (uint32_t g = 0; g < G; ++g) if (snap.status[g].state == GROVE_GANG_REJECTED) classes.push_back(snap.gangs[g].priority);
    std::sort(classes.begin(), classes.end(), std::greater<int32_t>());
    classes.erase(std::unique(classes.begin(), classes.end()), classes.end());
    auto mark = [&](int32_t p) { for (uint32_t r = 0; r < n_running; ++r) evict[r] = !gone[r] && running[r].priority < p; };
    if (!classes.empty()) mark(classes.front());
    if (!classes.empty() && standing()) {
      rc = ensure_armed(); if (rc) return rc;
      for (int32_t p : classes) {
        mark(p);
        if (!standing()) break;
        std::vector<uint32_t> members;   // (one priority: submission order is rank order)
        for (uint32_t g = 0; g < G; ++g)
          if (snap.status[g].state == GROVE_GANG_REJECTED && snap.gangs[g].priority == p) members.push_back(g);
        rc = run_class(members, limit, GROVE_STATUS_PREEMPTOR, true); if (rc) return rc;
      }
    }
  }
  if (restore.armed) {
    restore.armed = false;
    rc = restore.put_back(); if (rc) return rc;
  }
  st0.kernel_launches += 1;   // k_reclaim_check
  return publish_reclaim(e, snap.status, snap.place, extra, snap.sstat, st0, std::move(victims), stats);
}

int32_t grove_run_cycle_preempt(grove_engine_t* e, const grove_running_gang_t* running, uint32_t n_running,
                                const grove_holding_t* holdings, uint32_t n_holdings, grove_cycle_stats_t* stats) {
  if (!e || (n_running && !running) || (n_holdings && !holdings)) return GROVE_ERR_INVALID_ARG;
  if (e->sp_members) return refuse_spread(e, "grove_run_cycle_preempt");
  if (e->qu_members) return refuse_queues(e, "grove_run_cycle_preempt");
  if (!e->fc_gangs.empty()) return refuse_fences(e, "grove_run_cycle_preempt");
  if (e->bp_members) return refuse_binpack(e, "grove_run_cycle_preempt");
  if (e->im_enrolled) return refuse_imex(e, "grove_run_cycle_preempt");
  NoDiagnosis no_diag{e};
  if (e->wide) return refuse_wide(e, "grove_run_cycle_preempt");
  int32_t rc = check_ready(e);
  if (rc) return rc;
  rc = check_running(e, running, n_running, holdings, n_holdings);
  if (rc) return rc;
  return reclaim_cycle(e, nullptr, running, n_running, holdings, nullptr, nullptr, true, stats);
}

int32_t grove_run_cycle_reuse_preempt(grove_engine_t* e, const uint32_t* replaces, uint32_t n_gangs, const grove_running_gang_t* running,
                                      uint32_t n_running, const grove_holding_t* holdings, uint32_t n_holdings, grove_cycle_stats_t* stats) {
  if (!e || (n_gangs && !replaces) || (n_running && !running) || (n_holdings && !holdings)) return GROVE_ERR_INVALID_ARG;
  if (e->sp_members) return refuse_spread(e, "grove_run_cycle_reuse_preempt");
  if (e->qu_members) return refuse_queues(e, "grove_run_cycle_reuse_preempt");
  if (!e->fc_gangs.empty()) return refuse_fences(e, "grove_run_cycle_reuse_preempt");
  if (e->bp_members) return refuse_binpack(e, "grove_run_cycle_reuse_preempt");
  if (e->im_enrolled) return refuse_imex(e, "grove_run_cycle_reuse_preempt");
  NoDiagnosis no_diag{e};
  if (e->wide) return refuse_wide(e, "grove_run_cycle_reuse_preempt");
  const int32_t rc = check_reuse_inputs(e, replaces, n_gangs, running, n_running, holdings, n_holdings);
  if (rc) return rc;
  return reclaim_cycle(e, replaces, running, n_running, holdings, nullptr, nullptr, true, stats);
}

// The checks grove_run_cycle_preempt_queues and grove_run_cycle_reclaim_queues share.  First the sets the entries refuse (a refusal
// here leaves grove_diagnose as it was) ...
static int32_t check_queue_sets(grove_engine* e, const char* entry) {
  if (e->sp_members) return refuse_spread(e, entry);
  if (!e->fc_gangs.empty()) return refuse_fences(e, entry);
  if (e->bp_members) return refuse_binpack(e, entry);
  if (e->im_enrolled) return refuse_imex(e, entry);
  if (!e->qu_given) { e->err = std::string(entry) + ": no queue set given for the current submission (grove_set_queues)"; return GROVE_ERR_STATE; }
  if (e->fs_given) { e->err = std::string(entry) + ": not supported while a fair-share set is in place (grove_set_fair_share)"; return GROVE_ERR_STATE; }
  return GROVE_OK;
}

// ... then the submission, the running gangs, and what the running gangs of each queue hold, within its used
static int32_t check_queue_running(grove_engine* e, const char* entry, const grove_running_gang_t* running, uint32_t n_running,
                                   const grove_holding_t* holdings, uint32_t n_holdings, const uint32_t* running_queue) {
  const std::string kEntry(entry);
  if (e->wide) return refuse_wide(e, entry);
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  const int32_t rc = check_running(e, running, n_running, holdings, n_holdings);
  if (rc) return rc;
  const std::vector<grove_queue_t>& queues = e->qu_queues;
  const uint32_t NQ = uint32_t(queues.size());
  std::vector<std::array<int64_t, 3>> run_use(NQ, {0, 0, 0});
  for (uint32_t r = 0; r < n_running; ++r) {
    const uint32_t q = running_queue[r];
    if (q == GROVE_NONE_U32) continue;
    if (q >= NQ) { e->err = kEntry + ": running_queue names a queue out of range"; return GROVE_ERR_INVALID_ARG; }
    const std::array<int64_t, 3> u = usage_of(running[r], holdings);
    for (int k = 0; k < 3; ++k) run_use[q][k] += u[k];
  }
  for (uint32_t q = 0; q < NQ; ++q)
    for (int k = 0; k < 3; ++k)
      if (uint64_t(run_use[q][k]) > queues[q].used[k]) { e->err = kEntry + ": the running gangs of a queue hold more than its used"; return GROVE_ERR_INVALID_ARG; }
  return GROVE_OK;
}

int32_t grove_run_cycle_preempt_queues(grove_engine_t* e, const grove_running_gang_t* running, uint32_t n_running,
                                       const grove_holding_t* holdings, uint32_t n_holdings, const uint32_t* running_queue,
                                       grove_cycle_stats_t* stats) {
  if (!e || (n_running && (!running || !running_queue)) || (n_holdings && !holdings)) return GROVE_ERR_INVALID_ARG;
  int32_t rc = check_queue_sets(e, "grove_run_cycle_preempt_queues");
  if (rc) return rc;
  NoDiagnosis no_diag{e};
  rc = check_queue_running(e, "grove_run_cycle_preempt_queues", running, n_running, holdings, n_holdings, running_queue);
  if (rc) return rc;
  return reclaim_cycle(e, nullptr, running, n_running, holdings, running_queue, nullptr, true, stats);
}

// grove_run_cycle_reclaim_queues, and with priority grove_run_cycle_reclaim_preempt_queues: the same inputs, the same refusals
static int32_t reclaim_queues_entry(grove_engine* e, const char* entry, const grove_queue_quota_t* quotas, uint32_t n_queues,
                                    const grove_running_gang_t* running, uint32_t n_running, const grove_holding_t* holdings,
                                    uint32_t n_holdings, const uint32_t* running_queue, bool priority, grove_cycle_stats_t* stats) {
  if (!e || (n_queues && !quotas) || (n_running && (!running || !running_queue)) || (n_holdings && !holdings)) return GROVE_ERR_INVALID_ARG;
  int32_t rc = check_queue_sets(e, entry);
  if (rc) return rc;
  NoDiagnosis no_diag{e};
  rc = check_queue_running(e, entry, running, n_running, holdings, n_holdings, running_queue);
  if (rc) return rc;
  if (n_queues != e->qu_queues.size()) { e->err = std::string(entry) + ": n_queues is not the number of queues of the set"; return GROVE_ERR_INVALID_ARG; }
  return reclaim_cycle(e, nullptr, running, n_running, holdings, running_queue, quotas, priority, stats);
}

int32_t grove_run_cycle_reclaim_queues(grove_engine_t* e, const grove_queue_quota_t* quotas, uint32_t n_queues,
                                       const grove_running_gang_t* running, uint32_t n_running, const grove_holding_t* holdings,
                                       uint32_t n_holdings, const uint32_t* running_queue, grove_cycle_stats_t* stats) {
  return reclaim_queues_entry(e, "grove_run_cycle_reclaim_queues", quotas, n_queues, running, n_running, holdings, n_holdings,
                              running_queue, false, stats);
}

int32_t grove_run_cycle_reclaim_preempt_queues(grove_engine_t* e, const grove_queue_quota_t* quotas, uint32_t n_queues,
                                               const grove_running_gang_t* running, uint32_t n_running, const grove_holding_t* holdings,
                                               uint32_t n_holdings, const uint32_t* running_queue, grove_cycle_stats_t* stats) {
  return reclaim_queues_entry(e, "grove_run_cycle_reclaim_preempt_queues", quotas, n_queues, running, n_running, holdings, n_holdings,
                              running_queue, true, stats);
}

// ---------------------------------------------------------------------------------------------
// Fair-share order (include/grove_place.h "fair-share order"; DESIGN.md section 1; kernels in fairshare.cuh).  The turn order
// depends on which gangs are admitted, so the cycle is a fixed point: run the queue cycle in order O_i, compute O_{i+1} = O(R_i)
// from its outcomes on the device, and start the next queue cycle at the first turn d where the two differ -- every turn before d
// is final.  Each later cycle is a sub-submission of the turns from d on, in that order (one priority, so that its rank is its
// order), over the node table at d (the last cycle's table with what the turns from d on took given back) and a queue set whose
// `used` are the loads at d.  Per iteration the host reads d and then the order from d on.
// ---------------------------------------------------------------------------------------------
int32_t grove_set_fair_share(grove_engine_t* e, const grove_queue_quota_t* quotas, uint32_t n_queues) {
  if (!e || (n_queues && !quotas)) return GROVE_ERR_INVALID_ARG;
  if (e->in_cycle) return fail(e, GROVE_ERR_STATE, "cycle in flight");
  if (!e->qu_given) return fail(e, GROVE_ERR_STATE, "grove_set_fair_share: no queue set given for the current submission (grove_set_queues)");
  if (n_queues != e->qu_queues.size()) return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_fair_share: n_queues is not the number of queues of the set");
  std::vector<uint8_t> inner(n_queues, 0);
  for (uint32_t q = 0; q < n_queues; ++q) if (e->qu_queues[q].parent != GROVE_NONE_U32) inner[e->qu_queues[q].parent] = 1;
  for (uint32_t g = 0; g < e->G; ++g)
    if (e->qu_gang_queue[g] != GROVE_NONE_U32 && inner[e->qu_gang_queue[g]])
      return fail(e, GROVE_ERR_INVALID_ARG, "grove_set_fair_share: a gang sits in a queue that has children (members must be in leaf queues)");
  e->fs_quotas.assign(quotas, quotas + n_queues);
  e->fs_given = true; e->fs_have_order = false;
  return GROVE_OK;
}

int32_t grove_get_turn_order(grove_engine_t* e, uint32_t* out, uint32_t cap) {
  if (!e || (e->G && !out)) return GROVE_ERR_INVALID_ARG;
  if (!e->fs_have_order) return fail(e, GROVE_ERR_STATE, "grove_get_turn_order: no fair-share cycle since the last submission");
  if (cap < e->G) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  if (e->G) std::memcpy(out, e->fs_order.data(), sizeof(uint32_t) * e->G);
  return GROVE_OK;
}

int32_t grove_get_fair_share_stats(grove_engine_t* e, grove_fair_share_stats_t* out) {
  if (!e || !out) return GROVE_ERR_INVALID_ARG;
  if (!e->fs_have_order) return fail(e, GROVE_ERR_STATE, "grove_get_fair_share_stats: no fair-share cycle since the last submission");
  *out = e->fs_stats;
  return GROVE_OK;
}

static FsTree fs_tree(const grove_engine* e) {
  return FsTree{e->d_fs_parent.p, e->d_fs_depth.p, e->d_fs_load0.p, e->d_fs_quota.p, e->d_fs_leaf.p, e->d_fs_rank.p};
}

// The tables of O(R) for the current submission and queue set, uploaded once per cycle, and the scratch of its scans and sorts.
// -> the depth of the deepest tree node (the pseudo-queue has depth 1)
static int32_t fs_tables(grove_engine* e, const std::vector<uint32_t>& rank, uint32_t* max_depth) {
  const std::vector<grove_queue_t>& queues = e->qu_queues;
  const uint32_t G = e->G, NQ = uint32_t(queues.size()), NT = NQ + 2;
  std::vector<uint32_t> parent(NT, NQ + 1), leaf(G);
  std::vector<uint8_t> depth(NT, 1);
  std::vector<long long> load(size_t(NT) * 3, 0);
  std::vector<unsigned long long> quota(size_t(NT) * 3, GROVE_QUEUE_UNLIMITED);
  depth[NQ + 1] = 0;
  *max_depth = 1;
  for (uint32_t q = 0; q < NQ; ++q) {
    if (queues[q].parent != GROVE_NONE_U32) { parent[q] = queues[q].parent; depth[q] = uint8_t(depth[parent[q]] + 1); }
    *max_depth = std::max<uint32_t>(*max_depth, depth[q]);
    for (int k = 0; k < 3; ++k) { load[q * 3 + k] = (long long)std::min<uint64_t>(queues[q].used[k], uint64_t(1) << 62); quota[q * 3 + k] = e->fs_quotas[q].deserved[k]; }
  }
  for (uint32_t q = NQ; q-- > 0;)
    if (queues[q].parent != GROVE_NONE_U32) for (int k = 0; k < 3; ++k) load[queues[q].parent * 3 + k] += load[q * 3 + k];
  for (uint32_t g = 0; g < G; ++g) leaf[g] = e->qu_gang_queue[g] == GROVE_NONE_U32 ? NQ : e->qu_gang_queue[g];
  auto up = [e](auto& d, const auto& h) -> cudaError_t {
    cudaError_t c = d.ensure(std::max<size_t>(h.size(), 1));
    if (c == cudaSuccess && !h.empty()) c = cudaMemcpyAsync(d.p, h.data(), sizeof(h[0]) * h.size(), cudaMemcpyHostToDevice, e->stream);
    return c;
  };
  CU_TRY(e, up(e->d_fs_parent, parent)); CU_TRY(e, up(e->d_fs_depth, depth)); CU_TRY(e, up(e->d_fs_load0, load));
  CU_TRY(e, up(e->d_fs_quota, quota)); CU_TRY(e, up(e->d_fs_leaf, leaf)); CU_TRY(e, up(e->d_fs_rank, rank));
  CU_TRY(e, e->d_fs_owner.ensure(G)); CU_TRY(e, e->d_fs_vals.ensure(G)); CU_TRY(e, e->d_fs_prev.ensure(G)); CU_TRY(e, e->d_fs_first.ensure(1));
  CU_TRY(e, e->d_fs_keys.ensure(G)); CU_TRY(e, e->d_fs_keys2.ensure(G));
  CU_TRY(e, e->d_fs_use.ensure(G)); CU_TRY(e, e->d_fs_useq.ensure(G)); CU_TRY(e, e->d_fs_before.ensure(G));
  CU_TRY(e, e->h_fs_order.ensure(G));
  size_t t0 = 0, t1 = 0, t2 = 0;
  CU_TRY(e, cub::DeviceScan::ExclusiveScanByKey(nullptr, t0, e->d_fs_owner.p, e->d_fs_useq.p, e->d_fs_before.p, FsSum{}, FsUse{}, G,
                                                ::cuda::std::equal_to<>{}, e->stream));
  CU_TRY(e, cub::DeviceScan::InclusiveScanByKey(nullptr, t1, e->d_fs_owner.p, e->d_fs_keys.p, e->d_fs_keys2.p, FsMax{}, G,
                                                ::cuda::std::equal_to<>{}, e->stream));
  CU_TRY(e, cub::DeviceMergeSort::StableSortPairs(nullptr, t2, e->d_fs_keys.p, e->d_fs_vals.p, G, FsSortLess{}, e->stream));
  CU_TRY(e, e->d_fs_tmp.ensure(std::max<size_t>(std::max(t0, std::max(t1, t2)), 1)));
  CU_TRY(e, cudaStreamSynchronize(e->stream));   // (pageable sources)
  return GROVE_OK;
}

// O(use) into d_fs_vals: every leaf's sequence in rank order, then per tree level, deepest first, the load of each element's node
// at its turn (segmented exclusive scan), its key, the key's prefix max along the node's sequence (segmented inclusive scan), and
// the parents' sequences (stable sort by (parent, key)).  Then, unless first is null (the cycle's first order, with nothing to
// compare against), *first = the first position where the order differs from the one in d_fs_prev (G: none), which is all the
// host reads.  *ms: the device time of it all, in events.
static int32_t fs_order(grove_engine* e, uint32_t max_depth, const std::vector<FsUse>& use, uint32_t* first, float* ms) {
  const uint32_t G = uint32_t(use.size()), nb = (G + 255) / 256;   // (the whole submission: e->G is that of the last sub-cycle)
  const cudaStream_t s = e->stream;
  const FsTree t = fs_tree(e);
  FsKey* a = e->d_fs_keys.p;
  FsKey* b = e->d_fs_keys2.p;
  uint32_t* vals = e->d_fs_vals.p;
  size_t tmp = e->d_fs_tmp.cap;
  CU_TRY(e, cudaMemcpyAsync(e->d_fs_use.p, use.data(), sizeof(FsUse) * G, cudaMemcpyHostToDevice, s));
  CU_TRY(e, cudaEventRecord(e->ev[0], s));
  k_fs_init<<<nb, 256, 0, s>>>(t, G, a, vals);
  CU_TRY(e, cudaGetLastError());
  CU_TRY(e, cub::DeviceMergeSort::StableSortPairs(e->d_fs_tmp.p, tmp, a, vals, G, FsSortLess{}, s));
  for (uint32_t d = max_depth; d >= 1; --d) {
    k_fs_gather<<<nb, 256, 0, s>>>(G, a, vals, e->d_fs_use.p, e->d_fs_owner.p, e->d_fs_useq.p);
    CU_TRY(e, cudaGetLastError());
    tmp = e->d_fs_tmp.cap;
    CU_TRY(e, cub::DeviceScan::ExclusiveScanByKey(e->d_fs_tmp.p, tmp, e->d_fs_owner.p, e->d_fs_useq.p, e->d_fs_before.p, FsSum{}, FsUse{}, G,
                                                  ::cuda::std::equal_to<>{}, s));
    k_fs_key<<<nb, 256, 0, s>>>(t, G, d, e->d_fs_owner.p, vals, e->d_fs_before.p, a);
    CU_TRY(e, cudaGetLastError());
    tmp = e->d_fs_tmp.cap;
    CU_TRY(e, cub::DeviceScan::InclusiveScanByKey(e->d_fs_tmp.p, tmp, e->d_fs_owner.p, a, b, FsMax{}, G, ::cuda::std::equal_to<>{}, s));
    tmp = e->d_fs_tmp.cap;
    CU_TRY(e, cub::DeviceMergeSort::StableSortPairs(e->d_fs_tmp.p, tmp, b, vals, G, FsSortLess{}, s));
    std::swap(a, b);
  }
  if (first) {
    const uint32_t none = G;
    CU_TRY(e, cudaMemcpyAsync(e->d_fs_first.p, &none, sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    k_fs_diff<<<nb, 256, 0, s>>>(G, vals, e->d_fs_prev.p, e->d_fs_first.p);
    CU_TRY(e, cudaGetLastError());
    CU_TRY(e, cudaMemcpyAsync(first, e->d_fs_first.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    e->launches += 1;
  }
  CU_TRY(e, cudaEventRecord(e->ev[1], s));
  CU_TRY(e, cudaStreamSynchronize(s));
  CU_TRY(e, cudaEventElapsedTime(ms, e->ev[0], e->ev[1]));
  e->launches += 2 + 5 * max_depth;
  return GROVE_OK;
}

// the order O(use) from position d on, into order[d..G), and kept in d_fs_prev for the next comparison
static int32_t fs_take_order(grove_engine* e, uint32_t d, std::vector<uint32_t>& order) {
  const uint32_t G = uint32_t(order.size());
  CU_TRY(e, cudaMemcpyAsync(e->h_fs_order.p, e->d_fs_vals.p + d, sizeof(uint32_t) * (G - d), cudaMemcpyDeviceToHost, e->stream));
  CU_TRY(e, cudaMemcpyAsync(e->d_fs_prev.p, e->d_fs_vals.p, sizeof(uint32_t) * G, cudaMemcpyDeviceToDevice, e->stream));
  CU_TRY(e, cudaStreamSynchronize(e->stream));
  std::copy(e->h_fs_order.p, e->h_fs_order.p + (G - d), order.begin() + d);
  return GROVE_OK;
}

static int32_t fair_share_cycle(grove_engine* e, grove_cycle_stats_t* stats) {
  int32_t rc = check_ready(e);
  if (rc) return rc;
  if (e->bp_members) return refuse_binpack(e, "grove_run_cycle with a fair-share set");
  if (e->im_enrolled) return refuse_imex(e, "grove_run_cycle with a fair-share set");
  if (e->sp_members) return refuse_spread(e, "grove_run_cycle with a fair-share set");
  if (!e->fc_gangs.empty()) return refuse_fences(e, "grove_run_cycle with a fair-share set");
  if (!e->qu_given) return fail(e, GROVE_ERR_STATE, "grove_run_cycle: the fair-share set has no queue set (grove_set_queues)");
  struct Diag { grove_engine* e; ~Diag() { e->diag = grove_engine::kDiagFairShare; } } diag_guard{e};
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  const uint32_t G = e->G;
  const std::vector<grove_queue_t> queues = e->qu_queues;
  const std::vector<uint32_t> gang_queue = e->qu_gang_queue;
  const std::vector<grove_queue_quota_t> quotas = e->fs_quotas;
  const uint32_t NQ = uint32_t(queues.size());
  std::vector<uint32_t> by_rank(G), rank(G);
  std::iota(by_rank.begin(), by_rank.end(), 0u);
  std::stable_sort(by_rank.begin(), by_rank.end(), [e](uint32_t a, uint32_t b) { return e->gangs[a].priority > e->gangs[b].priority; });
  for (uint32_t k = 0; k < G; ++k) rank[by_rank[k]] = k;
  if (std::all_of(gang_queue.begin(), gang_queue.end(), [](uint32_t q) { return q == GROVE_NONE_U32; })) {
    rc = run_cycle(e, stats);   // no member: every share is 0 and the order is rank order
    if (rc) return rc;
    e->fs_order = by_rank; e->fs_stats = grove_fair_share_stats_t{1, 0}; e->fs_have_order = true;
    return GROVE_OK;
  }
  Snapshot snap;
  snap.gangs.assign(e->gangs.data(), e->gangs.data() + G);
  snap.cliques.assign(e->cliques.data(), e->cliques.data() + e->Q);
  snap.scopes.assign(e->scopes.data(), e->scopes.data() + e->S);
  snap.status.assign(G, grove_gang_status_t{});
  snap.sstat.assign(std::max<uint32_t>(e->S, 1), grove_scope_status_t{});
  // U of the first order: R_min of every member
  std::vector<FsUse> use(G, FsUse{});
  for (uint32_t g = 0; g < G; ++g) {
    if (gang_queue[g] == GROVE_NONE_U32) continue;
    for (uint32_t c = 0; c < snap.gangs[g].n_cliques; ++c) {
      const grove_clique_t& q = snap.cliques[snap.gangs[g].clique_off + c];
      use[g].v[0] += (long long)q.min_replicas * q.req_cpu_milli; use[g].v[1] += (long long)q.min_replicas * q.req_mem_mib;
      use[g].v[2] += (long long)q.min_replicas * q.req_gpu;
    }
  }
  uint32_t max_depth = 1;
  rc = fs_tables(e, rank, &max_depth);
  if (rc) return rc;
  // whatever goes wrong from here, the handle goes back to the caller's submission, queue set and fair-share set on the starting
  // node table (the fair-share set only when the queue set could be put back)
  struct Keep {
    grove_engine* e; const std::vector<grove_queue_quota_t>* q;
    ~Keep() { if (e->qu_given) { e->fs_quotas = *q; e->fs_given = true; } }
  } keep{e, &quotas};
  CU_TRY(e, e->d_rc_base.ensure(e->Npad));
  CU_TRY(e, cudaMemcpyAsync(e->d_rc_base.p, e->d_nres.p, sizeof(uint4) * e->Npad, cudaMemcpyDeviceToDevice, e->stream));
  Restore restore{e, &snap, &queues, &gang_queue, true};
  const uint64_t launches0 = e->launches;
  uint32_t d = 0, iterations = 0, first = 0;
  uint64_t rerun = 0;
  std::vector<uint32_t> order(G), pos(G);
  std::vector<std::vector<grove_placement_t>> pl(G);
  grove_cycle_stats_t st0{};
  float ms_order = 0.f;
  rc = fs_order(e, max_depth, use, nullptr, &ms_order); if (rc) return rc;
  rc = fs_take_order(e, 0, order); if (rc) return rc;
  st0.kernel_launches += e->launches - launches0;
  st0.ms_total += ms_order;
  for (;;) {
    ++iterations;
    if (iterations > 1) rerun += G - d;
    for (uint32_t p = 0; p < G; ++p) pos[order[p]] = p;
    // the queue loads at turn d: own used plus what the members admitted before d charged (members sit in leaves)
    std::vector<grove_queue_t> cq(queues);
    for (uint32_t p = 0; p < d; ++p) {
      const uint32_t g = order[p];
      if (snap.status[g].state == GROVE_GANG_ADMITTED && gang_queue[g] != GROVE_NONE_U32)
        for (int k = 0; k < 3; ++k) cq[gang_queue[g]].used[k] += uint64_t(use[g].v[k]);
    }
    // a gang from d on whose base had its turn before d and was not admitted -- or is itself such a gang -- comes back
    // BASE_REJECTED without a turn of the engine; a gated one is skipped first, as always
    std::vector<uint8_t> dropped(G, 0);
    for (bool more = true; more;) {
      more = false;
      for (uint32_t p = d; p < G; ++p) {
        const uint32_t g = order[p], b = snap.gangs[g].base_gang;
        if (dropped[g] || (snap.gangs[g].flags & GROVE_GANG_GATED) || b == GROVE_NONE_U32) continue;
        if ((pos[b] < d && snap.status[b].state != GROVE_GANG_ADMITTED) || dropped[b]) { dropped[g] = 1; more = true; }
      }
    }
    std::vector<uint32_t> sub_of(G, GROVE_NONE_U32), sub_queue;
    for (uint32_t p = d, k = 0; p < G; ++p) if (!dropped[order[p]]) sub_of[order[p]] = k++;
    Sub sub;
    for (uint32_t p = d; p < G; ++p) {
      const uint32_t g = order[p];
      pl[g].clear(); use[g] = FsUse{};
      if (dropped[g]) {
        grove_gang_status_t o{};
        o.state = GROVE_GANG_BASE_REJECTED; o.level = GROVE_LEVEL_NONE; o.domain_node = GROVE_NONE_U32;
        snap.status[g] = o;
        for (uint32_t si = 0; si < snap.gangs[g].n_scopes; ++si)
          snap.sstat[snap.gangs[g].scope_off + si] = grove_scope_status_t{GROVE_LEVEL_NONE, {0, 0, 0}, GROVE_NONE_U32};
        continue;
      }
      grove_gang_t& x = add_gang(e, snap, g, sub);
      x.priority = 0;   // one priority: the sub-submission's rank is its order, the turn order from d on
      const uint32_t b = snap.gangs[g].base_gang;
      if (b != GROVE_NONE_U32 && pos[b] >= d) x.base_gang = sub_of[b];   // (before d: admitted, so no base to wait for)
      sub_queue.push_back(gang_queue[g]);
    }
    if (!sub.ids.empty()) {
      rc = submit_sub(e, sub); if (rc) return rc;
      rc = install_queues(e, cq.data(), NQ, sub_queue.data()); if (rc) return rc;
      grove_cycle_stats_t stp{};
      rc = run_cycle(e, &stp); if (rc) return rc;
      accumulate(st0, stp);
      std::vector<grove_scope_status_t> ssp;
      rc = sub_scope_domains(e, sub, ssp); if (rc) return rc;
      for (uint32_t k = 0; k < sub.ids.size(); ++k) {
        const uint32_t g = sub.ids[k];
        const grove_gang_status_t sp = e->h_status.p[k];
        merge_gang(snap, sub, k, sp, ssp);
        if (sp.state != GROVE_GANG_ADMITTED) continue;
        std::vector<uint32_t> nodes; std::vector<Res> u;
        placed(e, snap, sub, k, nodes, u, pl[g]);
        for (const Res& r : u) { use[g].v[0] += r.cpu; use[g].v[1] += r.mem; use[g].v[2] += r.gpu; }
      }
    }
    // the order these outcomes give; the turns before `first` are final
    const uint64_t l0 = e->launches;
    rc = fs_order(e, max_depth, use, &first, &ms_order); if (rc) return rc;
    st0.kernel_launches += e->launches - l0;
    st0.ms_total += ms_order;
    if (first >= G) break;
    if (first <= d) return fail(e, GROVE_ERR_STATE, "fair-share order: the fixed point did not advance");
    // the node table at `first`: what the turns from there on took goes back (the same gangs in either order)
    std::vector<std::pair<uint32_t, Res>> back;
    for (uint32_t p = first; p < G; ++p) {
      const uint32_t g = order[p];
      if (snap.status[g].state != GROVE_GANG_ADMITTED) continue;
      for (const grove_placement_t& x : pl[g]) {
        const grove_clique_t& q = snap.cliques[x.clique];
        back.push_back({e->inv[x.node], Res{q.req_cpu_milli, q.req_mem_mib, q.req_gpu, 1}});
      }
    }
    rc = patch_nodes(e, back, st0); if (rc) return rc;
    rc = fs_take_order(e, first, order); if (rc) return rc;
    d = first;
  }
  restore.armed = false;
  rc = restore.put_back(); if (rc) return rc;
  // the outputs: placements grouped by gang in submission order
  std::vector<grove_placement_t> place;
  uint32_t admitted = 0, rejected = 0;
  for (uint32_t g = 0; g < G; ++g) {
    snap.status[g].placement_off = uint32_t(place.size());
    if (snap.status[g].state == GROVE_GANG_ADMITTED) { place.insert(place.end(), pl[g].begin(), pl[g].end()); ++admitted; }
    else if (snap.status[g].state == GROVE_GANG_REJECTED || snap.status[g].state == GROVE_GANG_BASE_REJECTED) ++rejected;
  }
  st0.gangs_admitted = admitted; st0.gangs_rejected = rejected;
  rc = publish_reclaim(e, snap.status, place, std::vector<std::vector<grove_placement_t>>(G), snap.sstat, st0, {}, stats);
  if (rc) return rc;
  e->fs_order = std::move(order);
  e->fs_stats = grove_fair_share_stats_t{iterations, uint32_t(std::min<uint64_t>(rerun, UINT32_MAX))};
  e->fs_have_order = true;
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// Consolidation (include/grove_place.h "consolidation"; DESIGN.md section 1; kernels in consolidate.cuh).  The ordinary pass, then
// per target b: the device keeps F aside and builds W from the running gangs' CSR, sums b's capacities per domain over both
// (k_fence_have) and ranks the qualifying domains (k_consol_rank).  A try is a one-gang cycle over the masked W; when b fits, the
// rows of F at its nodes come back, the displaced set is chosen here, F' is patched in and X's spec rows run as one cycle.  The
// node table stays on the device throughout: a rolled-back try is a copy of F back into place.
// ---------------------------------------------------------------------------------------------
int32_t grove_run_cycle_consolidate(grove_engine_t* e, const uint32_t* targets, uint32_t n_targets, const uint32_t* spec_of,
                                    const grove_running_gang_t* running, uint32_t n_running, const grove_holding_t* holdings,
                                    uint32_t n_holdings, grove_cycle_stats_t* stats) {
  if (!e || (n_targets && !targets) || (n_running && (!running || !spec_of)) || (n_holdings && !holdings)) return GROVE_ERR_INVALID_ARG;
  if (e->sp_members) return refuse_spread(e, "grove_run_cycle_consolidate");
  if (e->qu_members) return refuse_queues(e, "grove_run_cycle_consolidate");
  if (!e->fc_gangs.empty()) return refuse_fences(e, "grove_run_cycle_consolidate");
  if (e->bp_members) return refuse_binpack(e, "grove_run_cycle_consolidate");
  if (e->im_enrolled) return refuse_imex(e, "grove_run_cycle_consolidate");
  NoDiagnosis no_diag{e};
  if (e->wide) return refuse_wide(e, "grove_run_cycle_consolidate");
  if (n_targets > GROVE_MAX_CONSOLIDATE_TARGETS) return fail(e, GROVE_ERR_LIMIT, "grove_run_cycle_consolidate: more than GROVE_MAX_CONSOLIDATE_TARGETS targets");
  int32_t rc = check_ready(e);
  if (rc) return rc;
  const uint32_t G = e->G, N = e->N, nblk = (N + 255) / 256;
  std::vector<uint8_t> role(G, 0);   // 1: a target, 2: a spec row
  for (uint32_t k = 0; k < n_targets; ++k) {
    if (targets[k] >= G) return fail(e, GROVE_ERR_INVALID_ARG, "grove_run_cycle_consolidate: target out of range");
    if (role[targets[k]]) return fail(e, GROVE_ERR_INVALID_ARG, "grove_run_cycle_consolidate: a target is named twice");
    role[targets[k]] = 1;
  }
  for (uint32_t r = 0; r < n_running; ++r) {
    const uint32_t s = spec_of[r];
    if (s == GROVE_NONE_U32) continue;
    if (s >= G) return fail(e, GROVE_ERR_INVALID_ARG, "grove_run_cycle_consolidate: spec row out of range");
    if (role[s] == 1) return fail(e, GROVE_ERR_INVALID_ARG, "grove_run_cycle_consolidate: a spec row is also a target");
    if (role[s] == 2) return fail(e, GROVE_ERR_INVALID_ARG, "grove_run_cycle_consolidate: a spec row is named twice");
    if (!(e->gangs[s].flags & GROVE_GANG_GATED)) return fail(e, GROVE_ERR_INVALID_ARG, "grove_run_cycle_consolidate: a spec row must carry GROVE_GANG_GATED");
    role[s] = 2;
  }
  rc = check_running(e, running, n_running, holdings, n_holdings);
  if (rc) return rc;
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  ReclaimCsr csr{};
  rc = upload_running(e, running, n_running, holdings, &csr);
  if (rc) return rc;

  // 1. the ordinary pass
  grove_cycle_stats_t st0{};
  rc = grove_run_cycle(e, &st0);
  if (rc) return rc;
  Snapshot snap;
  rc = snapshot(e, &snap);
  if (rc) return rc;
  const std::vector<grove_gang_t>& gangs = snap.gangs;
  std::vector<uint32_t> order(targets, targets + n_targets);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {   // rank order: priority desc, index asc
    return gangs[a].priority != gangs[b].priority ? gangs[a].priority > gangs[b].priority : a < b;
  });
  std::vector<uint8_t> gone(std::max<uint32_t>(n_running, 1), 1);   // not movable, or moved this cycle
  for (uint32_t r = 0; r < n_running; ++r) gone[r] = spec_of[r] == GROVE_NONE_U32;
  auto movable = [&](int32_t p) {   // is M (the standing movable gangs of priority <= p) non-empty?
    for (uint32_t r = 0; r < n_running; ++r) if (!gone[r] && running[r].priority <= p) return true;
    return false;
  };
  std::vector<grove_move_t> moves;
  std::vector<std::vector<grove_placement_t>> extra(G);   // placements of the consolidated targets and the moved spec rows
  bool any = false;
  for (uint32_t b : order) any |= snap.status[b].state == GROVE_GANG_REJECTED && movable(gangs[b].priority);
  if (any) {
    CU_TRY(e, cudaMemcpyAsync(e->d_rc_base.p, e->d_nres.p, sizeof(uint4) * e->Npad, cudaMemcpyDeviceToDevice, e->stream));
    Restore restore{e, &snap, nullptr, nullptr};
    CU_TRY(e, e->d_cs_view.ensure(e->Npad)); CU_TRY(e, e->d_cs_rank.ensure(1 + 2 * kConsolTries)); CU_TRY(e, e->d_cs_zero.ensure(1));
    CU_TRY(e, cudaMemsetAsync(e->d_cs_zero.p, 0, sizeof(uint32_t), e->stream));   // k_fence_have's gang index and offset: 0
    // running gangs by node (caller order), for the choice of the displaced set
    const RunningByNode at = running_by_node(N, running, n_running, holdings);
    std::vector<int32_t> slot(N, -1);   // node (caller order) -> its row in `rows` during a try
    for (uint32_t b : order) {
      const int32_t p = gangs[b].priority;
      if (snap.status[b].state != GROVE_GANG_REJECTED || !movable(p)) continue;
      // 2. b as a submission of its own (anchor pinned to the ordinary pass's, no gating); F aside, W = F + what M holds
      Sub bsub;
      const grove_gang_t& x = add_gang(e, snap, b, bsub);
      rc = submit_sub(e, bsub); if (rc) return rc;
      CU_TRY(e, cudaMemcpyAsync(e->d_rc_gone.p, gone.data(), gone.size(), cudaMemcpyHostToDevice, e->stream));
      k_consol_view<<<nblk, 256, 0, e->stream>>>(e->d_nres.p, e->d_rc_real.p, e->d_cs_view.p, csr, N, p);
      CU_TRY(e, cudaGetLastError());
      st0.kernel_launches += 1;
      // 3. the candidate domains
      std::vector<std::pair<uint32_t, uint32_t>> tries;
      if (x.level == GROVE_LEVEL_NONE) {
        tries.push_back({0u, N});
      } else {
        rc = build_ginfo(e); if (rc) return rc;
        const size_t words = size_t(x.n_cliques) * e->n_dom[x.level];
        CU_TRY(e, e->d_cs_have.ensure(std::max<size_t>(2 * words, 1)));
        CU_TRY(e, cudaMemsetAsync(e->d_cs_have.p, 0, sizeof(uint32_t) * 2 * words, e->stream));
        Topo tf = make_topo(e), tw = tf;
        tw.nres = e->d_cs_view.p;
        const Tables tb = make_tables(e);
        k_fence_have<<<dim3(e->Npad / 256, 1), 256, 0, e->stream>>>(tf, tb, e->d_cs_zero.p, e->d_cs_zero.p, e->d_cs_have.p);
        k_fence_have<<<dim3(e->Npad / 256, 1), 256, 0, e->stream>>>(tw, tb, e->d_cs_zero.p, e->d_cs_zero.p, e->d_cs_have.p + words);
        k_consol_rank<<<1, 1024, 0, e->stream>>>(tf, tb, 0u, e->inv[x.anchor_node], e->d_cs_have.p, e->d_cs_have.p + words, e->d_cs_rank.p);
        CU_TRY(e, cudaGetLastError());
        st0.kernel_launches += 3;
        uint32_t rk[1 + 2 * kConsolTries];
        CU_TRY(e, cudaMemcpyAsync(rk, e->d_cs_rank.p, sizeof(rk), cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(e, cudaStreamSynchronize(e->stream));
        for (uint32_t t = 0; t < rk[0]; ++t) tries.push_back({rk[1 + 2 * t], rk[2 + 2 * t]});
      }
      bool committed = false, b_loaded = true;
      for (const auto& [lo, hi] : tries) {
        // 4. evaluate b against W with every node outside D unschedulable
        if (!b_loaded) { rc = submit_sub(e, bsub); if (rc) return rc; b_loaded = true; }
        k_consol_mask<<<nblk, 256, 0, e->stream>>>(e->d_cs_view.p, e->d_nres.p, N, lo, hi);
        CU_TRY(e, cudaGetLastError());
        grove_cycle_stats_t stb{};
        rc = grove_run_cycle(e, &stb); if (rc) return rc;
        accumulate(st0, stb); st0.kernel_launches += 1;
        const grove_gang_status_t sb = e->h_status.p[0];
        if (sb.state != GROVE_GANG_ADMITTED) continue;
        std::vector<grove_scope_status_t> ssb;
        rc = sub_scope_domains(e, bsub, ssb); if (rc) return rc;
        // b's usage, and the rows of F at its nodes
        std::vector<uint32_t> nodes_b; std::vector<Res> use, rows;
        std::vector<grove_placement_t> plb;
        placed(e, snap, bsub, 0, nodes_b, use, plb);
        rc = read_rows(e, nodes_b, rows, st0); if (rc) return rc;
        for (size_t j = 0; j < nodes_b.size(); ++j) slot[nodes_b[j]] = int32_t(j);
        // the displaced set: node by node, while F plus what X holds does not cover U, the victim rule of the reclaim pass over M
        std::vector<uint32_t> X;
        std::vector<uint8_t> in_x(std::max<uint32_t>(n_running, 1), 0);
        for (size_t j = 0; j < nodes_b.size(); ++j) {
          while (!rows[j].covers(use[j])) {
            const uint32_t v = choose_victim(at, nodes_b[j], running, [&](uint32_t r) { return !gone[r] && !in_x[r] && running[r].priority <= p; });
            if (v == GROVE_NONE_U32) return fail(e, GROVE_ERR_STATE, "consolidation: a target's node cannot be covered");
            in_x[v] = 1; X.push_back(v);
            for (uint32_t h = 0; h < running[v].n_holdings; ++h) {
              const grove_holding_t& y = holdings[running[v].holding_off + h];
              if (slot[y.node] >= 0) rows[slot[y.node]].add(held(y));
            }
          }
        }
        for (uint32_t n : nodes_b) slot[n] = -1;
        // F' = F + what X holds - U, patched into a copy of F
        {
          std::vector<std::pair<uint32_t, Res>> d;   // (sorted node, change)
          for (size_t j = 0; j < nodes_b.size(); ++j) { Res c; c.add(use[j], -1); d.push_back({e->inv[nodes_b[j]], c}); }
          for (uint32_t r : X)
            for (uint32_t h = 0; h < running[r].n_holdings; ++h) {
              const grove_holding_t& y = holdings[running[r].holding_off + h];
              d.push_back({e->inv[y.node], held(y)});
            }
          CU_TRY(e, cudaMemcpyAsync(e->d_nres.p, e->d_rc_real.p, sizeof(uint4) * e->Npad, cudaMemcpyDeviceToDevice, e->stream));
          rc = patch_nodes(e, d, st0); if (rc) return rc;
        }
        // relocate X: its spec rows as one sequential pass (running priority desc, running index asc), each with its own anchor
        std::vector<uint32_t> xs(X);
        std::sort(xs.begin(), xs.end(), [&](uint32_t a, uint32_t c) { return running[a].priority != running[c].priority ? running[a].priority > running[c].priority : a < c; });
        Sub xsub;
        for (uint32_t r : xs) {
          grove_gang_t& y = add_gang(e, snap, spec_of[r], xsub);
          y.priority = running[r].priority; y.flags &= uint16_t(~GROVE_GANG_GATED);
        }
        std::vector<grove_scope_status_t> ssx;
        if (!xs.empty()) {
          rc = submit_sub(e, xsub); if (rc) return rc;
          b_loaded = false;
          grove_cycle_stats_t stx{};
          rc = grove_run_cycle(e, &stx); if (rc) return rc;
          accumulate(st0, stx);
          bool all = true;
          for (uint32_t k = 0; k < xs.size(); ++k) all &= e->h_status.p[k].state == GROVE_GANG_ADMITTED;
          if (!all) continue;   // rolled back: the next try starts from the view again, and F is still aside
          rc = sub_scope_domains(e, xsub, ssx); if (rc) return rc;
        }
        // commit: the device table is F' minus the relocated gangs' usage
        grove_gang_status_t ob = sb;
        ob.reserved0 = GROVE_STATUS_CONSOLIDATED;
        merge_gang(snap, bsub, 0, ob, ssb);
        extra[b] = std::move(plb);
        for (uint32_t k = 0; k < xs.size(); ++k) {
          std::vector<uint32_t> nodes_x; std::vector<Res> use_x;
          placed(e, snap, xsub, k, nodes_x, use_x, extra[xsub.ids[k]]);
          grove_gang_status_t o = e->h_status.p[k];
          o.reserved0 = GROVE_STATUS_MOVED;
          merge_gang(snap, xsub, k, o, ssx);
        }
        for (uint32_t r : X) { gone[r] = 1; moves.push_back(grove_move_t{r, b}); }
        st0.gangs_admitted += 1 + uint32_t(X.size()); st0.gangs_rejected -= 1;
        committed = true;
        break;
      }
      if (!committed) {   // every try rolled back: F back into place
        CU_TRY(e, cudaMemcpyAsync(e->d_nres.p, e->d_rc_real.p, sizeof(uint4) * e->Npad, cudaMemcpyDeviceToDevice, e->stream));
      }
    }
    // the handle goes back to the caller's submission; the device table is F after every commit
    restore.armed = false;
    rc = restore.put_back(); if (rc) return rc;
  }
  st0.kernel_launches += 1;   // k_reclaim_check
  rc = publish_reclaim(e, snap.status, snap.place, extra, snap.sstat, st0, {}, stats);
  if (rc) return rc;
  e->moves = std::move(moves);
  return GROVE_OK;
}

int32_t grove_get_moves(grove_engine_t* e, grove_move_t* out, uint32_t cap, uint32_t* n_out) {
  if (!e || !n_out) return GROVE_ERR_INVALID_ARG;
  if (!e->have_results) return fail(e, GROVE_ERR_STATE, "no completed cycle");
  *n_out = uint32_t(e->moves.size());
  if (!out) return GROVE_OK;
  if (cap < e->moves.size()) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  std::memcpy(out, e->moves.data(), sizeof(grove_move_t) * e->moves.size());
  return GROVE_OK;
}

// ---------------------------------------------------------------------------------------------
// Multi-GPU score pass (BASELINE.json north_star: "the node-state table shards across GPUs only when the synthetic cluster
// exceeds single-GPU capacity, with one NCCL all-reduce over NVLink of the per-shard gang-feasibility bitmasks").  The object
// that outgrows a GPU is the Q x N score matrix, so THAT is what shards: every rank holds the (small) node table, builds K1 +
// K2 for its node range only -- cut at top-level domain boundaries, so every candidate domain of a gang lies in one shard --
// and contributes one int32[G + Q] vector of per-shard feasibility counts and capacity counts; their SUM over the ranks (the
// one collective, issued by the caller on its own communicator) says which gangs cannot fit anywhere in the snapshot.
// ---------------------------------------------------------------------------------------------
int32_t grove_shard_range(grove_engine_t* e, uint32_t* lo, uint32_t* hi) {
  if (!e || !lo || !hi) return GROVE_ERR_INVALID_ARG;
  if (!e->nodes_loaded) return fail(e, GROVE_ERR_STATE, "no node snapshot loaded");
  *lo = e->shard_lo; *hi = e->shard_hi;
  return GROVE_OK;
}

int32_t grove_run_score_pass(grove_engine_t* e, float* ms) {
  if (!e) return GROVE_ERR_INVALID_ARG;
  if (ms) *ms = 0.f;
  if (e->wide) return refuse_wide(e, "grove_run_score_pass");
  int32_t rc = cycle_begin(e);   // allocations, derived gang tables, state resets: the pass leaves the handle ready for a cycle
  if (rc) return rc;
  CycleGuard guard{e};
  e->score_pass_valid = false; e->score_valid = false;
  if (e->G == 0 || e->Q == 0) { e->in_cycle = false; guard.armed = false; return GROVE_OK; }
  const Topo tp = make_topo(e); const Tables tb = make_tables(e); const Relax rx = make_relax(e);
  const uint32_t c0 = e->shard_lo >> 4, c1 = (e->shard_hi + 15u) >> 4, cpr = c1 > c0 ? c1 - c0 : 0u;
  const size_t tstride = size_t(cpr) << 4;
  if (e->d_T.ensure(std::max<size_t>(size_t(e->Q) * tstride, 1)) != cudaSuccess) { (void)cudaGetLastError(); return fail(e, GROVE_ERR_OOM, "score matrix shard does not fit in device memory"); }
  CU_TRY(e, cudaEventRecord(e->ev_s0, e->stream));
  rc = build_cap_tables(e, tp, tb, rx);   // K1: fit bitmap + capacities of every signature over the loaded snapshot
  if (rc) return rc;
  CU_TRY(e, e->d_F0.ensure(std::max<size_t>(size_t(e->n_sigs) * e->words, 1)));
  CU_TRY(e, cudaMemcpyAsync(e->d_F0.p, e->d_F.p, sizeof(uint32_t) * size_t(e->n_sigs) * e->words, cudaMemcpyDeviceToDevice, e->stream));
  if (cpr) k_score<<<dim3(1, std::min<uint32_t>(e->Q, 65535u)), 256, 0, e->stream>>>(tp, tb, e->d_F0.p, e->d_T.p, e->Q, c0, cpr, tstride);   // K2, this shard's columns
  CU_TRY(e, cudaGetLastError());
  CU_TRY(e, cudaEventRecord(e->ev_s1, e->stream));
  CU_TRY(e, cudaEventSynchronize(e->ev_s1));
  float t = 0; cudaEventElapsedTime(&t, e->ev_s0, e->ev_s1);
  if (ms) *ms = t;
  e->last.ms_score = t;
  e->in_cycle = false; guard.armed = false;
  e->score_pass_valid = true; e->t_c0 = c0; e->t_cpr = cpr;
  return GROVE_OK;
}

int32_t grove_shard_summary_device(grove_engine_t* e, void* d_out, uint32_t cap_words) {
  if (!e || !d_out) return GROVE_ERR_INVALID_ARG;
  if (e->wide) return refuse_wide(e, "grove_shard_summary_device");
  if (!e->score_pass_valid) return fail(e, GROVE_ERR_STATE, "no score pass over the loaded snapshot");
  if (cap_words < e->G + e->Q) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  const Topo tp = make_topo(e); const Tables tb = make_tables(e);
  CU_TRY(e, e->d_sig_sum.ensure(std::max<uint32_t>(e->n_sigs, 1)));
  if (e->n_sigs) k_sig_range_sum<<<e->n_sigs, 256, 0, e->stream>>>(tp, e->d_cap8.p, e->shard_lo, e->shard_hi, e->d_sig_sum.p);
  k_shard_summary<<<std::max(1u, std::min((e->G * 32 + 255) / 256, e->n_sm * 8u)), 256, 0, e->stream>>>(tp, tb, e->d_cap8.p, e->d_capsum.p, e->d_sig_sum.p, e->shard_lo, e->shard_hi,
                                                                                                   static_cast<int32_t*>(d_out));
  CU_TRY(e, cudaGetLastError());
  CU_TRY(e, cudaStreamSynchronize(e->stream));   // the caller's collective runs on its own stream
  return GROVE_OK;
}

// ---- introspection for parity tests ----
int32_t grove_debug_get_perm(grove_engine_t* e, uint32_t* sorted_to_caller, uint32_t cap) {
  if (!e || !sorted_to_caller) return GROVE_ERR_INVALID_ARG;
  if (!e->nodes_loaded) return fail(e, GROVE_ERR_STATE, "no node snapshot loaded");
  if (cap < e->N) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  std::memcpy(sorted_to_caller, e->perm.data(), sizeof(uint32_t) * e->N);
  return GROVE_OK;
}

// K1 over the cycle-start snapshot is recomputed on request (the engine's own table follows the committed state)
int32_t grove_debug_get_fit_row(grove_engine_t* e, uint32_t clique, uint32_t* words, uint32_t cap_words) {
  if (!e || !words) return GROVE_ERR_INVALID_ARG;
  if (!e->have_results || clique >= e->Q) return fail(e, GROVE_ERR_STATE, "no completed cycle / bad clique");
  const uint32_t w = (e->N + 31) / 32;
  if (cap_words < w) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  { int32_t rc = grove_build_score_matrix(e, nullptr); if (rc) return rc; }
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  // the fit row of the cycle-start snapshot is the support of the score row
  std::vector<uint8_t> row(e->N);
  CU_TRY(e, cudaMemcpy(row.data(), e->d_T.p + size_t(clique) * e->Npad, e->N, cudaMemcpyDeviceToHost));
  std::memset(words, 0, sizeof(uint32_t) * w);
  for (uint32_t n = 0; n < e->N; ++n) if (row[n]) words[n >> 5] |= 1u << (n & 31);
  return GROVE_OK;
}

int32_t grove_debug_get_score_row(grove_engine_t* e, uint32_t clique, uint8_t* bytes, uint32_t cap_bytes) {
  if (!e || !bytes) return GROVE_ERR_INVALID_ARG;
  if (e->score_pass_valid) {   // after a score pass: this handle's shard of the row, zeros outside it
    if (clique >= e->Q) return fail(e, GROVE_ERR_STATE, "bad clique");
    if (cap_bytes < e->N) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
    CU_TRY(e, cudaSetDevice(e->cfg.device));
    std::memset(bytes, 0, e->N);
    const size_t first = size_t(e->t_c0) << 4, width = size_t(e->t_cpr) << 4;
    const size_t cnt = first < e->N ? std::min<size_t>(width, e->N - first) : 0;
    if (cnt) CU_TRY(e, cudaMemcpy(bytes + first, e->d_T.p + size_t(clique) * width, cnt, cudaMemcpyDeviceToHost));
    return GROVE_OK;
  }
  if (!e->have_results || clique >= e->Q) return fail(e, GROVE_ERR_STATE, "no completed cycle / bad clique");
  if (cap_bytes < e->N) return fail(e, GROVE_ERR_LIMIT, "output buffer too small");
  { int32_t rc = grove_build_score_matrix(e, nullptr); if (rc) return rc; }
  CU_TRY(e, cudaSetDevice(e->cfg.device));
  CU_TRY(e, cudaMemcpy(bytes, e->d_T.p + size_t(clique) * e->Npad, e->N, cudaMemcpyDeviceToHost));
  return GROVE_OK;
}

}  // extern "C"
