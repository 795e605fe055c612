/*
 * grove_place.h -- C ABI of libgrove_place.so, the H100 (sm_90a) gang-placement engine.
 *
 * This is the drop-in boundary for the scheduling-cycle hot path named in
 * BASELINE.json (resource fit -> topology score -> all-or-nothing gang
 * admission).  The reference (ai-dynamo/grove @ 08ad3b37) ships no scheduler
 * and no FFI; what it pins is the INPUT contract (the PodGang CRD) and the
 * plug-in seam a scheduler hangs off.  Every entry point below names the
 * reference interface it stands in for:
 *
 *   grove_engine_create / _destroy   scheduler.Backend.Init()
 *                                    operator/internal/scheduler/types.go:41-43
 *   grove_load_nodes / _update_nodes node snapshot a scheduler session takes of
 *                                    Node.status.allocatable + topology labels;
 *                                    generator: operator/hack/infra_manager/kwok.py:55-117
 *                                    level schema: operator/internal/scheduler/kai/topology.go:103-135
 *   grove_submit_gangs               scheduler.Backend.SyncPodGang(ctx, *PodGang)
 *                                    operator/internal/scheduler/types.go:45-47
 *                                    payload = PodGangSpec, scheduler/api/core/v1alpha1/podgang.go:51-131
 *   grove_run_cycle                  the scheduling cycle itself (absent from the
 *                                    reference tree; KAI-Scheduler v0.14.0, operator/go.mod:11).
 *                                    Result = the SEQUENTIAL pass: gangs one at a time in (priority desc,
 *                                    submission index asc) order, each against the state the earlier ones left
 *                                    (PriorityClassName, podgang.go:62-64); the engine reaches it by parallel
 *                                    relaxation (DESIGN.md section 1), bit-identical to oracle/grove_oracle_seq.c
 *   grove_get_placements             Pod.spec.nodeName bindings, counted back by
 *                                    operator/internal/controller/podclique/reconcilestatus.go:134-141
 *   grove_get_gang_status            PodGangStatus{Phase,PlacementScore},
 *                                    scheduler/api/core/v1alpha1/podgang.go:141-150,182-190
 *   grove_get_scope_domains          the topology domain chosen for every TopologyConstraintGroupConfig
 *                                    (podgang.go:120-131) -- what a binder needs to explain a placement
 *   grove_diagnose                   why a REJECTED gang did not fit: the message of the Unschedulable
 *                                    PodScheduled condition a pending pod carries
 *
 * cgo rules honoured: plain pointers + sizes only, every input array is copied
 * before the call returns (no Go pointer is retained), outputs go to
 * caller-owned buffers, there are no callbacks.  A handle is NOT thread-safe:
 * one cycle in flight per handle; distinct handles are independent.
 *
 * There is no CPU fallback behind this ABI.  If no CUDA device is usable
 * grove_engine_create fails with GROVE_ERR_NO_DEVICE.
 */
#ifndef GROVE_PLACE_H
#define GROVE_PLACE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GROVE_ABI_VERSION 2u

#define GROVE_MAX_LEVELS 4u          /* topology levels, index 0 = broadest (GREP-244 README.md:143) */
#define GROVE_LEVEL_NONE 0xFFu       /* "no pack constraint at this scope" */
#define GROVE_DOM_ABSENT 0xFFFFFFFFu /* node lacks the label of that level (GREP-244 README.md:65) */
#define GROVE_NONE_U32 0xFFFFFFFFu
#define GROVE_MAX_GANG_PODS 128u     /* sum of replicas over a gang's cliques */
#define GROVE_MAX_WIDE_GANG_PODS 2048u /* sum of replicas over a gang's cliques, wide submissions (grove_submit_gangs_wide) */
#define GROVE_MAX_GANG_CLIQUES 32u
#define GROVE_MAX_GANG_SCOPES 32u
#define GROVE_MAX_NODES (1u << 24)

/* error codes (all entry points return 0 on success, <0 on error) */
#define GROVE_OK 0
#define GROVE_ERR_INVALID_ARG (-1)
#define GROVE_ERR_NO_DEVICE (-2)
#define GROVE_ERR_CUDA (-3)
#define GROVE_ERR_LIMIT (-4)
#define GROVE_ERR_STATE (-5)
#define GROVE_ERR_OOM (-6)

/* ---- node-state table: 32 B per node -------------------------------------------------------- */
#define GROVE_NODE_SCHEDULABLE 0x1u               /* not cordoned / Ready */
#define GROVE_NODE_CLASS_SHIFT 8u                 /* bits 8..11: selector class id 0..15 */
#define GROVE_NODE_CLASS_MASK 0xF00u
typedef struct grove_node {
  uint32_t free_cpu_milli; /* allocatable - requested, millicores */
  uint32_t free_mem_mib;   /* MiB */
  uint16_t free_gpu;       /* nvidia.com/gpu */
  uint16_t free_pods;      /* pod slots left */
  uint32_t flags;          /* GROVE_NODE_SCHEDULABLE | class << 8 */
  uint32_t dom[GROVE_MAX_LEVELS]; /* interned label value per level, or GROVE_DOM_ABSENT */
} grove_node_t;

/* ---- gang-request tables -------------------------------------------------------------------- */
/* one PodGroup (PodClique) of a PodGang: podgang.go:75-91 */
typedef struct grove_clique {
  uint32_t req_cpu_milli; /* per-pod request */
  uint32_t req_mem_mib;
  uint16_t req_gpu;
  uint8_t min_replicas;   /* PodGroup.MinReplicas: gang-guaranteed */
  uint8_t replicas;       /* len(PodReferences) >= min_replicas: surplus is best effort (podgang.go:80-83) */
  uint16_t class_mask;    /* bit c set <=> node selector class c is acceptable (nodeSelector+tolerations) */
  uint8_t level;          /* PodGroup.TopologyConstraint Required level index, or GROVE_LEVEL_NONE */
  uint8_t scope;          /* bits 0..4: index of the owning scope inside the gang (non-decreasing over the gang's
                             cliques); bits 5..7: Preferred level index + 1, 0 = none (GROVE_CLIQUE_SCOPE_PREF) */
} grove_clique_t;
#define GROVE_CLIQUE_SCOPE(x) ((uint32_t)(x) & 0x1Fu)
#define GROVE_CLIQUE_PREFERRED(x) ((((uint32_t)(x)) >> 5) ? (((uint32_t)(x)) >> 5) - 1u : (uint32_t)GROVE_LEVEL_NONE)
#define GROVE_CLIQUE_SCOPE_PREF(scope, pref) \
  ((uint8_t)(((scope) & 0x1Fu) | (((pref) == GROVE_LEVEL_NONE ? 0u : (uint32_t)(pref) + 1u) << 5)))

/* one TopologyConstraintGroupConfig (podgang.go:120-131), or the implicit scope of loose PodGroups */
typedef struct grove_scope {
  uint16_t first_clique;  /* relative to the gang's clique_off */
  uint16_t n_cliques;
  uint8_t level;          /* Required level index, or GROVE_LEVEL_NONE */
  uint8_t preferred1;     /* Preferred level index + 1 (deeper than `level`), 0 = none: zero-filled records
                             written against the earlier layout keep their meaning */
  uint8_t reserved[2];
} grove_scope_t;

#define GROVE_GANG_GATED 0x1u /* pods still carry the grove.io/podgang-pending-creation gate: skip */
typedef struct grove_gang {
  uint32_t clique_off;    /* into the cliques array of the same submission */
  uint32_t scope_off;     /* into the scopes array */
  uint16_t n_cliques;
  uint16_t n_scopes;
  int32_t priority;       /* PriorityClass value (PodGangSpec.PriorityClassName resolved, podgang.go:62-64):
                             gangs are placed strictly in (priority desc, submission index asc) order */
  uint32_t anchor_node;   /* caller's node index to score distance against (ReuseReservationRef hint,
                             podgang.go:66-71), or GROVE_NONE_U32 = engine derives hash(gang index) % N */
  uint32_t base_gang;     /* scaled gang: index of its base gang in this submission (gated behind it,
                             pod/syncflow.go:319-358), or GROVE_NONE_U32.  Considered at its own turn: admitted
                             only if the base gang was admitted EARLIER in this cycle's order, else
                             GROVE_GANG_BASE_REJECTED (it waits for the next cycle, like its gated pods do) */
  uint8_t level;          /* PodGangSpec.TopologyConstraint Required level index, or GROVE_LEVEL_NONE */
  uint8_t preferred;      /* PackConstraint.Preferred level index (podgang.go:110-117): best effort, tried before
                             falling back level by level up to `level`; deeper than `level`; or GROVE_LEVEL_NONE */
  uint16_t flags;
  uint32_t reserved;
} grove_gang_t;

/* ---- outputs -------------------------------------------------------------------------------- */
/* one bound pod: the r-th entry of a clique binds that clique's r-th PodReference */
typedef struct grove_placement {
  uint32_t clique; /* global clique index in the submission */
  uint32_t node;   /* caller's node index (position in the grove_load_nodes array) */
} grove_placement_t;

#define GROVE_GANG_PENDING 0u       /* never seen by a cycle */
#define GROVE_GANG_ADMITTED 1u      /* all MinReplicas bound (Scheduled=True) */
#define GROVE_GANG_REJECTED 2u      /* no feasible domain at its turn: Unschedulable, nothing bound */
#define GROVE_GANG_GATED_SKIP 3u    /* GROVE_GANG_GATED set */
#define GROVE_GANG_BASE_REJECTED 4u /* base gang not admitted before this gang's turn */
typedef struct grove_gang_status {
  uint8_t state;
  uint8_t level;           /* level of the domain the whole gang was packed into (its Required level, or the deeper
                              Preferred level that held), GROVE_LEVEL_NONE = the whole cluster / not admitted */
  uint16_t reserved0;      /* flags: GROVE_STATUS_PREEMPTOR = admitted by the reclaim pass of grove_run_cycle_preempt,
                              GROVE_STATUS_SPREAD_SKEWED = a SOFT spread member placed outside its allowed domains,
                              GROVE_STATUS_FENCING = a REJECTED fencing gang whose fence held (grove_set_fences),
                              GROVE_STATUS_OVER_LIMIT / GROVE_STATUS_SURPLUS_CAPPED = a queue member held back by its queue
                              chain's limits (grove_set_queues), GROVE_STATUS_RECLAIMER = admitted by the class pass of
                              grove_run_cycle_reclaim_queues (or the reclaim pass of
                              grove_run_cycle_reclaim_preempt_queues, whose preempt pass sets GROVE_STATUS_PREEMPTOR),
                              GROVE_STATUS_SURPLUS_ONLY = with GROVE_STATUS_PREEMPTOR, admitted by the surplus pass of
                              grove_run_cycle_preempt_elastic; else 0 */
  uint16_t score_num;      /* PlacementScore = score_num / score_den (podgang.go:187-189): over the gang, its scopes and
                              its cliques that carry a pack constraint, (levels honoured) / (levels asked for), where
                              asked = Preferred if set else Required; 1/1 when nothing was asked or everything held;
                              0/0 when not admitted */
  uint16_t score_den;
  uint32_t n_pods;         /* pods bound (>= sum MinReplicas when admitted) */
  uint32_t placement_off;  /* first entry in grove_get_placements output */
  uint32_t domain_node;    /* caller index of the first node (topology order) of that gang domain, or GROVE_NONE_U32 */
  uint32_t reserved1[3];
} grove_gang_status_t;

/* chosen domain of one scope (same indexing as the scopes array of the submission) */
typedef struct grove_scope_status {
  uint8_t level;           /* level of the domain the scope's cliques share; GROVE_LEVEL_NONE = no own domain (packed in
                              the gang's domain) or gang not admitted */
  uint8_t reserved[3];
  uint32_t domain_node;    /* caller index of the first node (topology order) of that domain, or GROVE_NONE_U32 */
} grove_scope_status_t;

typedef struct grove_config {
  uint32_t abi_version;  /* GROVE_ABI_VERSION */
  int32_t device;        /* CUDA ordinal */
  uint32_t n_levels;     /* 1..GROVE_MAX_LEVELS */
  uint32_t window;       /* gangs beyond the settled prefix that relax concurrently; 0 = default.  A tuning knob:
                            results do not depend on it */
  uint32_t rank;         /* multi-GPU: this handle's rank ... */
  uint32_t world;        /* ... of `world` handles driving the same cycle; 0 or 1 = single GPU */
  uint32_t reserved[2];
} grove_config_t;

typedef struct grove_cycle_stats {
  uint32_t rounds;           /* relaxation rounds the engine took (an implementation figure, not a result) */
  uint32_t gangs_admitted;
  uint32_t gangs_rejected;   /* REJECTED + BASE_REJECTED */
  uint32_t pods_bound;
  uint64_t pairs_evaluated;  /* (clique,node) pairs through fit+score (K1/K2 over the cycle-start snapshot) */
  uint64_t kernel_launches;
  uint64_t evaluations;      /* gang evaluations (K3) over all rounds; >= gangs considered */
  float ms_fit;              /* CUDA-event device time: K1 + capacity tables */
  float ms_score;            /* K2 (beside the relaxation, on its own stream) */
  float ms_admit;            /* relaxation rounds: evaluate / publish / detect / settle */
  float ms_commit;           /* output compaction */
  float ms_total;            /* first launch -> last kernel done */
  float reserved;
} grove_cycle_stats_t;

typedef struct grove_engine grove_engine_t;

int32_t grove_engine_create(const grove_config_t* cfg, grove_engine_t** out);
void grove_engine_destroy(grove_engine_t* e);
const char* grove_last_error(grove_engine_t* e);
uint32_t grove_abi_version(void);

/* full snapshot; copied (host -> device) before return */
int32_t grove_load_nodes(grove_engine_t* e, const grove_node_t* nodes, uint32_t n);
/* churn deltas: replace free_* and flags of nodes idx[i] (labels must not change) */
int32_t grove_update_nodes(grove_engine_t* e, const uint32_t* idx, const grove_node_t* recs, uint32_t n);
/* read back the engine's current node table in caller order (after commits) */
int32_t grove_get_nodes(grove_engine_t* e, grove_node_t* out, uint32_t cap);

int32_t grove_submit_gangs(grove_engine_t* e, const grove_gang_t* gangs, uint32_t n_gangs,
                           const grove_clique_t* cliques, uint32_t n_cliques,
                           const grove_scope_t* scopes, uint32_t n_scopes);

/* ---- wide submissions: PodGangs of up to GROVE_MAX_WIDE_GANG_PODS pods ------------------------------------------
 * counts[q] replaces the 8-bit min_replicas / replicas of clique q (those fields are ignored).  Everything else is
 * validated as by grove_submit_gangs, with min_replicas <= replicas and at most GROVE_MAX_WIDE_GANG_PODS pods per gang.
 * A submission is WIDE when some gang has more than GROVE_MAX_GANG_PODS pods or some clique more than 255 replicas;
 * one within the old limits behaves exactly as if it had come through grove_submit_gangs.  A wide submission is
 * scheduled by grove_run_cycle and read back by every getter and grove_build_score_matrix; grove_run_cycle_preempt,
 * grove_run_cycle_reuse, grove_run_cycle_reuse_preempt, grove_run_score_pass and grove_shard_summary_device refuse it
 * with GROVE_ERR_LIMIT. */
typedef struct grove_clique_count {
  uint16_t min_replicas;  /* PodGroup.MinReplicas */
  uint16_t replicas;      /* len(PodReferences) >= min_replicas */
} grove_clique_count_t;
int32_t grove_submit_gangs_wide(grove_engine_t* e, const grove_gang_t* gangs, uint32_t n_gangs,
                                const grove_clique_t* cliques, const grove_clique_count_t* counts, uint32_t n_cliques,
                                const grove_scope_t* scopes, uint32_t n_scopes);

/* blocking: fit -> score -> admit -> commit; on return every gang is decided */
int32_t grove_run_cycle(grove_engine_t* e, grove_cycle_stats_t* stats);

int32_t grove_get_placements(grove_engine_t* e, grove_placement_t* out, uint32_t cap, uint32_t* n_out);
int32_t grove_get_gang_status(grove_engine_t* e, grove_gang_status_t* out, uint32_t cap);
int32_t grove_get_scope_domains(grove_engine_t* e, grove_scope_status_t* out, uint32_t cap);

/* ---- preemption / reclaim ------------------------------------------------------------------------
 * The API reserves it (PodGangConditionTypeDisruptionTarget, podgang.go:166-170: "PodGang is preempted by a higher priority
 * PodGang"; PriorityClassName podgang.go:62-64); the arithmetic is ours (DESIGN.md section 1, "Reclaim pass").  RUNNING gangs
 * (admitted by earlier cycles) are handed in with what they hold per node.  After the ordinary pass every REJECTED gang, in
 * order rank, is evaluated once more against the RECLAIM VIEW of its priority p -- free resources plus everything held by
 * running gangs of priority < p that are still standing (E(p)) -- and skipped while E(p) is empty.  If it fits, it is admitted
 * (GROVE_STATUS_PREEMPTOR) and, node by
 * node in the order of its placement, running gangs are evicted WHOLE (lowest priority first, then highest running index)
 * until the node's free resources cover what it puts there; everything an evicted gang held anywhere returns to the free
 * pool.  grove_get_victims lists (running gang, preemptor) pairs: the caller sets DisruptionTarget on them. */
typedef struct grove_holding {
  uint32_t node;          /* caller's node index */
  uint32_t cpu_milli, mem_mib;
  uint16_t gpu, pods;
} grove_holding_t;
typedef struct grove_running_gang {
  int32_t priority;
  uint32_t holding_off;   /* into the holdings array */
  uint32_t n_holdings;
  uint32_t reserved;
} grove_running_gang_t;
typedef struct grove_victim {
  uint32_t running;       /* index into the running array */
  uint32_t preemptor;     /* gang index of the submission */
} grove_victim_t;
#define GROVE_STATUS_PREEMPTOR 0x1u /* grove_gang_status_t.reserved0: admitted by the reclaim pass */
/* ordinary pass + reclaim pass; outputs through the usual getters (statuses, placements, scope domains, node table = free
 * resources after evictions and admissions).  GROVE_ERR_INVALID_ARG when a running gang's holdings lie outside the holdings
 * array, a holding lies on a node out of range, or free + the holdings of every running gang overflows a field of a node
 * record. */
int32_t grove_run_cycle_preempt(grove_engine_t* e, const grove_running_gang_t* running, uint32_t n_running,
                                const grove_holding_t* holdings, uint32_t n_holdings, grove_cycle_stats_t* stats);
int32_t grove_get_victims(grove_engine_t* e, grove_victim_t* out, uint32_t cap, uint32_t* n_out);

/* ---- elastic reclaim ------------------------------------------------------------------------------
 * The reclaim pass, shrinking running gangs to their MinReplicas before evicting any whole (DESIGN.md section 1, "Elastic
 * reclaim").  The reference pins the contract (PodGroup.MinReplicas, podgang.go:80-83: "guaranteed gang scheduling is only
 * provided for MinReplicas"); the arithmetic is ours.  Inputs are those of grove_run_cycle_preempt plus the SURPLUS PODS: one
 * record per pod of a running gang above its PodGroup's MinReplicas, a gang's pods in the order it gives them up (for Grove the
 * highest PodReference index first).  A surplus pod is part of its gang's holdings on its node and takes 1 pod slot plus its cpu,
 * mem and gpu.  F is the free table; E(p) the standing running gangs of a priority below p.  A taken surplus pod is gone, its
 * gang keeps standing.
 *   1. The ordinary pass: grove_run_cycle.
 *   2. Every priority p of a gang still REJECTED, descending, while E(p) is non-empty; its members are its REJECTED gangs in rank
 *      order, each evaluated once as grove_run_cycle_preempt evaluates it (K3, same candidate order, ordinary-pass anchor).
 *      Pass 1, only when some untaken surplus pod of E(p) stands: each member against F + the untaken surplus pods of E(p),
 *      skipped once none stands; admitted: GROVE_STATUS_PREEMPTOR | GROVE_STATUS_SURPLUS_ONLY, and it takes surplus pods only.
 *      Pass 2, the members pass 1 did not admit: each against F + what the standing gangs of E(p) still hold (holdings minus their
 *      taken pods), skipped once E(p) is empty; admitted: GROVE_STATUS_PREEMPTOR.
 *   3. The node step of an admitted g, node by node in the order its placement first names them, need = what g puts there:
 *      while F does not cover need: if F + the untaken surplus pods there of the standing gangs of E(p) covers it, take such pods
 *      one at a time until F does (the gang by the victim rule -- lowest priority, then highest running index -- then its
 *      first-listed untaken pod on the node) and stop; else evict WHOLE, by the victim rule, the next gang of E(p) that still holds
 *      something on the node: everything it still holds anywhere, its untaken surplus pods included, returns to F.  Then F -= need.
 * grove_get_victims lists the whole-gang evictions, grove_get_surplus_victims the (surplus pod, preemptor) pairs, each in
 * eviction order; a gang that lost pods is not a victim unless it was later evicted whole.  With n_surplus == 0 every output
 * equals grove_run_cycle_preempt's.  Refusals: those of grove_run_cycle_preempt, with the same codes; GROVE_ERR_INVALID_ARG for a
 * surplus pod whose running gang or node is out of range, or a (running gang, node) whose surplus pods add up to more than its
 * holdings there in cpu, mem, gpu or pods.  grove_diagnose refuses the cycle that follows.  grove_get_surplus_victims returns
 * GROVE_ERR_STATE before any cycle and 0 pairs after a cycle of any other entry. */
typedef struct grove_surplus_pod {   /* 20 B */
  uint32_t running;                  /* index into the running array */
  uint32_t node;                     /* caller's node index */
  uint32_t cpu_milli, mem_mib;
  uint16_t gpu;
  uint16_t reserved;
} grove_surplus_pod_t;
typedef struct grove_surplus_victim {
  uint32_t pod;                      /* index into the surplus array */
  uint32_t preemptor;                /* gang index of the submission */
} grove_surplus_victim_t;
#define GROVE_STATUS_SURPLUS_ONLY 0x100u /* grove_gang_status_t.reserved0: a preemptor admitted by pass 1 of
                                            grove_run_cycle_preempt_elastic (it evicted surplus pods only) */
int32_t grove_run_cycle_preempt_elastic(grove_engine_t* e, const grove_running_gang_t* running, uint32_t n_running,
                                        const grove_holding_t* holdings, uint32_t n_holdings,
                                        const grove_surplus_pod_t* surplus, uint32_t n_surplus, grove_cycle_stats_t* stats);
int32_t grove_get_surplus_victims(grove_engine_t* e, grove_surplus_victim_t* out, uint32_t cap, uint32_t* n_out);

/* ---- reservation reuse ---------------------------------------------------------------------------
 * The API names it (PodGangSpec.ReuseReservationRef, podgang.go:65-71: "During updates, an operator can suggest to reuse the
 * reservation of the previous PodGang for a newer version of the PodGang resource"); the arithmetic is ours (DESIGN.md section
 * 1, "Reservation reuse").  RUNNING gangs are handed in as for grove_run_cycle_preempt (the loaded node table does not include
 * what they hold).  replaces[g] (one entry per submitted gang) is the running gang that gang g is the new version of, or
 * GROVE_NONE_U32; a running gang is replaced by at most one gang.  The cycle is the ordinary sequential pass, except that a
 * gang g with a predecessor is evaluated against free + H_g, where the hold H_g starts as the predecessor's holdings and no other
 * gang ever sees it.  Admitted with usage U (per node and resource): free -= (U - H_g)+ and H_g = (H_g - U)+ -- the new version
 * uses its own reservation first.  Rejected, GATED_SKIP or BASE_REJECTED: nothing changes, the predecessor keeps running.  When
 * the pass ends every admitted replacement's predecessor is gone: free += H_g.  Outputs through the usual getters; the node
 * table is the free table after all that.  GROVE_ERR_INVALID_ARG when n_gangs is not the submitted count, replaces[] names a
 * running gang out of range or one twice, a holding lies on a node out of range, or free + all holds overflows a field of a
 * node record.  No reclaim pass. */
int32_t grove_run_cycle_reuse(grove_engine_t* e, const uint32_t* replaces, uint32_t n_gangs,
                              const grove_running_gang_t* running, uint32_t n_running,
                              const grove_holding_t* holdings, uint32_t n_holdings, grove_cycle_stats_t* stats);

/* ---- reuse with reclaim ---------------------------------------------------------------------------
 * Reservation reuse and the reclaim pass in one cycle (DESIGN.md section 1, "Reuse with reclaim").  Inputs as for
 * grove_run_cycle_reuse.  The ordinary pass is grove_run_cycle_reuse; every predecessor of an admitted new version is then
 * released and can never be a victim.  Every gang it left REJECTED is then reconsidered in order rank as by
 * grove_run_cycle_preempt, against free + E(p) (what the standing running gangs of a priority below p hold), skipped while E(p)
 * is empty.  A gang g with a predecessor r that still stands:
 *   - r's priority >= p: g also sees r's holdings H_r, nobody else does; admitted, it uses H_r first on every node, then evicts;
 *     r is released (not a victim) and (H_r - U)+ returns to the free table after the last gang of priority p;
 *   - r's priority < p: r is an ordinary evictable gang; admitted, g releases r first (everything it held returns at once, r is
 *     not a victim), then evicts as usual.
 * Preemptors carry GROVE_STATUS_PREEMPTOR; grove_get_victims lists (running gang, preemptor) pairs.  GROVE_ERR_INVALID_ARG for
 * the inputs grove_run_cycle_reuse rejects, with the same reasons; the overflow check covers free + the holdings of every
 * running gang. */
int32_t grove_run_cycle_reuse_preempt(grove_engine_t* e, const uint32_t* replaces, uint32_t n_gangs,
                                      const grove_running_gang_t* running, uint32_t n_running,
                                      const grove_holding_t* holdings, uint32_t n_holdings, grove_cycle_stats_t* stats);

/* ---- diagnosis of rejected gangs ------------------------------------------------------------------
 * Why each REJECTED gang of the last grove_run_cycle did not fit (DESIGN.md section 1, "Diagnosis"): the Unschedulable message
 * Kubernetes schedulers give a pending pod.  Gang g is judged against V_g = the node table the cycle left plus the usage of
 * every admitted gang ranked after g, i.e. the table the sequential pass evaluated g against.  Per clique q of g, over all N
 * nodes of V_g: nodes_fit = nodes where K1 fit(q, n) holds; every other node is counted once, under the first predicate it
 * fails in the order of the fields below; pods_fit = sum over the fit nodes of the pods of q that fit there, exactly
 * (min over resources with a request of floor(free / request), and the free pod slots).  Per gang, at its Required level l
 * (the whole cluster is one domain when it has none): domains = the level-l domains, domains_ok = those in which every clique
 * with MinReplicas > 0 finds MinReplicas pods on its own, and the verdict.  Gangs in any other state, and their cliques, get
 * all-zero records.  The cycle's outputs are not touched.  GROVE_ERR_STATE when there is no completed cycle, when the last
 * cycle was grove_run_cycle_preempt / _reuse / _reuse_preempt, or when grove_load_nodes*, grove_update_nodes or
 * grove_submit_gangs* was called since; GROVE_ERR_LIMIT when cap_g < gangs submitted or cap_q < cliques submitted. */
#define GROVE_DIAG_NONE 0u          /* the gang was not REJECTED */
#define GROVE_DIAG_CLIQUE_SHORT 1u  /* a clique's pods_fit < MinReplicas: it fits nowhere in the cluster (`clique` names it) */
#define GROVE_DIAG_NO_DOMAIN 2u     /* every clique fits the cluster, but no level-l domain holds each clique's MinReplicas */
#define GROVE_DIAG_NO_JOINT_FIT 3u  /* domains_ok > 0 (or no Required level), yet no placement holds all cliques together:
                                       shared nodes, or the Required levels of scopes / cliques inside those domains */
typedef struct grove_gang_diag {   /* 16 B */
  uint8_t verdict;        /* GROVE_DIAG_* */
  uint8_t level;          /* the gang's Required level, GROVE_LEVEL_NONE = none (0 when not REJECTED) */
  uint16_t clique;        /* GROVE_DIAG_CLIQUE_SHORT: first short clique, relative to the gang's clique_off; else 0 */
  uint32_t domains;       /* level-l domains (nodes lacking the label are in none); 1 without a Required level */
  uint32_t domains_ok;    /* domains in which every clique with MinReplicas > 0 has MinReplicas pods fitting on its own */
  uint32_t reserved;
} grove_gang_diag_t;
typedef struct grove_clique_diag {   /* 40 B */
  uint32_t nodes_fit;     /* nodes where fit(q, n) holds */
  uint32_t unschedulable; /* not schedulable */
  uint32_t selector;      /* selector class not accepted by the clique's class_mask */
  uint32_t labels;        /* lacks a label down to the deepest Required level binding the clique */
  uint32_t cpu, mem, gpu; /* free < request */
  uint32_t pods;          /* no free pod slot */
  uint64_t pods_fit;      /* sum over nodes of the pods of the clique that fit */
} grove_clique_diag_t;
int32_t grove_diagnose(grove_engine_t* e, grove_gang_diag_t* gangs, uint32_t cap_g, grove_clique_diag_t* cliques, uint32_t cap_q);

/* ---- topology spread ---------------------------------------------------------------------------------
 * The replicas of one PodCliqueSet spread over topology domains (DESIGN.md section 1, "Topology spread"; Kubernetes
 * TopologySpreadConstraint at PodGang granularity).  A spread group s has a level l_s, a max_skew >= 1 and a mode.  Each
 * submitted gang belongs to at most one group (gang_group[g], or GROVE_NONE_U32); a member's gang Required level is l_s or
 * deeper, so an admitted member lies in exactly one level-l_s domain A(g), and it has a clique with MinReplicas > 0.  Seeds
 * are running replicas of a group, each counted in the level-l_s domain of its node (nowhere when the node lacks that label).
 * At member g's turn in the sequential pass: c(A) = seeds in A + members of s ranked before g that were admitted into A;
 * E_g = the level-l_s domains holding a schedulable node whose selector class some clique of g accepts; m = min over E_g of
 * c(A); A is ALLOWED iff A is in E_g and c(A) + 1 - m <= max_skew.
 *   GROVE_SPREAD_HARD (DoNotSchedule): a candidate domain outside every allowed A is infeasible; none feasible -> REJECTED.
 *   GROVE_SPREAD_SOFT (ScheduleAnyway): the allowed candidates first (the usual order, Preferred levels included); if none
 *   fits, the disallowed ones.  A gang admitted by that second walk carries GROVE_STATUS_SPREAD_SKEWED.
 * Everything else is the ordinary pass.  Call after grove_submit_gangs and before grove_run_cycle; the next
 * grove_submit_gangs* or grove_load_nodes* clears the set, grove_update_nodes keeps it.  GROVE_ERR_INVALID_ARG for a wrong
 * n_gangs, a group index out of range, a level >= n_levels, a bad mode, max_skew 0, a member without a gang Required level at
 * l_s or deeper, a member with no MinReplicas > 0, a seed on a node or group out of range; GROVE_ERR_LIMIT for a wide
 * submission, and when the members' allowed-domain rows (one bit per member and domain of its group's level) would exceed 1 GB;
 * GROVE_ERR_STATE before nodes are loaded and gangs submitted.  While a set with members is in place grove_run_cycle_preempt / _reuse / _reuse_preempt return
 * GROVE_ERR_STATE, and grove_diagnose returns GROVE_ERR_STATE after such a cycle.  A set without members changes nothing. */
#define GROVE_SPREAD_HARD 1u            /* DoNotSchedule */
#define GROVE_SPREAD_SOFT 2u            /* ScheduleAnyway */
#define GROVE_STATUS_SPREAD_SKEWED 0x2u /* grove_gang_status_t.reserved0: a SOFT member placed outside its allowed domains */
typedef struct grove_spread {
  uint8_t level;
  uint8_t mode;           /* GROVE_SPREAD_HARD or GROVE_SPREAD_SOFT */
  uint16_t max_skew;      /* >= 1 */
  uint32_t reserved;
} grove_spread_t;
typedef struct grove_spread_seed {
  uint32_t group;
  uint32_t node;          /* caller's node index */
} grove_spread_seed_t;
int32_t grove_set_spread(grove_engine_t* e, const grove_spread_t* groups, uint32_t n_groups,
                         const uint32_t* gang_group, uint32_t n_gangs,
                         const grove_spread_seed_t* seeds, uint32_t n_seeds);

/* ---- fences -------------------------------------------------------------------------------------------
 * A rejected gang keeps the gangs ranked after it out of the domain closest to fitting it, so that a large gang is not starved
 * by smaller ones that take every node freed (DESIGN.md section 1, "Fences"; the backfill-with-reservation of batch schedulers).
 * `gangs` names the FENCING gangs of the current submission; each has a gang Required level l.  F0 is the node table the cycle
 * starts from, rank = (priority desc, submission index asc).
 *   Picks, fixed at cycle start, in rank order: for each level-l domain D (nodes lacking the label are in none) and each clique q
 *   with MinReplicas > 0, have_q(D) = sum over n in D of min(cap(q, n), MinReplicas_q), cap = grove_diagnose's exact capacity on
 *   F0 (0 where K1 fit fails); shortfall(D) = sum over q of max(0, MinReplicas_q - have_q(D)).  The gang picks the D of least
 *   shortfall among the level-l domains that share no node with an earlier pick, ties by its candidate order at level l
 *   (descending min(closeness(first node, anchor), l + 1), then ascending rotated index); none left: no pick.
 *   The pass: the sequential pass, except that a gang sees every node of an ACTIVE fence of a gang ranked before it as
 *   unschedulable (K1 fit fails).  A fence is active when its gang was evaluated and came out REJECTED; an admitted, gated or
 *   BASE_REJECTED gang fences nothing.
 *   Outputs: a REJECTED gang with an active fence carries GROVE_STATUS_FENCING in reserved0, level = l and domain_node = the
 *   caller index of the fenced domain's first node.  Everything else is what the pass gives; fences leave no trace in the node
 *   table.
 * Call after grove_submit_gangs and before grove_run_cycle; the next grove_submit_gangs* or grove_load_nodes* clears the set,
 * grove_update_nodes keeps it.  GROVE_ERR_INVALID_ARG for an index out of range, a duplicate, or a gang without a gang Required
 * level; GROVE_ERR_LIMIT for more than GROVE_MAX_FENCES gangs, for a wide submission, and when the per-domain sums (fencing gangs x
 * cliques x domains of their level, 4 B each) would exceed 1 GB; GROVE_ERR_STATE before nodes are loaded and gangs submitted.
 * While a non-empty set is in place grove_run_cycle_preempt / _reuse / _reuse_preempt return GROVE_ERR_STATE, so does
 * grove_run_cycle with a spread set with members, and grove_diagnose returns GROVE_ERR_STATE after a fenced cycle.  An empty set
 * changes nothing. */
#define GROVE_MAX_FENCES 64u
#define GROVE_STATUS_FENCING 0x4u       /* grove_gang_status_t.reserved0: a REJECTED gang whose fence held at the end of the cycle */
int32_t grove_set_fences(grove_engine_t* e, const uint32_t* gangs, uint32_t n);

/* ---- bin-packing ---------------------------------------------------------------------------------------
 * A member starts its search at the fullest domain that can hold it, so that empty domains stay empty for large gangs (DESIGN.md
 * section 1, "Bin-packing"; KAI-Scheduler's default bin-pack placement).  level_of[g] is the pack level b of submitted gang g, or
 * GROVE_LEVEL_NONE when g is not a member; b < n_levels, and b is the gang's Required level or deeper when it has one.
 *   Picks, on F0 (the table the cycle starts from), for every member on its own: the candidates are the level-b domains (nodes
 *   lacking the label are in none); S_D = the 64-bit sums of free cpu, mem, gpu and pods over the SCHEDULABLE nodes of D.  D qualifies
 *   when every clique q with MinReplicas m_q > 0 has sum over n in D of cap(q, n) >= m_q (grove_diagnose's exact capacity, 0 where
 *   K1 fit fails), and sum over q of m_q * request_q <= S_D for cpu, mem and gpu, and sum of m_q <= S_D.pods.  The pick is the
 *   qualifying D of least (S_D.gpu, S_D.cpu, S_D.mem, first node in topology order); none: the member keeps its default anchor.
 *   The cycle: the cycle that would run otherwise (grove_run_cycle, or the queue cycle with a queue set), with each picked member's
 *   anchor_node replaced by the caller index of its pick's first node.  Nothing else changes.
 * grove_get_binpack_picks: per gang of the last cycle that ran with a set, the caller index of the first node of its pick, or
 * GROVE_NONE_U32 (not a member, or no qualifying domain); GROVE_ERR_STATE before such a cycle.
 * Call after grove_submit_gangs and before the cycle; the next grove_submit_gangs* or grove_load_nodes* clears the set,
 * grove_update_nodes keeps it (the picks are made again each cycle).  A set without members changes nothing.  GROVE_ERR_INVALID_ARG
 * for a wrong n_gangs, b >= n_levels, or b above the gang's Required level; GROVE_ERR_LIMIT for a wide submission; GROVE_ERR_STATE
 * before nodes are loaded and gangs submitted.  While a set with members is in place grove_run_cycle_preempt / _reuse /
 * _reuse_preempt / _preempt_queues / _consolidate return GROVE_ERR_STATE, and so does grove_run_cycle with a spread set with
 * members or a fence set.  grove_diagnose accepts a bin-packing cycle; grove_build_score_matrix scores against the anchors the
 * last cycle used.  Members that share a pick depend on one another, so a cycle with members relaxes at most 128 gangs at a time
 * unless grove_config_t.window says otherwise (DESIGN.md section 1, "Bin-packing": the measured cost). */
int32_t grove_set_binpack(grove_engine_t* e, const uint8_t* level_of, uint32_t n_gangs);
int32_t grove_get_binpack_picks(grove_engine_t* e, uint32_t* out, uint32_t cap);

/* ---- ComputeDomain exclusivity -------------------------------------------------------------------------
 * A node's GPUs take part in at most one IMEX channel, hence one NVIDIA ComputeDomain (CD), at a time: pods of MNNVL-enrolled
 * PodGroups of different CDs never share a node (DESIGN.md section 1, "ComputeDomain exclusivity"; Grove's auto-MNNVL).
 * cd[q] (one per submitted clique) is the CD of clique q's pods, a caller-interned id, or GROVE_CD_NONE when q is not enrolled.
 * owner0[n] (one per loaded node, caller order) is the CD that holds node n's IMEX channel when the cycle starts, GROVE_CD_NONE,
 * or GROVE_CD_NO_IMEX (the node has no IMEX driver).
 * The sequential pass is unchanged except at gang g's turn: owner(n) = owner0[n] if that is not GROVE_CD_NONE, else the CD of the
 * enrolled pods that gangs ranked before g put on n in this cycle (at most one), else GROVE_CD_NONE.  An enrolled clique q of g
 * fails K1 fit on n unless owner(n) is GROVE_CD_NONE or cd[q] (MinReplicas and surplus alike); cliques that are not enrolled are
 * unaffected.  Candidate order, anchors, gating, the base-gang rule and PlacementScore do not change.  All enrolled cliques of a
 * gang share one CD; a scaled gang carries its base gang's CD, so it may join the nodes its base holds.
 * grove_get_compute_domain_owners: per loaded node (caller order), its owner at the end of the last cycle that ran with a set:
 * owner0, plus the CD of every admitted gang's enrolled pods -- the next cycle's owner0.  GROVE_ERR_STATE before such a cycle.
 * Call after grove_submit_gangs and before the cycle; the next grove_submit_gangs* or grove_load_nodes* clears the set,
 * grove_update_nodes keeps it.  A set without an enrolled clique runs the ordinary cycle; the owners are then owner0.
 * GROVE_ERR_INVALID_ARG for n_cliques / n_nodes other than the counts submitted / loaded, GROVE_CD_NO_IMEX as a clique's CD, or an
 * enrolled clique with req_gpu == 0; GROVE_ERR_LIMIT for two CDs in one gang or a wide submission; GROVE_ERR_STATE before nodes
 * are loaded and gangs submitted.  While a set with an enrolled clique is in place grove_run_cycle_preempt / _reuse /
 * _reuse_preempt / _preempt_queues / _consolidate return GROVE_ERR_STATE, and so does grove_run_cycle with a spread set with
 * members, a fence set, a queue set with members or a bin-packing set with members; grove_diagnose returns GROVE_ERR_STATE after
 * such a cycle. */
#define GROVE_CD_NONE GROVE_NONE_U32    /* not enrolled / no CD holds the node */
#define GROVE_CD_NO_IMEX 0xFFFFFFFEu    /* owner0: the node has no IMEX driver (no enrolled pod may land on it) */
int32_t grove_set_compute_domains(grove_engine_t* e, const uint32_t* cd, uint32_t n_cliques, const uint32_t* owner0, uint32_t n_nodes);
int32_t grove_get_compute_domain_owners(grove_engine_t* e, uint32_t* out, uint32_t cap);

/* ---- consolidation ------------------------------------------------------------------------------------
 * Running gangs are relocated so that a blocked gang fits, and only when every relocated gang finds a new place (DESIGN.md
 * section 1, "Consolidation"; after KAI-Scheduler's consolidation action).  Running gangs and holdings are as for
 * grove_run_cycle_preempt (the loaded node table does not include what they hold).  spec_of[r] (one entry per running gang) is
 * the row of the current submission that restates running gang r's PodGang, which makes r MOVABLE, or GROVE_NONE_U32.  A spec row
 * carries GROVE_GANG_GATED (so the ordinary pass skips it), its base_gang is ignored, it is named at most once and is not a
 * target.  `targets` names up to GROVE_MAX_CONSOLIDATE_TARGETS submitted gangs.  F is the free table, rank = (priority desc,
 * submission index asc).
 *   1. The ordinary pass: grove_run_cycle on the submission; F is the table it leaves.
 *   2. Every target b it left REJECTED, in rank order: M = the movable running gangs of priority <= p_b not moved this cycle
 *      (empty: skip b), W = F + what the gangs of M hold.
 *   3. Candidates: the level-l domains (l = b's gang Required level) in which every clique of b with MinReplicas m > 0 finds m pods
 *      over W (grove_diagnose's exact capacities), in the order of their shortfall over F (as grove_set_fences computes it), ties
 *      by the fences' candidate order; at most GROVE_CONSOLIDATE_TRIES of them.  Without a Required level: the whole cluster.
 *   4. A try on D: b is evaluated with its ordinary-pass anchor against W with every node outside D unschedulable; it does not
 *      fit: next D.  It fits with usage U: walking its nodes in the order its placement first names them, while F plus what X holds
 *      does not cover U on the node, one more gang of M holding there joins the displaced set X (lowest priority first, then the
 *      highest running index).  X's spec rows run as one sequential pass (rank = running priority desc, running index asc; each
 *      keeps its own anchor) against F + what X holds - U.  All admitted: commit -- F is what that pass leaves, b is ADMITTED with
 *      GROVE_STATUS_CONSOLIDATED, every spec row of X is ADMITTED with GROVE_STATUS_MOVED and its new placement and scope domains,
 *      grove_get_moves lists (r, b) for each member; no more tries for b.  Otherwise nothing changes and the next D is tried.
 * Outputs through the usual getters; the node table is F after all commits.  GROVE_ERR_LIMIT for a wide submission or more than
 * GROVE_MAX_CONSOLIDATE_TARGETS targets; GROVE_ERR_STATE while a spread set with members or a non-empty fence set is in place;
 * GROVE_ERR_INVALID_ARG for a target or spec row out of range or named twice, a spec row that is not gated or is a target, holdings
 * out of range, or free + holdings overflowing a field of a node record.  grove_diagnose refuses the cycle that follows. */
#define GROVE_MAX_CONSOLIDATE_TARGETS 16u
#define GROVE_CONSOLIDATE_TRIES 4u
#define GROVE_STATUS_CONSOLIDATED 0x8u  /* grove_gang_status_t.reserved0: a target admitted by the consolidation pass */
#define GROVE_STATUS_MOVED 0x10u        /* grove_gang_status_t.reserved0: the spec row of a running gang that was relocated */
typedef struct grove_move {
  uint32_t running;       /* index into the running array */
  uint32_t target;        /* gang index of the submission it made room for */
} grove_move_t;
int32_t grove_run_cycle_consolidate(grove_engine_t* e, const uint32_t* targets, uint32_t n_targets,
                                    const uint32_t* spec_of, const grove_running_gang_t* running, uint32_t n_running,
                                    const grove_holding_t* holdings, uint32_t n_holdings, grove_cycle_stats_t* stats);
int32_t grove_get_moves(grove_engine_t* e, grove_move_t* out, uint32_t cap, uint32_t* n_out);

/* ---- queue limits --------------------------------------------------------------------------------------
 * Hierarchical queues bound what each tenant holds (DESIGN.md section 1, "Queue limits"; after KAI-Scheduler's Queue `limit`).
 * Queue i has a parent (< i, or GROVE_NONE_U32; chains at most GROVE_MAX_QUEUE_DEPTH deep), limit[r] per resource r (cpu milli,
 * mem MiB, gpu; GROVE_QUEUE_UNLIMITED = none) and used[r], what the running gangs of exactly this queue hold.  A queue's load is
 * its own used plus that of all its descendants.  gang_queue[g] is the queue of submitted gang g, or GROVE_NONE_U32; chain(g) is
 * that queue and its ancestors.  rank = (priority desc, submission index asc); R_min(g) = sum over g's cliques of MinReplicas *
 * request; U(h) = the usage of h's placement, surplus included.
 * The sequential pass is unchanged except at a member g, after the gating and base-gang rules, at its turn:
 *   1. For each Q in chain(g): H_Q[r] = limit_Q[r] - load_Q[r] - sum of U(h)[r] over the members h ranked before g that were
 *      admitted and have Q in chain(h) (signed 64-bit).
 *   2. If R_min(g)[r] > H_Q[r] for some r with R_min(g)[r] > 0 and some Q in chain(g) with a finite limit_Q[r], g is REJECTED
 *      without evaluation and carries GROVE_STATUS_OVER_LIMIT.
 *   3. Otherwise H(g)[r] = min of H_Q[r] over chain(g) (finite limits only), rem = H(g) - R_min(g); clique by clique in order,
 *      s_q = min(replicas_q - MinReplicas_q, floor(rem[r] / req_q[r]) over the r with req_q[r] > 0 and a finite limit), at least
 *      0, rem -= s_q * req_q.  g is evaluated as always as if clique q had MinReplicas_q + s_q replicas.  Admitted with some
 *      s_q < replicas_q - MinReplicas_q: GROVE_STATUS_SURPLUS_CAPPED.
 *   4. An admitted member charges U(g) to every queue of its chain.
 * Call after grove_submit_gangs and before grove_run_cycle; the next grove_submit_gangs* or grove_load_nodes* clears the set,
 * grove_update_nodes keeps it.  A set without members changes nothing.  GROVE_ERR_INVALID_ARG for a wrong n_gangs, a parent at or
 * after its own index, a queue index out of range; GROVE_ERR_LIMIT for more than GROVE_MAX_QUEUES queues, a chain deeper than
 * GROVE_MAX_QUEUE_DEPTH, a wide submission; GROVE_ERR_STATE before nodes are loaded and gangs submitted.  While a set with members
 * is in place grove_run_cycle_preempt / _reuse / _reuse_preempt / _consolidate return GROVE_ERR_STATE, and so does grove_run_cycle
 * with a spread set with members or a fence set.  grove_diagnose accepts a queue cycle; a gang carrying GROVE_STATUS_OVER_LIMIT
 * gets an all-zero record. */
#define GROVE_MAX_QUEUES 4096u
#define GROVE_MAX_QUEUE_DEPTH 4u
#define GROVE_QUEUE_UNLIMITED 0xFFFFFFFFFFFFFFFFull
#define GROVE_STATUS_OVER_LIMIT 0x20u      /* REJECTED by its queue chain's headroom, not evaluated */
#define GROVE_STATUS_SURPLUS_CAPPED 0x40u  /* ADMITTED with fewer best-effort pods allowed than it asked for */
typedef struct grove_queue {
  uint32_t parent;                  /* < own index, or GROVE_NONE_U32 */
  uint32_t reserved;
  uint64_t limit[3];                /* cpu milli, mem MiB, gpu; GROVE_QUEUE_UNLIMITED = none */
  uint64_t used[3];                 /* held by the running gangs of exactly this queue */
} grove_queue_t;
int32_t grove_set_queues(grove_engine_t* e, const grove_queue_t* queues, uint32_t n_queues,
                         const uint32_t* gang_queue, uint32_t n_gangs);

/* ---- reclaim within queue limits -----------------------------------------------------------------------
 * The reclaim pass on a queue cycle: a gang its queue chain turns away can evict lower-priority gangs of the same queues
 * (DESIGN.md section 1, "Reclaim within queue limits"; after KAI-Scheduler's preempt action).  Runs on the queue set that
 * grove_set_queues gave the current submission (a set without members counts).  Running gangs and holdings are as for
 * grove_run_cycle_preempt; running_queue[r] is the queue of running gang r, or GROVE_NONE_U32, and what the running gangs of queue
 * q hold (cpu, mem, gpu summed over their holdings) must not exceed used(q).  E(p) = the standing running gangs of a priority below p.
 *   1. The ordinary pass: grove_run_cycle with the queue set.  The load of each queue is then its starting load plus U of the
 *      admitted members in its subtree.
 *   2. Every gang it left REJECTED (OVER_LIMIT ones included) is reconsidered once, in rank order, while E(p) is non-empty: against
 *      the node view free + what E(p) holds, and the queue limits with load'_Q = load_Q - what the gangs of E(p) whose queue lies in
 *      Q's subtree hold.  Admitted: GROVE_STATUS_PREEMPTOR, ORed with GROVE_STATUS_SURPLUS_CAPPED; rejected again: its ordinary-pass
 *      status, flags included.
 *   3. Victims of an admitted g: (a) node by node, as grove_run_cycle_preempt evicts; (b) for each Q of chain(g), leaf first, while
 *      load_Q[r] > limit_Q[r] for a resource r with U(g)[r] > 0 and a finite limit, one whole gang of E(p) in Q's subtree that holds
 *      some of such a resource, lowest priority first, then highest running index.  An eviction returns the victim's holdings to the
 *      free table and takes its usage off every queue of its chain.  grove_get_victims lists (victim, preemptor) in eviction order.
 * Outputs through the usual getters; the queue set stays in place.  GROVE_ERR_STATE without a queue set given since the last
 * submission, with a spread set with members or a non-empty fence set; GROVE_ERR_LIMIT for a wide submission; GROVE_ERR_INVALID_ARG
 * for the inputs grove_run_cycle_preempt rejects, a running_queue entry out of range, or running usage of a queue above its used.
 * grove_diagnose refuses the cycle that follows. */
int32_t grove_run_cycle_preempt_queues(grove_engine_t* e, const grove_running_gang_t* running, uint32_t n_running,
                                       const grove_holding_t* holdings, uint32_t n_holdings,
                                       const uint32_t* running_queue, grove_cycle_stats_t* stats);

/* ---- reclaim across queues -----------------------------------------------------------------------------
 * A queue below its deserved quota takes room back from queues above theirs, whatever the priorities (DESIGN.md section 1,
 * "Reclaim across queues"; after KAI-Scheduler's reclaim action and Queue `spec.resources.*.quota`).  Inputs are those of
 * grove_run_cycle_preempt_queues plus one quota row per queue of the set: deserved[r] per resource (cpu milli, mem MiB, gpu;
 * GROVE_QUEUE_UNLIMITED = KAI's quota -1, the queue deserves whatever it holds).  cap_X = min(limit_X, deserved_X) per resource.
 * load_X is as in "reclaim within queue limits", kept up to date as gangs are evicted and admitted; the victim order is lowest
 * priority first, then the highest running index; a running gang stands until it is evicted.
 *   1. The ordinary pass: grove_run_cycle with the queue set.
 *   2. Classes: every queue Q that is the queue of a gang the ordinary pass left REJECTED (OVER_LIMIT ones included), in ascending
 *      order of share_Q at the start of the pass = the max over resources x with a finite deserved_Q[x] of load_Q[x] / deserved_Q[x]
 *      (0/0 = 0, l/0 = +inf for l > 0, no finite quota = 0; compared exactly), ties by queue index.  Members M(Q): those gangs, in
 *      rank order.
 *   3. The donor set E(Q), fixed when class Q starts.  For a queue X and a standing running gang r of X's subtree, P_X(r) = what
 *      the standing running gangs r' of X's subtree with r' no later than r in victim order hold; ok_X(r): load_X[x] - P_X(r)[x] >=
 *      deserved_X[x] on every resource x that r holds with a finite deserved_X[x]; over_X(r): there is such an x.
 *      D(r, Q) = chain(queue(r)) \ chain(Q).  r is in E(Q) when it has a queue, neither queue(r) nor Q lies in the other's chain,
 *      ok_X(r) holds for every X of D(r, Q) and over_X(r) for some.  An empty E(Q) skips the class.
 *   4. The members, one at a time in rank order, against the node view free + what E(Q) holds and the queue rules of
 *      "queue limits" with load'_X = load_X - what the gangs of E(Q) in X's subtree hold and cap in place of limit.  Admitted:
 *      GROVE_STATUS_RECLAIMER, ORed with GROVE_STATUS_SURPLUS_CAPPED; rejected again: its ordinary-pass status, flags included.
 *   5. Victims of an admitted g, from the standing gangs of E(Q) only: (a) node by node, as grove_run_cycle_preempt evicts; (b) for
 *      each X of chain(Q), leaf first, while load_X[r] > cap_X[r] for a resource r with U(g)[r] > 0 and a finite cap, the first gang
 *      in victim order of E(Q) in X's subtree that holds some of such a resource.  An eviction returns the victim's holdings to the
 *      free table and takes its usage off every queue of its chain.  grove_get_victims lists (victim, reclaimer) in eviction order.
 * A victim never lies in its reclaimer's queue, an ancestor or its subtree, and may outrank its reclaimer.  Outputs through the
 * usual getters; the queue set stays in place.  Refusals are those of grove_run_cycle_preempt_queues, plus GROVE_ERR_INVALID_ARG
 * when n_queues is not the set's number of queues.  grove_diagnose refuses the cycle that follows. */
#define GROVE_STATUS_RECLAIMER 0x80u /* grove_gang_status_t.reserved0: admitted by grove_run_cycle_reclaim_queues's class pass */
typedef struct grove_queue_quota {
  uint64_t deserved[3];             /* cpu milli, mem MiB, gpu; GROVE_QUEUE_UNLIMITED = whatever the queue holds */
} grove_queue_quota_t;
int32_t grove_run_cycle_reclaim_queues(grove_engine_t* e, const grove_queue_quota_t* quotas, uint32_t n_queues,
                                       const grove_running_gang_t* running, uint32_t n_running,
                                       const grove_holding_t* holdings, uint32_t n_holdings,
                                       const uint32_t* running_queue, grove_cycle_stats_t* stats);

/* ---- reclaim, then preempt, across and within queues ---------------------------------------------------
 * Both queue eviction passes in one cycle, in KAI-Scheduler's order: its reclaim action, then its preempt action (DESIGN.md
 * section 1, "Reclaim, then preempt").  Inputs, the queue set it runs on and the victim order are those of
 * grove_run_cycle_reclaim_queues.
 *   1. The ordinary pass: grove_run_cycle with the queue set.
 *   2. The reclaim pass: steps 2-5 of "reclaim across queues" (queue classes in ascending share at the start of the pass, donor
 *      sets E(Q), cap = min(limit, deserved), the node step and then the queue step).  Admitted: GROVE_STATUS_RECLAIMER, ORed
 *      with GROVE_STATUS_SURPLUS_CAPPED.
 *   3. The preempt pass: steps 2-3 of "reclaim within queue limits" from the state step 2 leaves (its free table, its queue
 *      loads, its standing set).  Every gang still REJECTED -- OVER_LIMIT ones, members of skipped or unsuccessful queue classes
 *      and gangs without a queue included; a reclaimer never -- is reconsidered once, in rank order, while E(p) (the standing
 *      running gangs of a priority below p) is non-empty, under the queue LIMITS.  Admitted: GROVE_STATUS_PREEMPTOR, ORed with
 *      GROVE_STATUS_SURPLUS_CAPPED; rejected again: its ordinary-pass status, flags included.
 * grove_get_victims lists every eviction in order, those of step 2 first; the flag of the gang named in a pair says which pass
 * chose it.  Outputs through the usual getters; the queue set stays in place.  Refusals are those of
 * grove_run_cycle_reclaim_queues, with the same codes; grove_diagnose refuses the cycle that follows. */
int32_t grove_run_cycle_reclaim_preempt_queues(grove_engine_t* e, const grove_queue_quota_t* quotas, uint32_t n_queues,
                                               const grove_running_gang_t* running, uint32_t n_running,
                                               const grove_holding_t* holdings, uint32_t n_holdings,
                                               const uint32_t* running_queue, grove_cycle_stats_t* stats);

/* ---- fair-share order ----------------------------------------------------------------------------------
 * The queue cycle's turns go by fair share: the queue furthest below its deserved quota takes the next turn (DESIGN.md section 1,
 * "Fair-share order"; after KAI-Scheduler's allocate action, which takes the next job from the queue with the lowest share).
 * grove_set_fair_share gives one quota row per queue of the set grove_set_queues gave the current submission.  With it in place,
 * grove_run_cycle runs the queue cycle ("queue limits", rules 1-4) with one change, the turn order:
 *   share_X = max over resources x with a finite deserved_X[x] of load_X[x] / deserved_X[x] (0/0 = 0, l/0 = +inf for l > 0, no
 *   finite quota = 0; compared exactly), load_X taken at the turn: its starting load plus U of every member of X's subtree
 *   admitted earlier in the cycle.  The gangs with no queue form one more top-level pseudo-queue of share 0.  The next gang is
 *   next(root): for a leaf, its first waiting gang in rank order; for an inner node, next(C) of the child C that still has a
 *   waiting gang with the smallest (share_C, rank(next(C))).
 * Each turn is then the queue cycle's: gated gangs are skipped, a scaled gang needs its base admitted at an earlier turn, the gate
 * and the surplus caps read "ranked before g" as "took its turn before g", and K3 runs with the gang's ordinary anchor.  Every
 * member must sit in a leaf queue (GROVE_ERR_INVALID_ARG otherwise).  The set is cleared with the queue set (next
 * grove_submit_gangs* / grove_load_nodes* / grove_set_queues) and kept by grove_update_nodes.  Refused: n_queues other than the
 * set's queue count (GROVE_ERR_INVALID_ARG); no queue set (GROVE_ERR_STATE).  While it is in place, grove_run_cycle with a
 * bin-packing set with members, an enrolled ComputeDomain, a spread set with members or a fence set, and
 * grove_run_cycle_{preempt,reclaim,reclaim_preempt}_queues, return GROVE_ERR_STATE; so does grove_diagnose after the cycle.
 * grove_get_turn_order: the gangs in the order they had their turn (GROVE_ERR_STATE before a fair-share cycle);
 * grove_get_fair_share_stats: the queue cycles the engine ran to find that order and how many turns they ran again. */
typedef struct grove_fair_share_stats {
  uint32_t iterations;    /* relaxation cycles run (the first over every gang, each later one over the turns from the first changed one) */
  uint32_t turns_rerun;   /* turns the cycles after the first ran again */
} grove_fair_share_stats_t;
int32_t grove_set_fair_share(grove_engine_t* e, const grove_queue_quota_t* quotas, uint32_t n_queues);
int32_t grove_get_turn_order(grove_engine_t* e, uint32_t* out, uint32_t cap);
int32_t grove_get_fair_share_stats(grove_engine_t* e, grove_fair_share_stats_t* out);

/* ---- over-quota weight ---------------------------------------------------------------------------------
 * A queue's fair share is its deserved quota plus a slice of the capacity nobody deserves, divided among siblings by their
 * over-quota weights and capped by what each asks for (DESIGN.md section 1, "Over-quota weight"; after KAI-Scheduler's proportion
 * plugin and Queue `spec.resources.*.overQuotaWeight`).  grove_set_over_quota gives one weight row per queue of the set
 * grove_set_queues gave the current submission.  With it in place, grove_run_cycle with a fair-share set,
 * grove_run_cycle_reclaim_queues and the reclaim pass of grove_run_cycle_reclaim_preempt_queues behave exactly as if the caller had
 * passed the fair shares as the deserved quotas (shares, caps and donor sets); the preempt pass and every entry that takes no
 * quotas do not read it.  The fair shares are computed once per call, at its start, per resource r, from the call's deserved
 * quotas; every quantity below saturates at 2^62:
 *   C[r] = the free r of the schedulable nodes of the table the call starts from + the load of every top-level queue (own used
 *   plus its descendants').  demand_X[r] = load_X[r] + replicas * request[r] of every clique of every gang not GROVE_GANG_GATED
 *   whose queue lies in X's subtree (surplus pods count).  The root's pool is C; at a parent with pool P each child c takes:
 *     deserved_c[r] unlimited: fair_c[r] = GROVE_QUEUE_UNLIMITED, and t_c = min(demand_c, limit_c) of P, which c's children divide;
 *     otherwise base_c = min(deserved_c, demand_c, limit_c), need_c = min(demand_c, limit_c) - base_c.
 *   R = max(0, P - sum of bases - sum of t).  Then, while a round gives something: A = the finite children with need_c > 0 and
 *   w_c > 0, W = sum of their weights, each gets g_c = min(need_c, floor(R * w_c / W)), R -= sum g, need_c -= g_c.  The leftover
 *   (R < |A|) goes one unit each to the members of A in (w desc, queue index asc) order while R > 0.  fair_c = base_c + what c
 *   got; c's children divide it.
 * The set is cleared with the queue set (next grove_submit_gangs* / grove_load_nodes* / grove_set_queues) and kept by
 * grove_update_nodes.  Refused: n_queues other than the set's queue count or a null row pointer with n_queues > 0
 * (GROVE_ERR_INVALID_ARG); no queue set (GROVE_ERR_STATE).  grove_get_fair_shares writes 3 values per queue (cpu milli, mem MiB,
 * gpu): the fair shares the last call that ran with weights computed (GROVE_QUEUE_UNLIMITED where deserved is); GROVE_ERR_STATE
 * before such a call since the set was given, GROVE_ERR_LIMIT when cap_queues is below the queue count. */
typedef struct grove_queue_weight {   /* 16 B */
  uint32_t over_quota[3];             /* cpu, mem, gpu; KAI's default is 1, 0 = the queue gets no share of the surplus */
  uint32_t reserved;
} grove_queue_weight_t;
int32_t grove_set_over_quota(grove_engine_t* e, const grove_queue_weight_t* w, uint32_t n_queues);
int32_t grove_get_fair_shares(grove_engine_t* e, uint64_t* out, uint32_t cap_queues);

/* K2: the topology-distance score matrix T[clique][node] = fit ? 1 + levels shared with the gang's anchor : 0 (u8) over the
 * snapshot the last cycle started from -- what a scheduler's Score extension point would hand out.  The admission does
 * not read it (its visiting order comes from the anchor's domain ranges), so it is built on request; GROVE_TUNE_SCORE=1
 * builds it every cycle beside the admission.  *ms (nullable): device time of the kernel. */
int32_t grove_build_score_matrix(grove_engine_t* e, float* ms);

/* ---- multi-GPU score pass (north_star: node-range shards + one all-reduce of per-shard feasibility) -------------
 * A handle created with grove_config_t.world = W > 1 and rank = r builds K1 + K2 (fit / score matrix) only for ITS node range:
 * the topology-sorted node table cut at top-level domain boundaries into W ranges of about equal size (every handle loads the
 * whole -- small -- node table; the Q x N score matrix is what outgrows a GPU).  grove_run_score_pass: K1 + K2 over the loaded
 * snapshot for the submitted gangs, no admission; *ms (nullable) = device time.  grove_shard_summary_device writes int32[G + Q]
 * into the caller's DEVICE buffer: [g] = domains of gang g's Required level starting in the shard in which each of its cliques
 * finds MinReplicas worth of capacity (0 for gangs without a Required level), [G + q] = pods of clique q that fit on the
 * shard's nodes.  The caller sums the vectors of all ranks with ONE all-reduce (NCCL over NVLink; gloo in the CPU tests) and
 * reads cluster-wide feasibility off the sum: a gang with a Required level and sum 0, or a clique whose summed capacity is
 * below MinReplicas, cannot be admitted from this snapshot.  With world <= 1 the shard is the whole table. */
int32_t grove_shard_range(grove_engine_t* e, uint32_t* lo, uint32_t* hi); /* topology-sorted node indices [lo, hi) */
int32_t grove_run_score_pass(grove_engine_t* e, float* ms);
int32_t grove_shard_summary_device(grove_engine_t* e, void* d_out, uint32_t cap_words);

/* ---- device-resident variants (inputs already in HBM; used by bench.py `value`) -------------- */
/* d_nodes: device pointer to n grove_node_t in caller order, labels identical to the last load.  Read ASYNCHRONOUSLY on the
 * engine's stream: the buffer must stay valid and unchanged until the next blocking call on the handle (grove_run_cycle,
 * grove_run_score_pass, grove_get_nodes) has returned. */
int32_t grove_load_nodes_device(grove_engine_t* e, const void* d_nodes, uint32_t n);

/* ---- introspection for the parity tests (sorted node order; see DESIGN.md "Data layout") ------ */
int32_t grove_debug_get_perm(grove_engine_t* e, uint32_t* sorted_to_caller, uint32_t cap);
/* K1 / K2 output over the cycle-start snapshot: fit bitmap row (ceil(n/32) words) and score row (n bytes) of one clique */
int32_t grove_debug_get_fit_row(grove_engine_t* e, uint32_t clique, uint32_t* words, uint32_t cap_words);
int32_t grove_debug_get_score_row(grove_engine_t* e, uint32_t clique, uint8_t* bytes, uint32_t cap_bytes);
#ifdef __cplusplus
}
#endif
#endif /* GROVE_PLACE_H */
