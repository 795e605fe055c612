// grove_host.hpp -- host side above the C ABI, in C++ because the reference is compiled code (Go) and
// no Go toolchain exists in this image.  It mirrors, name for name, the reference interfaces that sit
// either side of the placement hot path:
//
//   PodGang / PodGroup / TopologyConstraint ...   scheduler/api/core/v1alpha1/podgang.go:51-190
//   Backend / TopologyAwareSchedBackend           operator/internal/scheduler/types.go:37-96
//   ComputeExpectedPodGangs (the producer)        operator/internal/controller/podcliqueset/components/podgang/syncflow.go:145-371
//   name generation                               operator/api/common/namegen.go:70-117
//   CreatePodGroupsForPodGang                     .../components/podgang/podgang.go:165-186
//   isBasePodGangScheduled / scheduling gates     operator/internal/controller/podclique/components/pod/syncflow.go:255-358
//
// (all paths relative to ai-dynamo/grove).  Error convention: Go returns `error`; here every fallible
// call returns std::optional<Error> (nullopt == nil), and Error carries the GroveError fields
// (operator/internal/errors/errors.go:41-86).
#pragma once
#include <cstdint>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <array>
#include <map>
#include <mutex>
#include <thread>
#include <optional>
#include <string>
#include <vector>

#include "../../../include/grove_place.h"

namespace grove::host {

// ---- errors ------------------------------------------------------------------------------------
struct Error {
  std::string code;       // e.g. "ERR_SYNC_PODGANG"
  std::string operation;  // e.g. "SyncPodGang"
  std::string message;
};
using Err = std::optional<Error>;

// ---- scheduler/api/core/v1alpha1/podgang.go ------------------------------------------------------
struct NamespacedName { std::string Namespace, Name; };                              // :133-139
struct TopologyPackConstraint { std::optional<std::string> Required, Preferred; };   // :101-118 (label KEYS)
struct TopologyConstraint { std::optional<TopologyPackConstraint> PackConstraint; }; // :93-99
struct PodGroup {                                                                    // :75-91
  std::string Name;
  std::vector<NamespacedName> PodReferences;
  int32_t MinReplicas = 0;
  std::optional<TopologyConstraint> Topology;
};
struct TopologyConstraintGroupConfig {                                               // :120-131
  std::string Name;
  std::vector<std::string> PodGroupNames;
  std::optional<TopologyConstraint> Topology;
};
struct PodGangSpec {                                                                 // :51-72
  std::vector<PodGroup> PodGroups;
  std::optional<TopologyConstraint> Topology;
  std::vector<TopologyConstraintGroupConfig> TopologyConstraintGroupConfigs;
  std::string PriorityClassName;
  std::optional<NamespacedName> ReuseReservationRef;
};
enum class PodGangPhase { Pending, Starting, Running };                              // :141-150
struct PodGangStatus {                                                               // :182-190
  PodGangPhase Phase = PodGangPhase::Pending;
  bool Scheduled = false;                 // condition PodGangConditionTypeScheduled :155
  std::string ScheduledReason;            // "" | "Unschedulable" | "BaseNotScheduled" | "Gated"
  std::string ScheduledMessage;           // condition message (why a PodGang cannot be handed to the engine)
  std::optional<double> PlacementScore;   // :187-189
  uint32_t UnboundPods = 0;               // best-effort pods (beyond MinReplicas) of a scheduled PodGang that found no node
  bool DisruptionTarget = false;          // condition PodGangConditionTypeDisruptionTarget :166-170, reason 1: "PodGang is preempted
  std::string DisruptionMessage;          // by a higher priority PodGang" -- names the preemptor; the caller terminates the pods
  std::vector<NamespacedName> EvictedPods;  // elastic preemption: pods above their PodGroup's MinReplicas that a higher priority
                                            // PodGang took; the caller terminates them, the PodGang keeps running
};
struct PodGang {
  std::string Namespace, Name;
  std::map<std::string, std::string> Labels;  // grove.io/scheduler-name etc.
  PodGangSpec Spec;
  PodGangStatus Status;
  // not part of the CRD: what the pod template of each PodGroup requests (a scheduler reads it from the Pods)
  struct Requests {
    uint32_t cpu_milli = 0, mem_mib = 0; uint16_t gpu = 0; std::map<std::string, std::string> nodeSelector; std::vector<std::string> tolerationKeys;
    // auto-MNNVL: the resourceClaimTemplateName of the pod template's `mnnvl-claim` entry, i.e. the ComputeDomain its pods join;
    // empty = not enrolled (the operator injects the claim only into GPU containers: a PodGroup without GPUs is never enrolled)
    std::string ComputeDomain;
  };
  std::map<std::string, Requests> PodGroupRequests;  // by PodGroup name
  std::string BasePodGangName;                        // scaled PodGang: gated behind this one (syncflow.go:319-358)
  bool Gated = false;                                 // pods still carry grove.io/podgang-pending-creation
};

// ---- operator/api/core/v1alpha1: the slice of PodCliqueSet the producer reads ----------------------
struct TopologyLevel { std::string Domain, Key; };                                   // clustertopology.go:111-124
struct PackDomain { std::string packDomain; };                                       // TopologyConstraint{PackDomain}
struct PodCliqueTemplateSpec {
  std::string Name;
  int32_t Replicas = 1;
  std::optional<int32_t> MinAvailable;          // defaulted to Replicas (defaulting/podcliqueset.go:74-83)
  std::optional<PackDomain> Topology;
  PodGang::Requests Requests;
};
struct PodCliqueScalingGroupConfig {
  std::string Name;
  std::vector<std::string> CliqueNames;
  std::optional<int32_t> Replicas;               // kubebuilder default 1 (podcliqueset.go:308-309)
  std::optional<int32_t> MinAvailable;           // kubebuilder default 1 (podcliqueset.go:321-322)
  std::optional<PackDomain> Topology;
};
struct PodCliqueSet {
  std::string Namespace = "default", Name;
  int32_t Replicas = 1;
  std::vector<PodCliqueTemplateSpec> Cliques;
  std::vector<PodCliqueScalingGroupConfig> PodCliqueScalingGroupConfigs;
  std::optional<PackDomain> Topology;
  std::string PriorityClassName;
};

// ---- namegen.go ------------------------------------------------------------------------------------
std::string GeneratePodCliqueName(const std::string& owner, int replica, const std::string& pclqTemplateName);  // :70-72
std::string GeneratePodCliqueScalingGroupName(const std::string& pcs, int replica, const std::string& name);    // :76-78
std::string GenerateBasePodGangName(const std::string& pcs, int replica);                                       // :82-84
std::string CreatePodGangNameFromPCSGFQN(const std::string& pcsgFQN, int scaledPodGangIndex);                   // :88-90

// ---- the producer (syncflow.go) ----------------------------------------------------------------------
struct PclqInfo {            // syncflow.go:776-783
  std::string fqn;
  int32_t replicas = 0, minAvailable = 0;
  std::optional<TopologyConstraint> topologyConstraint;
  std::string templateName;
};
struct PodGangInfo {         // syncflow.go:763-774
  std::string fqn;
  std::optional<TopologyConstraint> topologyConstraint;
  std::vector<PclqInfo> pclqs;
  std::vector<TopologyConstraintGroupConfig> pcsgTopologyConstraints;
  std::string baseFqn;       // "" for base PodGangs
};
// applies the defaulting webhook's MinAvailable := Replicas, then computeExpectedPodGangs
Err ComputeExpectedPodGangs(const PodCliqueSet& pcs, const std::vector<TopologyLevel>& topologyLevels, bool tasEnabled,
                            std::vector<PodGangInfo>* out);
// buildResource + createPodGroupsForPodGang (podgang.go:128-186); pod names are <pclq>-<ordinal>, sorted
PodGang BuildPodGang(const PodCliqueSet& pcs, const PodGangInfo& info);

// ---- webhook rule the packing relies on (webhook/admission/pcs/validation/topologyconstraints.go:195-268) ----
// A parent's pack domain must not be narrower than a child's (PodCliqueSet vs PodClique, PodCliqueSet vs
// PodCliqueScalingGroup, PodCliqueScalingGroup vs its PodCliques); domains unknown to the ClusterTopology are skipped.
// One FieldError per violating pair, in the reference's order, with the reference's field paths.
struct FieldError { std::string field, message; };
std::vector<FieldError> ValidateHierarchicalTopologyConstraints(const PodCliqueSet& pcs, const std::vector<std::string>& clusterTopologyDomains);

// ---- the gang predicate (podclique/components/pod/syncflow.go:316-358) ---------------------------------------
// A base PodGang is "scheduled" when every PodGroup has ScheduledReplicas >= MinReplicas; scaled PodGangs stay gated
// until then.  base == nullptr (PodGang not found) and a PodGroup without a PodClique status are errors: the caller
// requeues, as the reference does for every Get failure.  scheduledReplicas: PodClique name -> Status.ScheduledReplicas
// (podclique/reconcilestatus.go:134-141).
Err IsBasePodGangScheduled(const PodGang* base, const std::map<std::string, int32_t>& scheduledReplicas, bool* scheduled);

// What the bindings turn into on the way back (podclique/reconcilestatus.go:134-141, 255-274): ScheduledReplicas = pods of
// the PodClique with PodScheduled=True, and the PodCliqueScheduled condition on it.
struct Condition { std::string Type, Status, Reason, Message; };
Condition ComputePodCliqueScheduledCondition(int32_t scheduledReplicas, int32_t minAvailable);
// bindings of one cycle -> ScheduledReplicas per PodClique (pod names are <pclq fqn>-<ordinal>)
std::map<std::string, int32_t> CountScheduledReplicas(const std::vector<struct Binding>& bindings);

// Which pods reach a scheduler at all (checkAndRemovePodSchedulingGates, pod/syncflow.go:255-312): a pod loses its
// grove.io/podgang-pending-creation gate when it carries the gate, is already listed in its PodGang's PodReferences,
// and its PodGang is a base PodGang or its base PodGang is scheduled.  basePodGangName empty = the pod's PodGang is a
// base PodGang.  *removed: the gate is removed now; *skipped: the pod keeps its gate and is counted as skipped.
Err CheckPodSchedulingGate(bool podHasGate, bool podListedInPodGang, const std::string& basePodGangName, const PodGang* base,
                           const std::map<std::string, int32_t>& scheduledReplicas, bool* removed, bool* skipped);

// ---- nodes ------------------------------------------------------------------------------------------
struct Node {   // the slice of corev1.Node + bound Pods a scheduler snapshots; shape of kwok.py:74-117
  std::string Name;
  std::map<std::string, std::string> Labels;
  uint32_t alloc_cpu_milli = 0, alloc_mem_mib = 0; uint16_t alloc_gpu = 0, alloc_pods = 110;
  uint32_t used_cpu_milli = 0, used_mem_mib = 0; uint16_t used_gpu = 0, used_pods = 0;
  bool Unschedulable = false;                 // cordon
  std::vector<std::string> TaintKeys;         // NoSchedule taints
  std::string ComputeDomain;                  // the ComputeDomain whose pods hold the node's IMEX channel, as observed ("" = none seen)
  bool ImexCapable = true;                    // false: the node runs no IMEX driver (no enrolled pod may land on it)
};

struct Binding { std::string PodNamespace, PodName, NodeName; };   // Pod.spec.nodeName

// ---- operator/internal/scheduler/types.go ---------------------------------------------------------------
class Backend {                                                                       // :37-58
 public:
  virtual ~Backend() = default;
  virtual std::string Name() const = 0;
  virtual Err Init() = 0;
  virtual Err SyncPodGang(const PodGang& podGang) = 0;          // read-only on the cache-owned object
  virtual Err OnPodGangDelete(const PodGang& podGang) = 0;
  virtual void PreparePod(std::string* schedulerName) const = 0; // sets pod.spec.schedulerName
  virtual Err ValidatePodCliqueSet(const PodCliqueSet& pcs) const = 0;
};
struct GroupVersionResource { std::string Group, Version, Resource; };                // schema.GroupVersionResource
class TopologyAwareSchedBackend {                                                     // :64-96
 public:
  virtual ~TopologyAwareSchedBackend() = default;
  virtual GroupVersionResource TopologyGVR() const = 0;                               // :65-68
  virtual std::string TopologyResourceName(const std::string& clusterTopologyName) const = 0;
  virtual Err SyncTopology(const std::vector<TopologyLevel>& levels) = 0;
  virtual Err OnTopologyDelete() = 0;
  // (inSync, message)
  virtual std::pair<bool, std::string> CheckTopologyDrift(const std::vector<TopologyLevel>& levels) const = 0;
};

// a PodCliqueSet's topology spread (Kubernetes TopologySpreadConstraint at PodGang granularity; DESIGN.md section 1)
struct TopologySpread {
  std::string LevelKey;                               // a level of the ClusterTopology: the replicas spread over its domains
  int32_t MaxSkew = 1;                                // >= 1
  std::string WhenUnsatisfiable = "DoNotSchedule";    // or "ScheduleAnyway"
};

// a KAI queue's hard limits (scheduling.run.ai/v2 Queue: spec.parentQueue, spec.resources.{cpu,memory,gpu}.limit; DESIGN.md
// section 1 "Queue limits"), in the engine's units: millicores, MiB, GPUs.  nullopt = no limit (KAI's -1).  The deserved quota
// (spec.resources.{cpu,memory,gpu}.quota; DESIGN.md section 1 "Reclaim across queues") in the same units; nullopt = KAI's -1, the
// queue deserves whatever it holds.  Only SetReclaimAcrossQueues reads it.  The over-quota weight
// (spec.resources.{cpu,memory,gpu}.overQuotaWeight; DESIGN.md section 1 "Over-quota weight"): the queue's share of the capacity
// nobody deserves relative to its siblings; nullopt = 1, KAI's default.  Only SetOverQuotaWeights reads it.
struct Queue {
  std::string Parent;                            // "" = a root queue; otherwise a queue set earlier
  std::optional<uint64_t> CpuMilli, MemMiB, Gpu;
  std::optional<uint64_t> DeservedCpuMilli, DeservedMemMiB, DeservedGpu;
  std::optional<uint32_t> OverQuotaWeightCpu, OverQuotaWeightMem, OverQuotaWeightGpu;
};

// packed tables of one cycle, as handed to libgrove_place.so
struct Tables {
  std::vector<grove_node_t> nodes;
  std::vector<grove_gang_t> gangs;
  std::vector<grove_clique_t> cliques;
  std::vector<grove_clique_count_t> counts;             // clique row -> MinReplicas / replicas (what grove_submit_gangs_wide reads)
  std::vector<grove_scope_t> scopes;
  std::vector<std::string> gangNames;                 // row -> PodGang "<ns>/<name>"
  std::vector<std::pair<uint32_t, uint32_t>> cliqueOf; // clique row -> (gang row, PodGroup index in Spec.PodGroups)
  std::vector<uint8_t> remainder;                       // gang row -> 1: unbound pods of an already scheduled PodGang (MinReplicas 0)
  std::vector<uint32_t> refBase;                        // clique row -> first PodReference its placement entries bind (remainders)
  std::map<std::string, std::string> skipped;           // PodGang "<ns>/<name>" -> why it was left out of this pass
  // topology spread (SetTopologySpread): the groups, each gang row's group (GROVE_NONE_U32: none), the running replicas
  std::vector<grove_spread_t> spreadGroups;
  std::vector<uint32_t> spreadOf;
  std::vector<grove_spread_seed_t> spreadSeeds;
  std::vector<std::string> spreadSet;                   // group -> "<ns>/<PodCliqueSet>"
  // queue limits (SetQueue): the queues (parents first) with what the running PodGangs of each hold, each gang row's queue
  // (GROVE_NONE_U32: none)
  std::vector<grove_queue_t> queues;
  std::vector<grove_queue_quota_t> quotas;              // per queue of `queues`, its deserved quota
  std::vector<grove_queue_weight_t> weights;            // per queue of `queues`, its over-quota weights
  std::vector<std::string> queueNames;
  std::vector<uint32_t> queueOf;
  // consolidation (SetConsolidation): rows [specRow, gangs.size()) are gated rows restating running PodGangs, which makes them
  // movable (grove_run_cycle_consolidate's spec rows); specRow == gangs.size() when there are none
  uint32_t specRow = 0;
};

// The `gpu` scheduler backend: the third case of newBackendForProfile (manager/manager.go:35-52).
class GpuBackend : public Backend, public TopologyAwareSchedBackend {
 public:
  static constexpr const char* kName = "gpu-scheduler";
  explicit GpuBackend(int device = 0, std::string classLabelKey = "node_role.e2e.grove.nvidia.com");
  ~GpuBackend() override;
  std::string Name() const override { return kName; }
  Err Init() override;                       // creates the engine handle; fails (no fallback) without a CUDA device
  Err SyncPodGang(const PodGang& podGang) override;
  Err OnPodGangDelete(const PodGang& podGang) override;
  void PreparePod(std::string* schedulerName) const override { *schedulerName = kName; }
  Err ValidatePodCliqueSet(const PodCliqueSet& pcs) const override;
  // this backend keeps no topology CR of its own: the ordered level keys of the ClusterTopology ARE its topology
  // (kai/topology.go:40-46 returns KAI's CRD here); the CT controller's dynamic watch lands on the ClusterTopology itself
  GroupVersionResource TopologyGVR() const override { return {"grove.io", "v1alpha1", "clustertopologies"}; }
  std::string TopologyResourceName(const std::string& ct) const override { return ct; }
  Err SyncTopology(const std::vector<TopologyLevel>& levels) override;
  Err OnTopologyDelete() override;
  std::pair<bool, std::string> CheckTopologyDrift(const std::vector<TopologyLevel>& levels) const override;

  // encode the pending PodGangs + a node snapshot into packed tables (no GPU needed; unit-testable)
  Err Encode(const std::vector<Node>& nodes, Tables* out) const;
  // one scheduling cycle: Encode -> grove_load_nodes / submit / run_cycle -> bindings + PodGang statuses
  Err RunCycle(const std::vector<Node>& nodes, std::vector<Binding>* bindings, std::map<std::string, PodGangStatus>* statuses,
               grove_cycle_stats_t* stats = nullptr);
  size_t Pending() const { std::lock_guard<std::mutex> l(mu_); return pending_.size(); }   // PodGangs with unbound pods (unscheduled, or scheduled with a remainder)
  size_t Unscheduled() const { std::lock_guard<std::mutex> l(mu_); return pending_.size() - bound_.size(); }
  void SetPriorityClass(const std::string& name, int32_t value) { std::lock_guard<std::mutex> l(mu_); priorityClasses_[name] = value; }
  // Preemption (podgang.go:166-170): with it on, a cycle is grove_run_cycle_preempt -- PodGangs this backend scheduled earlier
  // are the RUNNING gangs (priority + what they hold per node, remembered from their bindings); a PodGang the ordinary pass
  // rejects may evict running PodGangs of a lower priority.  Victims come back in `statuses` with DisruptionTarget set and
  // are forgotten here: the caller deletes their pods (the node snapshot of the next cycle shows the resources as free).
  void SetPreemption(bool on) { std::lock_guard<std::mutex> l(mu_); preemption_ = on; }
  // Elastic preemption (PodGroup.MinReplicas, podgang.go:80-83; DESIGN.md section 1 "Elastic reclaim"): with it and SetPreemption
  // on, and no reservation reuse, queue or consolidation switch, a cycle with running PodGangs is grove_run_cycle_preempt_elastic:
  // the bound pods of each running PodGroup beyond MinReplicas (highest PodReference index first) are surplus, and a preemptor
  // takes those before it evicts any PodGang whole.  A PodGang that lost pods keeps running, is not a DisruptionTarget, and comes
  // back in `statuses` with EvictedPods naming them; their holdings are forgotten here.  Off by default.
  void SetElasticPreemption(bool on) { std::lock_guard<std::mutex> l(mu_); elastic_ = on; }
  // Reservation reuse (ReuseReservationRef, podgang.go:65-71): with it on, a PodGang whose ReuseReservationRef names a running
  // PodGang is that gang's new version and the cycle is grove_run_cycle_reuse -- it may use what its predecessor holds, nobody
  // else may.  Once it is admitted the predecessor is forgotten as running (the caller deletes its pods; a later OnPodGangDelete
  // of it releases nothing twice).  The anchor hint stays either way.  Off by default; a cycle with both this and preemption on
  // fails.
  void SetReservationReuse(bool on) { std::lock_guard<std::mutex> l(mu_); reuse_ = on; }
  // Reuse with reclaim: with it on, a cycle with running PodGangs is grove_run_cycle_reuse_preempt -- reservation reuse as
  // above, then the reclaim pass, in which a rejected new version may also use its predecessor's reservation -- whatever
  // SetPreemption and SetReservationReuse say.  Admitted new versions forget their predecessor (not disrupted); victims get
  // DisruptionTarget naming their preemptor and are forgotten.  Off by default; with it off the other two switches work as
  // before: either one alone, and both together fail.
  void SetReclaimWithReuse(bool on) { std::lock_guard<std::mutex> l(mu_); reclaimReuse_ = on; }
  // Preemption within queue limits: with it and SetPreemption on (reservation reuse and reuse with reclaim off), queue members are
  // no longer kept out of a pass with preemption; a pass with members is grove_run_cycle_preempt_queues, whose running gangs'
  // queues are the ones their PodGangs were scheduled in.  A member its queue chain turns away may then evict lower-priority
  // PodGangs of its own queues; victims get DisruptionTarget naming their preemptor, as with preemption.  Off by default.
  void SetPreemptionWithinQueues(bool on) { std::lock_guard<std::mutex> l(mu_); preemptQueues_ = on; }
  // Reclaim across queues (KAI's reclaim action; DESIGN.md section 1 "Reclaim across queues"): with it on (reservation reuse and
  // reuse with reclaim off), queue members stay in the pass and a pass with members and running PodGangs is
  // grove_run_cycle_reclaim_queues, with each Queue's deserved quota and each running PodGang's queue the one it was scheduled in.
  // A queue below its quota may then evict running PodGangs of queues above theirs, whatever the priorities; victims get
  // DisruptionTarget naming the reclaimer and its queue.  Off by default; a cycle with both this and SetPreemptionWithinQueues on
  // fails.
  void SetReclaimAcrossQueues(bool on) { std::lock_guard<std::mutex> l(mu_); reclaimQueues_ = on; }
  // Reclaim, then preempt (KAI's reclaim action, then its preempt action; DESIGN.md section 1 "Reclaim, then preempt"): with it
  // and SetPreemption on (reservation reuse and reuse with reclaim off), queue members stay in the pass and a pass with members
  // and running PodGangs is grove_run_cycle_reclaim_preempt_queues, whatever SetReclaimAcrossQueues and
  // SetPreemptionWithinQueues say.  Victims of the reclaim pass get DisruptionTarget naming the reclaimer and its queue, those of
  // the preempt pass naming their preemptor.  Off by default.
  void SetReclaimThenPreempt(bool on) { std::lock_guard<std::mutex> l(mu_); reclaimThenPreempt_ = on; }
  // Fair-share order (KAI's allocate order; DESIGN.md section 1 "Fair-share order"): with it on, a pass with queue members and no
  // preemption, reservation reuse or consolidation runs the queue cycle with grove_set_fair_share and each Queue's deserved quota:
  // the next turn goes to the queue furthest below its quota, priority orders PodGangs only inside a queue.  Members must sit in
  // leaf queues (a cycle with a member in a parent queue fails).  Bin-packing is not applied in such a pass.  Off by default.
  void SetFairShareOrder(bool on) { std::lock_guard<std::mutex> l(mu_); fairShare_ = on; }
  // Over-quota weight (KAI's proportion plugin; DESIGN.md section 1 "Over-quota weight"): with it on, every cycle that runs with
  // quotas -- SetReclaimAcrossQueues, SetReclaimThenPreempt, SetFairShareOrder -- sets each Queue's over-quota weights
  // (grove_set_over_quota), so that a queue's fair share, its deserved quota plus its weighted slice of the capacity nobody
  // deserves, stands in for the deserved quota.  Off by default; off behaves exactly as before.
  void SetOverQuotaWeights(bool on) { std::lock_guard<std::mutex> l(mu_); overQuota_ = on; }
  // the fair shares (cpu milli, mem MiB, gpu; GROVE_QUEUE_UNLIMITED where the deserved quota is unlimited) of the last cycle that
  // ran with weights, by queue name, as KAI reports them in queue status; empty before such a cycle
  std::map<std::string, std::array<uint64_t, 3>> FairShares() const { std::lock_guard<std::mutex> l(mu_); return fairShares_; }
  // Large PodGangs: with it on, PodGangs of up to GROVE_MAX_WIDE_GANG_PODS pods (PodGroups of up to as many) are encoded and a
  // cycle submits through grove_submit_gangs_wide; ValidatePodCliqueSet accepts base PodGangs of that size.  The running-gang
  // cycles (preemption, reservation reuse, reuse with reclaim) do not take such PodGangs: while one of those switches is on too,
  // a PodGang beyond GROVE_MAX_GANG_PODS pods or 255 replicas stays out of the pass, Unschedulable with a reason that says so.
  // Off by default; off behaves exactly as before.
  void SetLargePodGangs(bool on) { std::lock_guard<std::mutex> l(mu_); large_ = on; }
  // Unschedulable messages: with it on, after an ordinary cycle (no running-gang cycle: no preemption, reservation reuse or
  // reuse with reclaim) the ScheduledMessage of every rejected PodGang says why, from grove_diagnose: the first PodGroup that
  // fits nowhere in the cluster with the nodes each predicate turned away, or how many domains of the PodGang's Required level
  // hold each PodGroup's MinReplicas.  Off by default (the message stays empty, as before).
  void SetExplainUnschedulable(bool on) { std::lock_guard<std::mutex> l(mu_); explain_ = on; }
  // the message for one rejected PodGang row of `t` from its diagnosis records (levels: the ClusterTopology's, broadest first)
  static std::string ExplainRejection(const Tables& t, const PodGang& pg, uint32_t row, const grove_gang_diag_t& gd,
                                      const grove_clique_diag_t* cliques, const std::vector<TopologyLevel>& levels);
  // Topology spread: the pending BASE PodGangs (no BasePodGangName) whose app.kubernetes.io/part-of label names the PodCliqueSet
  // `pcsName` spread over the domains of `spread.LevelKey` (grove_set_spread); the running base PodGangs of the set that this
  // backend scheduled count where they landed.  A member must have a Required level at or below that level and a PodGroup with
  // MinReplicas > 0; other PodGangs of the set are packed as usual and not counted.  A DoNotSchedule member rejected at its turn
  // gets a ScheduledMessage that names the spread; a ScheduleAnyway member placed outside the allowed domains is scheduled with a
  // message that says so.  With preemption, reservation reuse or reuse with reclaim on, or in a pass with a PodGang beyond the
  // ordinary limits (SetLargePodGangs), members stay out of the pass, Unschedulable with a reason.  nullopt removes the set's
  // spread.  Off by default (no set has one).
  Err SetTopologySpread(const std::string& pcsName, std::optional<TopologySpread> spread);
  // Starvation guard (grove_set_fences; DESIGN.md section 1 "Fences"): counts, per pending PodGang, the consecutive cycles it came
  // back Unschedulable (REJECTED; a gated or base-not-scheduled cycle neither counts nor resets, a scheduled one resets).  Each
  // cycle the <= maxGangs highest-ranked PodGangs with a Required level that were rejected at least afterCycles times fence a
  // domain: while one of them stays rejected, the PodGangs ranked after it are kept out of the domain of its Required level that
  // was closest to fitting it, so that the nodes freed there accumulate for it.  A fencing PodGang's ScheduledMessage names the
  // level and the label value of that domain.  In a pass with preemption, reservation reuse or topology spread members, or with a
  // PodGang beyond the ordinary limits (SetLargePodGangs), nothing is fenced (the counts go on).  maxGangs = 0 turns it off (the
  // default); afterCycles >= 1, maxGangs <= GROVE_MAX_FENCES.
  Err SetStarvationGuard(uint32_t afterCycles, uint32_t maxGangs);
  // Bin-packing (grove_set_binpack; DESIGN.md section 1 "Bin-packing"): with the key of a topology level, every PodGang of an
  // ordinary or queue pass starts its search at the fullest domain of that level -- or of its own Required level when that is
  // deeper -- that can hold it on the cycle's node table, so that empty domains stay empty for large PodGangs.  A preference, not a
  // constraint: in a pass with preemption, reservation reuse, consolidation, topology spread members, fences or a PodGang beyond the
  // ordinary limits (SetLargePodGangs) the pass runs without it, and so does every pass while the key names no level of the
  // topology.  An empty key (the default) turns it off.
  void SetBinPacking(const std::string& levelKey) { std::lock_guard<std::mutex> l(mu_); binpackKey_ = levelKey; }
  // ComputeDomain exclusivity (grove_set_compute_domains; DESIGN.md section 1 "ComputeDomain exclusivity"): a node's GPUs take part
  // in one IMEX channel at a time, so the pods of an enrolled PodGroup (Requests::ComputeDomain) land only on nodes no other
  // ComputeDomain holds.  A node's holder when the pass starts is Node::ComputeDomain, else the ComputeDomain of the enrolled pods
  // this backend bound there for a PodGang that still runs; a node that is not ImexCapable takes no enrolled pod.  A PodGang whose
  // PodGroups name two ComputeDomains stays out of the pass (Unschedulable, with the reason), and so does every enrolled PodGang
  // while preemption, reservation reuse, consolidation, the starvation guard, bin-packing, topology spread members, queue members
  // or a PodGang beyond the ordinary limits could be in the pass.  Off (the default): the pass is as before.
  void SetComputeDomainExclusivity(bool on) { std::lock_guard<std::mutex> l(mu_); imex_ = on; }
  // Consolidation (grove_run_cycle_consolidate; DESIGN.md section 1 "Consolidation"): the spec of every PodGang this backend
  // scheduled is remembered, and each running PodGang it scheduled whole (nothing left pending) is restated as a gated row, which
  // makes it movable.  Each cycle the <= maxTargets highest-ranked pending PodGangs rejected at least afterCycles times in a row
  // (counted as the starvation guard counts) are the targets: running PodGangs of their priority or below are relocated out of the
  // domain closest to fitting one when every relocated PodGang is admitted elsewhere.  A moved PodGang comes back in `statuses`
  // with DisruptionTarget set and a message naming the PodGang it made room for; it is forgotten as running (the caller deletes
  // its pods), and when it is synced again it is anchored at the first node of the placement the cycle planned for it.  A
  // consolidated PodGang's ScheduledMessage names the PodGangs that were moved.  Only in a pass without preemption, reservation
  // reuse, topology spread members or PodGangs beyond the ordinary limits.  maxTargets = 0 turns it off (the default);
  // afterCycles >= 1, maxTargets <= GROVE_MAX_CONSOLIDATE_TARGETS; it cannot be on together with the starvation guard.
  Err SetConsolidation(uint32_t afterCycles, uint32_t maxTargets);
  // Queue limits (grove_set_queues; DESIGN.md section 1 "Queue limits"): a pending PodGang whose kai.scheduler/queue label names
  // a queue set here is a member of it (a label naming an unknown queue makes it a non-member); what the PodGangs this backend
  // scheduled hold counts against their queue and its ancestors.  A member whose queue chain has no room for its MinReplicas is
  // Unschedulable with a ScheduledMessage naming the first queue of its chain (leaf first) and the resource that had no room, with
  // limit and load; a scheduled member whose best-effort pods the limits held back says how many.  With preemption, reservation
  // reuse, reuse with reclaim, consolidation or the starvation guard on, or in a pass with topology spread members or a PodGang
  // beyond the ordinary limits, members stay out of the pass, Unschedulable with a reason.  A parent must be set before its
  // children, chains are at most GROVE_MAX_QUEUE_DEPTH deep; nullopt removes a queue (not one that is a parent).  Off by default.
  Err SetQueue(const std::string& name, std::optional<Queue> queue);
  // the ScheduledMessages of the queue members of one cycle of `t` (gs, pl: its statuses and placements)
  static std::map<std::string, std::string> QueueMessages(const Tables& t, const std::vector<grove_gang_status_t>& gs,
                                                          const std::vector<grove_placement_t>& pl);
  static constexpr const char* kQueueLabel = "kai.scheduler/queue";
  static constexpr const char* kPartOfLabel = "app.kubernetes.io/part-of";
  size_t Running() const { std::lock_guard<std::mutex> l(mu_); return running_.size(); }
  // why a PodGang cannot be handed to the engine (limits of the packed tables), or empty.  SyncPodGang accepts every
  // PodGang -- the reference's reconciler would requeue forever on an error -- and RunCycle reports these as
  // Unschedulable with this message instead of failing the pass for everybody (ADVICE round 1).
  static std::string WhyNotEncodable(const PodGang& pg);
  // the same under the limits of a large-PodGang backend (large = true: GROVE_MAX_WIDE_GANG_PODS pods per PodGang and PodGroup)
  static std::string WhyNotEncodable(const PodGang& pg, bool large);

  // The cycle loop of the backend (INTEGRATION.md section 2): SyncPodGang / OnPodGangDelete are called concurrently by
  // the PodGang reconcilers (controller/podgang/register.go:34-36, MaxConcurrentReconciles) and only touch the pending
  // set under the mutex; ONE thread takes node snapshots, runs cycles on the engine handle (not thread-safe) and hands
  // bindings + statuses to the binder callback.
  using SnapshotFn = std::function<std::vector<Node>()>;
  using BindFn = std::function<void(const std::vector<Binding>&, const std::map<std::string, PodGangStatus>&, const grove_cycle_stats_t&)>;
  Err Start(SnapshotFn snapshot, BindFn bind, std::chrono::milliseconds period);
  void Stop();
  uint64_t Cycles() const { return cycles_.load(); }

 private:
  int device_;
  std::string classKey_;
  std::vector<TopologyLevel> levels_;
  std::map<std::string, PodGang> pending_;   // "<ns>/<name>" -> copy (the cache-owned object is never retained)
  std::map<std::string, int32_t> priorityClasses_;
  std::map<std::string, std::string> lastNode_;  // scheduled PodGang -> a node it landed on (ReuseReservationRef hint)
  std::map<std::string, std::vector<uint32_t>> bound_;  // scheduled PodGang still pending with unbound pods -> pods bound per PodGroup
  struct Held { std::string node; uint32_t cpu_milli = 0, mem_mib = 0; uint16_t gpu = 0, pods = 0; };
  // a pod this backend bound for a running PodGang: its PodGroup, PodReference index and what it takes on its node
  struct BoundPod { NamespacedName ref; uint32_t group = 0, index = 0; std::string node; uint32_t cpu_milli = 0, mem_mib = 0; uint16_t gpu = 0; };
  // cdOn: node -> the ComputeDomain of its enrolled pods there; pods, minReplicas: its bound pods and every PodGroup's MinReplicas
  // (elastic preemption)
  struct RunningGang {
    int32_t priority = 0; std::vector<Held> held; std::map<std::string, std::string> cdOn;
    std::vector<BoundPod> pods; std::vector<int32_t> minReplicas;
  };
  std::map<std::string, RunningGang> running_;   // PodGangs scheduled by this backend and not deleted since
  bool preemption_ = false;
  bool elastic_ = false;
  bool reuse_ = false;
  bool reclaimReuse_ = false;
  bool preemptQueues_ = false;
  bool reclaimQueues_ = false;
  bool reclaimThenPreempt_ = false;
  bool fairShare_ = false;
  bool overQuota_ = false;
  std::map<std::string, std::array<uint64_t, 3>> fairShares_;   // FairShares()
  bool large_ = false;
  bool explain_ = false;
  std::string binpackKey_;                             // bin-packing level (off: empty)
  bool imex_ = false;                                  // ComputeDomain exclusivity
  uint32_t guardAfter_ = 1, guardMax_ = 0;             // starvation guard (off: guardMax_ == 0)
  std::map<std::string, uint32_t> rejectedFor_;        // pending PodGang -> consecutive Unschedulable cycles
  uint32_t consAfter_ = 1, consMax_ = 0;               // consolidation (off: consMax_ == 0)
  std::map<std::string, PodGang> specOf_;              // scheduled PodGang -> its spec (what a gated row restating it encodes)
  std::map<std::string, std::string> moveAnchor_;      // moved PodGang -> the first node of its planned placement (anchor)
  std::map<std::string, TopologySpread> spread_;       // PodCliqueSet name -> its spread
  std::map<std::string, std::string> setOf_;           // scheduled base PodGang -> "<ns>/<PodCliqueSet>" (its part-of label)
  std::map<std::string, Queue> queues_;                // queue name -> its limits
  std::map<std::string, std::string> queueOf_;         // scheduled PodGang -> its queue (kai.scheduler/queue label)
  grove_engine_t* engine_ = nullptr;
  uint32_t engineLevels_ = 0;
  mutable std::mutex mu_;        // pending set, bindings, levels: everything SyncPodGang / OnPodGangDelete / SyncTopology touch
  std::mutex cycleMu_;           // one cycle at a time on the engine handle
  std::thread loop_;
  std::condition_variable cv_;
  bool stop_ = false;
  std::atomic<uint64_t> cycles_{0};
  // restate: running PodGangs to append as gated spec rows (consolidation), after every pending row
  Err EncodeLocked(const std::vector<Node>& nodes, Tables* out, const std::vector<std::string>* restate = nullptr) const;
};

}  // namespace grove::host
