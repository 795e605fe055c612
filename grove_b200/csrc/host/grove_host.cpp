// grove_host.cpp -- see grove_host.hpp.  Host-side mirror of the reference interfaces around the
// placement hot path; the placement itself happens behind the C ABI (libgrove_place.so).
#include "grove_host.hpp"

#include <algorithm>
#include <array>
#include <cstdint>
#include <set>

namespace grove::host {

static Error mkerr(const char* code, const char* op, std::string msg) { return Error{code, op, std::move(msg)}; }

// ---- namegen.go ------------------------------------------------------------------------------------
std::string GeneratePodCliqueName(const std::string& owner, int replica, const std::string& t) {
  return owner + "-" + std::to_string(replica) + "-" + t;
}
std::string GeneratePodCliqueScalingGroupName(const std::string& pcs, int replica, const std::string& name) {
  return pcs + "-" + std::to_string(replica) + "-" + name;
}
std::string GenerateBasePodGangName(const std::string& pcs, int replica) { return pcs + "-" + std::to_string(replica); }
std::string CreatePodGangNameFromPCSGFQN(const std::string& pcsgFQN, int idx) { return pcsgFQN + "-" + std::to_string(idx); }

// ---- producer: syncflow.go:145-371 -------------------------------------------------------------------
// createTopologyPackConstraint (syncflow.go:349-371): packDomain -> node-label key through the ordered
// ClusterTopology levels; TAS disabled, no constraint, or an unknown domain => nil.  Only Required is set.
static std::optional<TopologyConstraint> createTopologyPackConstraint(const std::vector<TopologyLevel>& levels, bool tas,
                                                                      const std::optional<PackDomain>& req) {
  if (!tas || !req) return std::nullopt;
  for (const auto& l : levels)
    if (l.Domain == req->packDomain) {
      TopologyConstraint tc;
      tc.PackConstraint = TopologyPackConstraint{l.Key, std::nullopt};
      return tc;
    }
  return std::nullopt;  // stale domain: the reference logs and nullifies the constraint
}

static const PodCliqueTemplateSpec* findClique(const PodCliqueSet& pcs, const std::string& name) {
  for (const auto& c : pcs.Cliques) if (c.Name == name) return &c;
  return nullptr;
}
static const PodCliqueScalingGroupConfig* findScalingGroupForClique(const PodCliqueSet& pcs, const std::string& clique) {
  for (const auto& g : pcs.PodCliqueScalingGroupConfigs)
    if (std::find(g.CliqueNames.begin(), g.CliqueNames.end(), clique) != g.CliqueNames.end()) return &g;
  return nullptr;
}

// buildPodCliqueInfo (syncflow.go:335-345); MinAvailable defaulted as the webhook does (defaulting/podcliqueset.go:74-83)
static PclqInfo buildPodCliqueInfo(const std::vector<TopologyLevel>& levels, bool tas, const PodCliqueTemplateSpec& t, const std::string& fqn) {
  PclqInfo p;
  p.fqn = fqn; p.replicas = t.Replicas; p.minAvailable = t.MinAvailable.value_or(t.Replicas); p.templateName = t.Name;
  p.topologyConstraint = createTopologyPackConstraint(levels, tas, t.Topology);
  return p;
}

Err ComputeExpectedPodGangs(const PodCliqueSet& pcs, const std::vector<TopologyLevel>& levels, bool tas, std::vector<PodGangInfo>* out) {
  out->clear();
  // base PodGang per PCS replica: standalone cliques + PCSG replicas [0, minAvailable) (syncflow.go:172-275)
  for (int r = 0; r < pcs.Replicas; ++r) {
    PodGangInfo pg;
    pg.fqn = GenerateBasePodGangName(pcs.Name, r);
    pg.topologyConstraint = createTopologyPackConstraint(levels, tas, pcs.Topology);
    for (const auto& t : pcs.Cliques)
      if (!findScalingGroupForClique(pcs, t.Name))
        pg.pclqs.push_back(buildPodCliqueInfo(levels, tas, t, GeneratePodCliqueName(pcs.Name, r, t.Name)));
    for (const auto& cfg : pcs.PodCliqueScalingGroupConfigs) {
      const int minAvailable = cfg.MinAvailable.value_or(1);
      const std::string pcsgFQN = GeneratePodCliqueScalingGroupName(pcs.Name, r, cfg.Name);
      for (int ri = 0; ri < minAvailable; ++ri) {
        std::vector<std::string> fqns;
        for (const auto& cn : cfg.CliqueNames) {
          const PodCliqueTemplateSpec* t = findClique(pcs, cn);
          if (!t) return mkerr("ERR_SYNC_PODGANG", "ComputeExpectedPodGangs",
                               "PodCliqueScalingGroup \"" + cfg.Name + "\" references a PodClique \"" + cn + "\" that does not exist in the PodCliqueSet");
          const std::string fqn = GeneratePodCliqueName(pcsgFQN, ri, cn);
          pg.pclqs.push_back(buildPodCliqueInfo(levels, tas, *t, fqn));
          fqns.push_back(fqn);
        }
        if (tas && cfg.Topology) {  // one TopologyConstraintGroupConfig per PCSG replica (syncflow.go:262-271)
          TopologyConstraintGroupConfig gc;
          gc.Name = pcsgFQN + "-" + std::to_string(ri);
          gc.PodGroupNames = fqns;
          gc.Topology = createTopologyPackConstraint(levels, tas, cfg.Topology);
          pg.pcsgTopologyConstraints.push_back(std::move(gc));
        }
      }
    }
    out->push_back(std::move(pg));
  }
  // scaled PodGang per PCSG replica >= minAvailable (syncflow.go:277-333)
  for (int r = 0; r < pcs.Replicas; ++r)
    for (const auto& cfg : pcs.PodCliqueScalingGroupConfigs) {
      const std::string pcsgFQN = GeneratePodCliqueScalingGroupName(pcs.Name, r, cfg.Name);
      const int replicas = cfg.Replicas.value_or(1), minAvailable = cfg.MinAvailable.value_or(1);
      for (int idx = 0, pr = minAvailable; idx < replicas - minAvailable; ++idx, ++pr) {
        PodGangInfo pg;
        pg.fqn = CreatePodGangNameFromPCSGFQN(pcsgFQN, idx);
        pg.baseFqn = GenerateBasePodGangName(pcs.Name, r);
        for (const auto& cn : cfg.CliqueNames) {
          const PodCliqueTemplateSpec* t = findClique(pcs, cn);
          if (!t) return mkerr("ERR_SYNC_PODGANG", "ComputeExpectedPodGangs", "PodCliqueScalingGroup references unknown PodClique \"" + cn + "\"");
          pg.pclqs.push_back(buildPodCliqueInfo(levels, tas, *t, GeneratePodCliqueName(pcsgFQN, pr, cn)));
        }
        // PCSG constraint if set, else fall back to the PCS constraint (syncflow.go:311-324)
        if (tas) pg.topologyConstraint = cfg.Topology ? createTopologyPackConstraint(levels, tas, cfg.Topology)
                                                      : createTopologyPackConstraint(levels, tas, pcs.Topology);
        out->push_back(std::move(pg));
      }
    }
  return std::nullopt;
}

PodGang BuildPodGang(const PodCliqueSet& pcs, const PodGangInfo& info) {
  PodGang pg;
  pg.Namespace = pcs.Namespace; pg.Name = info.fqn;
  pg.Labels["grove.io/scheduler-name"] = GpuBackend::kName;
  pg.Spec.Topology = info.topologyConstraint;
  pg.Spec.TopologyConstraintGroupConfigs = info.pcsgTopologyConstraints;
  pg.Spec.PriorityClassName = pcs.PriorityClassName;
  pg.BasePodGangName = info.baseFqn;
  for (const auto& p : info.pclqs) {  // createPodGroupsForPodGang (podgang.go:165-186)
    PodGroup g;
    g.Name = p.fqn; g.MinReplicas = p.minAvailable; g.Topology = p.topologyConstraint;
    for (int i = 0; i < p.replicas; ++i) g.PodReferences.push_back({pcs.Namespace, p.fqn + "-" + std::to_string(i)});
    std::sort(g.PodReferences.begin(), g.PodReferences.end(), [](const NamespacedName& a, const NamespacedName& b) { return a.Name < b.Name; });
    pg.Spec.PodGroups.push_back(std::move(g));
    if (const PodCliqueTemplateSpec* t = findClique(pcs, p.templateName)) pg.PodGroupRequests[p.fqn] = t->Requests;
  }
  return pg;
}

// ---- GpuBackend ----------------------------------------------------------------------------------------
GpuBackend::GpuBackend(int device, std::string classLabelKey) : device_(device), classKey_(std::move(classLabelKey)) {}
GpuBackend::~GpuBackend() { Stop(); if (engine_) grove_engine_destroy(engine_); }

Err GpuBackend::Init() {
  if (levels_.empty()) return std::nullopt;  // the engine is created once the topology is known (SyncTopology)
  if (engine_ && engineLevels_ == levels_.size()) return std::nullopt;
  if (engine_) { grove_engine_destroy(engine_); engine_ = nullptr; }
  grove_config_t cfg{};
  cfg.abi_version = GROVE_ABI_VERSION; cfg.device = device_; cfg.n_levels = uint32_t(levels_.size());
  const int32_t rc = grove_engine_create(&cfg, &engine_);
  if (rc != GROVE_OK) { engine_ = nullptr; return mkerr("ERR_INIT_BACKEND", "Init", "grove_engine_create failed with " + std::to_string(rc) + " (there is no CPU fallback)"); }
  engineLevels_ = uint32_t(levels_.size());
  return std::nullopt;
}

Err GpuBackend::SyncTopology(const std::vector<TopologyLevel>& levels) {
  if (levels.empty() || levels.size() > GROVE_MAX_LEVELS)
    return mkerr("ERR_SYNC_TOPOLOGY", "SyncTopology", "the engine supports 1.." + std::to_string(GROVE_MAX_LEVELS) + " topology levels");
  std::lock_guard<std::mutex> l(mu_);
  levels_ = levels;  // ordered broadest -> narrowest, as desiredKAITopologyLevels hands them over (kai/topology.go:103-135)
  return std::nullopt;
}
Err GpuBackend::OnTopologyDelete() { std::lock_guard<std::mutex> l(mu_); levels_.clear(); return std::nullopt; }
std::pair<bool, std::string> GpuBackend::CheckTopologyDrift(const std::vector<TopologyLevel>& levels) const {
  std::lock_guard<std::mutex> l(mu_);
  if (levels.size() != levels_.size()) return {false, "level count differs"};
  for (size_t i = 0; i < levels.size(); ++i)
    if (levels[i].Key != levels_[i].Key) return {false, "level " + std::to_string(i) + " key " + levels_[i].Key + " != " + levels[i].Key};
  return {true, ""};
}

std::vector<FieldError> ValidateHierarchicalTopologyConstraints(const PodCliqueSet& pcs, const std::vector<std::string>& domains) {
  std::vector<FieldError> errs;
  auto index = [&domains](const std::string& d) { auto it = std::find(domains.begin(), domains.end(), d); return it == domains.end() ? -1 : int(it - domains.begin()); };
  auto violation = [&index](const std::string& parent, const std::string& child) {   // hasHierarchyViolation :195-202
    const int p = index(parent), c = index(child);
    return p != -1 && c != -1 && p > c;
  };
  auto msg = [](const std::string& pd, const std::string& pkind, const std::string& pname, const std::string& cd, const std::string& ckind, const std::string& cname) {
    const std::string who = pname.empty() ? pkind : pkind + " '" + pname + "'";
    return who + " topology constraint domain '" + pd + "' is narrower than " + ckind + " '" + cname + "' topology constraint domain '" + cd + "'";
  };
  const std::string root = "spec.template";
  if (pcs.Topology) {
    const std::string& pd = pcs.Topology->packDomain;
    for (const auto& c : pcs.Cliques)
      if (c.Topology && violation(pd, c.Topology->packDomain))
        errs.push_back({root + ".topologyConstraint", msg(pd, "PodCliqueSet", "", c.Topology->packDomain, "PodClique", c.Name)});
    for (const auto& g : pcs.PodCliqueScalingGroupConfigs)
      if (g.Topology && violation(pd, g.Topology->packDomain))
        errs.push_back({root + ".topologyConstraint", msg(pd, "PodCliqueSet", "", g.Topology->packDomain, "PodCliqueScalingGroup", g.Name)});
  }
  for (size_t i = 0; i < pcs.PodCliqueScalingGroupConfigs.size(); ++i) {
    const auto& g = pcs.PodCliqueScalingGroupConfigs[i];
    if (!g.Topology) continue;
    for (const auto& cn : g.CliqueNames) {
      auto it = std::find_if(pcs.Cliques.begin(), pcs.Cliques.end(), [&cn](const PodCliqueTemplateSpec& t) { return t.Name == cn; });
      if (it != pcs.Cliques.end() && it->Topology && violation(g.Topology->packDomain, it->Topology->packDomain))
        errs.push_back({root + ".podCliqueScalingGroups[" + std::to_string(i) + "].topologyConstraint",
                        msg(g.Topology->packDomain, "PodCliqueScalingGroup", g.Name, it->Topology->packDomain, "PodClique", it->Name)});
    }
  }
  return errs;
}

Err GpuBackend::ValidatePodCliqueSet(const PodCliqueSet& pcs) const {
  std::vector<std::string> domains;
  for (const auto& l : levels_) domains.push_back(l.Domain);
  if (auto errs = ValidateHierarchicalTopologyConstraints(pcs, domains); !errs.empty())
    return mkerr("ERR_VALIDATE_PCS", "ValidatePodCliqueSet", errs[0].field + ": " + errs[0].message);
  std::vector<PodGangInfo> infos;
  if (auto e = ComputeExpectedPodGangs(pcs, levels_, true, &infos)) return e;
  bool large;
  { std::lock_guard<std::mutex> l(mu_); large = large_; }
  const int maxPods = int(large ? GROVE_MAX_WIDE_GANG_PODS : GROVE_MAX_GANG_PODS);
  for (const auto& pg : infos) {
    int pods = 0;
    for (const auto& p : pg.pclqs) pods += p.replicas;
    if (pg.pclqs.size() > GROVE_MAX_GANG_CLIQUES || pods > maxPods || pg.pcsgTopologyConstraints.size() + 1 > GROVE_MAX_GANG_SCOPES)
      return mkerr("ERR_VALIDATE_PCS", "ValidatePodCliqueSet", "PodGang " + pg.fqn + " exceeds the gpu-scheduler limits (32 PodCliques / 32 constraint groups / " +
                                                                   std::to_string(maxPods) + " pods per PodGang)");
  }
  return std::nullopt;
}

Err GpuBackend::SyncPodGang(const PodGang& podGang) {
  std::lock_guard<std::mutex> l(mu_);   // called concurrently by the PodGang reconcilers (podgang/register.go:34-36)
  pending_[podGang.Namespace + "/" + podGang.Name] = podGang;  // a copy: the cache-owned object is neither mutated nor retained
  return std::nullopt;
}
Err IsBasePodGangScheduled(const PodGang* base, const std::map<std::string, int32_t>& scheduledReplicas, bool* scheduled) {
  *scheduled = false;
  if (!base) return mkerr("ERR_GET_PODGANG", "Sync", "failed to get base PodGang");
  for (const auto& g : base->Spec.PodGroups) {
    auto it = scheduledReplicas.find(g.Name);
    if (it == scheduledReplicas.end())
      return mkerr("ERR_GET_PODCLIQUE", "Sync", "failed to get PodClique " + g.Name + " in namespace " + base->Namespace + " for base PodGang readiness check");
    if (it->second < g.MinReplicas) return std::nullopt;  // not scheduled yet: a legitimate state, no error
  }
  *scheduled = true;
  return std::nullopt;
}

Condition ComputePodCliqueScheduledCondition(int32_t scheduledReplicas, int32_t minAvailable) {
  const std::string counts = "expected at least: " + std::to_string(minAvailable) + ", found: " + std::to_string(scheduledReplicas);
  if (scheduledReplicas < minAvailable) return {"PodCliqueScheduled", "False", "InsufficientScheduledPods", "Insufficient scheduled pods. " + counts};
  return {"PodCliqueScheduled", "True", "SufficientScheduledPods", "Sufficient scheduled pods found. " + counts};
}

std::map<std::string, int32_t> CountScheduledReplicas(const std::vector<Binding>& bindings) {
  std::map<std::string, int32_t> n;
  for (const auto& b : bindings) n[b.PodName.substr(0, b.PodName.rfind('-'))]++;
  return n;
}

Err CheckPodSchedulingGate(bool podHasGate, bool podListedInPodGang, const std::string& basePodGangName, const PodGang* base,
                           const std::map<std::string, int32_t>& scheduledReplicas, bool* removed, bool* skipped) {
  *removed = false; *skipped = false;
  bool baseScheduled = true;   // computed once per PodClique, before any pod is looked at (syncflow.go:259-269)
  if (!basePodGangName.empty()) {
    if (auto e = IsBasePodGangScheduled(base, scheduledReplicas, &baseScheduled))
      return mkerr("ERR_REMOVE_POD_SCHEDULING_GATE", "Sync", "failed to check if base PodGang is scheduled for PodClique: " + e->message);
  }
  if (!podHasGate) return std::nullopt;                                 // nothing to do, not a skip
  if (!podListedInPodGang) { *skipped = true; return std::nullopt; }    // not yet in PodGang.Spec.PodGroups[].PodReferences
  if (!baseScheduled) { *skipped = true; return std::nullopt; }         // scaled PodGang behind an unscheduled base
  *removed = true;
  return std::nullopt;
}

Err GpuBackend::OnPodGangDelete(const PodGang& podGang) {
  std::lock_guard<std::mutex> l(mu_);
  const std::string key = podGang.Namespace + "/" + podGang.Name;
  pending_.erase(key); bound_.erase(key); running_.erase(key); setOf_.erase(key); rejectedFor_.erase(key);
  specOf_.erase(key); moveAnchor_.erase(key); queueOf_.erase(key);
  return std::nullopt;
}

Err GpuBackend::SetQueue(const std::string& name, std::optional<Queue> queue) {
  std::lock_guard<std::mutex> l(mu_);
  if (name.empty()) return mkerr("ERR_SYNC_PODGANG", "SetQueue", "a queue needs a name");
  if (!queue) {
    for (const auto& [n, q] : queues_)
      if (q.Parent == name) return mkerr("ERR_SYNC_PODGANG", "SetQueue", "queue " + name + " is the parent of queue " + n);
    queues_.erase(name);
    return std::nullopt;
  }
  uint32_t depth = 1;
  for (std::string p = queue->Parent; !p.empty(); p = queues_.at(p).Parent) {
    if (p == name) return mkerr("ERR_SYNC_PODGANG", "SetQueue", "queue " + name + " would be its own ancestor");
    if (!queues_.count(p)) return mkerr("ERR_SYNC_PODGANG", "SetQueue", "queue " + name + ": parent queue " + p + " is not set");
    if (++depth > GROVE_MAX_QUEUE_DEPTH) return mkerr("ERR_SYNC_PODGANG", "SetQueue", "queue " + name + ": chain deeper than GROVE_MAX_QUEUE_DEPTH");
  }
  for (const auto& [n, q] : queues_)   // a queue that is a parent keeps its place in the tree
    if (q.Parent == name && queues_.at(name).Parent != queue->Parent)
      return mkerr("ERR_SYNC_PODGANG", "SetQueue", "queue " + name + " is the parent of queue " + n + ": its parent cannot change");
  if (!queues_.count(name) && queues_.size() >= GROVE_MAX_QUEUES) return mkerr("ERR_SYNC_PODGANG", "SetQueue", "more than GROVE_MAX_QUEUES queues");
  queues_[name] = *queue;
  return std::nullopt;
}

Err GpuBackend::SetStarvationGuard(uint32_t afterCycles, uint32_t maxGangs) {
  std::lock_guard<std::mutex> l(mu_);
  if (afterCycles < 1) return mkerr("ERR_SYNC_PODGANG", "SetStarvationGuard", "afterCycles must be at least 1");
  if (maxGangs > GROVE_MAX_FENCES) return mkerr("ERR_SYNC_PODGANG", "SetStarvationGuard", "maxGangs exceeds GROVE_MAX_FENCES");
  if (maxGangs && consMax_) return mkerr("ERR_SYNC_PODGANG", "SetStarvationGuard", "the starvation guard and consolidation cannot both be on");
  guardAfter_ = afterCycles; guardMax_ = maxGangs;
  return std::nullopt;
}

Err GpuBackend::SetConsolidation(uint32_t afterCycles, uint32_t maxTargets) {
  std::lock_guard<std::mutex> l(mu_);
  if (afterCycles < 1) return mkerr("ERR_SYNC_PODGANG", "SetConsolidation", "afterCycles must be at least 1");
  if (maxTargets > GROVE_MAX_CONSOLIDATE_TARGETS) return mkerr("ERR_SYNC_PODGANG", "SetConsolidation", "maxTargets exceeds GROVE_MAX_CONSOLIDATE_TARGETS");
  if (maxTargets && guardMax_) return mkerr("ERR_SYNC_PODGANG", "SetConsolidation", "the starvation guard and consolidation cannot both be on");
  consAfter_ = afterCycles; consMax_ = maxTargets;
  return std::nullopt;
}

Err GpuBackend::SetTopologySpread(const std::string& pcsName, std::optional<TopologySpread> spread) {
  std::lock_guard<std::mutex> l(mu_);
  if (!spread) { spread_.erase(pcsName); return std::nullopt; }
  if (spread->LevelKey.empty()) return mkerr("ERR_SYNC_PODGANG", "SetTopologySpread", "topology spread of " + pcsName + ": no level key");
  if (spread->MaxSkew < 1 || spread->MaxSkew > 0xFFFF) return mkerr("ERR_SYNC_PODGANG", "SetTopologySpread", "topology spread of " + pcsName + ": maxSkew out of range");
  if (spread->WhenUnsatisfiable != "DoNotSchedule" && spread->WhenUnsatisfiable != "ScheduleAnyway")
    return mkerr("ERR_SYNC_PODGANG", "SetTopologySpread", "topology spread of " + pcsName + ": whenUnsatisfiable must be DoNotSchedule or ScheduleAnyway");
  spread_[pcsName] = *spread;
  return std::nullopt;
}

std::string GpuBackend::WhyNotEncodable(const PodGang& pg) { return WhyNotEncodable(pg, false); }

std::string GpuBackend::WhyNotEncodable(const PodGang& pg, bool large) {
  const size_t maxRep = large ? GROVE_MAX_WIDE_GANG_PODS : 255u, maxPods = large ? GROVE_MAX_WIDE_GANG_PODS : GROVE_MAX_GANG_PODS;
  if (pg.Spec.PodGroups.empty()) return "spec.podgroups: a PodGang needs at least one PodGroup";
  if (pg.Spec.PodGroups.size() > GROVE_MAX_GANG_CLIQUES) return "spec.podgroups: more than " + std::to_string(GROVE_MAX_GANG_CLIQUES) + " PodGroups";
  if (pg.Spec.TopologyConstraintGroupConfigs.size() + 1 > GROVE_MAX_GANG_SCOPES) return "spec.topologyConstraintGroupConfigs: more than " + std::to_string(GROVE_MAX_GANG_SCOPES - 1) + " group configs";
  size_t pods = 0;
  for (const auto& p : pg.Spec.PodGroups) {
    if (p.MinReplicas < 0 || size_t(p.MinReplicas) > maxRep) return "spec.podgroups[" + p.Name + "].minReplicas: must be within 0.." + std::to_string(maxRep);
    if (p.PodReferences.size() > maxRep) return "spec.podgroups[" + p.Name + "].podReferences: more than " + std::to_string(maxRep) + " pods";
    if (size_t(p.MinReplicas) > p.PodReferences.size()) return "spec.podgroups[" + p.Name + "].minReplicas: exceeds the pods referenced";
    pods += p.PodReferences.size();
  }
  if (pods > maxPods) return "spec.podgroups: more than " + std::to_string(maxPods) + " pods in one PodGang";
  for (const auto& gc : pg.Spec.TopologyConstraintGroupConfigs)
    for (const auto& n : gc.PodGroupNames)
      if (std::none_of(pg.Spec.PodGroups.begin(), pg.Spec.PodGroups.end(), [&n](const PodGroup& p) { return p.Name == n; }))
        return "spec.topologyConstraintGroupConfigs[" + gc.Name + "].podGroupNames: unknown PodGroup " + n;
  return "";
}

Err GpuBackend::Encode(const std::vector<Node>& nodes, Tables* out) const {
  std::lock_guard<std::mutex> l(mu_);
  return EncodeLocked(nodes, out);
}

Err GpuBackend::EncodeLocked(const std::vector<Node>& nodes, Tables* out, const std::vector<std::string>* restate) const {
  *out = Tables{};
  if (levels_.empty()) return mkerr("ERR_SYNC_PODGANG", "Encode", "no ClusterTopology levels synced");
  const uint32_t L = uint32_t(levels_.size());
  // nodes: interned label value per level; selector class from one label key; taints per class
  std::vector<std::map<std::string, uint32_t>> intern(L);
  std::map<std::string, uint32_t> classOf;  // label value -> class id (0 = label absent)
  std::vector<std::set<std::string>> classTaints(1);
  std::vector<std::string> classValue(1, "");
  out->nodes.resize(nodes.size());
  for (size_t i = 0; i < nodes.size(); ++i) {
    const Node& n = nodes[i];
    grove_node_t& r = out->nodes[i];
    r.free_cpu_milli = n.alloc_cpu_milli > n.used_cpu_milli ? n.alloc_cpu_milli - n.used_cpu_milli : 0;
    r.free_mem_mib = n.alloc_mem_mib > n.used_mem_mib ? n.alloc_mem_mib - n.used_mem_mib : 0;
    r.free_gpu = uint16_t(n.alloc_gpu > n.used_gpu ? n.alloc_gpu - n.used_gpu : 0);
    r.free_pods = uint16_t(n.alloc_pods > n.used_pods ? n.alloc_pods - n.used_pods : 0);
    uint32_t cls = 0;
    if (auto it = n.Labels.find(classKey_); it != n.Labels.end()) {
      auto [ci, fresh] = classOf.emplace(it->second, uint32_t(classOf.size() + 1));
      if (fresh) { classTaints.emplace_back(); classValue.push_back(it->second); }
      cls = ci->second;
      if (cls > 15) return mkerr("ERR_SYNC_PODGANG", "Encode", "more than 15 values of the selector-class label " + classKey_);
    }
    for (const auto& t : n.TaintKeys) classTaints[cls].insert(t);
    r.flags = (n.Unschedulable ? 0u : GROVE_NODE_SCHEDULABLE) | (cls << GROVE_NODE_CLASS_SHIFT);
    for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) {
      r.dom[l] = GROVE_DOM_ABSENT;
      if (l >= L) continue;
      if (auto it = n.Labels.find(levels_[l].Key); it != n.Labels.end())
        r.dom[l] = intern[l].emplace(it->second, uint32_t(intern[l].size())).first->second;
    }
  }
  // (Required, Preferred) label keys -> level indices; a Preferred level that is not deeper than the Required
  // one adds nothing (best effort, podgang.go:110-117) and is dropped
  auto levelOf = [this](const std::optional<TopologyConstraint>& tc, uint8_t* lvl, uint8_t* pref) -> Err {
    *lvl = GROVE_LEVEL_NONE; *pref = GROVE_LEVEL_NONE;
    if (!tc || !tc->PackConstraint) return std::nullopt;
    // a key that is no (longer a) level of the synced ClusterTopology is dropped, not an error: the operator does the same
    // for a pack domain it cannot find (createTopologyPackConstraint, syncflow.go:349-371, logs and returns nil)
    auto find = [this](const std::string& key, const char*, uint8_t* o) -> Err {
      for (size_t l = 0; l < levels_.size(); ++l) if (levels_[l].Key == key) { *o = uint8_t(l); return std::nullopt; }
      return std::nullopt;
    };
    if (tc->PackConstraint->Required) if (auto e = find(*tc->PackConstraint->Required, "Required", lvl)) return e;
    if (tc->PackConstraint->Preferred) if (auto e = find(*tc->PackConstraint->Preferred, "Preferred", pref)) return e;
    if (*pref != GROVE_LEVEL_NONE && *lvl != GROVE_LEVEL_NONE && *pref <= *lvl) *pref = GROVE_LEVEL_NONE;
    return std::nullopt;
  };
  // Row order: PodGangs that still have to get their minimum (key order), then the REMAINDERS of scheduled PodGangs:
  // pods that found no node when the gang was admitted stay Pending and are retried with MinReplicas 0 (the gang
  // guarantee is met), after everybody's minimum -- what the e2e suites wait for step by step
  // (gang_scheduling_test.go GS5-GS12).  A remainder carries no placement of its own, so it is only resubmitted for
  // PodGangs without pack constraints (with constraints its pods would have to rejoin the domains chosen earlier).
  auto constrained = [](const PodGang& pg) {
    auto has = [](const std::optional<TopologyConstraint>& tc) { return tc && tc->PackConstraint && (tc->PackConstraint->Required || tc->PackConstraint->Preferred); };
    if (has(pg.Spec.Topology)) return true;
    for (const auto& gc : pg.Spec.TopologyConstraintGroupConfigs) if (has(gc.Topology)) return true;
    for (const auto& p : pg.Spec.PodGroups) if (has(p.Topology)) return true;
    return false;
  };
  // The best-effort pods of a PodGang that is not scheduled yet follow the same route: it goes in as its minimum
  // only, and its surplus as a remainder row gated behind it (base_gang) -- minimums of every gang before anybody's
  // surplus, which is what the suites' step descriptions say happens (GS8 :583, GS10 :779, GS12 :1023).
  auto hasSurplus = [](const PodGang& pg) { for (const auto& p : pg.Spec.PodGroups) if (int64_t(p.PodReferences.size()) > p.MinReplicas) return true; return false; };
  // PodGangs the packed tables cannot hold are left out of the pass (and so is a scaled PodGang behind one); everybody else
  // is scheduled as usual
  // (a large PodGang -- SetLargePodGangs -- only when no running-gang cycle may run: those take no wide submission)
  const bool runningCycles = preemption_ || reuse_ || reclaimReuse_ || reclaimQueues_;
  for (const auto& kv : pending_) {
    std::string why = WhyNotEncodable(kv.second, large_);
    if (why.empty() && large_ && runningCycles) {
      const std::string narrow = WhyNotEncodable(kv.second, false);
      if (!narrow.empty()) why = narrow + ": large PodGangs are not scheduled while preemption or reservation reuse is on";
    }
    if (!why.empty()) out->skipped[kv.first] = why;
  }
  // topology spread: the base PodGangs of a set with a spread.  The running-gang cycles and wide submissions take no spread set:
  // while one of them may run, the members stay out of the pass
  auto spreadSetOf = [this](const PodGang& pg) -> const TopologySpread* {
    if (!pg.BasePodGangName.empty()) return nullptr;
    auto it = pg.Labels.find(kPartOfLabel);
    if (it == pg.Labels.end()) return nullptr;
    auto sp = spread_.find(it->second);
    return sp == spread_.end() ? nullptr : &sp->second;
  };
  if (!spread_.empty()) {
    bool wideAny = false;
    if (large_) for (const auto& kv : pending_) wideAny |= !out->skipped.count(kv.first) && !WhyNotEncodable(kv.second, false).empty();
    if (runningCycles || wideAny)
      for (const auto& kv : pending_)
        if (!out->skipped.count(kv.first) && spreadSetOf(kv.second))
          out->skipped[kv.first] = runningCycles ? "topology spread is not applied while preemption or reservation reuse is on"
                                                 : "topology spread is not applied in a pass with PodGangs beyond the ordinary limits";
  }
  // queue limits: the members of a known queue.  The running-gang cycles, consolidation, fences, spread sets and wide submissions
  // take no queue set: while one of them may run, the members stay out of the pass
  auto queueOfPg = [this](const PodGang& pg) -> std::string {
    auto it = pg.Labels.find(kQueueLabel);
    return it != pg.Labels.end() && queues_.count(it->second) ? it->second : std::string();
  };
  if (!queues_.empty()) {
    bool wideAny = false, spreadAny = false;
    for (const auto& kv : pending_) {
      if (out->skipped.count(kv.first)) continue;
      wideAny |= large_ && !WhyNotEncodable(kv.second, false).empty();
      spreadAny |= spreadSetOf(kv.second) != nullptr;
    }
    // grove_run_cycle_preempt_queues / grove_run_cycle_reclaim_queues / grove_run_cycle_reclaim_preempt_queues
    const bool withinQueues = (reclaimQueues_ || ((preemptQueues_ || reclaimThenPreempt_) && preemption_)) && !reuse_ && !reclaimReuse_;
    const char* why = runningCycles && !withinQueues ? "queue limits are not applied while preemption or reservation reuse is on"
                      : consMax_ ? "queue limits are not applied while consolidation is on"
                      : guardMax_ ? "queue limits are not applied while the starvation guard is on"
                      : spreadAny ? "queue limits are not applied in a pass with topology spread members"
                      : wideAny ? "queue limits are not applied in a pass with PodGangs beyond the ordinary limits" : nullptr;
    if (why)
      for (const auto& kv : pending_)
        if (!out->skipped.count(kv.first) && !queueOfPg(kv.second).empty()) out->skipped[kv.first] = why;
  }
  // ComputeDomain exclusivity: one ComputeDomain per PodGang, and only in a pass that can take the set (grove_set_compute_domains
  // is refused with the running-gang entries, the other sets' members and wide submissions): otherwise the enrolled PodGangs stay out
  if (imex_) {
    auto cdOf = [](const PodGang& pg, bool* two) {   // the ComputeDomain of its enrolled PodGroups ("" = none)
      std::string cd; *two = false;
      for (const auto& grp : pg.Spec.PodGroups) {
        auto it = pg.PodGroupRequests.find(grp.Name);
        if (it == pg.PodGroupRequests.end() || it->second.ComputeDomain.empty() || !it->second.gpu) continue;
        if (!cd.empty() && cd != it->second.ComputeDomain) *two = true;
        cd = it->second.ComputeDomain;
      }
      return cd;
    };
    bool wideAny = false, spreadAny = false, queueAny = false;
    for (const auto& kv : pending_) {
      if (out->skipped.count(kv.first)) continue;
      wideAny |= large_ && !WhyNotEncodable(kv.second, false).empty();
      spreadAny |= spreadSetOf(kv.second) != nullptr;
      queueAny |= !queueOfPg(kv.second).empty();
    }
    const char* why = runningCycles ? "ComputeDomain exclusivity is not applied while preemption or reservation reuse is on"
                      : consMax_ ? "ComputeDomain exclusivity is not applied while consolidation is on"
                      : guardMax_ ? "ComputeDomain exclusivity is not applied while the starvation guard is on"
                      : !binpackKey_.empty() ? "ComputeDomain exclusivity is not applied while bin-packing is on"
                      : spreadAny ? "ComputeDomain exclusivity is not applied in a pass with topology spread members"
                      : queueAny ? "ComputeDomain exclusivity is not applied in a pass with queue members"
                      : wideAny ? "ComputeDomain exclusivity is not applied in a pass with PodGangs beyond the ordinary limits" : nullptr;
    for (const auto& kv : pending_) {
      if (out->skipped.count(kv.first)) continue;
      bool two = false;
      const std::string cd = cdOf(kv.second, &two);
      if (two) out->skipped[kv.first] = "the PodGroups of this PodGang name two ComputeDomains (MNNVL groups); one per PodGang is supported";
      else if (!cd.empty() && why) out->skipped[kv.first] = why;
    }
  }
  for (const auto& kv : pending_)
    if (!out->skipped.count(kv.first) && !kv.second.BasePodGangName.empty() && out->skipped.count(kv.second.Namespace + "/" + kv.second.BasePodGangName))
      out->skipped[kv.first] = "base PodGang " + kv.second.BasePodGangName + " cannot be scheduled: " + out->skipped[kv.second.Namespace + "/" + kv.second.BasePodGangName];
  std::vector<const std::string*> order;
  for (const auto& kv : pending_) if (!bound_.count(kv.first) && !out->skipped.count(kv.first)) order.push_back(&kv.first);
  const size_t nFull = order.size();
  for (const auto& kv : pending_) {
    if (out->skipped.count(kv.first)) continue;
    const bool scheduled = bound_.count(kv.first) != 0;
    if (!constrained(kv.second) && (scheduled || hasSurplus(kv.second))) order.push_back(&kv.first);
  }
  std::map<std::string, uint32_t> row;  // PodGang key -> gang row (PodGangs still to be scheduled only: what a base_gang can name)
  for (size_t i = 0; i < nFull; ++i) row.emplace(*order[i], uint32_t(i));
  std::map<std::string, uint32_t> nodeIndex;
  for (size_t i = 0; i < nodes.size(); ++i) nodeIndex[nodes[i].Name] = uint32_t(i);
  std::map<std::string, uint32_t> groupOf;   // "<ns>/<PodCliqueSet>" -> spread group
  auto spreadGroup = [&](const std::string& ns, const std::string& pcs, const TopologySpread& sp) -> uint32_t {
    uint8_t lvl = GROVE_LEVEL_NONE;
    for (size_t l = 0; l < levels_.size(); ++l) if (levels_[l].Key == sp.LevelKey) lvl = uint8_t(l);
    if (lvl == GROVE_LEVEL_NONE) return GROVE_NONE_U32;   // not a level of the synced ClusterTopology: dropped, as a pack domain is
    auto [it, fresh] = groupOf.emplace(ns + "/" + pcs, uint32_t(out->spreadGroups.size()));
    if (fresh) {
      grove_spread_t g{}; g.level = lvl; g.max_skew = uint16_t(sp.MaxSkew);
      g.mode = sp.WhenUnsatisfiable == "ScheduleAnyway" ? GROVE_SPREAD_SOFT : GROVE_SPREAD_HARD;
      out->spreadGroups.push_back(g); out->spreadSet.push_back(it->first);
    }
    return it->second;
  };
  // consolidation: the running PodGangs to restate come last, as gated rows that bind all their pods (MinReplicas = replicas)
  const size_t nRows = order.size();
  if (restate) for (const std::string& key : *restate) order.push_back(&key);
  out->specRow = uint32_t(nRows);
  for (size_t oi = 0; oi < order.size(); ++oi) {
    const std::string& key = *order[oi];
    const bool spec = oi >= nRows;
    const PodGang& pg = spec ? specOf_.at(key) : pending_.at(key);
    const bool remainder = !spec && oi >= nFull;
    const bool split = !spec && !remainder && !constrained(pg) && hasSurplus(pg);  // this row carries the minimum only
    std::vector<uint32_t> minOnly;                                                 // surplus row of an unscheduled PodGang: its minimum is row `row[key]`
    const std::vector<uint32_t>* done = nullptr;                                   // pods covered elsewhere, per PodGroup
    if (remainder) {
      if (auto it = bound_.find(key); it != bound_.end()) done = &it->second;
      else { for (const auto& p : pg.Spec.PodGroups) minOnly.push_back(uint32_t(std::max<int32_t>(0, p.MinReplicas))); done = &minOnly; }
    }
    grove_gang_t g{};
    g.clique_off = uint32_t(out->cliques.size()); g.scope_off = uint32_t(out->scopes.size());
    g.anchor_node = GROVE_NONE_U32; g.base_gang = GROVE_NONE_U32; g.preferred = GROVE_LEVEL_NONE;
    g.flags = pg.Gated || spec ? GROVE_GANG_GATED : 0;
    if (auto e = levelOf(pg.Spec.Topology, &g.level, &g.preferred)) return e;
    if (auto it = priorityClasses_.find(pg.Spec.PriorityClassName); it != priorityClasses_.end()) g.priority = it->second;
    if (!spec && !remainder && !pg.BasePodGangName.empty())   // a base that is already scheduled gates nothing
      if (auto it = row.find(pg.Namespace + "/" + pg.BasePodGangName); it != row.end()) g.base_gang = it->second;
    if (remainder && !minOnly.empty()) g.base_gang = row.at(key);   // surplus of a PodGang whose minimum is in this very pass
    if (remainder) {  // stay close to where the gang landed
      if (auto it = lastNode_.find(key); it != lastNode_.end()) if (auto nt = nodeIndex.find(it->second); nt != nodeIndex.end()) g.anchor_node = nt->second;
    } else if (spec) {  // a restated running PodGang: anchored where it runs
      if (auto it = lastNode_.find(key); it != lastNode_.end()) if (auto nt = nodeIndex.find(it->second); nt != nodeIndex.end()) g.anchor_node = nt->second;
    } else if (auto mv = moveAnchor_.find(key); mv != moveAnchor_.end()) {   // moved by consolidation: where the cycle planned it
      if (auto nt = nodeIndex.find(mv->second); nt != nodeIndex.end()) g.anchor_node = nt->second;
    } else if (pg.Spec.ReuseReservationRef) {  // locality hint: score distance against where that PodGang was placed
      auto it = lastNode_.find(pg.Spec.ReuseReservationRef->Namespace + "/" + pg.Spec.ReuseReservationRef->Name);
      if (it != lastNode_.end()) if (auto nt = nodeIndex.find(it->second); nt != nodeIndex.end()) g.anchor_node = nt->second;
    }
    // scopes: the loose PodGroups first (one implicit scope), then one scope per TopologyConstraintGroupConfig
    std::set<std::string> grouped;
    for (const auto& gc : pg.Spec.TopologyConstraintGroupConfigs) for (const auto& n : gc.PodGroupNames) grouped.insert(n);
    struct ScopeRows { uint8_t first, pref; std::vector<uint32_t> second; };  // (Required level, Preferred level, PodGroup indices)
    std::vector<ScopeRows> scopes;
    std::vector<uint32_t> loose;
    auto left = [&](uint32_t i) { return pg.Spec.PodGroups[i].PodReferences.size() - (done ? (*done)[i] : 0u); };
    for (uint32_t i = 0; i < pg.Spec.PodGroups.size(); ++i) if (!grouped.count(pg.Spec.PodGroups[i].Name) && (!remainder || left(i))) loose.push_back(i);
    if (!loose.empty()) scopes.push_back({uint8_t(GROVE_LEVEL_NONE), uint8_t(GROVE_LEVEL_NONE), loose});
    for (const auto& gc : pg.Spec.TopologyConstraintGroupConfigs) {
      uint8_t lvl, pref; if (auto e = levelOf(gc.Topology, &lvl, &pref)) return e;
      std::vector<uint32_t> members;
      for (const auto& n : gc.PodGroupNames) {
        auto it = std::find_if(pg.Spec.PodGroups.begin(), pg.Spec.PodGroups.end(), [&n](const PodGroup& p) { return p.Name == n; });
        if (it == pg.Spec.PodGroups.end()) return mkerr("ERR_SYNC_PODGANG", "Encode", "group config " + gc.Name + " names unknown PodGroup " + n);
        const uint32_t gi = uint32_t(it - pg.Spec.PodGroups.begin());
        if (!remainder || left(gi)) members.push_back(gi);
      }
      if (!members.empty()) scopes.push_back({lvl, pref, members});
    }
    uint32_t rel = 0, pods = 0;
    for (size_t si = 0; si < scopes.size(); ++si) {
      grove_scope_t s{}; s.first_clique = uint16_t(rel); s.n_cliques = uint16_t(scopes[si].second.size()); s.level = scopes[si].first;
      s.preferred1 = scopes[si].pref == GROVE_LEVEL_NONE ? uint8_t(0) : uint8_t(scopes[si].pref + 1);
      out->scopes.push_back(s);
      for (uint32_t gi : scopes[si].second) {
        const PodGroup& p = pg.Spec.PodGroups[gi];
        grove_clique_t c{};
        PodGang::Requests rq;
        if (auto it = pg.PodGroupRequests.find(p.Name); it != pg.PodGroupRequests.end()) rq = it->second;
        c.req_cpu_milli = rq.cpu_milli; c.req_mem_mib = rq.mem_mib; c.req_gpu = rq.gpu;
        const size_t maxRep = large_ ? GROVE_MAX_WIDE_GANG_PODS : 255u;
        if (p.MinReplicas < 0 || size_t(p.MinReplicas) > maxRep || p.PodReferences.size() > maxRep || size_t(p.MinReplicas) > p.PodReferences.size())
          return mkerr("ERR_SYNC_PODGANG", "Encode", "PodGroup " + p.Name + ": MinReplicas / PodReferences out of range");
        grove_clique_count_t n{uint16_t(p.MinReplicas), uint16_t(p.PodReferences.size())};
        if (remainder) { n.min_replicas = 0; n.replicas = uint16_t(left(gi)); }
        if (split) n.replicas = n.min_replicas;
        if (spec) n.min_replicas = n.replicas;
        // the 8-bit fields are what grove_submit_gangs reads; grove_submit_gangs_wide reads the counts row
        c.min_replicas = uint8_t(std::min<uint32_t>(n.min_replicas, 255u)); c.replicas = uint8_t(std::min<uint32_t>(n.replicas, 255u));
        uint8_t cpref;
        if (auto e = levelOf(p.Topology, &c.level, &cpref)) return e;
        c.scope = GROVE_CLIQUE_SCOPE_PREF(uint32_t(si), cpref);
        // class mask: classes whose label value satisfies the nodeSelector and whose taints are all tolerated
        uint16_t mask = 0;
        auto sel = rq.nodeSelector.find(classKey_);
        for (uint32_t cl = 0; cl < classValue.size(); ++cl) {
          if (sel != rq.nodeSelector.end() && (cl == 0 || classValue[cl] != sel->second)) continue;
          bool tolerated = true;
          for (const auto& t : classTaints[cl]) tolerated &= std::find(rq.tolerationKeys.begin(), rq.tolerationKeys.end(), t) != rq.tolerationKeys.end();
          if (tolerated) mask |= uint16_t(1u << cl);
        }
        c.class_mask = mask;
        out->cliques.push_back(c);
        out->counts.push_back(n);
        out->cliqueOf.push_back({uint32_t(out->gangs.size()), gi});
        out->refBase.push_back(done ? (*done)[gi] : 0u);
        pods += n.replicas; ++rel;
      }
    }
    if (rel == 0 || rel > GROVE_MAX_GANG_CLIQUES || scopes.size() > GROVE_MAX_GANG_SCOPES || pods > (large_ ? GROVE_MAX_WIDE_GANG_PODS : GROVE_MAX_GANG_PODS))
      return mkerr("ERR_SYNC_PODGANG", "Encode", "PodGang " + key + " exceeds the gpu-scheduler limits");
    g.n_cliques = uint16_t(rel); g.n_scopes = uint16_t(scopes.size());
    uint32_t grp = GROVE_NONE_U32;
    if (const TopologySpread* sp = remainder || spec ? nullptr : spreadSetOf(pg)) {
      bool need = false;
      for (size_t k = out->counts.size() - rel; k < out->counts.size(); ++k) need |= out->counts[k].min_replicas > 0;
      const uint32_t s = spreadGroup(pg.Namespace, pg.Labels.at(kPartOfLabel), *sp);
      if (s != GROVE_NONE_U32 && need && g.level != GROVE_LEVEL_NONE && g.level >= out->spreadGroups[s].level) grp = s;
    }
    out->spreadOf.push_back(grp);
    const std::string qn = spec ? std::string() : queueOfPg(pg);   // (a gated spec row is never evaluated)
    out->queueOf.push_back(qn.empty() ? GROVE_NONE_U32 : uint32_t(std::distance(queues_.begin(), queues_.find(qn))));
    out->gangs.push_back(g);
    out->gangNames.push_back(key);
    out->remainder.push_back(remainder ? 1 : 0);
  }
  // the running replicas of the sets being spread: where the base PodGangs this backend scheduled landed
  if (std::any_of(out->spreadOf.begin(), out->spreadOf.end(), [](uint32_t x) { return x != GROVE_NONE_U32; }))
    for (const auto& [key, set] : setOf_) {
      auto gi = groupOf.find(set);
      auto ln = lastNode_.find(key);
      if (gi == groupOf.end() || ln == lastNode_.end() || row.count(key)) continue;
      if (auto nt = nodeIndex.find(ln->second); nt != nodeIndex.end()) out->spreadSeeds.push_back(grove_spread_seed_t{gi->second, nt->second});
    }
  else { out->spreadGroups.clear(); out->spreadSet.clear(); }
  // the queue table, parents first (ordered by depth, then name), with what the running PodGangs of each queue hold
  if (std::any_of(out->queueOf.begin(), out->queueOf.end(), [](uint32_t x) { return x != GROVE_NONE_U32; })) {
    auto depth = [this](const std::string& n) { uint32_t d = 0; for (std::string p = queues_.at(n).Parent; !p.empty(); p = queues_.at(p).Parent) ++d; return d; };
    std::vector<std::string> names;
    for (const auto& kv : queues_) names.push_back(kv.first);
    std::stable_sort(names.begin(), names.end(), [&](const std::string& a, const std::string& b) { return depth(a) < depth(b); });
    std::map<std::string, uint32_t> idx;
    for (uint32_t i = 0; i < names.size(); ++i) idx[names[i]] = i;
    for (const std::string& n : names) {
      const Queue& q = queues_.at(n);
      grove_queue_t r{};
      r.parent = q.Parent.empty() ? GROVE_NONE_U32 : idx.at(q.Parent);
      r.limit[0] = q.CpuMilli.value_or(GROVE_QUEUE_UNLIMITED); r.limit[1] = q.MemMiB.value_or(GROVE_QUEUE_UNLIMITED); r.limit[2] = q.Gpu.value_or(GROVE_QUEUE_UNLIMITED);
      out->queues.push_back(r);
      out->quotas.push_back(grove_queue_quota_t{{q.DeservedCpuMilli.value_or(GROVE_QUEUE_UNLIMITED), q.DeservedMemMiB.value_or(GROVE_QUEUE_UNLIMITED),
                                                 q.DeservedGpu.value_or(GROVE_QUEUE_UNLIMITED)}});
    }
    for (const auto& [key, qn] : queueOf_) {
      auto it = idx.find(qn); auto rg = running_.find(key);
      if (it == idx.end() || rg == running_.end()) continue;
      for (const Held& h : rg->second.held) { out->queues[it->second].used[0] += h.cpu_milli; out->queues[it->second].used[1] += h.mem_mib; out->queues[it->second].used[2] += h.gpu; }
    }
    std::vector<uint32_t> byName(queues_.size());   // queueOf holds positions in queues_ (by name): renumber
    { uint32_t k = 0; for (const auto& kv : queues_) byName[k++] = idx.at(kv.first); }
    for (uint32_t& x : out->queueOf) if (x != GROVE_NONE_U32) x = byName[x];
    out->queueNames = names;
  } else out->queueOf.assign(out->queueOf.size(), GROVE_NONE_U32);
  return std::nullopt;
}

Err GpuBackend::RunCycle(const std::vector<Node>& nodes, std::vector<Binding>* bindings, std::map<std::string, PodGangStatus>* statuses,
                         grove_cycle_stats_t* stats) {
  std::lock_guard<std::mutex> cycle(cycleMu_);   // the engine handle is not thread-safe: one cycle at a time
  bindings->clear(); statuses->clear();
  if (stats) *stats = grove_cycle_stats_t{};
  Tables t;
  std::map<std::string, PodGang> snap;            // the PodGangs of this pass: reconcilers may add / delete others meanwhile
  bool large = false, explain = false;
  uint32_t guardAfter = 1, guardMax = 0;
  std::map<std::string, uint32_t> rejectedFor;
  std::vector<TopologyLevel> levels;
  std::vector<std::string> restate;               // consolidation: the running PodGangs restated as gated spec rows
  std::vector<grove_running_gang_t> crun; std::vector<grove_holding_t> cheld;
  std::vector<uint32_t> targets, specOf;          // consolidation: target rows; spec row of each running gang of crun
  {
    std::lock_guard<std::mutex> l(mu_);
    large = large_; explain = explain_; levels = levels_;
    guardAfter = guardAfter_; guardMax = guardMax_; rejectedFor = rejectedFor_;
    if (pending_.empty()) return std::nullopt;
    if (auto e = Init()) return e;
    if (!engine_) return mkerr("ERR_SYNC_PODGANG", "RunCycle", "no ClusterTopology synced");
    // consolidation runs in an ordinary pass only: every running PodGang scheduled whole is movable
    const bool consOn = consMax_ && !preemption_ && !reuse_ && !reclaimReuse_;
    if (consOn)
      for (const auto& kv : running_)
        if (!pending_.count(kv.first) && specOf_.count(kv.first) && WhyNotEncodable(specOf_.at(kv.first), false).empty()) restate.push_back(kv.first);
    if (auto e = EncodeLocked(nodes, &t, consOn ? &restate : nullptr)) return e;
    snap = pending_;
    if (t.specRow < t.gangs.size()) {   // the targets: as the starvation guard counts; none, or a pass that takes no consolidation: no spec rows
      bool wide = false;
      for (const grove_gang_t& g : t.gangs) {
        uint32_t pods = 0;
        for (uint32_t c = g.clique_off; c < g.clique_off + g.n_cliques; ++c) { const uint32_t rep = t.counts[c].replicas; pods += rep; wide |= rep > 255u; }
        wide |= pods > GROVE_MAX_GANG_PODS;
      }
      if (!wide && t.spreadGroups.empty()) {
        for (uint32_t g = 0; g < t.specRow; ++g) {
          auto it = rejectedFor_.find(t.gangNames[g]);
          if (!t.remainder[g] && it != rejectedFor_.end() && it->second >= consAfter_) targets.push_back(g);
        }
        std::stable_sort(targets.begin(), targets.end(), [&](uint32_t a, uint32_t b) { return t.gangs[a].priority > t.gangs[b].priority; });
        if (targets.size() > consMax_) targets.resize(consMax_);
      }
      if (targets.empty()) {   // drop the spec rows (they come last)
        const uint32_t r = t.specRow, q = t.gangs[r].clique_off, sc = t.gangs[r].scope_off;
        t.gangs.resize(r); t.gangNames.resize(r); t.remainder.resize(r); t.spreadOf.resize(r); t.queueOf.resize(r);
        t.cliques.resize(q); t.counts.resize(q); t.cliqueOf.resize(q); t.refBase.resize(q); t.scopes.resize(sc);
      } else {   // the movable running PodGangs with what they hold (holdings on nodes that left the snapshot are dropped)
        std::map<std::string, uint32_t> nodeIdx;
        for (uint32_t i = 0; i < nodes.size(); ++i) nodeIdx[nodes[i].Name] = i;
        for (uint32_t k = 0; k < restate.size(); ++k) {
          const RunningGang& rg = running_.at(restate[k]);
          grove_running_gang_t r{rg.priority, uint32_t(cheld.size()), 0u, 0u};
          for (const auto& h : rg.held) {
            auto it = nodeIdx.find(h.node);
            if (it == nodeIdx.end()) continue;
            cheld.push_back(grove_holding_t{it->second, h.cpu_milli, h.mem_mib, h.gpu, h.pods}); ++r.n_holdings;
          }
          crun.push_back(r); specOf.push_back(t.specRow + k);
        }
      }
    }
  }
  const bool consolidate = !targets.empty();
  for (const auto& kv : t.skipped) { PodGangStatus s; s.ScheduledReason = "Unschedulable"; s.ScheduledMessage = kv.second; (*statuses)[kv.first] = s; }
  if (t.gangs.empty()) return std::nullopt;
  auto chk = [this](int32_t rc, const char* what) -> Err {
    if (rc == GROVE_OK) return std::nullopt;
    return mkerr("ERR_SYNC_PODGANG", what, std::string(grove_last_error(engine_)) + " (" + std::to_string(rc) + ")");
  };
  if (auto e = chk(grove_load_nodes(engine_, t.nodes.data(), uint32_t(t.nodes.size())), "grove_load_nodes")) return e;
  if (large) {
    if (auto e = chk(grove_submit_gangs_wide(engine_, t.gangs.data(), uint32_t(t.gangs.size()), t.cliques.data(), t.counts.data(),
                                             uint32_t(t.cliques.size()), t.scopes.data(), uint32_t(t.scopes.size())), "grove_submit_gangs_wide")) return e;
  } else if (auto e = chk(grove_submit_gangs(engine_, t.gangs.data(), uint32_t(t.gangs.size()), t.cliques.data(), uint32_t(t.cliques.size()),
                                             t.scopes.data(), uint32_t(t.scopes.size())), "grove_submit_gangs")) return e;
  const bool spread = !t.spreadGroups.empty();   // (Encode keeps groups only when a row is a member)
  if (spread)
    if (auto e = chk(grove_set_spread(engine_, t.spreadGroups.data(), uint32_t(t.spreadGroups.size()), t.spreadOf.data(), uint32_t(t.spreadOf.size()),
                                      t.spreadSeeds.data(), uint32_t(t.spreadSeeds.size())), "grove_set_spread")) return e;
  if (!t.queues.empty())   // (Encode keeps the queue table only when a row is a member, and only in a pass that takes one)
    if (auto e = chk(grove_set_queues(engine_, t.queues.data(), uint32_t(t.queues.size()), t.queueOf.data(), uint32_t(t.queueOf.size())), "grove_set_queues")) return e;
  grove_cycle_stats_t st{};
  // running PodGangs -> the reclaim pass's / reservation reuse's tables (holdings on nodes that left the snapshot are dropped)
  std::vector<grove_running_gang_t> run; std::vector<grove_holding_t> held; std::vector<std::string> runNames;
  bool preempt = false, reuse = false, both = false;   // both: SetReclaimWithReuse, one grove_run_cycle_reuse_preempt
  bool acrossQueues = false;                           // SetReclaimAcrossQueues with queue members: grove_run_cycle_reclaim_queues
  bool thenPreempt = false;                            // SetReclaimThenPreempt with queue members: grove_run_cycle_reclaim_preempt_queues
  bool fairShare = false;                              // SetFairShareOrder with queue members: the queue cycle in fair-share order
  std::vector<uint32_t> replaces;   // reservation reuse: per gang row, the running gang it is the new version of
  {
    std::lock_guard<std::mutex> l(mu_);
    if (preemption_ && reuse_ && !reclaimReuse_) return mkerr("ERR_SYNC_PODGANG", "RunCycle", "preemption and reservation reuse cannot both be on");
    const bool reclaimThenPreempt = reclaimThenPreempt_ && preemption_;   // (whatever the two switches below say)
    if (reclaimQueues_ && preemptQueues_ && !reclaimThenPreempt)
      return mkerr("ERR_SYNC_PODGANG", "RunCycle", "reclaim across queues and preemption within queues cannot both be on");
    both = reclaimReuse_ && !running_.empty();
    // (Encode keeps queue members in the pass only when reuse and reuse with reclaim are off)
    thenPreempt = reclaimThenPreempt && !t.queues.empty() && !running_.empty();
    acrossQueues = !thenPreempt && reclaimQueues_ && !t.queues.empty() && !running_.empty();
    preempt = ((preemption_ || reclaimReuse_) && !running_.empty()) || acrossQueues;
    reuse = (reuse_ || reclaimReuse_) && !running_.empty();
    fairShare = fairShare_ && !t.queues.empty() && !both && !preempt && !reuse && !consolidate;
    if (preempt || reuse) {
      std::map<std::string, uint32_t> nodeIdx;
      for (uint32_t i = 0; i < nodes.size(); ++i) nodeIdx[nodes[i].Name] = i;
      for (const auto& kv : running_) {
        if (snap.count(kv.first)) continue;   // still pending with a remainder: not evictable while it is being placed
        grove_running_gang_t r{kv.second.priority, uint32_t(held.size()), 0u, 0u};
        for (const auto& h : kv.second.held) {
          auto it = nodeIdx.find(h.node);
          if (it == nodeIdx.end()) continue;
          held.push_back(grove_holding_t{it->second, h.cpu_milli, h.mem_mib, h.gpu, h.pods}); ++r.n_holdings;
        }
        run.push_back(r); runNames.push_back(kv.first);
      }
    }
    if (reuse) {   // the minimum row of a PodGang whose ReuseReservationRef names a running PodGang; one new version per running gang
      std::map<std::string, uint32_t> runIdx;
      for (uint32_t r = 0; r < runNames.size(); ++r) runIdx[runNames[r]] = r;
      std::vector<uint8_t> taken(run.size(), 0);
      replaces.assign(t.gangs.size(), GROVE_NONE_U32);
      for (uint32_t g = 0; g < t.gangs.size(); ++g) {
        const PodGang& pg = snap.at(t.gangNames[g]);
        if (t.remainder[g] || !pg.Spec.ReuseReservationRef) continue;
        auto it = runIdx.find(pg.Spec.ReuseReservationRef->Namespace + "/" + pg.Spec.ReuseReservationRef->Name);
        if (it == runIdx.end() || taken[it->second]) continue;
        taken[it->second] = 1; replaces[g] = it->second;
      }
      reuse = std::any_of(replaces.begin(), replaces.end(), [](uint32_t r) { return r != GROVE_NONE_U32; });
    }
  }
  bool wide = false;   // a row beyond the ordinary limits makes the submission wide, which takes no fence or bin-packing set
  for (const grove_gang_t& g : t.gangs) {
    uint32_t pods = 0;
    for (uint32_t c = g.clique_off; c < g.clique_off + g.n_cliques; ++c) {
      const uint32_t rep = large ? t.counts[c].replicas : t.cliques[c].replicas;
      pods += rep; wide |= rep > 255u;
    }
    wide |= pods > GROVE_MAX_GANG_PODS;
  }
  // the starvation guard: the highest-ranked rows (priority desc, row asc = the engine's rank) of the PodGangs rejected often
  // enough, in an ordinary pass only
  std::vector<uint32_t> fences;
  if (guardMax && !both && !reuse && !preempt && !spread) {
    std::vector<uint32_t> rows;
    for (uint32_t g = 0; g < t.gangs.size() && !wide; ++g) {
      auto it = rejectedFor.find(t.gangNames[g]);
      if (!t.remainder[g] && t.gangs[g].level != GROVE_LEVEL_NONE && it != rejectedFor.end() && it->second >= guardAfter) rows.push_back(g);
    }
    std::stable_sort(rows.begin(), rows.end(), [&](uint32_t a, uint32_t b) { return t.gangs[a].priority > t.gangs[b].priority; });
    if (rows.size() > guardMax) rows.resize(guardMax);
    fences = rows;
    if (!fences.empty())
      if (auto e = chk(grove_set_fences(engine_, fences.data(), uint32_t(fences.size())), "grove_set_fences")) return e;
  }
  // bin-packing: every row a member, at the level of the key or its own Required level when deeper, in an ordinary or queue pass
  if (!both && !reuse && !preempt && !consolidate && !spread && fences.empty() && !wide && !fairShare) {
    uint8_t lv = GROVE_LEVEL_NONE;
    {
      std::lock_guard<std::mutex> l(mu_);
      for (size_t i = 0; i < levels_.size() && !binpackKey_.empty(); ++i) if (levels_[i].Key == binpackKey_) lv = uint8_t(i);
    }
    if (lv != GROVE_LEVEL_NONE) {
      std::vector<uint8_t> packAt(t.gangs.size());
      for (size_t g = 0; g < t.gangs.size(); ++g) packAt[g] = t.gangs[g].level == GROVE_LEVEL_NONE ? lv : std::max(lv, t.gangs[g].level);
      if (auto e = chk(grove_set_binpack(engine_, packAt.data(), uint32_t(packAt.size())), "grove_set_binpack")) return e;
    }
  }
  // ComputeDomain exclusivity (Encode left enrolled rows only in a pass that takes the set): the ComputeDomain of every enrolled
  // clique row, and every node's holder -- the one observed, else the one of the enrolled pods this backend bound there for a
  // PodGang that still runs
  std::vector<std::string> cdName;   // clique row -> its ComputeDomain ("" = not enrolled)
  bool imexOn = false;
  { std::lock_guard<std::mutex> l(mu_); imexOn = imex_; }
  if (imexOn && !both && !reuse && !preempt && !consolidate) {
    cdName.assign(t.cliques.size(), std::string());
    bool any = false;
    for (uint32_t q = 0; q < t.cliques.size(); ++q) {
      const auto [grow, pgi] = t.cliqueOf[q];
      if (grow >= t.specRow || !t.cliques[q].req_gpu) continue;
      const PodGang& pg = snap.at(t.gangNames[grow]);
      auto it = pg.PodGroupRequests.find(pg.Spec.PodGroups[pgi].Name);
      if (it != pg.PodGroupRequests.end() && !it->second.ComputeDomain.empty()) { cdName[q] = it->second.ComputeDomain; any = true; }
    }
    if (any) {
      std::map<std::string, uint32_t> ids;
      auto id = [&ids](const std::string& name) { return ids.emplace(name, uint32_t(ids.size())).first->second; };
      std::vector<uint32_t> cd(t.cliques.size(), GROVE_CD_NONE), owner0(nodes.size(), GROVE_CD_NONE);
      for (uint32_t q = 0; q < t.cliques.size(); ++q) if (!cdName[q].empty()) cd[q] = id(cdName[q]);
      std::map<std::string, std::string> boundBy;   // node -> ComputeDomain of the enrolled pods this backend bound there
      {
        std::lock_guard<std::mutex> l(mu_);
        for (const auto& kv : running_) for (const auto& [node, c] : kv.second.cdOn) boundBy.emplace(node, c);
      }
      for (uint32_t n = 0; n < nodes.size(); ++n) {
        if (!nodes[n].ImexCapable) owner0[n] = GROVE_CD_NO_IMEX;
        else if (!nodes[n].ComputeDomain.empty()) owner0[n] = id(nodes[n].ComputeDomain);
        else if (auto it = boundBy.find(nodes[n].Name); it != boundBy.end()) owner0[n] = id(it->second);
      }
      if (auto e = chk(grove_set_compute_domains(engine_, cd.data(), uint32_t(cd.size()), owner0.data(), uint32_t(owner0.size())),
                       "grove_set_compute_domains")) return e;
    } else {
      cdName.clear();
    }
  }
  if (both) { if (auto e = chk(grove_run_cycle_reuse_preempt(engine_, replaces.data(), uint32_t(replaces.size()), run.data(), uint32_t(run.size()), held.data(), uint32_t(held.size()), &st), "grove_run_cycle_reuse_preempt")) return e; }
  else if (reuse) { if (auto e = chk(grove_run_cycle_reuse(engine_, replaces.data(), uint32_t(replaces.size()), run.data(), uint32_t(run.size()), held.data(), uint32_t(held.size()), &st), "grove_run_cycle_reuse")) return e; }
  else if (preempt && !t.queues.empty()) {   // (Encode keeps queue members in a pass with preemption only with SetPreemptionWithinQueues,
                                             // SetReclaimAcrossQueues or SetReclaimThenPreempt)
    std::vector<uint32_t> runQueue(run.size(), GROVE_NONE_U32);   // the queue each running PodGang was scheduled in
    {
      std::lock_guard<std::mutex> l(mu_);
      for (uint32_t r = 0; r < runNames.size(); ++r)
        if (auto it = queueOf_.find(runNames[r]); it != queueOf_.end())
          if (auto n = std::find(t.queueNames.begin(), t.queueNames.end(), it->second); n != t.queueNames.end()) runQueue[r] = uint32_t(n - t.queueNames.begin());
    }
    if (thenPreempt) {
      if (auto e = chk(grove_run_cycle_reclaim_preempt_queues(engine_, t.quotas.data(), uint32_t(t.quotas.size()), run.data(), uint32_t(run.size()),
                                                              held.data(), uint32_t(held.size()), runQueue.data(), &st), "grove_run_cycle_reclaim_preempt_queues")) return e;
    } else if (acrossQueues) {
      if (auto e = chk(grove_run_cycle_reclaim_queues(engine_, t.quotas.data(), uint32_t(t.quotas.size()), run.data(), uint32_t(run.size()), held.data(),
                                                      uint32_t(held.size()), runQueue.data(), &st), "grove_run_cycle_reclaim_queues")) return e;
    } else if (auto e = chk(grove_run_cycle_preempt_queues(engine_, run.data(), uint32_t(run.size()), held.data(), uint32_t(held.size()), runQueue.data(), &st),
                            "grove_run_cycle_preempt_queues")) return e;
  }
  else if (preempt) { if (auto e = chk(grove_run_cycle_preempt(engine_, run.data(), uint32_t(run.size()), held.data(), uint32_t(held.size()), &st), "grove_run_cycle_preempt")) return e; }
  else if (consolidate) {
    if (auto e = chk(grove_run_cycle_consolidate(engine_, targets.data(), uint32_t(targets.size()), specOf.data(), crun.data(), uint32_t(crun.size()),
                                                 cheld.data(), uint32_t(cheld.size()), &st), "grove_run_cycle_consolidate")) return e;
  }
  else {
    if (fairShare)
      if (auto e = chk(grove_set_fair_share(engine_, t.quotas.data(), uint32_t(t.quotas.size())), "grove_set_fair_share")) return e;
    if (auto e = chk(grove_run_cycle(engine_, &st), "grove_run_cycle")) return e;
  }
  if (stats) *stats = st;
  std::vector<grove_placement_t> pl(st.pods_bound + 1);
  uint32_t n = 0;
  if (auto e = chk(grove_get_placements(engine_, pl.data(), uint32_t(pl.size()), &n), "grove_get_placements")) return e;
  std::vector<grove_gang_status_t> gs(t.gangs.size());
  if (auto e = chk(grove_get_gang_status(engine_, gs.data(), uint32_t(gs.size())), "grove_get_gang_status")) return e;
  std::vector<uint32_t> seen(t.cliques.size(), 0);  // the r-th entry of a clique binds its r-th PodReference
  for (uint32_t i = 0; i < n; ++i) {
    const auto [grow, pgi] = t.cliqueOf[pl[i].clique];
    if (grow >= t.specRow) continue;   // a moved PodGang: the caller deletes its pods, it is scheduled anew when synced again
    const PodGang& pg = snap.at(t.gangNames[grow]);
    const PodGroup& grp = pg.Spec.PodGroups[pgi];
    const NamespacedName& pod = grp.PodReferences[t.refBase[pl[i].clique] + seen[pl[i].clique]++];
    bindings->push_back({pod.Namespace, pod.Name, nodes[pl[i].node].Name});
  }
  for (size_t g = 0; g < t.specRow; ++g) {
    PodGangStatus s;
    switch (gs[g].state) {
      case GROVE_GANG_ADMITTED:
        s.Phase = PodGangPhase::Starting; s.Scheduled = true;
        if (!t.remainder[g]) s.PlacementScore = double(gs[g].score_num) / double(gs[g].score_den);  // a remainder re-reports no score
        break;
      case GROVE_GANG_REJECTED: s.ScheduledReason = "Unschedulable"; break;
      case GROVE_GANG_BASE_REJECTED: s.ScheduledReason = "BaseNotScheduled"; break;
      case GROVE_GANG_GATED_SKIP: s.ScheduledReason = "Gated"; break;
      default: s.ScheduledReason = "Pending"; break;
    }
    if (t.remainder[g] && statuses->count(t.gangNames[g])) continue;   // the minimum row of the same PodGang already spoke
    (*statuses)[t.gangNames[g]] = s;
  }
  // topology spread: a DoNotSchedule member that found no room in the domains it was allowed, a ScheduleAnyway member placed
  // outside them (set after the diagnosis below, which refuses a spread cycle)
  std::map<std::string, std::string> spreadMsg;
  if (spread)
    for (uint32_t g = 0; g < gs.size(); ++g) {
      const uint32_t s = t.spreadOf[g];
      if (s == GROVE_NONE_U32) continue;
      const std::string key = levels[t.spreadGroups[s].level].Key, skew = std::to_string(t.spreadGroups[s].max_skew);
      if (gs[g].state == GROVE_GANG_REJECTED && t.spreadGroups[s].mode == GROVE_SPREAD_HARD)
        spreadMsg[t.gangNames[g]] = "topology spread of " + t.spreadSet[s] + " over " + key + " (maxSkew " + skew +
                                    ", DoNotSchedule): no " + key + " domain within the skew had room for this replica";
      if (gs[g].state == GROVE_GANG_ADMITTED && (gs[g].reserved0 & GROVE_STATUS_SPREAD_SKEWED))
        spreadMsg[t.gangNames[g]] = "topology spread of " + t.spreadSet[s] + " over " + key + " (maxSkew " + skew +
                                    ", ScheduleAnyway): no " + key + " domain within the skew had room; placed beyond it";
    }
  // why the rejected PodGangs did not fit (an ordinary cycle only: the running-gang cycles judge gangs against other views).  A
  // failed diagnosis leaves the messages empty: it never costs the cycle its bindings.
  if (explain && !both && !reuse && !preempt && !consolidate &&
      std::any_of(gs.begin(), gs.end(), [](const grove_gang_status_t& x) { return x.state == GROVE_GANG_REJECTED; })) {
    std::vector<grove_gang_diag_t> gd(gs.size());
    std::vector<grove_clique_diag_t> qd(t.cliques.size());
    if (grove_diagnose(engine_, gd.data(), uint32_t(gd.size()), qd.data(), uint32_t(qd.size())) == GROVE_OK)
      for (uint32_t g = 0; g < gs.size(); ++g)
        if (gs[g].state == GROVE_GANG_REJECTED && !t.remainder[g])
          (*statuses)[t.gangNames[g]].ScheduledMessage = ExplainRejection(t, snap.at(t.gangNames[g]), g, gd[g], qd.data(), levels);
  }
  for (const auto& [key, msg] : spreadMsg) (*statuses)[key].ScheduledMessage = msg;
  for (const auto& [key, msg] : QueueMessages(t, gs, pl)) (*statuses)[key].ScheduledMessage = msg;
  // consolidation: a moved PodGang is disrupted (the caller deletes its pods); a consolidated one names the PodGangs it moved
  std::vector<grove_move_t> moves;
  if (consolidate) {
    uint32_t nm = 0;
    if (auto e = chk(grove_get_moves(engine_, nullptr, 0, &nm), "grove_get_moves")) return e;
    moves.resize(nm + 1);
    if (auto e = chk(grove_get_moves(engine_, moves.data(), uint32_t(moves.size()), &nm), "grove_get_moves")) return e;
    moves.resize(nm);
    std::map<uint32_t, std::string> names;
    for (const grove_move_t& m : moves) {
      const std::string& key = restate[m.running];
      PodGangStatus s; s.Phase = PodGangPhase::Running; s.Scheduled = true;
      s.DisruptionTarget = true; s.DisruptionMessage = "moved to make room for PodGang " + t.gangNames[m.target];
      (*statuses)[key] = s;
      names[m.target] += (names[m.target].empty() ? "" : ", ") + key;
    }
    for (const auto& [g, who] : names) (*statuses)[t.gangNames[g]].ScheduledMessage = "scheduled by moving PodGangs " + who;
  }
  // the starvation guard's fences that held: the domain the PodGang keeps the PodGangs ranked after it out of
  for (uint32_t g : fences) {
    if (!(gs[g].reserved0 & GROVE_STATUS_FENCING) || gs[g].level >= levels.size()) continue;
    const TopologyLevel& lv = levels[gs[g].level];
    auto lab = nodes[gs[g].domain_node].Labels.find(lv.Key);
    (*statuses)[t.gangNames[g]].ScheduledMessage =
        "Unschedulable for " + std::to_string(rejectedFor.at(t.gangNames[g]) + 1) + " cycles in a row: " + lv.Domain + " " +
        (lab == nodes[gs[g].domain_node].Labels.end() ? std::string("?") : lab->second) +
        " is held for this PodGang; PodGangs ranked after it are kept out of it until it is scheduled";
  }
  // a scheduled PodGang leaves the pending set once every PodReference is bound; until then its unbound pods are retried
  // as a remainder (Encode).  Remember where gangs landed for ReuseReservationRef hints.
  auto constrained = [](const PodGang& pg) {
    auto has = [](const std::optional<TopologyConstraint>& tc) { return tc && tc->PackConstraint && (tc->PackConstraint->Required || tc->PackConstraint->Preferred); };
    if (has(pg.Spec.Topology)) return true;
    for (const auto& gc : pg.Spec.TopologyConstraintGroupConfigs) if (has(gc.Topology)) return true;
    for (const auto& p : pg.Spec.PodGroups) if (has(p.Topology)) return true;
    return false;
  };
  std::lock_guard<std::mutex> l(mu_);
  // the starvation guard's counts: consecutive Unschedulable cycles; a gated or base-not-scheduled cycle changes nothing
  for (uint32_t g = 0; g < t.specRow; ++g) {
    if (t.remainder[g] || !pending_.count(t.gangNames[g])) continue;
    if (gs[g].state == GROVE_GANG_REJECTED) ++rejectedFor_[t.gangNames[g]];
    else if (gs[g].state == GROVE_GANG_ADMITTED) rejectedFor_.erase(t.gangNames[g]);
  }
  if (preempt) {   // victims: DisruptionTarget on the PodGang (podgang.go:166-170), forgotten as running
    uint32_t nv = 0;
    if (auto e = chk(grove_get_victims(engine_, nullptr, 0, &nv), "grove_get_victims")) return e;
    std::vector<grove_victim_t> vs(nv + 1);
    if (auto e = chk(grove_get_victims(engine_, vs.data(), uint32_t(vs.size()), &nv), "grove_get_victims")) return e;
    for (uint32_t i = 0; i < nv; ++i) {
      PodGangStatus s; s.Phase = PodGangPhase::Running; s.Scheduled = true;
      s.DisruptionTarget = true;
      const uint32_t g = vs[i].preemptor;
      // (after both passes, the evictor's flag says which pass chose the victim)
      const bool reclaimed = acrossQueues || (thenPreempt && (gs[g].reserved0 & GROVE_STATUS_RECLAIMER));
      s.DisruptionMessage = reclaimed ? "reclaimed by PodGang " + t.gangNames[g] + " of queue " + t.queueNames[t.queueOf[g]]
                                         : "preempted by higher priority PodGang " + t.gangNames[g];
      (*statuses)[runNames[vs[i].running]] = s;
      running_.erase(runNames[vs[i].running]);
    }
  }
  // an admitted new version replaces its predecessor: the caller deletes the old pods, whose resources the cycle released.  (With
  // reclaim a predecessor that an earlier preemptor evicted is that one's victim and was forgotten above; it keeps its
  // DisruptionTarget.  A released one is not disrupted.)
  if (reuse && !replaces.empty())
    for (uint32_t i = 0; i < gs.size(); ++i)
      if (gs[i].state == GROVE_GANG_ADMITTED && replaces[i] != GROVE_NONE_U32) running_.erase(runNames[replaces[i]]);
  for (const grove_move_t& m : moves) {   // forgotten as running; anchored where this cycle planned it when synced again
    const std::string& key = restate[m.running];
    const grove_gang_status_t& ms = gs[t.specRow + m.running];
    running_.erase(key); specOf_.erase(key); lastNode_.erase(key);
    if (ms.n_pods) moveAnchor_[key] = nodes[pl[ms.placement_off].node].Name;
  }
  for (uint32_t i = 0; i < t.specRow; ++i) {
    if (gs[i].state != GROVE_GANG_ADMITTED) continue;
    const std::string& key = t.gangNames[i];
    auto pit = pending_.find(key);
    if (pit == pending_.end()) continue;   // deleted while the cycle ran
    const PodGang& pg = pit->second;
    specOf_[key] = pg; moveAnchor_.erase(key);
    {   // what the PodGang holds from now on (a remainder adds to what its minimum took)
      RunningGang& rg = running_[key];
      rg.priority = t.gangs[i].priority;
      for (uint32_t k = 0; k < gs[i].n_pods; ++k) {
        const grove_placement_t& e = pl[gs[i].placement_off + k];
        const grove_clique_t& q = t.cliques[e.clique];
        const std::string& nn = nodes[e.node].Name;
        auto it = std::find_if(rg.held.begin(), rg.held.end(), [&](const Held& h) { return h.node == nn; });
        if (it == rg.held.end()) { rg.held.push_back(Held{nn}); it = rg.held.end() - 1; }
        it->cpu_milli += q.req_cpu_milli; it->mem_mib += q.req_mem_mib; it->gpu = uint16_t(it->gpu + q.req_gpu); it->pods = uint16_t(it->pods + 1);
        if (!cdName.empty() && !cdName[e.clique].empty()) rg.cdOn[nn] = cdName[e.clique];   // its IMEX channel, while the PodGang runs
      }
    }
    if (gs[i].n_pods && !lastNode_.count(key)) lastNode_[key] = nodes[pl[gs[i].placement_off].node].Name;
    if (t.queueOf[i] != GROVE_NONE_U32) queueOf_[key] = t.queueNames[t.queueOf[i]];   // what it holds counts against its queue
    if (pg.BasePodGangName.empty())   // a replica of its PodCliqueSet from now on (topology spread counts it where it landed)
      if (auto it = pg.Labels.find(kPartOfLabel); it != pg.Labels.end()) setOf_[key] = pg.Namespace + "/" + it->second;
    std::vector<uint32_t>& done = bound_[key];
    done.resize(pg.Spec.PodGroups.size(), 0u);
    for (uint32_t c = t.gangs[i].clique_off; c < t.gangs[i].clique_off + t.gangs[i].n_cliques; ++c) done[t.cliqueOf[c].second] += seen[c];
    bool all = true; uint32_t unbound = 0;
    for (size_t k = 0; k < done.size(); ++k) {
      all &= done[k] >= pg.Spec.PodGroups[k].PodReferences.size();
      if (done[k] < pg.Spec.PodGroups[k].PodReferences.size()) unbound += uint32_t(pg.Spec.PodGroups[k].PodReferences.size()) - done[k];
    }
    // A PodGang WITH pack constraints is not resubmitted as a remainder (its best-effort pods would have to rejoin the
    // domains chosen for the gang): it is scheduled, leaves the pending set, and the status says how many of its
    // best-effort pods stayed Pending (ADVICE round 1: such gangs used to sit in the pending set for ever)
    if (!all && constrained(pg)) { (*statuses)[key].UnboundPods = unbound; all = true; }
    if (all) { pending_.erase(key); bound_.erase(key); }
  }
  return std::nullopt;
}

// The queue messages of a cycle, restated from its results in rank order (DESIGN.md section 1 "Queue limits"): the headroom each
// member met, from the queues' limits and loads and what the admitted members ranked before it took.
std::map<std::string, std::string> GpuBackend::QueueMessages(const Tables& t, const std::vector<grove_gang_status_t>& gs,
                                                             const std::vector<grove_placement_t>& pl) {
  std::map<std::string, std::string> msg;
  if (t.queues.empty()) return msg;
  static const char* kRes[3] = {"cpu (millicores)", "memory (MiB)", "GPUs"};
  const size_t nq = t.queues.size();
  std::vector<std::array<int64_t, 3>> load(nq);
  for (size_t q = 0; q < nq; ++q) for (int r = 0; r < 3; ++r) load[q][r] = int64_t(t.queues[q].used[r]);
  for (size_t q = nq; q-- > 0;)   // parents come first: a queue's load is its own and its descendants'
    if (t.queues[q].parent != GROVE_NONE_U32) for (int r = 0; r < 3; ++r) load[t.queues[q].parent][r] += load[q][r];
  std::vector<uint32_t> order;
  for (uint32_t g = 0; g < t.queueOf.size(); ++g) if (t.queueOf[g] != GROVE_NONE_U32) order.push_back(g);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return t.gangs[a].priority > t.gangs[b].priority; });
  auto finite = [&](size_t q, int r) { return t.queues[q].limit[r] != GROVE_QUEUE_UNLIMITED; };
  for (uint32_t g : order) {
    if (gs[g].state != GROVE_GANG_ADMITTED && gs[g].state != GROVE_GANG_REJECTED) continue;   // gated, or its base was not scheduled
    const grove_gang_t& gg = t.gangs[g];
    int64_t R[3] = {0, 0, 0};
    for (uint32_t c = gg.clique_off; c < gg.clique_off + gg.n_cliques; ++c) {
      const int64_t m = t.counts[c].min_replicas;
      R[0] += m * t.cliques[c].req_cpu_milli; R[1] += m * t.cliques[c].req_mem_mib; R[2] += m * t.cliques[c].req_gpu;
    }
    std::vector<uint32_t> chain;
    for (uint32_t q = t.queueOf[g]; q != GROVE_NONE_U32; q = t.queues[q].parent) chain.push_back(q);
    if (gs[g].reserved0 & GROVE_STATUS_OVER_LIMIT) {   // the first queue of the chain, leaf first, and the resource without room
      for (uint32_t q : chain) {
        int r = 0;
        while (r < 3 && !(finite(q, r) && R[r] > 0 && R[r] > int64_t(t.queues[q].limit[r]) - load[q][r])) ++r;
        if (r == 3) continue;
        msg[t.gangNames[g]] = "queue " + t.queueNames[q] + " has no room for this PodGang: " + kRes[r] + " limit " +
                              std::to_string(t.queues[q].limit[r]) + ", load " + std::to_string(load[q][r]) + ", MinReplicas need " + std::to_string(R[r]);
        break;
      }
      continue;
    }
    if (gs[g].state != GROVE_GANG_ADMITTED) continue;
    if (gs[g].reserved0 & GROVE_STATUS_SURPLUS_CAPPED) {   // s_q clique by clique, as the engine caps the surplus
      int64_t rem[3];
      bool fin[3] = {false, false, false};
      for (int r = 0; r < 3; ++r) {
        rem[r] = INT64_MAX;
        for (uint32_t q : chain) if (finite(q, r)) { fin[r] = true; rem[r] = std::min(rem[r], int64_t(t.queues[q].limit[r]) - load[q][r]); }
        if (fin[r]) rem[r] -= R[r];
      }
      int64_t held = 0;
      for (uint32_t c = gg.clique_off; c < gg.clique_off + gg.n_cliques; ++c) {
        const int64_t extra = int64_t(t.counts[c].replicas) - t.counts[c].min_replicas;
        const int64_t req[3] = {t.cliques[c].req_cpu_milli, t.cliques[c].req_mem_mib, t.cliques[c].req_gpu};
        int64_t sq = extra;
        for (int r = 0; r < 3; ++r) if (fin[r] && req[r] > 0) sq = rem[r] < 0 ? 0 : std::min(sq, rem[r] / req[r]);
        for (int r = 0; r < 3; ++r) if (fin[r]) rem[r] -= sq * req[r];
        held += extra - sq;
      }
      msg[t.gangNames[g]] = "queue limits held back " + std::to_string(held) + " best-effort pods of this PodGang";
    }
    for (uint32_t k = 0; k < gs[g].n_pods; ++k) {   // it charges what it took to every queue of its chain
      const grove_clique_t& c = t.cliques[pl[gs[g].placement_off + k].clique];
      for (uint32_t q : chain) { load[q][0] += c.req_cpu_milli; load[q][1] += c.req_mem_mib; load[q][2] += c.req_gpu; }
    }
  }
  return msg;
}

std::string GpuBackend::ExplainRejection(const Tables& t, const PodGang& pg, uint32_t row, const grove_gang_diag_t& gd,
                                         const grove_clique_diag_t* cliques, const std::vector<TopologyLevel>& levels) {
  const grove_gang_t& g = t.gangs[row];
  auto levelName = [&](uint32_t l) { return l < levels.size() ? levels[l].Domain : "level " + std::to_string(l); };
  if (gd.verdict == GROVE_DIAG_CLIQUE_SHORT) {
    const uint32_t q = g.clique_off + gd.clique;
    const grove_clique_diag_t& c = cliques[q];
    const grove_clique_t& rec = t.cliques[q];
    const grove_scope_t& sc = t.scopes[g.scope_off + GROVE_CLIQUE_SCOPE(rec.scope)];
    int deepest = -1;   // the deepest Required level binding the PodGroup: the label a node must carry
    for (uint32_t l : {uint32_t(g.level), uint32_t(sc.level), uint32_t(rec.level)}) if (l != GROVE_LEVEL_NONE) deepest = std::max(deepest, int(l));
    const std::pair<uint32_t, std::string> why[] = {
        {c.unschedulable, "unschedulable"}, {c.selector, "not matching the node selector"},
        {c.labels, "without the " + (deepest >= 0 && uint32_t(deepest) < levels.size() ? levels[deepest].Key : std::string("topology")) + " label"},
        {c.cpu, "insufficient cpu"}, {c.mem, "insufficient memory"}, {c.gpu, "insufficient nvidia.com/gpu"}, {c.pods, "too many pods"}};
    std::string parts;
    for (const auto& w : why) if (w.first) parts += (parts.empty() ? "" : ", ") + std::to_string(w.first) + " " + w.second;
    const uint32_t nodes = c.nodes_fit + c.unschedulable + c.selector + c.labels + c.cpu + c.mem + c.gpu + c.pods;
    return "PodGroup " + pg.Spec.PodGroups[t.cliqueOf[q].second].Name + ": " + std::to_string(c.nodes_fit) + "/" + std::to_string(nodes) +
           " nodes fit" + (parts.empty() ? "" : " (" + parts + ")") + "; " + std::to_string(c.pods_fit) + " of " +
           std::to_string(t.counts[q].min_replicas) + " pods fit in the cluster";
  }
  if (gd.verdict == GROVE_DIAG_NO_DOMAIN)
    return "no " + levelName(gd.level) + " holds every PodGroup's MinReplicas (0 of " + std::to_string(gd.domains) + ")";
  if (gd.verdict == GROVE_DIAG_NO_JOINT_FIT) {
    if (gd.level == GROVE_LEVEL_NONE) return "the cluster holds each PodGroup's MinReplicas alone, but not all of them together";
    return std::to_string(gd.domains_ok) + " of " + std::to_string(gd.domains) + " " + levelName(gd.level) +
           "s hold each PodGroup's MinReplicas alone, but not all of them together";
  }
  return "";
}

Err GpuBackend::Start(SnapshotFn snapshot, BindFn bind, std::chrono::milliseconds period) {
  std::lock_guard<std::mutex> l(mu_);
  if (loop_.joinable()) return mkerr("ERR_SYNC_PODGANG", "Start", "cycle loop already running");
  stop_ = false;
  loop_ = std::thread([this, snapshot, bind, period] {
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(mu_);
        if (cv_.wait_for(lk, period, [this] { return stop_; })) return;
        if (pending_.empty()) continue;
      }
      std::vector<Binding> b; std::map<std::string, PodGangStatus> st; grove_cycle_stats_t cs{};
      const std::vector<Node> nodes = snapshot();
      if (auto e = RunCycle(nodes, &b, &st, &cs)) continue;   // the next tick retries (the reconciler's requeue)
      cycles_.fetch_add(1);
      bind(b, st, cs);
    }
  });
  return std::nullopt;
}

void GpuBackend::Stop() {
  { std::lock_guard<std::mutex> l(mu_); stop_ = true; }
  cv_.notify_all();
  if (loop_.joinable()) loop_.join();
}

}  // namespace grove::host
