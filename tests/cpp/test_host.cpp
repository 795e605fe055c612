// Host-side mirror tests.  The producer cases are the reference's own table-driven vectors
// (ai-dynamo/grove operator/internal/controller/podcliqueset/components/podgang/syncflow_test.go:740-953
// TestComputeExpectedPodGangs and :965-1420 TestComputeExpectedPodGangsWithTopologyConstraints),
// transcribed: same inputs, same expected PodGang names, counts and topology keys.
//   test_host cpu   producer + encoder (no GPU)        test_host gpu   + GpuBackend cycles on cuda:0
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <set>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static PodCliqueTemplateSpec clq(const char* name, int replicas, int minAvail, const char* pack = nullptr) {
  PodCliqueTemplateSpec t; t.Name = name; t.Replicas = replicas; t.MinAvailable = minAvail;
  if (pack) t.Topology = PackDomain{pack};
  return t;
}
static PodCliqueScalingGroupConfig sg(const char* name, int replicas, int minAvail, std::vector<std::string> cliques, const char* pack = nullptr) {
  PodCliqueScalingGroupConfig g; g.Name = name; g.Replicas = replicas; g.MinAvailable = minAvail; g.CliqueNames = std::move(cliques);
  if (pack) g.Topology = PackDomain{pack};
  return g;
}
static std::set<std::string> names(const std::vector<PodGangInfo>& v, bool scaled) {
  std::set<std::string> s; for (const auto& p : v) if (p.baseFqn.empty() != scaled) s.insert(p.fqn); return s;
}
static std::string key(const std::optional<TopologyConstraint>& tc) {
  return (tc && tc->PackConstraint && tc->PackConstraint->Required) ? *tc->PackConstraint->Required : std::string();
}

static void test_compute_expected_podgangs() {  // syncflow_test.go:740-953
  struct Case { const char* name; int pcsReplicas; std::vector<PodCliqueTemplateSpec> pclqs; std::vector<PodCliqueScalingGroupConfig> pcsgs;
                size_t n; std::set<std::string> base, scaled; };
  std::vector<Case> cases = {
    {"Simple PCS with standalone PCLQs only", 2, {clq("worker", 3, 2)}, {}, 2, {"test-pcs-0", "test-pcs-1"}, {}},
    {"PCS with PCSG having minAvailable=1", 1, {clq("sg-worker", 2, 2)}, {sg("scaling-group", 3, 1, {"sg-worker"})}, 3, {"test-pcs-0"},
     {"test-pcs-0-scaling-group-0", "test-pcs-0-scaling-group-1"}},
    {"PCS with mixed standalone PCLQ and PCSG", 1, {clq("standalone", 2, 1), clq("scalable", 3, 2)}, {sg("sg", 4, 2, {"scalable"})}, 3,
     {"test-pcs-0"}, {"test-pcs-0-sg-0", "test-pcs-0-sg-1"}},
    {"Multiple PCS replicas with PCSG", 2, {clq("worker", 2, 1)}, {sg("worker-sg", 2, 1, {"worker"})}, 4, {"test-pcs-0", "test-pcs-1"},
     {"test-pcs-0-worker-sg-0", "test-pcs-1-worker-sg-0"}},
    {"PCSG with minAvailable equals replicas", 1, {clq("worker", 2, 2)}, {sg("sg", 2, 2, {"worker"})}, 1, {"test-pcs-0"}, {}},
    {"Multiple PCSGs in one PCS replica", 1, {clq("worker-a", 2, 2), clq("worker-b", 2, 2)},
     {sg("sg-a", 3, 1, {"worker-a"}), sg("sg-b", 2, 1, {"worker-b"})}, 4, {"test-pcs-0"},
     {"test-pcs-0-sg-a-0", "test-pcs-0-sg-a-1", "test-pcs-0-sg-b-0"}},
    {"Multiple cliques in one PCSG", 1, {clq("worker", 2, 2), clq("helper", 1, 1)}, {sg("sg", 3, 1, {"worker", "helper"})}, 3, {"test-pcs-0"},
     {"test-pcs-0-sg-0", "test-pcs-0-sg-1"}},
  };
  for (const auto& c : cases) {
    PodCliqueSet pcs; pcs.Name = "test-pcs"; pcs.Replicas = c.pcsReplicas; pcs.Cliques = c.pclqs; pcs.PodCliqueScalingGroupConfigs = c.pcsgs;
    std::vector<PodGangInfo> out;
    CHECK(!ComputeExpectedPodGangs(pcs, {}, false, &out));
    CHECK(out.size() == c.n);
    CHECK(names(out, false) == c.base);
    CHECK(names(out, true) == c.scaled);
    if (g_fail) std::fprintf(stderr, "  in case: %s\n", c.name);
  }
}

static void test_topology_constraints() {  // syncflow_test.go:965-1420
  const std::vector<TopologyLevel> levels = {{"zone", "topology.kubernetes.io/zone"}, {"rack", "topology.kubernetes.io/rack"}, {"host", "kubernetes.io/hostname"}};
  const std::string Z = levels[0].Key, R = levels[1].Key, H = levels[2].Key;
  auto run = [&](bool tas, const char* pcsPack, std::vector<PodCliqueTemplateSpec> pclqs, std::vector<PodCliqueScalingGroupConfig> pcsgs) {
    PodCliqueSet pcs; pcs.Name = "test-pcs"; pcs.Cliques = std::move(pclqs); pcs.PodCliqueScalingGroupConfigs = std::move(pcsgs);
    if (pcsPack) pcs.Topology = PackDomain{pcsPack};
    std::vector<PodGangInfo> out;
    CHECK(!ComputeExpectedPodGangs(pcs, levels, tas, &out));
    return out;
  };
  auto find = [](const std::vector<PodGangInfo>& v, const std::string& fqn) -> const PodGangInfo* { for (auto& p : v) if (p.fqn == fqn) return &p; return nullptr; };
  auto pclqKey = [](const PodGangInfo& pg, const std::string& fqn) { for (auto& p : pg.pclqs) if (p.fqn == fqn) return key(p.topologyConstraint); return std::string("<missing>"); };
  auto pcsgKey = [](const PodGangInfo& pg, const std::string& n) { for (auto& g : pg.pcsgTopologyConstraints) if (g.Name == n) return key(g.Topology); return std::string("<missing>"); };
  {  // no constraints anywhere
    auto o = run(true, nullptr, {clq("worker", 3, 2)}, {});
    CHECK(o.size() == 1 && key(o[0].topologyConstraint).empty() && o[0].pcsgTopologyConstraints.empty());
  }
  {  // PCS only
    auto o = run(true, "zone", {clq("worker", 3, 2)}, {});
    CHECK(o.size() == 1 && key(find(o, "test-pcs-0")->topologyConstraint) == Z);
  }
  {  // one of the PCLQs
    auto o = run(true, nullptr, {clq("router", 3, 2), clq("worker", 2, 1, "host")}, {});
    CHECK(o.size() == 1 && key(o[0].topologyConstraint).empty());
    CHECK(pclqKey(o[0], "test-pcs-0-worker") == H && pclqKey(o[0], "test-pcs-0-router").empty());
  }
  {  // all levels, standalone
    auto o = run(true, "zone", {clq("router", 3, 2, "zone"), clq("worker", 2, 1, "host")}, {});
    CHECK(key(o[0].topologyConstraint) == Z && pclqKey(o[0], "test-pcs-0-worker") == H && pclqKey(o[0], "test-pcs-0-router") == Z);
  }
  const std::vector<PodCliqueTemplateSpec> decode = {clq("decode-leader", 1, 1, "host"), clq("decode-worker", 5, 1, "host")};
  {  // PCS + PCSG
    auto o = run(true, "zone", decode, {sg("scaling-group", 2, 1, {"decode-leader", "decode-worker"}, "rack")});
    CHECK(o.size() == 2);
    const PodGangInfo* b = find(o, "test-pcs-0"); const PodGangInfo* s = find(o, "test-pcs-0-scaling-group-0");
    CHECK(b && s);
    if (b && s) {
      CHECK(key(b->topologyConstraint) == Z);
      CHECK(pclqKey(*b, "test-pcs-0-scaling-group-0-decode-leader") == H && pclqKey(*b, "test-pcs-0-scaling-group-0-decode-worker") == H);
      CHECK(pcsgKey(*b, "test-pcs-0-scaling-group-0") == R);
      CHECK(key(s->topologyConstraint) == R);  // scaled PodGang carries the PCSG constraint
      CHECK(pclqKey(*s, "test-pcs-0-scaling-group-1-decode-leader") == H && pclqKey(*s, "test-pcs-0-scaling-group-1-decode-worker") == H);
      CHECK(s->pcsgTopologyConstraints.empty());
    }
  }
  {  // standalone + PCSG, all levels
    std::vector<PodCliqueTemplateSpec> all = {clq("router", 1, 1, "zone")}; all.insert(all.end(), decode.begin(), decode.end());
    auto o = run(true, "zone", all, {sg("scaling-group", 2, 1, {"decode-leader", "decode-worker"}, "rack")});
    const PodGangInfo* b = find(o, "test-pcs-0");
    CHECK(o.size() == 2 && b && pclqKey(*b, "test-pcs-0-router") == Z && pcsgKey(*b, "test-pcs-0-scaling-group-0") == R);
  }
  {  // TAS disabled: nothing set anywhere
    std::vector<PodCliqueTemplateSpec> all = {clq("router", 1, 1, "zone")}; all.insert(all.end(), decode.begin(), decode.end());
    auto o = run(false, "zone", all, {sg("scaling-group", 2, 1, {"decode-leader", "decode-worker"}, "rack")});
    CHECK(o.size() == 2);
    for (const auto& pg : o) {
      CHECK(key(pg.topologyConstraint).empty() && pg.pcsgTopologyConstraints.empty());
      for (const auto& p : pg.pclqs) CHECK(key(p.topologyConstraint).empty());
    }
  }
  {  // PCSG without constraint: scaled PodGang falls back to the PCS constraint
    auto o = run(true, "zone", decode, {sg("scaling-group", 2, 1, {"decode-leader", "decode-worker"})});
    const PodGangInfo* b = find(o, "test-pcs-0"); const PodGangInfo* s = find(o, "test-pcs-0-scaling-group-0");
    CHECK(b && s && key(b->topologyConstraint) == Z && key(s->topologyConstraint) == Z && b->pcsgTopologyConstraints.empty());
  }
}

static std::vector<Node> e2e_nodes(int n, int cordoned = 0) {  // hack/e2e.yaml: 150 MiB nodes; zone 28 / block 14 / rack 7 / host
  std::vector<Node> v(n);
  for (int i = 0; i < n; ++i) {
    Node& nd = v[i];
    nd.Name = "kwok-node-" + std::to_string(i);
    nd.Labels = {{"topology.kubernetes.io/zone", "zone-" + std::to_string(i / 28)}, {"topology.kubernetes.io/block", "block-" + std::to_string(i / 14)},
                 {"topology.kubernetes.io/rack", "rack-" + std::to_string(i / 7)}, {"kubernetes.io/hostname", nd.Name},
                 {"node_role.e2e.grove.nvidia.com", "agent"}};
    nd.alloc_cpu_milli = 4000; nd.alloc_mem_mib = 150; nd.alloc_pods = 110;
    nd.TaintKeys = {"node_role.e2e.grove.nvidia.com"};
    nd.Unschedulable = i >= n - cordoned;
  }
  return v;
}
static const std::vector<TopologyLevel> kLevels = {{"zone", "topology.kubernetes.io/zone"}, {"block", "topology.kubernetes.io/block"},
                                                   {"rack", "topology.kubernetes.io/rack"}, {"host", "kubernetes.io/hostname"}};

static PodCliqueSet workload1() {  // e2e/yaml/workload1.yaml
  PodCliqueSet pcs; pcs.Name = "workload1";
  PodGang::Requests rq; rq.mem_mib = 80; rq.nodeSelector = {{"node_role.e2e.grove.nvidia.com", "agent"}}; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
  for (auto [n, r] : std::vector<std::pair<const char*, int>>{{"pc-a", 2}, {"pc-b", 1}, {"pc-c", 3}}) { auto c = clq(n, r, r); c.Requests = rq; pcs.Cliques.push_back(c); }
  pcs.PodCliqueScalingGroupConfigs = {sg("sg-x", 2, 2, {"pc-b", "pc-c"})};
  return pcs;
}

static void test_hierarchy_violations() {  // pcs/validation/topologyconstraints_test.go:228-357 (six vectors) and :410-457 (two)
  const std::vector<std::string> dom = {"region", "zone", "rack", "host", "numa"};
  const std::string PCS = "spec.template.topologyConstraint", SG0 = "spec.template.podCliqueScalingGroups[0].topologyConstraint";
  struct Case { const char* name; const char* pcs; std::vector<PodCliqueTemplateSpec> cliques; std::vector<PodCliqueScalingGroupConfig> sgs; std::vector<std::string> fields; };
  const std::vector<Case> cases = {
    {"PCS broader than PodClique", "zone", {clq("worker", 1, 1, "host")}, {}, {}},
    {"PCS narrower than PodClique", "host", {clq("worker", 1, 1, "zone")}, {}, {PCS}},
    {"PCS narrower than PCSG", "numa", {}, {sg("sg1", 1, 1, {"worker"}, "rack")}, {PCS}},
    {"PCSG narrower than PodClique", nullptr, {clq("worker", 1, 1, "zone")}, {sg("sg1", 1, 1, {"worker"}, "host")}, {SG0}},
    {"same level", "zone", {clq("worker", 1, 1, "zone")}, {}, {}},
    {"violations at several levels", "numa", {clq("worker1", 1, 1, "zone"), clq("worker2", 1, 1, "rack")}, {sg("sg1", 1, 1, {"worker1", "worker2"}, "host")},
     {PCS, PCS, PCS, SG0, SG0}},
  };
  for (const auto& c : cases) {
    PodCliqueSet pcs; pcs.Name = "t"; pcs.Cliques = c.cliques; pcs.PodCliqueScalingGroupConfigs = c.sgs;
    if (c.pcs) pcs.Topology = PackDomain{c.pcs};
    const auto errs = ValidateHierarchicalTopologyConstraints(pcs, dom);
    CHECK(errs.size() == c.fields.size());
    for (size_t i = 0; i < errs.size() && i < c.fields.size(); ++i) CHECK(errs[i].field == c.fields[i]);
  }
  const std::vector<std::string> custom = {"datacenter", "rack", "gpu-module", "host"};
  PodCliqueSet ok; ok.Topology = PackDomain{"datacenter"}; ok.Cliques = {clq("worker", 1, 1, "host")};
  CHECK(ValidateHierarchicalTopologyConstraints(ok, custom).empty());
  PodCliqueSet bad; bad.Topology = PackDomain{"host"}; bad.Cliques = {clq("worker", 1, 1, "datacenter")};
  CHECK(ValidateHierarchicalTopologyConstraints(bad, custom).size() == 1);
  PodCliqueSet unknown; unknown.Topology = PackDomain{"nvl-domain"}; unknown.Cliques = {clq("worker", 1, 1, "datacenter")};   // unknown domain: check skipped
  CHECK(ValidateHierarchicalTopologyConstraints(unknown, custom).empty());
  GpuBackend be; CHECK(!be.SyncTopology(kLevels));
  PodCliqueSet viol; viol.Name = "v"; viol.Topology = PackDomain{"host"}; viol.Cliques = {clq("worker", 1, 1, "zone")};
  CHECK(be.ValidatePodCliqueSet(viol).has_value());
}

static void test_is_base_podgang_scheduled() {  // podclique/components/pod/syncflow_test.go:323-372, the four vectors
  struct P { const char* name; int32_t minAvailable, scheduledReplicas; };
  struct Case { const char* name; bool exists; std::vector<P> pclqs; bool scheduled, error; };
  const std::vector<Case> cases = {
    {"all PodCliques meet MinAvailable", true, {{"simple1-0-pcb", 2, 2}, {"simple1-0-pcc", 1, 3}}, true, false},
    {"one PodClique below MinAvailable", true, {{"simple1-0-pcb", 2, 2}, {"simple1-0-pcc", 3, 2}}, false, false},
    {"base PodGang missing", false, {}, false, true},
    {"single PodClique", true, {{"simple1-0-pcb", 1, 1}}, true, false},
  };
  for (const auto& c : cases) {
    PodGang base; base.Namespace = "default"; base.Name = "simple1-0";
    std::map<std::string, int32_t> status;
    for (const auto& p : c.pclqs) { PodGroup g; g.Name = p.name; g.MinReplicas = p.minAvailable; base.Spec.PodGroups.push_back(g); status[p.name] = p.scheduledReplicas; }
    bool scheduled = true;
    auto e = IsBasePodGangScheduled(c.exists ? &base : nullptr, status, &scheduled);
    CHECK(e.has_value() == c.error);
    CHECK(scheduled == c.scheduled);
  }
  // a PodGroup whose PodClique cannot be read is an error too (requeue), not "unscheduled"
  PodGang base; base.Namespace = "default"; PodGroup g; g.Name = "x"; g.MinReplicas = 1; base.Spec.PodGroups.push_back(g);
  bool scheduled = true;
  CHECK(IsBasePodGangScheduled(&base, {}, &scheduled).has_value() && !scheduled);
}

static void test_pod_scheduling_gates() {  // podclique/components/pod/syncflow_test.go:40-125, the six vectors
  struct Case { const char* name; const char* podGang; bool baseExists, baseReady, hasGate, inPodGang, removed; int skipped; bool error; };
  const std::vector<Case> cases = {
    {"base PodGang pod: gate removed immediately", "simple1-0", true, false, true, true, true, 0, false},
    {"scaled PodGang pod, base not ready", "simple1-0-sga-2", true, false, true, true, false, 1, false},
    {"scaled PodGang pod, base ready", "simple1-0-sga-2", true, true, true, true, true, 0, false},
    {"scaled PodGang pod, base missing", "simple1-0-sga-3", false, false, true, true, false, 0, true},
    {"pod not in PodGang yet", "simple1-0-sga-2", true, true, true, false, false, 1, false},
    {"pod without gate", "simple1-0-sga-2", true, true, false, true, false, 0, false},
  };
  for (const auto& c : cases) {
    const bool scaled = std::string(c.podGang).find("-sga-") != std::string::npos;
    PodGang base; base.Namespace = "default"; base.Name = "simple1-0";
    PodGroup g; g.Name = "simple1-0-pcb"; g.MinReplicas = 2; base.Spec.PodGroups.push_back(g);
    std::map<std::string, int32_t> status = {{"simple1-0-pcb", c.baseReady ? 2 : 1}};
    bool removed = true, skipped = true;
    auto e = CheckPodSchedulingGate(c.hasGate, c.inPodGang, scaled ? "simple1-0" : "", c.baseExists ? &base : nullptr, status, &removed, &skipped);
    CHECK(e.has_value() == c.error);
    CHECK(removed == c.removed);
    CHECK(int(skipped) == c.skipped);
  }
}

static void test_scheduled_condition_and_counts() {  // podclique/reconcilestatus.go:134-141, 255-274
  auto c = ComputePodCliqueScheduledCondition(2, 3);
  CHECK(c.Type == "PodCliqueScheduled" && c.Status == "False" && c.Reason == "InsufficientScheduledPods");
  CHECK(c.Message == "Insufficient scheduled pods. expected at least: 3, found: 2");
  c = ComputePodCliqueScheduledCondition(3, 3);
  CHECK(c.Status == "True" && c.Reason == "SufficientScheduledPods" && c.Message == "Sufficient scheduled pods found. expected at least: 3, found: 3");
  const std::vector<Binding> b = {{"default", "w-0-pc-a-0", "n0"}, {"default", "w-0-pc-a-1", "n1"}, {"default", "w-0-sg-x-0-pc-c-10", "n2"}};
  const auto n = CountScheduledReplicas(b);
  CHECK(n.size() == 2 && n.at("w-0-pc-a") == 2 && n.at("w-0-sg-x-0-pc-c") == 1);
  // together with the gang predicate: bindings -> ScheduledReplicas -> is the base PodGang scheduled?
  PodGang base; base.Namespace = "default"; base.Name = "w-0";
  for (auto [name, mn] : std::vector<std::pair<const char*, int>>{{"w-0-pc-a", 2}, {"w-0-sg-x-0-pc-c", 1}}) { PodGroup g; g.Name = name; g.MinReplicas = mn; base.Spec.PodGroups.push_back(g); }
  bool scheduled = false;
  CHECK(!IsBasePodGangScheduled(&base, n, &scheduled) && scheduled);
}

static void test_encode() {
  GpuBackend be;
  CHECK(be.Name() == "gpu-scheduler");
  std::string sched; be.PreparePod(&sched); CHECK(sched == "gpu-scheduler");
  CHECK(!be.SyncTopology(kLevels));
  CHECK(be.CheckTopologyDrift(kLevels).first);
  auto drift = kLevels; drift[2].Key = "example.com/nvlink-domain";
  CHECK(!be.CheckTopologyDrift(drift).first);
  PodCliqueSet pcs = workload1(); pcs.Topology = PackDomain{"block"}; pcs.PodCliqueScalingGroupConfigs[0].Topology = PackDomain{"rack"};
  CHECK(!be.ValidatePodCliqueSet(pcs));
  std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
  CHECK(infos.size() == 1);
  for (const auto& i : infos) CHECK(!be.SyncPodGang(BuildPodGang(pcs, i)));
  CHECK(be.Pending() == 1);
  Tables t; CHECK(!be.Encode(e2e_nodes(10, 1), &t));
  CHECK(t.nodes.size() == 10 && t.gangs.size() == 1 && t.cliques.size() == 5 && t.scopes.size() == 3);
  CHECK(t.gangs[0].level == 1 && t.gangs[0].n_cliques == 5 && t.gangs[0].n_scopes == 3 && t.gangs[0].base_gang == GROVE_NONE_U32);
  CHECK(t.scopes[0].level == GROVE_LEVEL_NONE && t.scopes[0].n_cliques == 1);            // pc-a, loose
  CHECK(t.scopes[1].level == 2 && t.scopes[1].n_cliques == 2 && t.scopes[2].level == 2);  // sg-x replicas 0 and 1 -> rack
  CHECK(t.cliques[0].min_replicas == 2 && t.cliques[0].replicas == 2 && t.cliques[0].req_mem_mib == 80);
  CHECK(t.cliques[2].min_replicas == 3 && t.cliques[1].scope == 1 && t.cliques[4].scope == 2);
  CHECK(t.cliques[0].class_mask == 0x2);  // only the "agent" class, whose taint the pods tolerate
  CHECK((t.nodes[0].flags & GROVE_NODE_SCHEDULABLE) && !(t.nodes[9].flags & GROVE_NODE_SCHEDULABLE));
  CHECK(t.nodes[0].dom[0] == t.nodes[9].dom[0] && t.nodes[0].dom[2] != t.nodes[7].dom[2] && t.nodes[0].free_mem_mib == 150);
  // a Required key that is not (or no longer) a level of the synced topology is DROPPED, as the operator does for a pack
  // domain it cannot find (createTopologyPackConstraint, syncflow.go:349-371): the pass goes on for everybody
  PodGang bad = BuildPodGang(pcs, infos[0]); bad.Name = "bad"; bad.Spec.Topology = TopologyConstraint{TopologyPackConstraint{std::string("example.com/nope"), std::nullopt}};
  CHECK(!be.SyncPodGang(bad));
  CHECK(!be.Encode(e2e_nodes(10), &t));
  CHECK(t.gangs.size() == 2 && t.gangNames[0].find("bad") != std::string::npos && t.gangs[0].level == GROVE_LEVEL_NONE && t.gangs[1].level == 1);
  CHECK(!be.OnPodGangDelete(bad));
  // a PodGang the packed tables cannot hold is left out of the pass with a reason; SyncPodGang itself accepts it (an error
  // there would requeue the reconcile for ever), and the others are encoded as usual
  PodGang huge = BuildPodGang(pcs, infos[0]); huge.Name = "huge";
  for (int i = 0; i < 300; ++i) huge.Spec.PodGroups[0].PodReferences.push_back({"default", "huge-pod-" + std::to_string(i)});
  CHECK(!GpuBackend::WhyNotEncodable(huge).empty() && GpuBackend::WhyNotEncodable(bad).empty());
  CHECK(!be.SyncPodGang(huge));
  CHECK(!be.Encode(e2e_nodes(10), &t));
  CHECK(t.gangs.size() == 1 && t.skipped.size() == 1 && t.skipped.begin()->first.find("huge") != std::string::npos);
  CHECK(t.skipped.begin()->second.find("podReferences") != std::string::npos);
  CHECK(!be.OnPodGangDelete(huge));
  CHECK(be.TopologyGVR().Resource == "clustertopologies" && be.TopologyGVR().Group == "grove.io");
  // Preferred keys (podgang.go:110-117) become Preferred levels; one that is not deeper than Required is dropped
  PodGang pref = BuildPodGang(pcs, infos[0]); pref.Name = "zz-pref";  // rows follow the PodGang key order: after workload1-0
  pref.Spec.Topology = TopologyConstraint{TopologyPackConstraint{std::nullopt, kLevels[2].Key}};
  pref.Spec.TopologyConstraintGroupConfigs[0].Topology = TopologyConstraint{TopologyPackConstraint{kLevels[1].Key, kLevels[2].Key}};
  pref.Spec.TopologyConstraintGroupConfigs[1].Topology = TopologyConstraint{TopologyPackConstraint{kLevels[2].Key, kLevels[1].Key}};
  pref.Spec.PodGroups[0].Topology = TopologyConstraint{TopologyPackConstraint{std::nullopt, kLevels[3].Key}};
  CHECK(!be.SyncPodGang(pref));
  CHECK(!be.Encode(e2e_nodes(10), &t));
  CHECK(t.gangs.size() == 2 && t.gangs[1].level == GROVE_LEVEL_NONE && t.gangs[1].preferred == 2 && t.gangs[0].preferred == GROVE_LEVEL_NONE);
  CHECK(t.scopes[3].preferred1 == 0 && t.scopes[4].level == 1 && t.scopes[4].preferred1 == 3 && t.scopes[5].level == 2 && t.scopes[5].preferred1 == 0);
  CHECK(GROVE_CLIQUE_SCOPE(t.cliques[5].scope) == 0 && GROVE_CLIQUE_PREFERRED(t.cliques[5].scope) == 3);
  CHECK(GROVE_CLIQUE_SCOPE(t.cliques[6].scope) == 1 && GROVE_CLIQUE_PREFERRED(t.cliques[6].scope) == GROVE_LEVEL_NONE);
  CHECK(!be.OnPodGangDelete(pref));
  // engine limits surface in ValidatePodCliqueSet
  PodCliqueSet big; big.Name = "big"; big.Cliques = {clq("w", 200, 200)};
  CHECK(be.ValidatePodCliqueSet(big).has_value());
}

static void test_gpu_cycles() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  PodCliqueSet pcs = workload1();
  std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  // GS1 (gang_scheduling_test.go:34-74): 9 schedulable nodes -> nothing bound; 10 -> 10 pods on 10 distinct nodes
  for (const auto& i : infos) CHECK(!be.SyncPodGang(BuildPodGang(pcs, i)));
  CHECK(!be.RunCycle(e2e_nodes(10, 1), &b, &st));
  CHECK(b.empty() && st.size() == 1 && !st.begin()->second.Scheduled && st.begin()->second.ScheduledReason == "Unschedulable");
  CHECK(be.Pending() == 1);  // still pending: retried next cycle
  CHECK(!be.RunCycle(e2e_nodes(10), &b, &st));
  CHECK(b.size() == 10 && st.begin()->second.Scheduled && st.begin()->second.Phase == PodGangPhase::Starting);
  std::set<std::string> nodes, pods; for (auto& x : b) { nodes.insert(x.NodeName); pods.insert(x.PodName); }
  CHECK(nodes.size() == 10 && pods.size() == 10 && be.Pending() == 0);
  CHECK(st.begin()->second.PlacementScore && *st.begin()->second.PlacementScore > 0.0 && *st.begin()->second.PlacementScore <= 1.0);
  // TAS8 (topology_test.go:501-578): block -> rack -> host on 8 nodes
  PodCliqueSet tas; tas.Name = "tas-hierarchy"; tas.Topology = PackDomain{"block"};
  PodGang::Requests rq; rq.mem_mib = 40; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
  for (const char* n : {"prefill", "decode"}) { auto c = clq(n, 2, 2, "host"); c.Requests = rq; tas.Cliques.push_back(c); }
  tas.PodCliqueScalingGroupConfigs = {sg("inference-group", 2, 2, {"prefill", "decode"}, "rack")};
  CHECK(!ComputeExpectedPodGangs(tas, kLevels, true, &infos));
  for (const auto& i : infos) CHECK(!be.SyncPodGang(BuildPodGang(tas, i)));
  auto n8 = e2e_nodes(8);
  CHECK(!be.RunCycle(n8, &b, &st));
  CHECK(b.size() == 8 && st.begin()->second.Scheduled);
  std::map<std::string, std::set<std::string>> hostsOfClique, racksOfReplica;
  for (auto& x : b) {
    const std::string clique = x.PodName.substr(0, x.PodName.rfind('-'));  // <pclq fqn>-<ordinal>
    hostsOfClique[clique].insert(x.NodeName);
    const int idx = std::atoi(x.NodeName.c_str() + std::strlen("kwok-node-"));
    racksOfReplica[clique.substr(0, clique.rfind('-'))].insert(n8[idx].Labels.at("topology.kubernetes.io/rack"));
  }
  CHECK(hostsOfClique.size() == 4);
  for (auto& kv : hostsOfClique) CHECK(kv.second.size() == 1);   // every PodClique on one host
  CHECK(racksOfReplica.size() == 2);
  for (auto& kv : racksOfReplica) CHECK(kv.second.size() == 1);  // every PCSG replica in one rack
}

// GS5 + GS7 shape (gang_scheduling_test.go:277-285, 449-465) through the backend: workload2 (every minAvailable 1) while
// nodes are uncordoned step by step.  Pods of a scheduled PodGang that found no node stay pending and are retried.
static void test_gpu_min_replicas_then_remainder() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  PodCliqueSet pcs; pcs.Name = "workload2";
  PodGang::Requests rq; rq.mem_mib = 80; rq.nodeSelector = {{"node_role.e2e.grove.nvidia.com", "agent"}}; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
  for (auto [n, r] : std::vector<std::pair<const char*, int>>{{"pc-a", 2}, {"pc-b", 1}, {"pc-c", 3}}) { auto c = clq(n, r, 1); c.Requests = rq; pcs.Cliques.push_back(c); }
  pcs.PodCliqueScalingGroupConfigs = {sg("sg-x", 2, 1, {"pc-b", "pc-c"})};
  std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
  CHECK(infos.size() == 2);   // base (pc-a + sg-x-0) and the scaled gang of sg-x-1
  for (const auto& i : infos) CHECK(!be.SyncPodGang(BuildPodGang(pcs, i)));
  std::map<std::string, std::string> podNode;   // every binding so far
  auto cycle = [&](int cordoned) {
    auto nodes = e2e_nodes(14, cordoned);
    for (const auto& kv : podNode) for (auto& nd : nodes) if (nd.Name == kv.second) { nd.used_mem_mib += 80; nd.used_pods += 1; }
    std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
    CHECK(!be.RunCycle(nodes, &b, &st));
    for (const auto& x : b) { CHECK(!podNode.count(x.PodName)); podNode[x.PodName] = x.NodeName; }
    return b.size();
  };
  CHECK(cycle(12) == 0 && be.Unscheduled() == 2);                 // 2 free nodes < 3 = sum of the base gang's MinReplicas
  CHECK(cycle(11) == 3 && be.Unscheduled() == 1 && be.Pending() == 2);   // base scheduled with exactly its minimum; 3 of its pods wait
  CHECK(cycle(9) == 2 && be.Unscheduled() == 0 && be.Pending() == 2);    // the scaled gang's minimum (pc-b 1 + pc-c 1) goes before anyone's surplus
  CHECK(cycle(4) == 5 && be.Pending() == 0);                             // the five pods left over, as remainders
  std::set<std::string> nodes; for (const auto& kv : podNode) nodes.insert(kv.second);
  CHECK(podNode.size() == 10 && nodes.size() == 10);
}

// Preemption (podgang.go:166-170 DisruptionTarget, reason 1; PriorityClassName :62-64): six one-pod nodes full of a
// low-priority PodGang; a high-priority PodGang of two pods is unschedulable without it, evicts it WHOLE, and the victim comes
// back with the DisruptionTarget condition.  With preemption off the high-priority PodGang simply stays pending.
static void test_gpu_preemption() {
  for (const bool on : {false, true}) {
    GpuBackend be;
    CHECK(!be.SyncTopology(kLevels));
    CHECK(!be.Init());
    be.SetPreemption(on);
    be.SetPriorityClass("low", 0); be.SetPriorityClass("high", 1000);
    PodGang::Requests rq; rq.mem_mib = 80; rq.nodeSelector = {{"node_role.e2e.grove.nvidia.com", "agent"}}; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
    auto one = [&](const char* name, const char* prio, int replicas) {
      PodCliqueSet pcs; pcs.Name = name; pcs.PriorityClassName = prio;
      auto c = clq("w", replicas, replicas); c.Requests = rq; pcs.Cliques.push_back(c);
      std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
      CHECK(infos.size() == 1);
      return BuildPodGang(pcs, infos[0]);
    };
    std::map<std::string, std::string> podNode;
    auto cycle = [&](std::map<std::string, PodGangStatus>* st) {
      auto nodes = e2e_nodes(6);
      for (const auto& kv : podNode) for (auto& nd : nodes) if (nd.Name == kv.second) { nd.used_mem_mib += 80; nd.used_pods += 1; }
      std::vector<Binding> b;
      CHECK(!be.RunCycle(nodes, &b, st));
      for (const auto& x : b) podNode[x.PodName] = x.NodeName;
      return b.size();
    };
    std::map<std::string, PodGangStatus> st;
    const PodGang filler = one("filler", "low", 6);
    CHECK(!be.SyncPodGang(filler));
    CHECK(cycle(&st) == 6 && be.Running() == 1 && be.Pending() == 0);
    const PodGang urgent = one("urgent", "high", 2);
    CHECK(!be.SyncPodGang(urgent));
    const size_t bound = cycle(&st);
    const std::string fk = filler.Namespace + "/" + filler.Name, uk = urgent.Namespace + "/" + urgent.Name;
    if (!on) {
      CHECK(bound == 0 && st.at(uk).ScheduledReason == "Unschedulable" && !st.count(fk) && be.Running() == 1 && be.Pending() == 1);
      continue;
    }
    CHECK(bound == 2 && st.at(uk).Scheduled && be.Pending() == 0);
    CHECK(st.count(fk) && st.at(fk).DisruptionTarget && st.at(fk).DisruptionMessage.find(uk) != std::string::npos);
    CHECK(be.Running() == 1);   // the victim is forgotten, the preemptor runs
    // the two pods sit on nodes the victim held
    std::set<std::string> fillerNodes, urgentNodes;
    for (const auto& kv : podNode) (kv.first.find("urgent") != std::string::npos ? urgentNodes : fillerNodes).insert(kv.second);
    CHECK(urgentNodes.size() == 2);
    for (const auto& n : urgentNodes) CHECK(fillerNodes.count(n));
  }
}

// The backend's cycle loop (INTEGRATION.md section 2): several "reconcilers" call SyncPodGang concurrently
// (controller/podgang/register.go:34-36) while ONE thread snapshots nodes, runs cycles and binds.  A PodGang the tables
// cannot hold is reported Unschedulable with its reason and does not stop anybody else.
static void test_gpu_cycle_loop_with_concurrent_reconcilers() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  PodGang::Requests rq; rq.mem_mib = 80; rq.nodeSelector = {{"node_role.e2e.grove.nvidia.com", "agent"}}; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
  std::mutex mu; std::map<std::string, std::string> podNode; std::map<std::string, PodGangStatus> last;
  auto snapshot = [&] {
    auto nodes = e2e_nodes(28, 0);
    std::lock_guard<std::mutex> l(mu);
    for (const auto& kv : podNode) for (auto& nd : nodes) if (nd.Name == kv.second) { nd.used_mem_mib += 80; nd.used_pods += 1; }
    return nodes;
  };
  auto bind = [&](const std::vector<Binding>& b, const std::map<std::string, PodGangStatus>& st, const grove_cycle_stats_t&) {
    std::lock_guard<std::mutex> l(mu);
    for (const auto& x : b) { CHECK(!podNode.count(x.PodName)); podNode[x.PodName] = x.NodeName; }
    for (const auto& kv : st) last[kv.first] = kv.second;
  };
  CHECK(!be.Start(snapshot, bind, std::chrono::milliseconds(2)));
  CHECK(be.Start(snapshot, bind, std::chrono::milliseconds(2)).has_value());   // already running
  std::vector<std::thread> reconcilers;
  for (int t = 0; t < 4; ++t)
    reconcilers.emplace_back([&, t] {
      for (int k = 0; k < 3; ++k) {
        PodCliqueSet pcs; pcs.Name = "wl-" + std::to_string(t) + "-" + std::to_string(k);
        auto c = clq("pc", 2, 2); c.Requests = rq; pcs.Cliques.push_back(c);
        std::vector<PodGangInfo> infos;
        if (ComputeExpectedPodGangs(pcs, kLevels, true, &infos)) { ++g_fail; return; }
        for (const auto& i : infos) if (be.SyncPodGang(BuildPodGang(pcs, i))) ++g_fail;
        std::this_thread::sleep_for(std::chrono::milliseconds(1));
      }
    });
  { PodCliqueSet pcs; pcs.Name = "huge"; auto c = clq("pc", 2, 2); c.Requests = rq; pcs.Cliques.push_back(c);
    std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
    PodGang huge = BuildPodGang(pcs, infos[0]);
    for (int i = 0; i < 300; ++i) huge.Spec.PodGroups[0].PodReferences.push_back({"default", "huge-pod-" + std::to_string(i)});
    CHECK(!be.SyncPodGang(huge)); }
  for (auto& t : reconcilers) t.join();
  for (int spin = 0; spin < 2000 && be.Pending() > 1; ++spin) std::this_thread::sleep_for(std::chrono::milliseconds(1));
  be.Stop();
  std::lock_guard<std::mutex> l(mu);
  CHECK(be.Pending() == 1 && be.Cycles() >= 1);                      // only the oversized PodGang is left
  CHECK(podNode.size() == 24);                                       // 12 PodGangs x 2 pods, each bound exactly once
  std::set<std::string> used; for (const auto& kv : podNode) used.insert(kv.second);
  CHECK(used.size() == 24);                                          // 150 MiB nodes hold one 80 MiB pod each
  bool seen_huge = false;
  for (const auto& kv : last) if (kv.first.find("huge") != std::string::npos) { seen_huge = true; CHECK(!kv.second.Scheduled && kv.second.ScheduledReason == "Unschedulable" && !kv.second.ScheduledMessage.empty()); }
  CHECK(seen_huge);
}

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && std::strcmp(argv[1], "gpu") == 0;
  test_compute_expected_podgangs();
  test_topology_constraints();
  test_hierarchy_violations();
  test_is_base_podgang_scheduled();
  test_pod_scheduling_gates();
  test_scheduled_condition_and_counts();
  test_encode();
  if (gpu) { test_gpu_cycles(); test_gpu_min_replicas_then_remainder(); test_gpu_preemption(); test_gpu_cycle_loop_with_concurrent_reconcilers(); }
  else {  // without a CUDA device Init must fail loudly, never fall back
    GpuBackend be; be.SyncTopology(kLevels);
    auto e = be.Init();
    if (!e) std::fprintf(stderr, "note: a CUDA device is present; Init succeeded\n");
    else CHECK(e->message.find("no CPU fallback") != std::string::npos);
  }
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host tests ok (%s)\n", gpu ? "cpu+gpu" : "cpu");
  return 0;
}
