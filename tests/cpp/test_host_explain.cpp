// GpuBackend::SetExplainUnschedulable on cuda:0: with the switch off a rejected PodGang's status is what it always was (reason
// Unschedulable, empty message); with it on the message names the PodGroup and the predicates that turned nodes away, or the
// topology level no domain of which holds the PodGang; after a running-gang cycle (preemption) it stays empty.
#include <cstdio>
#include <map>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const std::vector<TopologyLevel> kLevels = {{"zone", "topology.kubernetes.io/zone"}, {"block", "topology.kubernetes.io/block"},
                                                   {"rack", "topology.kubernetes.io/rack"}, {"host", "kubernetes.io/hostname"}};

// hack/e2e.yaml's layout (zone 28 / block 14 / rack 7 / host), with room for `perNode` 80 MiB pods per node; the first
// `cordoned` nodes are cordoned
static std::vector<Node> nodes(int n, int perNode, int cordoned = 0) {
  std::vector<Node> v(n);
  for (int i = 0; i < n; ++i) {
    Node& nd = v[i];
    nd.Name = "kwok-node-" + std::to_string(i);
    nd.Labels = {{"topology.kubernetes.io/zone", "zone-" + std::to_string(i / 28)}, {"topology.kubernetes.io/block", "block-" + std::to_string(i / 14)},
                 {"topology.kubernetes.io/rack", "rack-" + std::to_string(i / 7)}, {"kubernetes.io/hostname", nd.Name},
                 {"node_role.e2e.grove.nvidia.com", "agent"}};
    nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 80u * uint32_t(perNode) + 70u; nd.alloc_pods = 110;
    nd.TaintKeys = {"node_role.e2e.grove.nvidia.com"};
    nd.Unschedulable = i < cordoned;
  }
  return v;
}

// e2e/yaml/workload1.yaml's base PodGang (Required block; 10 pods of 80 MiB), with `extra` more pods in PodGroup pc-a, whose
// MinReplicas becomes `mn`
static PodGang workload1(const std::string& name, int extra, int mn) {
  PodCliqueSet pcs; pcs.Name = "workload1";
  PodGang::Requests rq; rq.mem_mib = 80; rq.nodeSelector = {{"node_role.e2e.grove.nvidia.com", "agent"}}; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
  for (auto [n, r] : std::vector<std::pair<const char*, int>>{{"pc-a", 2}, {"pc-b", 1}, {"pc-c", 3}}) {
    PodCliqueTemplateSpec c; c.Name = n; c.Replicas = r; c.MinAvailable = r; c.Requests = rq; pcs.Cliques.push_back(c);
  }
  PodCliqueScalingGroupConfig g; g.Name = "sg-x"; g.Replicas = 2; g.MinAvailable = 2; g.CliqueNames = {"pc-b", "pc-c"};
  pcs.PodCliqueScalingGroupConfigs = {g};
  pcs.Topology = PackDomain{"block"};
  std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
  PodGang pg = BuildPodGang(pcs, infos[0]);
  pg.Name = name;
  for (int i = 0; i < extra; ++i) pg.Spec.PodGroups[0].PodReferences.push_back({"default", name + "-pc-a-" + std::to_string(i)});
  if (extra) pg.Spec.PodGroups[0].MinReplicas = mn;
  return pg;
}

static PodGangStatus cycle(GpuBackend& be, const PodGang& pg, const std::vector<Node>& ns) {
  CHECK(!be.SyncPodGang(pg));
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(ns, &b, &st));
  CHECK(st.count("default/" + pg.Name));
  return st["default/" + pg.Name];
}

static bool has(const std::string& s, const std::string& part) {
  const bool ok = s.find(part) != std::string::npos;
  if (!ok) std::fprintf(stderr, "  message \"%s\" lacks \"%s\"\n", s.c_str(), part.c_str());
  return ok;
}

int main() {
  {   // off: as before
    GpuBackend be;
    CHECK(!be.SyncTopology(kLevels) && !be.Init());
    const PodGangStatus s = cycle(be, workload1("w", 0, 0), nodes(28, 0, 4));
    CHECK(!s.Scheduled && s.ScheduledReason == "Unschedulable" && s.ScheduledMessage.empty());
  }
  {   // no node has the memory: the PodGroup, each predicate's count, and what fits of its MinReplicas
    GpuBackend be;
    be.SetExplainUnschedulable(true);
    CHECK(!be.SyncTopology(kLevels) && !be.Init());
    const PodGang pg = workload1("w", 0, 0);
    const PodGangStatus s = cycle(be, pg, nodes(28, 0, 4));
    CHECK(s.ScheduledReason == "Unschedulable");
    bool named = false;
    for (const auto& p : pg.Spec.PodGroups) named |= s.ScheduledMessage.rfind("PodGroup " + p.Name + ": ", 0) == 0;
    CHECK(named);
    CHECK(has(s.ScheduledMessage, ": 0/28 nodes fit (4 unschedulable, 24 insufficient memory); 0 of "));
    CHECK(has(s.ScheduledMessage, " pods fit in the cluster"));
  }
  {   // 200 pods of pc-a: 280 fit in the cluster, 140 in a block
    GpuBackend be;
    be.SetExplainUnschedulable(true); be.SetLargePodGangs(true);
    CHECK(!be.SyncTopology(kLevels) && !be.Init());
    const PodGangStatus s = cycle(be, workload1("big", 298, 200), nodes(28, 10));
    CHECK(s.ScheduledReason == "Unschedulable" && s.ScheduledMessage == "no block holds every PodGroup's MinReplicas (0 of 2)");
  }
  {   // 135 of pc-a and the 8 others: each fits a block alone, together they need 143 of a block's 140 pod slots
    GpuBackend be;
    be.SetExplainUnschedulable(true); be.SetLargePodGangs(true);
    CHECK(!be.SyncTopology(kLevels) && !be.Init());
    const PodGangStatus s = cycle(be, workload1("big", 298, 135), nodes(28, 10));
    CHECK(s.ScheduledReason == "Unschedulable" &&
          s.ScheduledMessage == "2 of 2 blocks hold each PodGroup's MinReplicas alone, but not all of them together");
  }
  {   // a running-gang cycle: the message stays empty
    GpuBackend be;
    be.SetExplainUnschedulable(true); be.SetPreemption(true);
    CHECK(!be.SyncTopology(kLevels) && !be.Init());
    CHECK(cycle(be, workload1("first", 0, 0), nodes(28, 40)).Scheduled);
    CHECK(be.Running() == 1);
    const PodGangStatus s = cycle(be, workload1("second", 0, 0), nodes(28, 0));
    CHECK(s.ScheduledReason == "Unschedulable" && s.ScheduledMessage.empty());
  }
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host explain tests ok\n");
  return 0;
}
