// GpuBackend with reuse with reclaim (SetReclaimWithReuse) on cuda:0.  Six e2e nodes (one 80 MiB pod each) are full with two
// running PodGangs of a low priority, serve-v1 and batch.  The next cycle carries serve-v2, whose ReuseReservationRef names
// serve-v1, and urgent, of a high priority.  In the same cycle serve-v2 is admitted onto serve-v1's nodes (a rolling update) and
// urgent preempts batch: batch gets DisruptionTarget naming urgent, serve-v1 is forgotten without it.  Preemption and reservation
// reuse turned on together, without the new switch, still fail.
#include <cstdio>
#include <set>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static std::vector<Node> e2e_nodes(int n) {  // hack/e2e.yaml: 150 MiB nodes; zone 28 / block 14 / rack 7 / host
  std::vector<Node> v(n);
  for (int i = 0; i < n; ++i) {
    Node& nd = v[i];
    nd.Name = "kwok-node-" + std::to_string(i);
    nd.Labels = {{"topology.kubernetes.io/zone", "zone-" + std::to_string(i / 28)}, {"topology.kubernetes.io/block", "block-" + std::to_string(i / 14)},
                 {"topology.kubernetes.io/rack", "rack-" + std::to_string(i / 7)}, {"kubernetes.io/hostname", nd.Name},
                 {"node_role.e2e.grove.nvidia.com", "agent"}};
    nd.alloc_cpu_milli = 4000; nd.alloc_mem_mib = 150; nd.alloc_pods = 110;
    nd.TaintKeys = {"node_role.e2e.grove.nvidia.com"};
  }
  return v;
}
static const std::vector<TopologyLevel> kLevels = {{"zone", "topology.kubernetes.io/zone"}, {"block", "topology.kubernetes.io/block"},
                                                   {"rack", "topology.kubernetes.io/rack"}, {"host", "kubernetes.io/hostname"}};

static PodGang one(const char* name, int replicas, const char* priorityClass) {
  PodGang::Requests rq; rq.mem_mib = 80; rq.nodeSelector = {{"node_role.e2e.grove.nvidia.com", "agent"}}; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
  PodCliqueSet pcs; pcs.Name = name; pcs.PriorityClassName = priorityClass;
  PodCliqueTemplateSpec c; c.Name = "w"; c.Replicas = replicas; c.MinAvailable = replicas; c.Requests = rq;
  pcs.Cliques.push_back(c);
  std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
  CHECK(infos.size() == 1);
  return BuildPodGang(pcs, infos[0]);
}

static std::string key(const PodGang& pg) { return pg.Namespace + "/" + pg.Name; }

static void test_rolling_update_and_preemption() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  be.SetPriorityClass("low", 0); be.SetPriorityClass("high", 10);
  be.SetReclaimWithReuse(true);
  std::map<std::string, std::string> podNode;   // pods the caller has not deleted -> node
  auto cycle = [&](std::map<std::string, PodGangStatus>* st) {
    auto nodes = e2e_nodes(6);
    for (const auto& kv : podNode) for (auto& nd : nodes) if (nd.Name == kv.second) { nd.used_mem_mib += 80; nd.used_pods += 1; }
    std::vector<Binding> b;
    CHECK(!be.RunCycle(nodes, &b, st));
    for (const auto& x : b) podNode[x.PodName] = x.NodeName;
    return b;
  };
  auto nodesOf = [&](const char* name) {
    std::set<std::string> s;
    for (const auto& kv : podNode) if (kv.first.find(name) != std::string::npos) s.insert(kv.second);
    return s;
  };
  std::map<std::string, PodGangStatus> st;
  const PodGang v1 = one("serve-v1", 3, "low"), batch = one("batch", 3, "low");
  CHECK(!be.SyncPodGang(v1)); CHECK(!be.SyncPodGang(batch));
  CHECK(cycle(&st).size() == 6 && be.Running() == 2 && be.Pending() == 0);
  const std::set<std::string> v1Nodes = nodesOf("serve-v1"), batchNodes = nodesOf("batch");
  PodGang v2 = one("serve-v2", 3, "low");
  v2.Spec.ReuseReservationRef = NamespacedName{v1.Namespace, v1.Name};
  const PodGang urgent = one("urgent", 2, "high");
  CHECK(!be.SyncPodGang(v2)); CHECK(!be.SyncPodGang(urgent));
  st.clear();
  const auto bound = cycle(&st);
  CHECK(bound.size() == 5);
  // the rolling update: serve-v2 on serve-v1's nodes; serve-v1 is forgotten, not disrupted
  CHECK(st.at(key(v2)).Scheduled && nodesOf("serve-v2") == v1Nodes);
  CHECK(!st.count(key(v1)) || !st.at(key(v1)).DisruptionTarget);
  // the preemption: urgent on batch's nodes; batch is disrupted, naming urgent
  CHECK(st.at(key(urgent)).Scheduled);
  std::set<std::string> urgentNodes = nodesOf("urgent");
  for (const auto& n : urgentNodes) CHECK(batchNodes.count(n));
  CHECK(st.count(key(batch)) && st.at(key(batch)).DisruptionTarget);
  CHECK(st.at(key(batch)).DisruptionMessage.find(key(urgent)) != std::string::npos);
  CHECK(be.Running() == 2 && be.Pending() == 0);   // serve-v2 and urgent
  // the caller deletes the old pods; deleting the forgotten PodGangs releases nothing twice
  CHECK(!be.OnPodGangDelete(v1)); CHECK(!be.OnPodGangDelete(batch));
  CHECK(be.Running() == 2);
}

static void test_old_switches_together_still_fail() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  be.SetPreemption(true); be.SetReservationReuse(true);
  CHECK(!be.SyncPodGang(one("serve-v1", 1, "low")));
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  auto e = be.RunCycle(e2e_nodes(6), &b, &st);
  CHECK(e && e->message.find("reservation reuse") != std::string::npos);
  be.SetReclaimWithReuse(true);   // the combined cycle takes over
  CHECK(!be.RunCycle(e2e_nodes(6), &b, &st));
  CHECK(b.size() == 1 && be.Running() == 1);
}

int main() {
  test_rolling_update_and_preemption();
  test_old_switches_together_still_fail();
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host reuse preempt tests ok\n");
  return 0;
}
