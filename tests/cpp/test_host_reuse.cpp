// GpuBackend with reservation reuse (ReuseReservationRef, podgang.go:65-71) on and off, on cuda:0.  Six e2e nodes (one 80 MiB pod
// each) are full with a running PodGang; its new version, of the same size, names it in ReuseReservationRef.  With reuse off the
// new version stays Unschedulable until the old pods are gone; with it on it is admitted onto the old version's nodes at once, the
// old version is forgotten as running, and deleting it afterwards releases nothing twice.  Reuse and preemption together fail.
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

static PodGang one(const char* name, int replicas) {
  PodGang::Requests rq; rq.mem_mib = 80; rq.nodeSelector = {{"node_role.e2e.grove.nvidia.com", "agent"}}; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
  PodCliqueSet pcs; pcs.Name = name;
  PodCliqueTemplateSpec c; c.Name = "w"; c.Replicas = replicas; c.MinAvailable = replicas; c.Requests = rq;
  pcs.Cliques.push_back(c);
  std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
  CHECK(infos.size() == 1);
  return BuildPodGang(pcs, infos[0]);
}

static void test_reuse(bool on) {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  be.SetReservationReuse(on);
  std::map<std::string, std::string> podNode;   // pods the caller has not deleted -> node
  auto cycle = [&](std::map<std::string, PodGangStatus>* st) {
    auto nodes = e2e_nodes(6);
    for (const auto& kv : podNode) for (auto& nd : nodes) if (nd.Name == kv.second) { nd.used_mem_mib += 80; nd.used_pods += 1; }
    std::vector<Binding> b;
    CHECK(!be.RunCycle(nodes, &b, st));
    for (const auto& x : b) podNode[x.PodName] = x.NodeName;
    return b.size();
  };
  std::map<std::string, PodGangStatus> st;
  const PodGang v1 = one("serve-v1", 6);
  CHECK(!be.SyncPodGang(v1));
  CHECK(cycle(&st) == 6 && be.Running() == 1 && be.Pending() == 0);
  std::set<std::string> v1Nodes;
  for (const auto& kv : podNode) v1Nodes.insert(kv.second);
  PodGang v2 = one("serve-v2", 6);
  v2.Spec.ReuseReservationRef = NamespacedName{v1.Namespace, v1.Name};
  CHECK(!be.SyncPodGang(v2));
  const std::string k1 = v1.Namespace + "/" + v1.Name, k2 = v2.Namespace + "/" + v2.Name;
  const size_t bound = cycle(&st);
  if (!on) {
    CHECK(bound == 0 && st.at(k2).ScheduledReason == "Unschedulable" && be.Running() == 1 && be.Pending() == 1);
    return;
  }
  CHECK(bound == 6 && st.at(k2).Scheduled && be.Pending() == 0);
  CHECK(be.Running() == 1);   // v2 runs, v1 is forgotten: the caller deletes its pods
  std::set<std::string> v2Nodes;
  for (const auto& kv : podNode) if (kv.first.find("serve-v2") != std::string::npos) v2Nodes.insert(kv.second);
  CHECK(v2Nodes == v1Nodes);
  CHECK(!be.OnPodGangDelete(v1));
  CHECK(be.Running() == 1 && be.Pending() == 0);
  // preemption and reuse together: the cycle fails
  be.SetPreemption(true);
  CHECK(!be.SyncPodGang(one("serve-extra", 1)));
  std::vector<Binding> b;
  auto e = be.RunCycle(e2e_nodes(6), &b, &st);
  CHECK(e && e->message.find("reservation reuse") != std::string::npos);
}

int main() {
  test_reuse(false);
  test_reuse(true);
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host reuse tests ok\n");
  return 0;
}
