// GpuBackend with preemption, elastic preemption off and on, on cuda:0.  Two 8-GPU nodes of one block are full: running PodGang A
// holds one with one 8-GPU pod, running PodGang B the other with two 4-GPU pods of a PodGroup with MinReplicas 1, so B's second
// pod is best effort.  Then P, of a higher priority, asks for one 4-GPU pod.  Off: P evicts A or B whole (DisruptionTarget).  On:
// P lands on B's node, B keeps running and is not disrupted, and its status names the pod the caller must terminate in
// EvictedPods; the backend forgets that pod's holdings.
#include <cstdio>
#include <set>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const std::vector<TopologyLevel> kLevels = {{"zone", "topology.kubernetes.io/zone"}, {"block", "topology.kubernetes.io/block"},
                                                   {"rack", "topology.kubernetes.io/rack"}, {"host", "kubernetes.io/hostname"}};

static std::vector<Node> gpu_nodes(int n) {   // one zone, one block, a rack per node
  std::vector<Node> v(n);
  for (int i = 0; i < n; ++i) {
    Node& nd = v[i];
    nd.Name = "gpu-node-" + std::to_string(i);
    nd.Labels = {{"topology.kubernetes.io/zone", "zone-0"}, {"topology.kubernetes.io/block", "block-0"},
                 {"topology.kubernetes.io/rack", "rack-" + std::to_string(i)}, {"kubernetes.io/hostname", nd.Name}};
    nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 524288; nd.alloc_gpu = 8; nd.alloc_pods = 110;
  }
  return v;
}

static PodGang gang(const char* name, int replicas, int minAvailable, uint16_t gpu, const char* priorityClass) {
  PodGang::Requests rq; rq.gpu = gpu;
  PodCliqueSet pcs; pcs.Name = name; pcs.PriorityClassName = priorityClass; pcs.Topology = PackDomain{"host"};
  PodCliqueTemplateSpec c; c.Name = "w"; c.Replicas = replicas; c.MinAvailable = minAvailable; c.Requests = rq;
  pcs.Cliques.push_back(c);
  std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
  CHECK(infos.size() == 1);
  return BuildPodGang(pcs, infos[0]);
}

static std::string key(const PodGang& pg) { return pg.Namespace + "/" + pg.Name; }

static void run(bool elastic) {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  be.SetPriorityClass("low", 0); be.SetPriorityClass("high", 5);
  be.SetPreemption(true); be.SetElasticPreemption(elastic);
  struct Placed { std::string node; uint16_t gpu; };
  std::map<std::string, Placed> pods;   // pods the caller has not terminated
  std::map<std::string, uint16_t> gpuOf;
  auto cycle = [&](std::map<std::string, PodGangStatus>* st) {
    auto nodes = gpu_nodes(2);
    for (const auto& kv : pods) for (auto& nd : nodes) if (nd.Name == kv.second.node) { nd.used_gpu += kv.second.gpu; nd.used_pods += 1; }
    std::vector<Binding> b;
    CHECK(!be.RunCycle(nodes, &b, st));
    for (const auto& x : b) pods[x.PodName] = Placed{x.NodeName, gpuOf.at(x.PodName)};
    return b;
  };
  auto note = [&](const PodGang& pg, uint16_t gpu) { for (const auto& r : pg.Spec.PodGroups[0].PodReferences) gpuOf[r.Name] = gpu; };
  const PodGang A = gang("a", 1, 1, 8, "low"), B = gang("b", 2, 1, 4, "low"), P = gang("p", 1, 1, 4, "high");
  note(A, 8); note(B, 4); note(P, 4);
  std::map<std::string, PodGangStatus> st;
  CHECK(!be.SyncPodGang(A)); CHECK(!be.SyncPodGang(B));
  CHECK(cycle(&st).size() == 3 && be.Running() == 2 && be.Pending() == 0);
  const std::string& b1 = B.Spec.PodGroups[0].PodReferences[1].Name;
  const std::string bNode = pods.at(b1).node;
  CHECK(pods.at(B.Spec.PodGroups[0].PodReferences[0].Name).node == bNode);
  CHECK(!be.SyncPodGang(P));
  st.clear();
  const auto bound = cycle(&st);
  CHECK(bound.size() == 1 && st.at(key(P)).Scheduled);
  if (elastic) {
    CHECK(bound[0].NodeName == bNode);
    CHECK(st.count(key(B)) && !st.at(key(B)).DisruptionTarget && st.at(key(B)).Phase == PodGangPhase::Running);
    CHECK(st.at(key(B)).EvictedPods.size() == 1 && st.at(key(B)).EvictedPods[0].Name == b1);
    CHECK(!st.count(key(A)) || !st.at(key(A)).DisruptionTarget);
    CHECK(be.Running() == 3);
    // the caller terminates the pod; the next cycle sees the node full again and has nothing to do
    pods.erase(b1);
    st.clear();
    CHECK(cycle(&st).empty() && be.Running() == 3);
  } else {
    const bool a = st.count(key(A)) && st.at(key(A)).DisruptionTarget, b = st.count(key(B)) && st.at(key(B)).DisruptionTarget;
    CHECK(a != b);
    const PodGang& victim = a ? A : B;
    CHECK(st.at(key(victim)).DisruptionMessage.find(key(P)) != std::string::npos && st.at(key(victim)).EvictedPods.empty());
    CHECK(be.Running() == 2);
  }
}

int main() {
  run(false);
  run(true);
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host preempt elastic tests ok\n");
  return 0;
}
