// GpuBackend with large PodGangs (SetLargePodGangs) off and on, on cuda:0.  The PodGang is workload1's base PodGang with 300
// more pods in PodGroup pc-a (310 pods, the one test_host.cpp shows being skipped); a second variant also asks for 260 of them
// as MinReplicas.  With the switch off it stays Unschedulable with the old reason; with it on it is scheduled and its bindings
// count its MinReplicas plus the surplus the nodes take; with preemption on as well it is skipped with a reason that says so.
#include <cstdio>
#include <map>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const std::vector<TopologyLevel> kLevels = {{"zone", "topology.kubernetes.io/zone"}, {"block", "topology.kubernetes.io/block"},
                                                   {"rack", "topology.kubernetes.io/rack"}, {"host", "kubernetes.io/hostname"}};

// hack/e2e.yaml's layout (zone 28 / block 14 / rack 7 / host), with room for `perNode` 80 MiB pods per node
static std::vector<Node> nodes(int n, int perNode) {
  std::vector<Node> v(n);
  for (int i = 0; i < n; ++i) {
    Node& nd = v[i];
    nd.Name = "kwok-node-" + std::to_string(i);
    nd.Labels = {{"topology.kubernetes.io/zone", "zone-" + std::to_string(i / 28)}, {"topology.kubernetes.io/block", "block-" + std::to_string(i / 14)},
                 {"topology.kubernetes.io/rack", "rack-" + std::to_string(i / 7)}, {"kubernetes.io/hostname", nd.Name},
                 {"node_role.e2e.grove.nvidia.com", "agent"}};
    nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 80u * uint32_t(perNode) + 70u; nd.alloc_pods = 110;
    nd.TaintKeys = {"node_role.e2e.grove.nvidia.com"};
  }
  return v;
}

static PodCliqueSet workload1(int pcaReplicas) {  // e2e/yaml/workload1.yaml, pc-a widened
  PodCliqueSet pcs; pcs.Name = "workload1";
  PodGang::Requests rq; rq.mem_mib = 80; rq.nodeSelector = {{"node_role.e2e.grove.nvidia.com", "agent"}}; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
  for (auto [n, r] : std::vector<std::pair<const char*, int>>{{"pc-a", pcaReplicas}, {"pc-b", 1}, {"pc-c", 3}}) {
    PodCliqueTemplateSpec c; c.Name = n; c.Replicas = r; c.MinAvailable = r; c.Requests = rq; pcs.Cliques.push_back(c);
  }
  PodCliqueScalingGroupConfig g; g.Name = "sg-x"; g.Replicas = 2; g.MinAvailable = 2; g.CliqueNames = {"pc-b", "pc-c"};
  pcs.PodCliqueScalingGroupConfigs = {g};
  pcs.Topology = PackDomain{"block"};
  return pcs;
}

// workload1's base PodGang with 300 more pods in pc-a (MinReplicas `mn` of its 302)
static PodGang huge(int mn) {
  PodCliqueSet pcs = workload1(2);
  std::vector<PodGangInfo> infos; CHECK(!ComputeExpectedPodGangs(pcs, kLevels, true, &infos));
  PodGang pg = BuildPodGang(pcs, infos[0]);
  pg.Name = "huge";
  for (int i = 0; i < 300; ++i) pg.Spec.PodGroups[0].PodReferences.push_back({"default", "huge-pc-a-" + std::to_string(i)});
  pg.Spec.PodGroups[0].MinReplicas = mn;
  return pg;
}

static std::map<std::string, int> perGroup(const std::vector<Binding>& b) {
  std::map<std::string, int> n;
  for (const auto& x : b) n[x.PodName.find("pc-a") != std::string::npos ? "pc-a" : "other"]++;
  return n;
}

static void test_off() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  const PodGang pg = huge(2);
  CHECK(GpuBackend::WhyNotEncodable(pg) == GpuBackend::WhyNotEncodable(pg, false) && !GpuBackend::WhyNotEncodable(pg).empty());
  CHECK(GpuBackend::WhyNotEncodable(pg, true).empty());
  CHECK(!be.SyncPodGang(pg));
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(nodes(28, 40), &b, &st));
  CHECK(b.empty() && st.at("default/huge").ScheduledReason == "Unschedulable");
  CHECK(st.at("default/huge").ScheduledMessage.find("more than 255 pods") != std::string::npos);
  CHECK(be.ValidatePodCliqueSet(workload1(200)).has_value());   // a 208-pod base PodGang exceeds 128
}

static void test_on(int mn, int perNode, size_t want, int wantPca) {
  GpuBackend be;
  be.SetLargePodGangs(true);
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  CHECK(!be.ValidatePodCliqueSet(workload1(200)));
  CHECK(be.ValidatePodCliqueSet(workload1(2100)).has_value());
  const PodGang pg = huge(mn);
  CHECK(!be.SyncPodGang(pg));
  Tables t;
  CHECK(!be.Encode(nodes(28, perNode), &t));
  CHECK(t.skipped.empty() && t.gangs.size() == 1 && t.counts.size() == t.cliques.size());
  CHECK(t.counts[0].replicas == 302 && t.counts[0].min_replicas == mn);
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(nodes(28, perNode), &b, &st));
  const PodGangStatus& s = st.at("default/huge");
  CHECK(s.Scheduled);
  CHECK(b.size() == want);
  const auto n = perGroup(b);
  CHECK(n.count("pc-a") && n.at("pc-a") == wantPca && n.at("other") == 8 && n.at("pc-a") >= mn);
  if (g_fail) std::fprintf(stderr, "  in test_on(%d, %d): %zu bindings, pc-a %d\n", mn, perNode, b.size(), n.count("pc-a") ? n.at("pc-a") : 0);
}

static void test_on_with_preemption() {
  GpuBackend be;
  be.SetLargePodGangs(true);
  be.SetPreemption(true);
  CHECK(!be.SyncTopology(kLevels));
  CHECK(!be.Init());
  CHECK(!be.SyncPodGang(huge(2)));
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(nodes(28, 40), &b, &st));
  CHECK(b.empty() && st.at("default/huge").ScheduledReason == "Unschedulable");
  CHECK(st.at("default/huge").ScheduledMessage.find("not scheduled while preemption") != std::string::npos);
}

int main() {
  test_off();
  // the gang is Required to one block (14 nodes): 40 pods a node hold all 310 pods; 20 a node hold 280 -- every MinReplicas
  // plus what the block has room for of pc-a's surplus
  test_on(2, 40, 310, 302);
  test_on(260, 40, 310, 302);
  test_on(260, 20, 280, 272);
  test_on_with_preemption();
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host large tests ok\n");
  return 0;
}
