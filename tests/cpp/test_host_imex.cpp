// GpuBackend with ComputeDomain exclusivity (SetComputeDomainExclusivity; DESIGN.md section 1 "ComputeDomain exclusivity") on cuda:0.
// Two 8-GPU nodes; PodCliqueSet replicas r1, r2, r3 of 4 x 1-GPU workers, each enrolled in its own ComputeDomain, and a CPU-only
// PodGang "a-front" that ranks first.  r1 and r2 start their search at the same node.  Off: the engine stacks them on that node,
// where the second IMEX channel would be refused.  On: one node each; r3 stays Unschedulable while both run (the holders come from
// this backend's own bindings: the snapshot reports none), and is scheduled on the node r1 held once r1 is deleted.  A PodGang
// whose PodGroups name two ComputeDomains stays out of the pass with the reason.  The passes run on the one engine handle the
// backend keeps, as the backend does in service; repeated cycles on one handle are a known defect on C4-sized inputs (DESIGN.md
// section 9, item 3), and these passes are a few rows on two nodes whose outcome each check states.
#include <cstdio>
#include <set>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const char* kBlock = "topology.kubernetes.io/block";
static const std::vector<TopologyLevel> kLevels = {{"block", kBlock}, {"host", "kubernetes.io/hostname"}};

static PodGang gang(const std::string& name, int pods, uint16_t gpu, const std::vector<std::string>& cds) {
  PodGang pg;
  pg.Namespace = "default"; pg.Name = name;
  pg.Labels = {{"grove.io/scheduler-name", GpuBackend::kName}};
  for (size_t k = 0; k < cds.size(); ++k) {
    PodGroup g; g.Name = name + "-w" + std::to_string(k); g.MinReplicas = pods;
    for (int i = 0; i < pods; ++i) g.PodReferences.push_back({"default", g.Name + "-" + std::to_string(i)});
    pg.Spec.PodGroups.push_back(g);
    PodGang::Requests rq; rq.gpu = gpu; rq.cpu_milli = 1000; rq.ComputeDomain = cds[k];
    pg.PodGroupRequests[g.Name] = rq;
  }
  return pg;
}

static std::vector<Node> snapshot(const int used[2]) {
  std::vector<Node> nodes(2);
  for (int n = 0; n < 2; ++n) {
    Node& nd = nodes[n];
    nd.Name = "node-0" + std::to_string(n);
    nd.Labels = {{kBlock, "block-0"}, {"kubernetes.io/hostname", nd.Name}};
    nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 1u << 20; nd.alloc_gpu = 8;
    nd.used_gpu = uint16_t(used[n]); nd.used_cpu_milli = uint32_t(used[n]) * 1000;
  }
  return nodes;
}

// one cycle; -> PodGang name -> the nodes its pods were bound to; the used GPUs follow the bindings
static std::map<std::string, std::set<std::string>> cycle(GpuBackend& be, int used[2], std::map<std::string, PodGangStatus>* st) {
  std::vector<Binding> b;
  CHECK(!be.RunCycle(snapshot(used), &b, st));
  std::map<std::string, std::set<std::string>> on;
  for (const Binding& x : b) {
    on[x.PodName.substr(0, x.PodName.find("-w"))].insert(x.NodeName);
    used[x.NodeName == "node-01"] += x.PodName.rfind("a-front", 0) == 0 ? 0 : 1;
  }
  return on;
}

int main() {
  for (bool on : {false, true}) {
    GpuBackend be;
    CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
    be.SetComputeDomainExclusivity(on);
    CHECK(!be.SyncPodGang(gang("a-front", 1, 0, {""})));      // row 0: r1 and r2 (rows 1, 2) both start at the first node
    CHECK(!be.SyncPodGang(gang("r1", 4, 1, {"pcs-0"})));
    CHECK(!be.SyncPodGang(gang("r2", 4, 1, {"pcs-1"})));
    int used[2] = {0, 0};
    std::map<std::string, PodGangStatus> st;
    auto placed = cycle(be, used, &st);
    CHECK(placed["r1"].size() == 1 && placed["r2"].size() == 1);
    if (!on) { CHECK(placed["r1"] == placed["r2"]); continue; }   // stacked: two ComputeDomains on one node
    CHECK(placed["r1"] != placed["r2"]);
    const std::string n1 = *placed["r1"].begin();
    // r3 while r1 and r2 run: both nodes are held (4 GPUs are still free on each), so it waits
    CHECK(!be.SyncPodGang(gang("r3", 4, 1, {"pcs-2"})));
    placed = cycle(be, used, &st);
    CHECK(placed.count("r3") == 0 && st["default/r3"].ScheduledReason == "Unschedulable");
    // r1 is deleted: its pods and its node's IMEX channel go; r3 is scheduled there
    CHECK(!be.OnPodGangDelete(gang("r1", 4, 1, {"pcs-0"})));
    used[n1 == "node-01"] -= 4;
    placed = cycle(be, used, &st);
    CHECK(st["default/r3"].Scheduled && placed["r3"] == std::set<std::string>({n1}));
    // a PodGang with two MNNVL groups stays out of the pass, with the reason
    CHECK(!be.SyncPodGang(gang("two", 1, 1, {"pcs-3", "pcs-4"})));
    placed = cycle(be, used, &st);
    CHECK(placed.count("two") == 0 && st["default/two"].ScheduledReason == "Unschedulable" &&
          st["default/two"].ScheduledMessage.find("two ComputeDomains") != std::string::npos);
  }
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host imex tests ok\n");
  return 0;
}
