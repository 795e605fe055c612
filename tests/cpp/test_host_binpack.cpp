// GpuBackend with bin-packing (SetBinPacking; DESIGN.md section 1 "Bin-packing") on cuda:0.  Four blocks of 8 nodes of 8 GPUs, two
// cycles.  Cycle 1: eight one-pod PodGangs of 8 GPUs packed in a block.  Cycle 2: "a-big" (8 pods of 8 GPUs packed in a block, a
// higher priority) and eight more one-pod PodGangs.  With bin-packing off the hash anchors leave a small PodGang in every block and
// a-big is not scheduled; with it on at block level the first eight fill block 0 and a-big is scheduled in one of the empty blocks.
#include <cstdio>
#include <set>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const char* kBlock = "topology.kubernetes.io/block";
static const std::vector<TopologyLevel> kLevels = {{"block", kBlock}, {"host", "kubernetes.io/hostname"}};

static std::string node_name(int i) { char b[16]; std::snprintf(b, sizeof b, "node-%02d", i); return b; }

static PodGang gang(const std::string& name, int pods, const std::string& priority) {
  PodGang pg;
  pg.Namespace = "default"; pg.Name = name;
  pg.Labels = {{"grove.io/scheduler-name", GpuBackend::kName}};
  PodGroup g; g.Name = name + "-w"; g.MinReplicas = pods;
  for (int i = 0; i < pods; ++i) g.PodReferences.push_back({"default", g.Name + "-" + std::to_string(i)});
  pg.Spec.PodGroups = {g};
  pg.Spec.Topology = TopologyConstraint{TopologyPackConstraint{std::string(kBlock), std::nullopt}};
  if (!priority.empty()) pg.Spec.PriorityClassName = priority;
  PodGang::Requests rq; rq.gpu = 8;
  pg.PodGroupRequests[g.Name] = rq;
  return pg;
}

// -> blocks the first cycle bound pods in; *big = a-big was scheduled in cycle 2
static std::set<int> run(bool binpack, bool* big) {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  be.SetPriorityClass("high", 10);
  if (binpack) be.SetBinPacking(kBlock);
  std::vector<int> used(32, 0);
  std::set<int> blocks;
  for (int cyc = 0; cyc < 2; ++cyc) {
    if (cyc == 1) CHECK(!be.SyncPodGang(gang("a-big", 8, "high")));
    for (int i = 0; i < 8; ++i) CHECK(!be.SyncPodGang(gang("s-" + std::to_string(cyc) + "-" + std::to_string(10 + i), 1, "")));
    std::vector<Node> nodes(32);
    for (int n = 0; n < 32; ++n) {
      Node& nd = nodes[n];
      nd.Name = node_name(n);
      nd.Labels = {{kBlock, "block-" + std::to_string(n / 8)}, {"kubernetes.io/hostname", nd.Name}};
      nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 1u << 20; nd.alloc_gpu = 8;
      nd.used_gpu = used[n];
    }
    std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
    CHECK(!be.RunCycle(nodes, &b, &st));
    for (const Binding& x : b) {
      const int n = std::stoi(x.NodeName.substr(5));
      used[n] = 8;
      if (cyc == 0) blocks.insert(n / 8);
    }
    if (cyc == 1) *big = st["default/a-big"].Scheduled;
  }
  return blocks;
}

int main() {
  bool big = true;
  CHECK(run(false, &big) == std::set<int>({0, 1, 2, 3}));   // the hash anchors scatter the small PodGangs
  CHECK(!big);
  big = false;
  CHECK(run(true, &big) == std::set<int>({0}));
  CHECK(big);
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host binpack tests ok\n");
  return 0;
}
