// GpuBackend with over-quota weights (SetOverQuotaWeights; DESIGN.md section 1 "Over-quota weight") on cuda:0, the two hand cases of
// tests/over_quota_cases.py with the switch on and off.  team-a and team-b each deserve 8 GPUs, with GPU over-quota weights 3 and 1.
//   Split 3:1 (SetFairShareOrder): six 8-GPU nodes, each team runs one 8-GPU PodGang, then submits four, team-b's of the higher
//   priority.  Fair shares 32 / 16: with the switch on three of team-a's and one of team-b's are scheduled, two and two with it off.
//   Reclaim beyond quota (SetReclaimAcrossQueues): four 8-GPU nodes, team-a runs one PodGang and team-b three, the cluster is full,
//   and team-a submits two.  Fair shares 20 / 12: with the switch on one team-a PodGang is scheduled and one team-b PodGang gets
//   DisruptionTarget; with it off team-a is at its quota and nothing moves.
#include <cstdio>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const std::vector<TopologyLevel> kLevels = {{"block", "topology.kubernetes.io/block"}, {"host", "kubernetes.io/hostname"}};

static PodGang gang(const std::string& name, const std::string& queue, const std::string& priorityClass) {
  PodGang pg;
  pg.Namespace = "default"; pg.Name = name;
  pg.Labels = {{"grove.io/scheduler-name", GpuBackend::kName}, {GpuBackend::kQueueLabel, queue}};
  pg.Spec.PriorityClassName = priorityClass;
  PodGroup g; g.Name = name + "-w"; g.MinReplicas = 1;
  g.PodReferences.push_back({"default", g.Name + "-0"});
  pg.Spec.PodGroups = {g};
  PodGang::Requests rq; rq.gpu = 8;
  pg.PodGroupRequests[g.Name] = rq;
  return pg;
}

static std::vector<Node> cluster(int n_nodes, const std::map<std::string, bool>& busy) {
  std::vector<Node> nodes(n_nodes);
  for (int n = 0; n < n_nodes; ++n) {
    Node& nd = nodes[n];
    nd.Name = "node-" + std::to_string(n);
    nd.Labels = {{"topology.kubernetes.io/block", "block-0"}, {"kubernetes.io/hostname", nd.Name}};
    nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 1u << 20; nd.alloc_gpu = 8;
    if (busy.count(nd.Name)) nd.used_gpu = 8;
  }
  return nodes;
}

static void teams(GpuBackend& be) {
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  be.SetPriorityClass("low", 0); be.SetPriorityClass("high", 10);
  Queue a, b;
  a.DeservedGpu = 8; b.DeservedGpu = 8;
  a.OverQuotaWeightGpu = 3;   // (cpu and memory: nullopt = 1)
  CHECK(!be.SetQueue("team-a", a)); CHECK(!be.SetQueue("team-b", b));
}

// -> how many of team-a's and team-b's new PodGangs the contested fair-share cycle schedules
static std::pair<int, int> split(bool weights) {
  GpuBackend be;
  teams(be);
  be.SetFairShareOrder(true);
  be.SetOverQuotaWeights(weights);
  CHECK(!be.SyncPodGang(gang("a-run", "team-a", "low"))); CHECK(!be.SyncPodGang(gang("b-run", "team-b", "high")));
  std::map<std::string, bool> busy;
  std::vector<Binding> bd; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(cluster(6, busy), &bd, &st));
  CHECK(bd.size() == 2);
  for (const Binding& x : bd) busy[x.NodeName] = true;
  for (int i = 0; i < 4; ++i) {
    CHECK(!be.SyncPodGang(gang("a-" + std::to_string(i), "team-a", "low")));
    CHECK(!be.SyncPodGang(gang("b-" + std::to_string(i), "team-b", "high")));
  }
  CHECK(!be.RunCycle(cluster(6, busy), &bd, &st));
  CHECK(bd.size() == 4);
  std::pair<int, int> got{0, 0};
  for (int i = 0; i < 4; ++i) {
    got.first += st["default/a-" + std::to_string(i)].Scheduled;
    got.second += st["default/b-" + std::to_string(i)].Scheduled;
  }
  const auto fs = be.FairShares();
  if (weights) CHECK(fs.size() == 2 && fs.at("team-a")[2] == 32 && fs.at("team-b")[2] == 16 && fs.at("team-a")[0] == GROVE_QUEUE_UNLIMITED);
  else CHECK(fs.empty());
  return got;
}

// -> (team-a PodGangs scheduled, team-b PodGangs disrupted) in the contested reclaim cycle
static std::pair<int, int> reclaim(bool weights) {
  GpuBackend be;
  teams(be);
  be.SetOverQuotaWeights(weights);
  CHECK(!be.SyncPodGang(gang("a-run", "team-a", "low")));
  for (const char* n : {"b-r0", "b-r1", "b-r2"}) CHECK(!be.SyncPodGang(gang(n, "team-b", "low")));
  std::map<std::string, bool> busy;
  std::vector<Binding> bd; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(cluster(4, busy), &bd, &st));
  CHECK(bd.size() == 4);
  for (const Binding& x : bd) busy[x.NodeName] = true;
  be.SetReclaimAcrossQueues(true);
  for (const char* n : {"a-0", "a-1"}) CHECK(!be.SyncPodGang(gang(n, "team-a", "low")));
  CHECK(!be.RunCycle(cluster(4, busy), &bd, &st));
  std::pair<int, int> got{0, 0};
  for (const char* n : {"default/a-0", "default/a-1"}) got.first += st.count(n) && st[n].Scheduled;
  for (const char* n : {"default/b-r0", "default/b-r1", "default/b-r2"}) got.second += st.count(n) && st[n].DisruptionTarget;
  CHECK(int(bd.size()) == got.first);
  const auto fs = be.FairShares();
  if (weights) CHECK(fs.size() == 2 && fs.at("team-a")[2] == 20 && fs.at("team-b")[2] == 12);
  else CHECK(fs.empty());
  return got;
}

int main() {
  CHECK((split(true) == std::pair<int, int>{3, 1}));
  CHECK((split(false) == std::pair<int, int>{2, 2}));
  CHECK((reclaim(true) == std::pair<int, int>{1, 1}));
  CHECK((reclaim(false) == std::pair<int, int>{0, 0}));
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host over-quota tests ok\n");
  return 0;
}
