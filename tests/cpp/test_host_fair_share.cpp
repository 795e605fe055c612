// GpuBackend with the fair-share order (SetFairShareOrder; DESIGN.md section 1 "Fair-share order") on cuda:0.  Four nodes of 8
// GPUs: team-b deserves 16 GPUs and already runs two 8-GPU PodGangs on two of them; team-a deserves 16 and holds none.  Each team
// then has two pending 8-GPU PodGangs, team-b's of the higher priority, for the two free nodes.  With the switch off team-b's are
// scheduled (priority decides); with it on team-a's are (team-a is furthest below its quota at every turn).
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

static std::vector<Node> cluster(const std::map<std::string, bool>& busy) {
  std::vector<Node> nodes(4);
  for (int n = 0; n < 4; ++n) {
    Node& nd = nodes[n];
    nd.Name = "node-" + std::to_string(n);
    nd.Labels = {{"topology.kubernetes.io/block", "block-0"}, {"kubernetes.io/hostname", nd.Name}};
    nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 1u << 20; nd.alloc_gpu = 8;
    if (busy.count(nd.Name)) nd.used_gpu = 8;
  }
  return nodes;
}

// -> the PodGangs scheduled in the contested cycle
static std::vector<std::string> contested(bool fair) {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  be.SetPriorityClass("low", 0); be.SetPriorityClass("high", 10);
  be.SetFairShareOrder(fair);
  Queue a, b;
  a.DeservedGpu = 16; b.DeservedGpu = 16;
  CHECK(!be.SetQueue("team-a", a)); CHECK(!be.SetQueue("team-b", b));
  // team-b's running PodGangs: scheduled by this backend, so they count in team-b's load
  for (const char* n : {"b-0", "b-1"}) CHECK(!be.SyncPodGang(gang(n, "team-b", "high")));
  std::map<std::string, bool> busy;
  std::vector<Binding> bd; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(cluster(busy), &bd, &st));
  CHECK(bd.size() == 2);
  for (const Binding& x : bd) busy[x.NodeName] = true;
  CHECK(busy.size() == 2);
  for (const char* n : {"a-0", "a-1"}) CHECK(!be.SyncPodGang(gang(n, "team-a", "low")));
  for (const char* n : {"b-2", "b-3"}) CHECK(!be.SyncPodGang(gang(n, "team-b", "high")));
  CHECK(!be.RunCycle(cluster(busy), &bd, &st));
  CHECK(bd.size() == 2);
  std::vector<std::string> got;
  for (const char* n : {"default/a-0", "default/a-1", "default/b-2", "default/b-3"})
    if (st.count(n) && st[n].Scheduled) got.push_back(n);
  return got;
}

int main() {
  const std::vector<std::string> off = contested(false), on = contested(true);
  CHECK((off == std::vector<std::string>{"default/b-2", "default/b-3"}));
  CHECK((on == std::vector<std::string>{"default/a-0", "default/a-1"}));
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host fair share tests ok\n");
  return 0;
}
