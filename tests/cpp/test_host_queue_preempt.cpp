// GpuBackend with preemption within queue limits (SetPreemptionWithinQueues; DESIGN.md section 1 "Reclaim within queue limits")
// on cuda:0.  Four nodes of 8 GPUs; queue team-a may hold 16 GPUs and two low-priority one-pod PodGangs of 8 GPUs hold them.  A
// high-priority PodGang of team-a arrives.  With preemption on and the switch off it stays out of the pass with the existing
// reason; with the switch on it is scheduled and exactly one team-a PodGang gets DisruptionTarget naming it.
#include <cstdio>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const std::vector<TopologyLevel> kLevels = {{"block", "topology.kubernetes.io/block"}, {"host", "kubernetes.io/hostname"}};

static PodGang gang(const std::string& name, const std::string& priorityClass) {
  PodGang pg;
  pg.Namespace = "default"; pg.Name = name;
  pg.Labels = {{"grove.io/scheduler-name", GpuBackend::kName}, {GpuBackend::kQueueLabel, "team-a"}};
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

static void team_a() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  be.SetPriorityClass("low", 0); be.SetPriorityClass("high", 10);
  Queue a; a.Gpu = 16;
  CHECK(!be.SetQueue("team-a", a));
  for (const char* n : {"a-0", "a-1"}) CHECK(!be.SyncPodGang(gang(n, "low")));
  std::map<std::string, bool> busy;
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(cluster(busy), &b, &st));
  CHECK(b.size() == 2);
  std::map<std::string, std::string> first;   // node -> the PodGang on it
  for (const Binding& x : b) { busy[x.NodeName] = true; first[x.NodeName] = "default/" + x.PodName.substr(0, 3); }
  be.SetPreemption(true);
  CHECK(!be.SyncPodGang(gang("a-hi", "high")));
  // the switch off: the member stays out of a pass with preemption
  CHECK(!be.RunCycle(cluster(busy), &b, &st));
  CHECK(b.empty() && !st["default/a-hi"].Scheduled);
  CHECK(st["default/a-hi"].ScheduledMessage.find("queue limits are not applied") == 0);
  // the switch on: scheduled, and exactly one team-a PodGang makes room in the queue; the other keeps its node
  be.SetPreemptionWithinQueues(true);
  CHECK(!be.RunCycle(cluster(busy), &b, &st));
  CHECK(b.size() == 1 && st["default/a-hi"].Scheduled);
  int disrupted = 0;
  for (const char* n : {"default/a-0", "default/a-1"})
    if (st.count(n) && st[n].DisruptionTarget) {
      ++disrupted;
      std::fprintf(stderr, "%s: %s\n", n, st[n].DisruptionMessage.c_str());
      CHECK(st[n].DisruptionMessage.find("default/a-hi") != std::string::npos);
    }
  CHECK(disrupted == 1);
  std::string kept;   // the node of the team-a PodGang that still runs
  for (const auto& [node, on] : first) if (!(st.count(on) && st[on].DisruptionTarget)) kept = node;
  CHECK(!kept.empty() && b.size() == 1 && b[0].NodeName != kept);
}

static void reuse_keeps_members_out() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  Queue a; a.Gpu = 16;
  CHECK(!be.SetQueue("team-a", a));
  be.SetPreemptionWithinQueues(true);
  be.SetReclaimWithReuse(true);
  CHECK(!be.SyncPodGang(gang("a-0", "")));
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(cluster({}), &b, &st));
  CHECK(b.empty() && st["default/a-0"].ScheduledMessage.find("queue limits are not applied") == 0);
}

int main() {
  team_a();
  reuse_keeps_members_out();
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host queue preemption tests ok\n");
  return 0;
}
