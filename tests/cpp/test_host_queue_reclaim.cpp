// GpuBackend with reclaim across queues (SetReclaimAcrossQueues; DESIGN.md section 1 "Reclaim across queues") on cuda:0.  Two
// nodes of 8 GPUs, full: team-b deserves 8 GPUs and runs two high-priority 8-GPU PodGangs; team-a deserves 8 and holds none.  A
// low-priority 8-GPU PodGang of team-a arrives.  With the switch off it stays Unschedulable; with it on it is scheduled and one
// team-b PodGang gets DisruptionTarget naming it and its queue.  A second team-a PodGang then stays pending: both teams are at
// their quota.
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
  std::vector<Node> nodes(2);
  for (int n = 0; n < 2; ++n) {
    Node& nd = nodes[n];
    nd.Name = "node-" + std::to_string(n);
    nd.Labels = {{"topology.kubernetes.io/block", "block-0"}, {"kubernetes.io/hostname", nd.Name}};
    nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 1u << 20; nd.alloc_gpu = 8;
    if (busy.count(nd.Name)) nd.used_gpu = 8;
  }
  return nodes;
}

static void starved_team() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  be.SetPriorityClass("low", 0); be.SetPriorityClass("high", 10);
  Queue a, b;
  a.DeservedGpu = 8; b.DeservedGpu = 8;
  CHECK(!be.SetQueue("team-a", a)); CHECK(!be.SetQueue("team-b", b));
  for (const char* n : {"b-0", "b-1"}) CHECK(!be.SyncPodGang(gang(n, "team-b", "high")));
  std::map<std::string, bool> busy;
  std::vector<Binding> bd; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(cluster(busy), &bd, &st));
  CHECK(bd.size() == 2);
  for (const Binding& x : bd) busy[x.NodeName] = true;
  CHECK(!be.SyncPodGang(gang("a-0", "team-a", "low")));
  // the switch off: the cluster is full and team-a's PodGang outranks nobody
  CHECK(!be.RunCycle(cluster(busy), &bd, &st));
  CHECK(bd.empty() && !st["default/a-0"].Scheduled);
  // the switch on: scheduled, and one team-b PodGang makes room although it outranks the reclaimer
  be.SetReclaimAcrossQueues(true);
  CHECK(!be.RunCycle(cluster(busy), &bd, &st));
  CHECK(bd.size() == 1 && st["default/a-0"].Scheduled);
  int disrupted = 0;
  for (const char* n : {"default/b-0", "default/b-1"})
    if (st.count(n) && st[n].DisruptionTarget) {
      ++disrupted;
      std::fprintf(stderr, "%s: %s\n", n, st[n].DisruptionMessage.c_str());
      CHECK(st[n].DisruptionMessage.find("default/a-0") != std::string::npos);
      CHECK(st[n].DisruptionMessage.find("team-a") != std::string::npos);
    }
  CHECK(disrupted == 1);
  // the victim's pods are deleted and a-0 runs on its node: both teams hold their quota of 8, a second team-a PodGang waits
  CHECK(!be.SyncPodGang(gang("a-1", "team-a", "low")));
  CHECK(!be.RunCycle(cluster(busy), &bd, &st));
  CHECK(bd.empty() && !st["default/a-1"].Scheduled);
  for (const char* n : {"default/b-0", "default/b-1"}) CHECK(!(st.count(n) && st[n].DisruptionTarget));
}

static void not_with_preemption_within_queues() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  Queue a; a.DeservedGpu = 8;
  CHECK(!be.SetQueue("team-a", a));
  be.SetReclaimAcrossQueues(true);
  be.SetPreemptionWithinQueues(true);
  CHECK(!be.SyncPodGang(gang("a-0", "team-a", "")));
  std::vector<Binding> bd; std::map<std::string, PodGangStatus> st;
  CHECK(be.RunCycle(cluster({}), &bd, &st).has_value());
}

int main() {
  starved_team();
  not_with_preemption_within_queues();
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host queue reclaim tests ok\n");
  return 0;
}
