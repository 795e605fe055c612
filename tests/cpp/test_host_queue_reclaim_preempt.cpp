// GpuBackend with reclaim, then preempt (SetReclaimThenPreempt; DESIGN.md section 1 "Reclaim, then preempt") on cuda:0.  Three
// full nodes of 8 GPUs.  team-b (quota 8) runs b-0 and b-1 at priority 5; team-c (limit 8, quota 8) runs c-low at priority 0;
// team-a (quota 8) holds nothing.  team-a submits a-0 (priority 0), team-c c-high (priority 9, only on c-low's node).  Reclaim
// across queues alone schedules a-0, preemption within queues alone c-high; with the new switch both are scheduled, and b-1 and
// c-low get DisruptionTarget naming their evictor.
#include <cstdio>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const std::vector<TopologyLevel> kLevels = {{"block", "topology.kubernetes.io/block"}, {"host", "kubernetes.io/hostname"}};

static const char* kPool = "pool";   // the selector-class label: one value per node

static PodGang gang(const std::string& name, const std::string& queue, const std::string& priorityClass, const std::string& pool = "") {
  PodGang pg;
  pg.Namespace = "default"; pg.Name = name;
  pg.Labels = {{"grove.io/scheduler-name", GpuBackend::kName}, {GpuBackend::kQueueLabel, queue}};
  pg.Spec.PriorityClassName = priorityClass;
  PodGroup g; g.Name = name + "-w"; g.MinReplicas = 1;
  g.PodReferences.push_back({"default", g.Name + "-0"});
  pg.Spec.PodGroups = {g};
  PodGang::Requests rq; rq.gpu = 8;
  if (!pool.empty()) rq.nodeSelector = {{kPool, pool}};
  pg.PodGroupRequests[g.Name] = rq;
  return pg;
}

static std::vector<Node> cluster(const std::map<std::string, bool>& busy) {
  std::vector<Node> nodes(3);
  for (int n = 0; n < 3; ++n) {
    Node& nd = nodes[n];
    nd.Name = "node-" + std::to_string(n);
    nd.Labels = {{"topology.kubernetes.io/block", "block-0"}, {"kubernetes.io/hostname", nd.Name}, {kPool, "pool-" + std::to_string(n)}};
    nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 1u << 20; nd.alloc_gpu = 8;
    if (busy.count(nd.Name)) nd.used_gpu = 8;
  }
  return nodes;
}

// 0: SetReclaimAcrossQueues only, 1: SetPreemptionWithinQueues only, 2: SetReclaimThenPreempt (with both older switches on too)
static void three_teams(int mode) {
  GpuBackend be(0, kPool);
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  be.SetPriorityClass("low", 0); be.SetPriorityClass("mid", 5); be.SetPriorityClass("high", 9);
  be.SetPreemption(true);
  Queue a, b, c;
  a.DeservedGpu = 8; b.DeservedGpu = 8; c.DeservedGpu = 8; c.Gpu = 8;
  CHECK(!be.SetQueue("team-a", a)); CHECK(!be.SetQueue("team-b", b)); CHECK(!be.SetQueue("team-c", c));
  if (mode == 0) be.SetReclaimAcrossQueues(true);
  if (mode == 1) be.SetPreemptionWithinQueues(true);
  if (mode == 2) { be.SetReclaimAcrossQueues(true); be.SetPreemptionWithinQueues(true); be.SetReclaimThenPreempt(true); }
  // the running PodGangs, one cycle each so that c-low lands on the last free node
  std::map<std::string, bool> busy;
  std::vector<Binding> bd; std::map<std::string, PodGangStatus> st;
  std::string cNode;
  for (auto [n, q, p] : {std::tuple{"b-0", "team-b", "mid"}, {"b-1", "team-b", "mid"}, {"c-low", "team-c", "low"}}) {
    CHECK(!be.SyncPodGang(gang(n, q, p)));
    CHECK(!be.RunCycle(cluster(busy), &bd, &st));
    CHECK(bd.size() == 1);
    for (const Binding& x : bd) { busy[x.NodeName] = true; if (std::string(n) == "c-low") cNode = x.NodeName; }
  }
  CHECK(busy.size() == 3);
  CHECK(!be.SyncPodGang(gang("a-0", "team-a", "low")));
  CHECK(!be.SyncPodGang(gang("c-high", "team-c", "high", "pool-" + cNode.substr(cNode.size() - 1))));
  CHECK(!be.RunCycle(cluster(busy), &bd, &st));
  const bool a0 = st["default/a-0"].Scheduled, cHigh = st["default/c-high"].Scheduled;
  std::fprintf(stderr, "mode %d: a-0 %d, c-high %d, %zu bindings\n", mode, int(a0), int(cHigh), bd.size());
  for (const char* n : {"default/b-0", "default/b-1", "default/c-low"})
    if (st.count(n) && st[n].DisruptionTarget) std::fprintf(stderr, "  %s: %s\n", n, st[n].DisruptionMessage.c_str());
  auto disrupted = [&](const char* n) { return st.count(n) && st[n].DisruptionTarget; };
  if (mode == 0) CHECK(a0 && !cHigh && bd.size() == 1);
  if (mode == 1) CHECK(!a0 && cHigh && bd.size() == 1);
  if (mode == 2) {
    CHECK(a0 && cHigh && bd.size() == 2);
    CHECK(!disrupted("default/b-0") && disrupted("default/b-1") && disrupted("default/c-low"));
    CHECK(st["default/b-1"].DisruptionMessage.find("reclaimed by PodGang default/a-0 of queue team-a") != std::string::npos);
    CHECK(st["default/c-low"].DisruptionMessage.find("preempted by higher priority PodGang default/c-high") != std::string::npos);
    for (const Binding& x : bd)
      if (x.PodName.rfind("c-high", 0) == 0) CHECK(x.NodeName == cNode);
  }
}

int main() {
  for (int mode = 0; mode < 3; ++mode) three_teams(mode);
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host queue reclaim-then-preempt tests ok\n");
  return 0;
}
