// GpuBackend with queue limits (SetQueue; DESIGN.md section 1 "Queue limits") on cuda:0.  Four nodes of 8 GPUs; queue team-a, a
// child of queue org, may hold 16 GPUs; three one-pod PodGangs of 8 GPUs are labelled kai.scheduler/queue=team-a.  With the queue
// set two are scheduled and the third is Unschedulable with a message that names team-a and GPUs; once one of the two is deleted
// the third is scheduled in the next cycle.  Without a queue all three are scheduled at once.  With preemption on, the members
// stay out of the pass with a reason.
#include <cstdio>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const std::vector<TopologyLevel> kLevels = {{"block", "topology.kubernetes.io/block"}, {"host", "kubernetes.io/hostname"}};

static PodGang gang(const std::string& name) {
  PodGang pg;
  pg.Namespace = "default"; pg.Name = name;
  pg.Labels = {{"grove.io/scheduler-name", GpuBackend::kName}, {GpuBackend::kQueueLabel, "team-a"}};
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

static void with_queue() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  CHECK(!be.SetQueue("org", Queue{}));
  Queue a; a.Parent = "org"; a.Gpu = 16;
  CHECK(!be.SetQueue("team-a", a));
  const PodGang g[3] = {gang("a-0"), gang("a-1"), gang("a-2")};
  for (const PodGang& x : g) CHECK(!be.SyncPodGang(x));
  std::map<std::string, bool> busy;
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(cluster(busy), &b, &st));
  CHECK(b.size() == 2);
  CHECK(st["default/a-0"].Scheduled && st["default/a-1"].Scheduled && !st["default/a-2"].Scheduled);
  const std::string m = st["default/a-2"].ScheduledMessage;
  std::fprintf(stderr, "a-2: %s\n", m.c_str());
  CHECK(st["default/a-2"].ScheduledReason == "Unschedulable");
  CHECK(m.find("queue team-a") != std::string::npos && m.find("GPUs limit 16, load 16") != std::string::npos);
  for (const Binding& x : b) busy[x.NodeName] = true;
  // a-0 leaves: its pod is gone from the snapshot, and team-a has room for a-2 again
  std::string node0;
  for (const Binding& x : b) if (x.PodName == "a-0-w-0") node0 = x.NodeName;
  busy.erase(node0);
  CHECK(!be.OnPodGangDelete(g[0]));
  CHECK(!be.RunCycle(cluster(busy), &b, &st));
  CHECK(b.size() == 1 && st["default/a-2"].Scheduled);
  // refusals: a queue's parent must be set first, a parent cannot be removed
  Queue orphan; orphan.Parent = "nobody";
  CHECK(be.SetQueue("team-b", orphan));
  CHECK(be.SetQueue("org", std::nullopt));
  CHECK(!be.SetQueue("team-a", std::nullopt));
  CHECK(!be.SetQueue("org", std::nullopt));
}

static void without_queue() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  for (const char* n : {"a-0", "a-1", "a-2"}) CHECK(!be.SyncPodGang(gang(n)));
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(cluster({}), &b, &st));
  CHECK(b.size() == 3);
  for (const char* n : {"default/a-0", "default/a-1", "default/a-2"}) CHECK(st[n].Scheduled && st[n].ScheduledMessage.empty());
}

static void members_stay_out_with_preemption() {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  Queue a; a.Gpu = 16;
  CHECK(!be.SetQueue("team-a", a));
  be.SetPreemption(true);
  CHECK(!be.SyncPodGang(gang("a-0")));
  std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
  CHECK(!be.RunCycle(cluster({}), &b, &st));
  CHECK(b.empty() && !st["default/a-0"].Scheduled);
  CHECK(st["default/a-0"].ScheduledMessage.find("queue limits are not applied") == 0);
}

int main() {
  with_queue();
  without_queue();
  members_stay_out_with_preemption();
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host queue tests ok\n");
  return 0;
}
