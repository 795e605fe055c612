// GpuBackend with the starvation guard (SetStarvationGuard; DESIGN.md section 1 "Fences") on cuda:0.  Four blocks of 8 nodes of
// 8 GPUs; when the first cycle starts every node but the last of each block runs a one-node pod of another tenant, which leaves in
// cycle 1 or 2.  Every cycle 14 one-pod PodGangs of 8 GPUs (no pack constraint) arrive and each runs two cycles once bound; those
// not bound are withdrawn.  PodGang "a-big" (8 pods of 8 GPUs packed in a block) ranks first at equal priority.  With the guard off
// the freed nodes are always taken by the small PodGangs and a-big is never scheduled in 20 cycles; with the guard on after one
// rejected cycle it fences a block, is scheduled in the third cycle, and the cycle in between carries the message that names it.
#include <cstdio>
#include <set>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static const char* kBlock = "topology.kubernetes.io/block";
static const std::vector<TopologyLevel> kLevels = {{"block", kBlock}, {"host", "kubernetes.io/hostname"}};

static std::string node_name(int i) { char b[16]; std::snprintf(b, sizeof b, "node-%02d", i); return b; }

static PodGang gang(const std::string& name, int pods, bool packed) {
  PodGang pg;
  pg.Namespace = "default"; pg.Name = name;
  pg.Labels = {{"grove.io/scheduler-name", GpuBackend::kName}};
  PodGroup g; g.Name = name + "-w"; g.MinReplicas = pods;
  for (int i = 0; i < pods; ++i) g.PodReferences.push_back({"default", g.Name + "-" + std::to_string(i)});
  pg.Spec.PodGroups = {g};
  if (packed) pg.Spec.Topology = TopologyConstraint{TopologyPackConstraint{std::string(kBlock), std::nullopt}};
  PodGang::Requests rq; rq.gpu = 8;
  pg.PodGroupRequests[g.Name] = rq;
  return pg;
}

// -> the cycle a-big was scheduled in (-1: never); messages[c] = a-big's ScheduledMessage in cycle c
static int run(bool guard, std::vector<std::string>* messages) {
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  if (guard) CHECK(!be.SetStarvationGuard(1, 1));
  std::vector<int> busyUntil(32, 0);
  for (int n = 0; n < 32; ++n) if (n % 8 != 7) busyUntil[n] = 1 + (n % 3 == 0);
  std::map<std::string, std::pair<int, PodGang>> small;   // bound small PodGang -> (cycle it leaves, its PodGang)
  CHECK(!be.SyncPodGang(gang("a-big", 8, true)));
  for (int cyc = 0; cyc < 20; ++cyc) {
    for (auto it = small.begin(); it != small.end();)
      if (it->second.first == cyc) { CHECK(!be.OnPodGangDelete(it->second.second)); it = small.erase(it); } else ++it;
    std::vector<PodGang> arrived;
    for (int i = 0; i < 14; ++i) { arrived.push_back(gang("s-" + std::to_string(100 + cyc) + "-" + std::to_string(10 + i), 1, false)); CHECK(!be.SyncPodGang(arrived.back())); }
    std::vector<Node> nodes(32);
    for (int n = 0; n < 32; ++n) {
      Node& nd = nodes[n];
      nd.Name = node_name(n);
      nd.Labels = {{kBlock, "block-" + std::to_string(n / 8)}, {"kubernetes.io/hostname", nd.Name}};
      nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 1u << 20; nd.alloc_gpu = 8;
      if (busyUntil[n] > cyc) nd.used_gpu = 8;
    }
    std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
    CHECK(!be.RunCycle(nodes, &b, &st));
    messages->push_back(st["default/a-big"].ScheduledMessage);
    if (st["default/a-big"].Scheduled) return cyc;
    for (const Binding& x : b) {
      const std::string pg = x.PodName.substr(0, x.PodName.size() - std::string("-w-0").size());
      busyUntil[std::stoi(x.NodeName.substr(5))] = cyc + 2;
      for (const PodGang& a : arrived) if (a.Name == pg) small[pg] = {cyc + 2, a};
    }
    for (const PodGang& a : arrived) if (!small.count(a.Name)) CHECK(!be.OnPodGangDelete(a));   // not bound: withdrawn
  }
  return -1;
}

int main() {
  std::vector<std::string> off, on;
  CHECK(run(false, &off) == -1);
  for (const auto& m : off) CHECK(m.find("held for this PodGang") == std::string::npos);
  const int at = run(true, &on);
  CHECK(at == 2);
  CHECK(on.size() == 3 && on[0].find("held for this PodGang") == std::string::npos);
  if (on.size() == 3) {
    std::fprintf(stderr, "cycle 1: %s\n", on[1].c_str());
    CHECK(on[1].find("Unschedulable for 2 cycles in a row: block block-") == 0 && on[1].find("held for this PodGang") != std::string::npos);
  }
  GpuBackend be;
  CHECK(be.SetStarvationGuard(0, 1));                  // afterCycles >= 1
  CHECK(be.SetStarvationGuard(1, GROVE_MAX_FENCES + 1));
  CHECK(!be.SetStarvationGuard(3, 0));                 // off
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host fence tests ok\n");
  return 0;
}
