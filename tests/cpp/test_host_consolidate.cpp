// GpuBackend with consolidation (SetConsolidation; DESIGN.md section 1 "Consolidation") on cuda:0.  Three blocks of 2 nodes of 8
// GPUs.  In cycle 0 the second node of every block is cordoned and three one-pod PodGangs of 8 GPUs (no pack constraint) are
// scheduled, one per block; they keep running.  From cycle 1 every node is schedulable and PodGang "a-big" (2 pods of 8 GPUs packed
// in a block) waits: every block has one free node.  With consolidation off it is never scheduled; with it on after one rejected
// cycle it is the target in cycle 2, one small PodGang moves to the free node of another block, a-big is scheduled, the moved
// PodGang carries DisruptionTarget naming a-big and a-big's message names it; synced again, the moved PodGang is scheduled in
// cycle 3.  Consolidation and the starvation guard cannot both be on.
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

struct Outcome {
  int scheduledAt = -1;                 // the cycle a-big was scheduled in (-1: never)
  std::string bigMessage;               // its ScheduledMessage then
  std::vector<std::string> disrupted;   // PodGangs with DisruptionTarget, and their messages
  bool movedRescheduled = false;        // the moved PodGang, synced again, was scheduled in the next cycle
};

static Outcome run(bool consolidation) {
  Outcome o;
  GpuBackend be;
  CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init());
  if (consolidation) CHECK(!be.SetConsolidation(1, 1));
  std::map<std::string, int> podNode;   // bound pod -> node
  std::map<std::string, PodGang> small;
  for (int i = 0; i < 3; ++i) { PodGang s = gang("s-" + std::to_string(i), 1, false); small[s.Name] = s; CHECK(!be.SyncPodGang(s)); }
  std::string moved;
  for (int cyc = 0; cyc < 6; ++cyc) {
    if (cyc == 1) CHECK(!be.SyncPodGang(gang("a-big", 2, true)));
    std::vector<Node> nodes(6);
    for (int n = 0; n < 6; ++n) {
      Node& nd = nodes[n];
      nd.Name = node_name(n);
      nd.Labels = {{kBlock, "block-" + std::to_string(n / 2)}, {"kubernetes.io/hostname", nd.Name}};
      nd.alloc_cpu_milli = 64000; nd.alloc_mem_mib = 1u << 20; nd.alloc_gpu = 8;
      nd.Unschedulable = cyc == 0 && n % 2 == 1;
    }
    for (const auto& [pod, n] : podNode) { nodes[n].used_gpu += 8; nodes[n].used_pods += 1; }
    std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
    CHECK(!be.RunCycle(nodes, &b, &st));
    for (const Binding& x : b) podNode[x.PodName] = std::stoi(x.NodeName.substr(5));
    for (const auto& [key, s] : st)
      if (s.DisruptionTarget) {
        o.disrupted.push_back(key + ": " + s.DisruptionMessage);
        moved = key.substr(std::string("default/").size());
        podNode.erase(moved + "-w-0");   // the caller deletes the moved PodGang's pods and syncs it again
        CHECK(!be.SyncPodGang(small.at(moved)));
      }
    if (cyc == 0) {
      std::set<int> blocks;
      for (const auto& [pod, n] : podNode) blocks.insert(n / 2);
      CHECK(podNode.size() == 3 && blocks.size() == 3);
    }
    if (o.scheduledAt >= 0 && !moved.empty() && st.count("default/" + moved) && st.at("default/" + moved).Scheduled &&
        !st.at("default/" + moved).DisruptionTarget) {
      o.movedRescheduled = true;
      break;
    }
    if (o.scheduledAt < 0 && st.count("default/a-big") && st.at("default/a-big").Scheduled) {
      o.scheduledAt = cyc; o.bigMessage = st.at("default/a-big").ScheduledMessage;
      if (moved.empty()) break;
    }
  }
  return o;
}

int main() {
  const Outcome off = run(false);
  CHECK(off.scheduledAt == -1 && off.disrupted.empty());
  const Outcome on = run(true);
  std::fprintf(stderr, "scheduled in cycle %d: %s\n", on.scheduledAt, on.bigMessage.c_str());
  for (const auto& d : on.disrupted) std::fprintf(stderr, "  %s\n", d.c_str());
  CHECK(on.scheduledAt == 2);
  CHECK(on.disrupted.size() == 1);
  if (on.disrupted.size() == 1) {
    CHECK(on.disrupted[0].find("default/s-") == 0);
    CHECK(on.disrupted[0].find("moved to make room for PodGang default/a-big") != std::string::npos);
    const std::string who = on.disrupted[0].substr(0, on.disrupted[0].find(':'));
    CHECK(on.bigMessage == "scheduled by moving PodGangs " + who);
  }
  CHECK(on.movedRescheduled);
  GpuBackend be;
  CHECK(be.SetConsolidation(0, 1));                                   // afterCycles >= 1
  CHECK(be.SetConsolidation(1, GROVE_MAX_CONSOLIDATE_TARGETS + 1));
  CHECK(!be.SetStarvationGuard(1, 1));
  CHECK(be.SetConsolidation(1, 1));                                   // not together with the starvation guard
  CHECK(!be.SetStarvationGuard(1, 0));
  CHECK(!be.SetConsolidation(1, 1));
  CHECK(be.SetStarvationGuard(1, 1));                                 // nor the other way round
  CHECK(!be.SetConsolidation(3, 0));                                  // off
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host consolidate tests ok\n");
  return 0;
}
