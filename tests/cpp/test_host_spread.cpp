// GpuBackend with topology spread (SetTopologySpread; DESIGN.md section 1 "Topology spread") on cuda:0, on the hack/e2e layout cut
// to two zones: 56 nodes of 150 MiB, four blocks of 14.  The replicas of one PodCliqueSet are one-pod base PodGangs of 80 MiB with
// a block Required level and the app.kubernetes.io/part-of label.  Four replicas land in four distinct blocks with the spread on
// (and are all scheduled with it off); a scale-out in a second cycle fills the blocks the first cycle left empty (the running
// replicas are the seeds); with one block full, DoNotSchedule leaves the fourth replica Unschedulable with a message that names the
// spread, and ScheduleAnyway places it in another block with a message that says so.
#include <cstdio>
#include <set>

#include "../../grove_b200/csrc/host/grove_host.hpp"

using namespace grove::host;

static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static std::vector<Node> e2e_nodes(int n) {  // hack/e2e.yaml: 150 MiB nodes; zone 28 / block 14 / rack 7 / host
  std::vector<Node> v(n);
  for (int i = 0; i < n; ++i) {
    Node& nd = v[i];
    nd.Name = "kwok-node-" + std::to_string(i);
    nd.Labels = {{"topology.kubernetes.io/zone", "zone-" + std::to_string(i / 28)}, {"topology.kubernetes.io/block", "block-" + std::to_string(i / 14)},
                 {"topology.kubernetes.io/rack", "rack-" + std::to_string(i / 7)}, {"kubernetes.io/hostname", nd.Name},
                 {"node_role.e2e.grove.nvidia.com", "agent"}};
    nd.alloc_cpu_milli = 4000; nd.alloc_mem_mib = 150; nd.alloc_pods = 110;
    nd.TaintKeys = {"node_role.e2e.grove.nvidia.com"};
  }
  return v;
}
static const std::vector<TopologyLevel> kLevels = {{"zone", "topology.kubernetes.io/zone"}, {"block", "topology.kubernetes.io/block"},
                                                   {"rack", "topology.kubernetes.io/rack"}, {"host", "kubernetes.io/hostname"}};
static const char* kBlock = "topology.kubernetes.io/block";

static PodGang replica(const std::string& pcs, int i) {   // base PodGang i of PodCliqueSet pcs: one 80 MiB pod, packed in a block
  PodGang pg;
  pg.Namespace = "default"; pg.Name = pcs + "-" + std::to_string(i);
  pg.Labels = {{"grove.io/scheduler-name", GpuBackend::kName}, {GpuBackend::kPartOfLabel, pcs}};
  PodGroup g; g.Name = pg.Name + "-w"; g.MinReplicas = 1; g.PodReferences = {{"default", pg.Name + "-w-0"}};
  pg.Spec.PodGroups = {g};
  pg.Spec.Topology = TopologyConstraint{TopologyPackConstraint{std::string(kBlock), std::nullopt}};
  PodGang::Requests rq; rq.mem_mib = 80; rq.nodeSelector = {{"node_role.e2e.grove.nvidia.com", "agent"}}; rq.tolerationKeys = {"node_role.e2e.grove.nvidia.com"};
  pg.PodGroupRequests[g.Name] = rq;
  return pg;
}

static int block_of(const std::string& node) { return std::stoi(node.substr(std::string("kwok-node-").size())) / 14; }

struct Cluster {
  GpuBackend be;
  std::map<std::string, std::string> podNode;   // pods bound so far -> node
  std::set<int> full;                           // blocks whose nodes are full
  Cluster() { CHECK(!be.SyncTopology(kLevels)); CHECK(!be.Init()); }
  std::map<std::string, PodGangStatus> cycle() {
    auto nodes = e2e_nodes(56);
    for (auto& nd : nodes) if (full.count(block_of(nd.Name))) nd.used_mem_mib = 150;
    for (const auto& kv : podNode) for (auto& nd : nodes) if (nd.Name == kv.second) { nd.used_mem_mib += 80; nd.used_pods += 1; }
    std::vector<Binding> b; std::map<std::string, PodGangStatus> st;
    CHECK(!be.RunCycle(nodes, &b, &st));
    for (const auto& x : b) podNode[x.PodName] = x.NodeName;
    return st;
  }
  std::vector<int> blocks(const std::string& pcs) {
    std::vector<int> out;
    for (const auto& kv : podNode) if (kv.first.rfind(pcs + "-", 0) == 0) out.push_back(block_of(kv.second));
    return out;
  }
};

static void four_replicas(bool on) {
  Cluster c;
  if (on) CHECK(!c.be.SetTopologySpread("serve", TopologySpread{kBlock, 1, "DoNotSchedule"}));
  for (int i = 0; i < 4; ++i) CHECK(!c.be.SyncPodGang(replica("serve", i)));
  auto st = c.cycle();
  CHECK(c.be.Pending() == 0 && c.podNode.size() == 4);
  const auto b = c.blocks("serve");
  if (on) CHECK(std::set<int>(b.begin(), b.end()).size() == 4);
}

static void scale_out() {
  Cluster c;
  CHECK(!c.be.SetTopologySpread("serve", TopologySpread{kBlock, 1, "DoNotSchedule"}));
  for (int i = 0; i < 2; ++i) CHECK(!c.be.SyncPodGang(replica("serve", i)));
  c.cycle();
  const auto b1 = c.blocks("serve");
  CHECK(b1.size() == 2 && b1[0] != b1[1]);
  for (int i = 2; i < 4; ++i) CHECK(!c.be.SyncPodGang(replica("serve", i)));
  c.cycle();
  const auto b2 = c.blocks("serve");
  CHECK(b2.size() == 4 && std::set<int>(b2.begin(), b2.end()).size() == 4);   // the second cycle took the two empty blocks
}

static void full_block(const char* when) {
  Cluster c;
  c.full = {3};
  CHECK(!c.be.SetTopologySpread("serve", TopologySpread{kBlock, 1, when}));
  for (int i = 0; i < 4; ++i) CHECK(!c.be.SyncPodGang(replica("serve", i)));
  auto st = c.cycle();
  const bool hard = std::string(when) == "DoNotSchedule";
  int unsched = 0, skewed = 0;
  for (const auto& kv : st) {
    if (kv.second.ScheduledReason == "Unschedulable") { ++unsched; CHECK(kv.second.ScheduledMessage.find("DoNotSchedule") != std::string::npos); }
    if (kv.second.Scheduled && !kv.second.ScheduledMessage.empty()) { ++skewed; CHECK(kv.second.ScheduledMessage.find("ScheduleAnyway") != std::string::npos); }
  }
  const auto b = c.blocks("serve");
  CHECK(std::find(b.begin(), b.end(), 3) == b.end());
  if (hard) CHECK(unsched == 1 && skewed == 0 && b.size() == 3 && c.be.Pending() == 1);
  else CHECK(unsched == 0 && skewed == 1 && b.size() == 4 && c.be.Pending() == 0);
}

static void validation_and_refusal() {
  Cluster c;
  CHECK(c.be.SetTopologySpread("serve", TopologySpread{kBlock, 0, "DoNotSchedule"}));
  CHECK(c.be.SetTopologySpread("serve", TopologySpread{kBlock, 1, "Sometimes"}));
  CHECK(!c.be.SetTopologySpread("serve", TopologySpread{kBlock, 1, "DoNotSchedule"}));
  c.be.SetPreemption(true);   // members stay out of the pass, with a reason; everybody else is scheduled
  CHECK(!c.be.SyncPodGang(replica("serve", 0)));
  CHECK(!c.be.SyncPodGang(replica("other", 0)));
  auto st = c.cycle();
  CHECK(st.at("default/serve-0").ScheduledReason == "Unschedulable" && st.at("default/serve-0").ScheduledMessage.find("topology spread") != std::string::npos);
  CHECK(st.at("default/other-0").Scheduled);
  c.be.SetPreemption(false);
  CHECK(!c.be.SetTopologySpread("serve", std::nullopt));
  st = c.cycle();
  CHECK(st.at("default/serve-0").Scheduled);
}

int main() {
  four_replicas(false);
  four_replicas(true);
  scale_out();
  full_block("DoNotSchedule");
  full_block("ScheduleAnyway");
  validation_and_refusal();
  if (g_fail) { std::fprintf(stderr, "%d check(s) failed\n", g_fail); return 1; }
  std::printf("host spread tests ok\n");
  return 0;
}
