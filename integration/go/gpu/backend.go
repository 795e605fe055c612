package gpu

// NOT COMPILED IN THE BUILD IMAGE (see place_cgo.go).  The logic below is what grove_b200/csrc/host/grove_host.cpp
// (`GpuBackend`) does in C++, where it is tested on the CPU (encoding) and on the GPU (cycles): same method names, same
// argument meaning, same error behaviour as the reference's Backend seam.

import (
	"context"
	"fmt"
	"math"
	"sort"
	"strings"
	"sync"
	"time"

	configv1alpha1 "github.com/ai-dynamo/grove/operator/api/config/v1alpha1"
	grovecorev1alpha1 "github.com/ai-dynamo/grove/operator/api/core/v1alpha1"
	"github.com/ai-dynamo/grove/operator/internal/scheduler"

	groveschedulerv1alpha1 "github.com/ai-dynamo/grove/scheduler/api/core/v1alpha1"
	corev1 "k8s.io/api/core/v1"
	"k8s.io/apimachinery/pkg/api/meta"
	metav1 "k8s.io/apimachinery/pkg/apis/meta/v1"
	"k8s.io/apimachinery/pkg/runtime"
	"k8s.io/apimachinery/pkg/runtime/schema"
	"k8s.io/client-go/tools/record"
	"sigs.k8s.io/controller-runtime/pkg/client"
)

// SchedulerNameGPU is the new entry of configv1alpha1.SupportedSchedulerNames (api/config/v1alpha1/types.go:54-66) and of
// the kubebuilder enum at :88-90.
const SchedulerNameGPU configv1alpha1.SchedulerName = "gpu-scheduler"

// engine limits (include/grove_place.h): PodGangs beyond them are reported Unschedulable, never an error from
// SyncPodGang -- the reconciler would requeue for ever (podgang/reconciler.go:86-89)
const (
	maxGangPods     = 128
	maxWideGangPods = 2048 // with largePodGangs: grove_submit_gangs_wide, 16-bit replica counts (GROVE_MAX_WIDE_GANG_PODS)
	maxGangCliques  = 32
	maxLevels       = 4
)

type schedulerBackend struct {
	client        client.Client
	scheme        *runtime.Scheme
	eventRecorder record.EventRecorder
	profile       configv1alpha1.SchedulerProfile

	mu       sync.Mutex                                  // pending set, level keys: everything the reconcilers touch
	pending  map[string]*groveschedulerv1alpha1.PodGang // "<ns>/<name>" -> deep copy (the cache-owned object is never retained)
	levels   []string                                    // ClusterTopology.Spec.Levels[].Key, broadest first
	running  map[string]runningGang                      // PodGangs scheduled by this backend: priority + holdings (reclaim pass)
	preempt  bool
	// elastic: with preempt also on and no queue or consolidation switch, a pass with running gangs is
	// grove_run_cycle_preempt_elastic: preemptors take the running gangs' pods beyond MinReplicas before evicting any gang whole
	// (GpuBackend::SetElasticPreemption in the C++ mirror)
	elastic bool
	// preemptQueues: with preempt also on, queue members stay in the pass and a pass with members is
	// grove_run_cycle_preempt_queues (GpuBackend::SetPreemptionWithinQueues in the C++ mirror)
	preemptQueues bool
	// reclaimQueues: queue members stay in the pass and a pass with members and running gangs is grove_run_cycle_reclaim_queues
	// with each queue's deserved quota (GpuBackend::SetReclaimAcrossQueues in the C++ mirror)
	reclaimQueues bool
	// reclaimThenPreempt: with preempt also on, queue members stay in the pass and a pass with members and running gangs is
	// grove_run_cycle_reclaim_preempt_queues, whatever preemptQueues and reclaimQueues say (GpuBackend::SetReclaimThenPreempt in
	// the C++ mirror)
	reclaimThenPreempt bool
	// fairShare: a pass with queue members and no preemption runs the queue cycle in fair-share order (grove_set_fair_share with
	// each queue's deserved quota; GpuBackend::SetFairShareOrder in the C++ mirror)
	fairShare bool
	// overQuota: the passes that run with quotas (reclaimQueues, reclaimThenPreempt, fairShare) also set each queue's over-quota
	// weights (grove_set_over_quota), so that its fair share stands in for its deserved quota; fairShares holds the shares the last
	// such pass used, by queue name (GpuBackend::SetOverQuotaWeights / FairShares in the C++ mirror)
	overQuota  bool
	fairShares map[string][3]uint64
	// largePodGangs: PodGangs of up to maxWideGangPods pods are encoded (a counts row per clique) and submitted through
	// grove_submit_gangs_wide.  The reclaim pass takes no such PodGang: with preempt also on, one beyond maxGangPods pods or 255
	// replicas is reported Unschedulable (GpuBackend::SetLargePodGangs in the C++ mirror).
	largePodGangs bool
	// explainUnschedulable: after an ordinary cycle the Unschedulable message of a rejected PodGang says why, from
	// grove_diagnose (GpuBackend::SetExplainUnschedulable in the C++ mirror); off, it is the fixed message of before.
	explainUnschedulable bool
	// spread: PodCliqueSet name -> its topology spread (SetTopologySpread); setOf: scheduled base PodGang -> its PodCliqueSet
	spread map[string]TopologySpread
	setOf  map[string]string
	// starvation guard (SetStarvationGuard): off while guardMax == 0; rejectedFor: pending PodGang -> consecutive Unschedulable cycles
	guardAfter, guardMax int
	// bin-packing (SetBinPacking): the level key every PodGang of an ordinary or queue pass packs at; off while empty
	binpackKey string
	// ComputeDomain exclusivity (SetComputeDomainExclusivity)
	imex bool
	rejectedFor          map[string]int
	// consolidation (SetConsolidation): off while consMax == 0; specOf: scheduled PodGang -> its spec (restated as a gated row to
	// make it movable); moveAnchor: moved PodGang -> the first node of the placement the cycle planned for it
	consAfter, consMax int
	specOf             map[string]*groveschedulerv1alpha1.PodGang
	moveAnchor         map[string]string
	// queue limits (SetQueue): queue name -> its limits; queueOf: scheduled PodGang -> its queue (kai.scheduler/queue label)
	queues  map[string]Queue
	queueOf map[string]string
	eng                  *engine
	stopLoop chan struct{}
}

// TopologySpread spreads the base PodGangs of one PodCliqueSet over the domains of a level (GpuBackend::SetTopologySpread in the
// C++ mirror; DESIGN.md section 1 "Topology spread").  WhenUnsatisfiable is "DoNotSchedule" or "ScheduleAnyway".
type TopologySpread struct {
	LevelKey          string
	MaxSkew           int32
	WhenUnsatisfiable string
}

// the label the producer puts on every PodGang of a PodCliqueSet (components/podgang/podgang.go:129), and the one that names the
// base PodGang of a scaled one (api/common/labels.go:35-37)
const (
	labelPartOf      = "app.kubernetes.io/part-of"
	labelBasePodGang  = "grove.io/base-podgang"
)

// SetElasticPreemption: with it and preemption on (no queue or consolidation switch), a pass with running PodGangs runs
// grove_run_cycle_preempt_elastic: the bound pods of each running PodGroup beyond MinReplicas are surplus, and a preemptor takes
// those before it evicts any PodGang whole (DESIGN.md section 1 "Elastic reclaim").  A PodGang that lost pods keeps running and
// is not a DisruptionTarget; the backend deletes those pods and forgets what they held.  Off by default.
func (b *schedulerBackend) SetElasticPreemption(on bool) {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.elastic = on
}

// SetPreemptionWithinQueues: with it and preemption on, queue members are no longer kept out of a pass with preemption, and a
// pass with members runs grove_run_cycle_preempt_queues: a member its queue chain turns away may evict lower-priority PodGangs of
// its own queues (DESIGN.md section 1 "Reclaim within queue limits").  The queue of each running PodGang is the one it was
// scheduled in.  Off by default.
func (b *schedulerBackend) SetPreemptionWithinQueues(on bool) {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.preemptQueues = on
}

// SetReclaimAcrossQueues: with it on, queue members stay in the pass, and a pass with members and running PodGangs runs
// grove_run_cycle_reclaim_queues with each Queue's deserved quota: a queue below its quota may evict running PodGangs of queues
// above theirs, whatever the priorities (DESIGN.md section 1 "Reclaim across queues").  Victims get DisruptionTarget naming the
// reclaimer.  Off by default; a cycle with both this and SetPreemptionWithinQueues on fails.
func (b *schedulerBackend) SetReclaimAcrossQueues(on bool) {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.reclaimQueues = on
}

// SetReclaimThenPreempt: with it and preemption on, queue members stay in the pass, and a pass with members and running PodGangs
// runs grove_run_cycle_reclaim_preempt_queues: reclaim across queues, then preemption within queue limits for every PodGang still
// pending, in one cycle as KAI-Scheduler runs its reclaim and preempt actions (DESIGN.md section 1 "Reclaim, then preempt").  It
// overrides SetReclaimAcrossQueues and SetPreemptionWithinQueues, whose combination then no longer fails.  Victims get
// DisruptionTarget naming the PodGang that evicted them.  Off by default.
func (b *schedulerBackend) SetReclaimThenPreempt(on bool) {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.reclaimThenPreempt = on
}

// SetFairShareOrder: with it on, a pass with queue members and no preemption runs the queue cycle in fair-share order, as
// KAI-Scheduler's allocate action orders its jobs: the next turn goes to the queue furthest below its deserved quota, priority
// orders PodGangs only inside a queue (DESIGN.md section 1 "Fair-share order").  Members must sit in leaf queues.  Bin-packing is
// not applied in such a pass.  Off by default.
func (b *schedulerBackend) SetFairShareOrder(on bool) {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.fairShare = on
}

// SetOverQuotaWeights: with it on, every pass that runs with quotas (SetReclaimAcrossQueues, SetReclaimThenPreempt,
// SetFairShareOrder) sets each queue's over-quota weights, as KAI-Scheduler's proportion plugin divides the capacity nobody
// deserves: a queue's fair share, its deserved quota plus its weighted slice of that capacity capped by what it asks for, stands
// in for its deserved quota (DESIGN.md section 1 "Over-quota weight").  Off by default; off behaves exactly as before.
func (b *schedulerBackend) SetOverQuotaWeights(on bool) {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.overQuota = on
}

// FairShares: the fair shares (cpu milli, mem MiB, gpu; unlimited where the deserved quota is) of the last pass that ran with
// over-quota weights, by queue name, as KAI reports them in queue status; empty before such a pass.
func (b *schedulerBackend) FairShares() map[string][3]uint64 {
	b.mu.Lock()
	defer b.mu.Unlock()
	out := make(map[string][3]uint64, len(b.fairShares))
	for k, v := range b.fairShares {
		out[k] = v
	}
	return out
}

// SetTopologySpread sets (nil: removes) the topology spread of PodCliqueSet pcs.  Its pending base PodGangs with a Required level
// at or below spread.LevelKey and a PodGroup with MinReplicas > 0 are members; the running ones this backend scheduled count
// where they landed.  With preemption on, or in a pass with a large PodGang, members stay out of the pass, Unschedulable.
func (b *schedulerBackend) SetTopologySpread(pcs string, spread *TopologySpread) error {
	b.mu.Lock()
	defer b.mu.Unlock()
	if b.spread == nil {
		b.spread, b.setOf = map[string]TopologySpread{}, map[string]string{}
	}
	if spread == nil {
		delete(b.spread, pcs)
		return nil
	}
	if spread.LevelKey == "" || spread.MaxSkew < 1 || spread.MaxSkew > 0xFFFF ||
		(spread.WhenUnsatisfiable != "DoNotSchedule" && spread.WhenUnsatisfiable != "ScheduleAnyway") {
		return fmt.Errorf("topology spread of %s: want a level key, maxSkew >= 1 and DoNotSchedule or ScheduleAnyway", pcs)
	}
	b.spread[pcs] = *spread
	return nil
}

// spreadSet: the PodCliqueSet whose spread pg is a member of, or ""
func (b *schedulerBackend) spreadSet(pg *groveschedulerv1alpha1.PodGang) string {
	if _, scaled := pg.Labels[labelBasePodGang]; scaled {
		return ""
	}
	if _, ok := b.spread[pg.Labels[labelPartOf]]; ok {
		return pg.Labels[labelPartOf]
	}
	return ""
}

// encodeSpread fills the spread tables of t for gang rows `rows`: one group per PodCliqueSet with a member, its running
// replicas as seeds.
func (b *schedulerBackend) encodeSpread(t *tables, rows []*groveschedulerv1alpha1.PodGang, levels []string, nodeIdx map[string]int) {
	groupOf := map[string]int{}
	t.spreadOf = make([]C.uint32_t, len(rows))
	members := 0
	for gi, pg := range rows {
		t.spreadOf[gi] = C.GROVE_NONE_U32
		set := b.spreadSet(pg)
		if set == "" {
			continue
		}
		sp := b.spread[set]
		lvl := levelIndex(levels, &sp.LevelKey)
		g := t.gangs[gi]
		need := false
		for q := int(g.clique_off); q < int(g.clique_off)+int(g.n_cliques); q++ {
			need = need || t.cliques[q].min_replicas > 0 // (a spread pass is never wide: the 8-bit counts hold)
		}
		if lvl == C.GROVE_LEVEL_NONE || g.level == C.GROVE_LEVEL_NONE || g.level < lvl || !need {
			continue // packed as usual, not counted
		}
		s, ok := groupOf[pg.Namespace+"/"+set]
		if !ok {
			s = len(t.spreadGroups)
			groupOf[pg.Namespace+"/"+set] = s
			mode := C.uint8_t(C.GROVE_SPREAD_HARD)
			if sp.WhenUnsatisfiable == "ScheduleAnyway" {
				mode = C.GROVE_SPREAD_SOFT
			}
			t.spreadGroups = append(t.spreadGroups, C.grove_spread_t{level: lvl, mode: mode, max_skew: C.uint16_t(sp.MaxSkew)})
		}
		t.spreadOf[gi] = C.uint32_t(s)
		members++
	}
	if members == 0 {
		t.spreadGroups, t.spreadOf = nil, nil
		return
	}
	for key, set := range b.setOf { // a running replica counts in the domain of a node it holds
		s, ok := groupOf[set]
		if !ok {
			continue
		}
		for node := range b.running[key].held {
			if n, ok := nodeIdx[node]; ok {
				t.spreadSeeds = append(t.spreadSeeds, C.grove_spread_seed_t{group: C.uint32_t(s), node: C.uint32_t(n)})
				break
			}
		}
	}
}

// Queue is a KAI queue's hard limits in the engine's units (millicores, MiB, GPUs; nil = no limit, KAI's -1), its deserved quota
// in the same units (spec.resources.*.quota; nil = KAI's -1, read only by SetReclaimAcrossQueues), its over-quota weights
// (spec.resources.*.overQuotaWeight; nil = 1, KAI's default, read only by SetOverQuotaWeights) and its parent ("" = a root
// queue).  GpuBackend::SetQueue in the C++ mirror; DESIGN.md section 1 "Queue limits", "Reclaim across queues" and "Over-quota
// weight".
type Queue struct {
	Parent                                                     string
	CpuMilli, MemMiB, Gpu                                      *uint64
	DeservedCpuMilli, DeservedMemMiB, DeservedGpu              *uint64
	OverQuotaWeightCpu, OverQuotaWeightMem, OverQuotaWeightGpu *uint32
}

const labelQueue = "kai.scheduler/queue"
const queueUnlimited = ^uint64(0)

// SetQueue sets (nil: removes) queue name.  A pending PodGang whose kai.scheduler/queue label names a set queue is a member: it is
// admitted only while its queue chain has room for its MinReplicas, and its best-effort pods are capped to what is left.  A parent
// is set before its children, chains are at most GROVE_MAX_QUEUE_DEPTH deep, a queue that is a parent is not removed.  With
// preemption, the starvation guard or consolidation on, or in a pass with topology spread members or large PodGangs, members stay
// out of the pass, Unschedulable with a reason.
func (b *schedulerBackend) SetQueue(name string, q *Queue) error {
	b.mu.Lock()
	defer b.mu.Unlock()
	if b.queues == nil {
		b.queues, b.queueOf = map[string]Queue{}, map[string]string{}
	}
	if name == "" {
		return fmt.Errorf("a queue needs a name")
	}
	if q == nil {
		for n, x := range b.queues {
			if x.Parent == name {
				return fmt.Errorf("queue %s is the parent of queue %s", name, n)
			}
		}
		delete(b.queues, name)
		return nil
	}
	depth := 1
	for p := q.Parent; p != ""; p = b.queues[p].Parent {
		if p == name {
			return fmt.Errorf("queue %s would be its own ancestor", name)
		}
		if _, ok := b.queues[p]; !ok {
			return fmt.Errorf("queue %s: parent queue %s is not set", name, p)
		}
		if depth++; depth > C.GROVE_MAX_QUEUE_DEPTH {
			return fmt.Errorf("queue %s: chain deeper than GROVE_MAX_QUEUE_DEPTH", name)
		}
	}
	for n, x := range b.queues {
		if old, ok := b.queues[name]; ok && x.Parent == name && old.Parent != q.Parent {
			return fmt.Errorf("queue %s is the parent of queue %s: its parent cannot change", name, n)
		}
	}
	if _, ok := b.queues[name]; !ok && len(b.queues) >= C.GROVE_MAX_QUEUES {
		return fmt.Errorf("more than GROVE_MAX_QUEUES queues")
	}
	b.queues[name] = *q
	return nil
}

// queueName: the set queue pg's label names, or ""
func (b *schedulerBackend) queueName(pg *groveschedulerv1alpha1.PodGang) string {
	if _, ok := b.queues[pg.Labels[labelQueue]]; ok {
		return pg.Labels[labelQueue]
	}
	return ""
}

// encodeQueues fills the queue tables of t for gang rows `rows`: the queues parents first (by depth, then name) with what the
// running PodGangs of each hold, and each row's queue.  Nothing when no row is a member.
func (b *schedulerBackend) encodeQueues(t *tables, rows []*groveschedulerv1alpha1.PodGang) {
	member := false
	for _, pg := range rows {
		member = member || b.queueName(pg) != ""
	}
	if !member {
		return
	}
	depth := func(n string) int {
		d := 0
		for p := b.queues[n].Parent; p != ""; p = b.queues[p].Parent {
			d++
		}
		return d
	}
	names := make([]string, 0, len(b.queues))
	for n := range b.queues {
		names = append(names, n)
	}
	sort.Slice(names, func(i, j int) bool {
		if di, dj := depth(names[i]), depth(names[j]); di != dj {
			return di < dj
		}
		return names[i] < names[j]
	})
	idx := make(map[string]int, len(names))
	for i, n := range names {
		idx[n] = i
	}
	lim := func(x *uint64) C.uint64_t {
		if x == nil {
			return C.uint64_t(queueUnlimited)
		}
		return C.uint64_t(*x)
	}
	for _, n := range names {
		q := b.queues[n]
		r := C.grove_queue_t{parent: C.GROVE_NONE_U32}
		if q.Parent != "" {
			r.parent = C.uint32_t(idx[q.Parent])
		}
		r.limit = [3]C.uint64_t{lim(q.CpuMilli), lim(q.MemMiB), lim(q.Gpu)}
		t.queues = append(t.queues, r)
		quota := C.grove_queue_quota_t{deserved: [3]C.uint64_t{lim(q.DeservedCpuMilli), lim(q.DeservedMemMiB), lim(q.DeservedGpu)}}
		if b.reclaimQueues || (b.reclaimThenPreempt && b.preempt) {
			t.quotas = append(t.quotas, quota)
		} else if b.fairShare && !b.preempt {
			t.fairShare = append(t.fairShare, quota)
		}
		if b.overQuota {
			wt := func(x *uint32) C.uint32_t {
				if x == nil {
					return 1
				}
				return C.uint32_t(*x)
			}
			t.weights = append(t.weights, C.grove_queue_weight_t{over_quota: [3]C.uint32_t{wt(q.OverQuotaWeightCpu), wt(q.OverQuotaWeightMem), wt(q.OverQuotaWeightGpu)}})
		}
	}
	for key, qn := range b.queueOf {
		i, ok := idx[qn]
		rg, running := b.running[key]
		if !ok || !running {
			continue
		}
		for _, h := range rg.held {
			t.queues[i].used[0] += C.uint64_t(h.cpuMilli)
			t.queues[i].used[1] += C.uint64_t(h.memMiB)
			t.queues[i].used[2] += C.uint64_t(h.gpu)
		}
	}
	for _, pg := range rows {
		if n := b.queueName(pg); n != "" {
			t.queueOf = append(t.queueOf, C.uint32_t(idx[n]))
		} else {
			t.queueOf = append(t.queueOf, C.GROVE_NONE_U32)
		}
	}
	t.queueNames = names
}

// queueMessages: the messages of the queue members of one cycle, restated from its results in rank order as
// GpuBackend::QueueMessages words them.
func queueMessages(t *tables, res *result, nRows int) map[int]string {
	msg := map[int]string{}
	if len(t.queues) == 0 {
		return msg
	}
	kRes := [3]string{"cpu (millicores)", "memory (MiB)", "GPUs"}
	load := make([][3]int64, len(t.queues))
	for q := range t.queues {
		for r := 0; r < 3; r++ {
			load[q][r] = int64(t.queues[q].used[r])
		}
	}
	for q := len(t.queues) - 1; q >= 0; q-- { // parents come first: a queue's load is its own and its descendants'
		if p := t.queues[q].parent; p != C.GROVE_NONE_U32 {
			for r := 0; r < 3; r++ {
				load[p][r] += load[q][r]
			}
		}
	}
	finite := func(q, r int) bool { return uint64(t.queues[q].limit[r]) != queueUnlimited }
	order := []int{}
	for g := 0; g < nRows; g++ {
		if t.queueOf[g] != C.GROVE_NONE_U32 {
			order = append(order, g)
		}
	}
	sort.SliceStable(order, func(i, j int) bool { return t.gangs[order[i]].priority > t.gangs[order[j]].priority }) // rank order
	for _, g := range order {
		st := res.status[g]
		if st.state != C.GROVE_GANG_ADMITTED && st.state != C.GROVE_GANG_REJECTED {
			continue
		}
		gg := t.gangs[g]
		var R [3]int64
		for c := int(gg.clique_off); c < int(gg.clique_off)+int(gg.n_cliques); c++ {
			m := int64(t.counts[c].min_replicas)
			R[0] += m * int64(t.cliques[c].req_cpu_milli)
			R[1] += m * int64(t.cliques[c].req_mem_mib)
			R[2] += m * int64(t.cliques[c].req_gpu)
		}
		chain := []int{}
		for q := t.queueOf[g]; q != C.GROVE_NONE_U32; q = t.queues[q].parent {
			chain = append(chain, int(q))
		}
		if st.reserved0&C.GROVE_STATUS_OVER_LIMIT != 0 { // the first queue of the chain, leaf first, and the resource without room
		find:
			for _, q := range chain {
				for r := 0; r < 3; r++ {
					if finite(q, r) && R[r] > 0 && R[r] > int64(t.queues[q].limit[r])-load[q][r] {
						msg[g] = fmt.Sprintf("queue %s has no room for this PodGang: %s limit %d, load %d, MinReplicas need %d",
							t.queueNames[q], kRes[r], uint64(t.queues[q].limit[r]), load[q][r], R[r])
						break find
					}
				}
			}
			continue
		}
		if st.state != C.GROVE_GANG_ADMITTED {
			continue
		}
		if st.reserved0&C.GROVE_STATUS_SURPLUS_CAPPED != 0 { // s_q clique by clique, as the engine caps the surplus
			var rem [3]int64
			var fin [3]bool
			for r := 0; r < 3; r++ {
				rem[r] = math.MaxInt64
				for _, q := range chain {
					if finite(q, r) {
						fin[r] = true
						if h := int64(t.queues[q].limit[r]) - load[q][r]; h < rem[r] {
							rem[r] = h
						}
					}
				}
				if fin[r] {
					rem[r] -= R[r]
				}
			}
			var heldBack int64
			for c := int(gg.clique_off); c < int(gg.clique_off)+int(gg.n_cliques); c++ {
				extra := int64(t.counts[c].replicas) - int64(t.counts[c].min_replicas)
				req := [3]int64{int64(t.cliques[c].req_cpu_milli), int64(t.cliques[c].req_mem_mib), int64(t.cliques[c].req_gpu)}
				sq := extra
				for r := 0; r < 3; r++ {
					if fin[r] && req[r] > 0 {
						if rem[r] < 0 {
							sq = 0
						} else if x := rem[r] / req[r]; x < sq {
							sq = x
						}
					}
				}
				for r := 0; r < 3; r++ {
					if fin[r] {
						rem[r] -= sq * req[r]
					}
				}
				heldBack += extra - sq
			}
			msg[g] = fmt.Sprintf("queue limits held back %d best-effort pods of this PodGang", heldBack)
		}
		for k := 0; k < int(st.n_pods); k++ { // it charges what it took to every queue of its chain
			c := t.cliques[res.placements[int(st.placement_off)+k].clique]
			for _, q := range chain {
				load[q][0] += int64(c.req_cpu_milli)
				load[q][1] += int64(c.req_mem_mib)
				load[q][2] += int64(c.req_gpu)
			}
		}
	}
	return msg
}

type runningGang struct {
	priority int32
	held     map[string]held // node name -> resources
}
type held struct {
	cpuMilli, memMiB uint32
	gpu, pods        uint16
}

var (
	_ scheduler.Backend                  = (*schedulerBackend)(nil)
	_ scheduler.TopologyAwareSchedBackend = (*schedulerBackend)(nil)
)

// New mirrors kai.New / kube.New (scheduler/kai/backend.go:46-55).
func New(cl client.Client, scheme *runtime.Scheme, rec record.EventRecorder, p configv1alpha1.SchedulerProfile) scheduler.Backend {
	return &schedulerBackend{client: cl, scheme: scheme, eventRecorder: rec, profile: p,
		pending: map[string]*groveschedulerv1alpha1.PodGang{}, running: map[string]runningGang{}}
}

func (b *schedulerBackend) Name() string { return string(SchedulerNameGPU) }

// Init creates nothing yet: the engine handle needs the level count, which arrives with SyncTopology.
func (b *schedulerBackend) Init() error {
	b.stopLoop = make(chan struct{})
	go b.loop(100 * time.Millisecond)
	return nil
}

// SyncPodGang is read-only on the cache-owned object (types.go:45-47): it copies the PodGang into the pending set.
func (b *schedulerBackend) SyncPodGang(_ context.Context, pg *groveschedulerv1alpha1.PodGang) error {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.pending[pg.Namespace+"/"+pg.Name] = pg.DeepCopy()
	return nil
}

func (b *schedulerBackend) OnPodGangDelete(_ context.Context, pg *groveschedulerv1alpha1.PodGang) error {
	b.mu.Lock()
	defer b.mu.Unlock()
	key := pg.Namespace + "/" + pg.Name
	delete(b.pending, key)
	delete(b.running, key) // its pods' resources show up as free in the next node snapshot
	delete(b.setOf, key)
	delete(b.queueOf, key)
	delete(b.rejectedFor, key)
	delete(b.specOf, key)
	delete(b.moveAnchor, key)
	return nil
}

// SetStarvationGuard fences, each cycle, the <= maxGangs highest-ranked pending PodGangs with a Required level that came back
// Unschedulable at least afterCycles cycles in a row (gated or base-not-scheduled cycles neither count nor reset): while one
// stays rejected, the PodGangs ranked after it are kept out of the domain closest to fitting it (grove_set_fences;
// GpuBackend::SetStarvationGuard in the C++ mirror).  Nothing is fenced with preemption on, with topology spread members or in a
// pass with a large PodGang.  maxGangs = 0 turns it off (the default).
func (b *schedulerBackend) SetStarvationGuard(afterCycles, maxGangs int) error {
	if afterCycles < 1 || maxGangs < 0 || maxGangs > int(C.GROVE_MAX_FENCES) {
		return fmt.Errorf("starvation guard: want afterCycles >= 1 and 0 <= maxGangs <= %d", int(C.GROVE_MAX_FENCES))
	}
	b.mu.Lock()
	defer b.mu.Unlock()
	if maxGangs > 0 && b.consMax > 0 {
		return fmt.Errorf("starvation guard: the starvation guard and consolidation cannot both be on")
	}
	b.guardAfter, b.guardMax = afterCycles, maxGangs
	return nil
}

// SetBinPacking makes every PodGang of an ordinary or queue pass start its search at the fullest domain of the level `levelKey`
// (or of its own Required level when that is deeper) that can hold it on the cycle's node table, so that empty domains stay empty
// for large PodGangs (grove_set_binpack; GpuBackend::SetBinPacking in the C++ mirror).  A preference, not a constraint: a pass with
// preemption, consolidation, topology spread members, fences or a large PodGang runs without it, and so does every pass while the
// key names no level of the topology.  An empty key (the default) turns it off.
func (b *schedulerBackend) SetBinPacking(levelKey string) {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.binpackKey = levelKey
}

// SetComputeDomainExclusivity keeps the pods of MNNVL-enrolled PodGroups (a pod's `mnnvl-claim` resource claim names the
// ComputeDomain through its resourceClaimTemplateName) off nodes that another ComputeDomain holds (grove_set_compute_domains;
// GpuBackend::SetComputeDomainExclusivity in the C++ mirror).  A node's holder when the pass starts is the ComputeDomain of the
// enrolled pods bound to it.  A PodGang whose PodGroups name two ComputeDomains stays out of the pass, and so does every enrolled
// PodGang in a pass with preemption, consolidation, the starvation guard, bin-packing, topology spread, queue limits or large
// PodGangs.  Off (the default): the pass is as before.
func (b *schedulerBackend) SetComputeDomainExclusivity(on bool) {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.imex = on
}

// mnnvlClaim is the resourceClaimTemplateName of the pod's `mnnvl-claim` entry, or "" (not enrolled)
func mnnvlClaim(pod *corev1.Pod) string {
	for _, c := range pod.Spec.ResourceClaims {
		if c.Name == "mnnvl-claim" && c.ResourceClaimTemplateName != nil {
			return *c.ResourceClaimTemplateName
		}
	}
	return ""
}

// SetConsolidation makes, each cycle, the <= maxTargets highest-ranked pending PodGangs that came back Unschedulable at least
// afterCycles cycles in a row (counted as the starvation guard counts) targets of grove_run_cycle_consolidate: running PodGangs
// this backend scheduled, restated as gated rows, are relocated out of the domain closest to fitting a target when every one of
// them is admitted elsewhere.  A moved PodGang gets DisruptionTarget naming the PodGang it made room for and is forgotten as
// running; synced again, it is anchored at the first node of its planned placement.  A consolidated PodGang's Scheduled message
// names the moved ones.  Only in a pass without preemption, topology spread members or large PodGangs; not together with the
// starvation guard (GpuBackend::SetConsolidation in the C++ mirror).  maxTargets = 0 turns it off (the default).
func (b *schedulerBackend) SetConsolidation(afterCycles, maxTargets int) error {
	if afterCycles < 1 || maxTargets < 0 || maxTargets > int(C.GROVE_MAX_CONSOLIDATE_TARGETS) {
		return fmt.Errorf("consolidation: want afterCycles >= 1 and 0 <= maxTargets <= %d", int(C.GROVE_MAX_CONSOLIDATE_TARGETS))
	}
	b.mu.Lock()
	defer b.mu.Unlock()
	if maxTargets > 0 && b.guardMax > 0 {
		return fmt.Errorf("consolidation: the starvation guard and consolidation cannot both be on")
	}
	b.consAfter, b.consMax = afterCycles, maxTargets
	return nil
}

// markMoved sets DisruptionTarget on a PodGang consolidation relocated (podgang.go:166-170); the caller's controllers delete its
// pods, and the PodGang is synced and scheduled again at its planned place.
func (b *schedulerBackend) markMoved(ctx context.Context, key string, target *groveschedulerv1alpha1.PodGang) {
	ns, name, _ := strings.Cut(key, "/")
	var pg groveschedulerv1alpha1.PodGang
	if err := b.client.Get(ctx, client.ObjectKey{Namespace: ns, Name: name}, &pg); err != nil {
		return
	}
	meta.SetStatusCondition(&pg.Status.Conditions, metav1.Condition{Type: string(groveschedulerv1alpha1.PodGangConditionTypeDisruptionTarget),
		Status: metav1.ConditionTrue, Reason: "Consolidated", Message: "moved to make room for PodGang " + target.Namespace + "/" + target.Name})
	_ = b.client.Status().Update(ctx, &pg)
}

// PreparePod keeps kube-scheduler away from the pod, as kai/backend.go:72-75 does.
func (b *schedulerBackend) PreparePod(pod *corev1.Pod) { pod.Spec.SchedulerName = b.Name() }

// ValidatePodCliqueSet rejects what the packed tables cannot hold, with the reference's field paths.
func (b *schedulerBackend) ValidatePodCliqueSet(_ context.Context, pcs *grovecorev1alpha1.PodCliqueSet) error {
	if n := len(pcs.Spec.Template.Cliques); n > maxGangCliques {
		return fmt.Errorf("spec.template.cliques: %d PodCliques, the %s backend packs at most %d per PodGang", n, b.Name(), maxGangCliques)
	}
	pods := int32(0)
	for _, c := range pcs.Spec.Template.Cliques {
		pods += c.Spec.Replicas
	}
	limit := int32(maxGangPods)
	if b.largePodGangs {
		limit = maxWideGangPods
	}
	if pods > limit {
		return fmt.Errorf("spec.template.cliques: %d pods in the base PodGang, the %s backend packs at most %d", pods, b.Name(), limit)
	}
	return nil
}

// ---- TopologyAwareSchedBackend (types.go:64-96): this backend keeps no topology CR of its own ----------------------
func (b *schedulerBackend) TopologyGVR() schema.GroupVersionResource {
	return schema.GroupVersionResource{Group: "grove.io", Version: "v1alpha1", Resource: "clustertopologies"}
}
func (b *schedulerBackend) TopologyResourceName(ct *grovecorev1alpha1.ClusterTopology) string { return ct.Name }

func (b *schedulerBackend) SyncTopology(_ context.Context, _ client.Client, ct *grovecorev1alpha1.ClusterTopology) error {
	keys := make([]string, 0, len(ct.Spec.Levels))
	for _, l := range ct.Spec.Levels {
		keys = append(keys, l.Key)
	}
	if len(keys) == 0 || len(keys) > maxLevels {
		return fmt.Errorf("ClusterTopology %s: %d levels, the %s backend takes 1..%d", ct.Name, len(keys), b.Name(), maxLevels)
	}
	b.mu.Lock()
	defer b.mu.Unlock()
	if b.eng != nil && len(keys) != len(b.levels) {
		b.eng.close()
		b.eng = nil
	}
	b.levels = keys
	if b.eng == nil {
		eng, err := newEngine(0, len(keys))
		if err != nil {
			return err
		}
		b.eng = eng
	}
	return nil
}

func (b *schedulerBackend) OnTopologyDelete(_ context.Context, _ client.Client, _ *grovecorev1alpha1.ClusterTopology) error {
	b.mu.Lock()
	defer b.mu.Unlock()
	b.levels = nil
	return nil
}

func (b *schedulerBackend) CheckTopologyDrift(_ context.Context, ct *grovecorev1alpha1.ClusterTopology,
	_ grovecorev1alpha1.SchedulerTopologyReference) (bool, string, int64, error) {
	b.mu.Lock()
	defer b.mu.Unlock()
	if len(b.levels) != len(ct.Spec.Levels) {
		return false, "level count differs", ct.Generation, nil
	}
	for i, l := range ct.Spec.Levels {
		if b.levels[i] != l.Key {
			return false, fmt.Sprintf("level %d: %q != %q", i, b.levels[i], l.Key), ct.Generation, nil
		}
	}
	return true, "", ct.Generation, nil
}

// ---- the cycle loop: ONE goroutine owns the engine handle ------------------------------------------------------------
func (b *schedulerBackend) loop(period time.Duration) {
	t := time.NewTicker(period)
	defer t.Stop()
	for {
		select {
		case <-b.stopLoop:
			return
		case <-t.C:
			if err := b.runCycle(context.Background()); err != nil {
				continue // the next tick retries (the reconciler's requeue)
			}
		}
	}
}

func levelIndex(levels []string, key *string) C.uint8_t {
	if key != nil {
		for i, k := range levels {
			if k == *key {
				return C.uint8_t(i)
			}
		}
	} // a key that is no longer a level is dropped, as createTopologyPackConstraint drops an unknown pack domain (syncflow.go:349-371)
	return C.GROVE_LEVEL_NONE
}

func required(tc *groveschedulerv1alpha1.TopologyConstraint) *string {
	if tc == nil || tc.PackConstraint == nil {
		return nil
	}
	return tc.PackConstraint.Required
}

// runCycle: snapshot Nodes + bound Pods -> tables -> engine.cycle -> bind pods, patch PodGang status, mark victims.
func (b *schedulerBackend) runCycle(ctx context.Context) error {
	b.mu.Lock()
	if b.eng == nil || len(b.pending) == 0 {
		b.mu.Unlock()
		return nil
	}
	snap := make([]*groveschedulerv1alpha1.PodGang, 0, len(b.pending))
	for _, pg := range b.pending {
		snap = append(snap, pg)
	}
	levels, eng, preempt, large, explain := b.levels, b.eng, b.preempt, b.largePodGangs, b.explainUnschedulable
	thenPreempt := b.reclaimThenPreempt && preempt
	if b.reclaimQueues && b.preemptQueues && !thenPreempt {
		b.mu.Unlock()
		return fmt.Errorf("reclaim across queues and preemption within queues cannot both be on")
	}
	imexOn := b.imex
	imexWhy := "" // a pass that takes no ComputeDomain set: the enrolled PodGangs stay out
	switch {
	case preempt:
		imexWhy = "ComputeDomain exclusivity is not applied while preemption is on"
	case b.consMax > 0:
		imexWhy = "ComputeDomain exclusivity is not applied while consolidation is on"
	case b.guardMax > 0:
		imexWhy = "ComputeDomain exclusivity is not applied while the starvation guard is on"
	case b.binpackKey != "":
		imexWhy = "ComputeDomain exclusivity is not applied while bin-packing is on"
	case len(b.queues) > 0:
		imexWhy = "ComputeDomain exclusivity is not applied while queue limits are set"
	}
	spreadOn := len(b.spread) > 0
	queuesOn := len(b.queues) > 0
	queueWhy := "" // a pass that takes no queue set: its members stay out
	switch {
	case preempt && !b.preemptQueues && !b.reclaimQueues && !thenPreempt:
		queueWhy = "queue limits are not applied while preemption is on"
	case b.consMax > 0:
		queueWhy = "queue limits are not applied while consolidation is on"
	case b.guardMax > 0:
		queueWhy = "queue limits are not applied while the starvation guard is on"
	}
	b.mu.Unlock()
	sort.Slice(snap, func(i, j int) bool { return snap[i].CreationTimestamp.Before(&snap[j].CreationTimestamp) }) // submission order

	var nodeList corev1.NodeList
	if err := b.client.List(ctx, &nodeList); err != nil {
		return err
	}
	var podList corev1.PodList
	if err := b.client.List(ctx, &podList); err != nil {
		return err
	}
	t, nodeNames := encodeNodes(nodeList.Items, podList.Items, levels) // allocatable - requests of bound pods; dom[l] = interned label value
	rows := make([]*groveschedulerv1alpha1.PodGang, 0, len(snap))
	wideAny := false // a wide submission takes no spread set
	spreadAny := false // a pass with spread members takes no queue set
	for _, pg := range snap {
		wideAny = wideAny || (large && whyNotEncodable(pg, false, false) != "")
		if spreadOn && !preempt {
			b.mu.Lock()
			spreadAny = spreadAny || b.spreadSet(pg) != ""
			b.mu.Unlock()
		}
	}
	if queueWhy == "" && spreadAny {
		queueWhy = "queue limits are not applied in a pass with topology spread members"
	}
	if queueWhy == "" && wideAny {
		queueWhy = "queue limits are not applied in a pass with large PodGangs"
	}
	if imexWhy == "" && spreadAny {
		imexWhy = "ComputeDomain exclusivity is not applied in a pass with topology spread members"
	}
	if imexWhy == "" && wideAny {
		imexWhy = "ComputeDomain exclusivity is not applied in a pass with large PodGangs"
	}
	podByKey := make(map[string]*corev1.Pod, len(podList.Items))
	for i := range podList.Items {
		podByKey[podList.Items[i].Namespace+"/"+podList.Items[i].Name] = &podList.Items[i]
	}
	groupCD := func(pg *groveschedulerv1alpha1.PodGang, pgi int) string { // the ComputeDomain of a PodGroup's pods ("" = none)
		for _, ref := range pg.Spec.PodGroups[pgi].PodReferences {
			if p, ok := podByKey[ref.Namespace+"/"+ref.Name]; ok {
				return mnnvlClaim(p)
			}
		}
		return ""
	}
	for _, pg := range snap {
		if why := whyNotEncodable(pg, large, preempt); why != "" { // large && preempt: within the old limits only
			b.setUnschedulable(ctx, pg, why)
			continue
		}
		if spreadOn && (preempt || wideAny) && b.spreadSet(pg) != "" {
			b.setUnschedulable(ctx, pg, "topology spread is not applied while preemption is on or in a pass with large PodGangs")
			continue
		}
		if queuesOn && queueWhy != "" {
			b.mu.Lock()
			member := b.queueName(pg) != ""
			b.mu.Unlock()
			if member {
				b.setUnschedulable(ctx, pg, queueWhy)
				continue
			}
		}
		if imexOn {
			cd, two := "", false
			for pgi := range pg.Spec.PodGroups {
				if c := groupCD(pg, pgi); c != "" {
					two = two || (cd != "" && cd != c)
					cd = c
				}
			}
			if two {
				b.setUnschedulable(ctx, pg, "the PodGroups of this PodGang name two ComputeDomains (MNNVL groups); one per PodGang is supported")
				continue
			}
			if cd != "" && imexWhy != "" {
				b.setUnschedulable(ctx, pg, imexWhy)
				continue
			}
		}
		b.encodeGang(t, pg, levels, podList.Items) // one grove_gang_t + its cliques / scopes; requests come from the pods
		rows = append(rows, pg)
	}
	nodeIdx := make(map[string]int, len(nodeNames))
	for i, n := range nodeNames {
		nodeIdx[n] = i
	}
	b.mu.Lock()
	for gi, pg := range rows { // moved by consolidation: anchored where the cycle planned it
		if n, ok := b.moveAnchor[pg.Namespace+"/"+pg.Name]; ok {
			if i, ok := nodeIdx[n]; ok {
				t.gangs[gi].anchor_node = C.uint32_t(i)
			}
		}
	}
	b.mu.Unlock()
	if spreadOn && !preempt && !wideAny {
		b.mu.Lock()
		b.encodeSpread(t, rows, levels, nodeIdx)
		b.mu.Unlock()
	}
	b.mu.Lock()
	if b.guardMax > 0 && !preempt && !wideAny && len(t.spreadGroups) == 0 { // the starvation guard, in an ordinary pass only
		cand := []int{}
		for gi, pg := range rows {
			if t.gangs[gi].level != C.GROVE_LEVEL_NONE && b.rejectedFor[pg.Namespace+"/"+pg.Name] >= b.guardAfter {
				cand = append(cand, gi)
			}
		}
		sort.SliceStable(cand, func(i, j int) bool { return t.gangs[cand[i]].priority > t.gangs[cand[j]].priority }) // rank order
		if len(cand) > b.guardMax {
			cand = cand[:b.guardMax]
		}
		for _, gi := range cand {
			t.fences = append(t.fences, C.uint32_t(gi))
		}
	}
	// consolidation, in an ordinary pass only: the targets as the starvation guard counts, and every running PodGang this backend
	// scheduled whole restated as a gated row after the pending ones (all its pods: MinReplicas = replicas)
	var moved []string // running gang of t.running -> PodGang key
	var runningKeys []string // preemption: running gang of t.running -> PodGang key
	if b.consMax > 0 && !preempt && !wideAny && len(t.spreadGroups) == 0 {
		for gi, pg := range rows {
			if b.rejectedFor[pg.Namespace+"/"+pg.Name] >= b.consAfter {
				t.targets = append(t.targets, C.uint32_t(gi))
			}
		}
		sort.SliceStable(t.targets, func(i, j int) bool { return t.gangs[t.targets[i]].priority > t.gangs[t.targets[j]].priority })
		if len(t.targets) > b.consMax {
			t.targets = t.targets[:b.consMax]
		}
		for key, rg := range b.running {
			spec, ok := b.specOf[key]
			if _, pending := b.pending[key]; len(t.targets) == 0 || pending || !ok || whyNotEncodable(spec, false, false) != "" {
				continue
			}
			row := len(t.gangs)
			b.encodeGang(t, spec, levels, podList.Items)
			t.gangs[row].flags |= C.GROVE_GANG_GATED
			for c := int(t.gangs[row].clique_off); c < int(t.gangs[row].clique_off)+int(t.gangs[row].n_cliques); c++ {
				t.cliques[c].min_replicas = t.cliques[c].replicas
				t.counts[c].min_replicas = t.counts[c].replicas
			}
			r := C.grove_running_gang_t{priority: C.int32_t(rg.priority), holding_off: C.uint32_t(len(t.holdings))}
			for node, h := range rg.held {
				if i, ok := nodeIdx[node]; ok { // holdings on nodes that left the snapshot are dropped
					t.holdings = append(t.holdings, C.grove_holding_t{node: C.uint32_t(i), cpu_milli: C.uint32_t(h.cpuMilli),
						mem_mib: C.uint32_t(h.memMiB), gpu: C.uint16_t(h.gpu), pods: C.uint16_t(h.pods)})
					r.n_holdings++
				}
			}
			t.running = append(t.running, r)
			t.specOf = append(t.specOf, C.uint32_t(row))
			moved = append(moved, key)
		}
		if len(moved) == 0 {
			t.targets = nil
		}
	}
	// bin-packing: every row a member, at the key's level or its own Required level when deeper, in an ordinary or queue pass
	fairShare := b.fairShare && !preempt && !b.reclaimQueues && queuesOn && queueWhy == ""
	if lv := levelIndex(levels, &b.binpackKey); b.binpackKey != "" && lv != C.GROVE_LEVEL_NONE && !preempt && !wideAny &&
		len(t.spreadGroups) == 0 && len(t.fences) == 0 && len(t.targets) == 0 && !fairShare {
		t.binpack = make([]C.uint8_t, len(t.gangs))
		for gi := range t.gangs {
			t.binpack[gi] = lv
			if req := t.gangs[gi].level; req != C.GROVE_LEVEL_NONE && req > lv {
				t.binpack[gi] = req
			}
		}
	}
	if queuesOn && queueWhy == "" {
		b.encodeQueues(t, rows)
		t.thenPreempt = thenPreempt
		if (preempt || b.reclaimQueues) && len(t.queues) > 0 { // the queue of every running gang of t.running (runningKeys: its PodGang), or none
			t.runningQueue = make([]C.uint32_t, len(t.running))
			for r := range t.running {
				t.runningQueue[r] = C.GROVE_NONE_U32
				if r < len(runningKeys) {
					for qi, n := range t.queueNames {
						if n == b.queueOf[runningKeys[r]] {
							t.runningQueue[r] = C.uint32_t(qi)
						}
					}
				}
			}
		}
	}
	// ComputeDomain exclusivity, in an ordinary pass: every enrolled GPU clique row's ComputeDomain, every node's holder (the
	// ComputeDomain of the enrolled pods bound to it)
	if imexOn && imexWhy == "" && len(t.targets) == 0 && len(t.fences) == 0 {
		ids := map[string]C.uint32_t{}
		id := func(name string) C.uint32_t {
			if v, ok := ids[name]; ok {
				return v
			}
			ids[name] = C.uint32_t(len(ids))
			return ids[name]
		}
		cd := make([]C.uint32_t, len(t.cliques))
		enrolled := false
		for c := range t.cliques {
			cd[c] = C.GROVE_CD_NONE
			if gi, pgi := cliqueOwner(t, c); gi < len(rows) && t.cliques[c].req_gpu > 0 {
				if name := groupCD(rows[gi], pgi); name != "" {
					cd[c], enrolled = id(name), true
				}
			}
		}
		if enrolled {
			owner0 := make([]C.uint32_t, len(nodeNames))
			for i := range owner0 {
				owner0[i] = C.GROVE_CD_NONE
			}
			for i := range podList.Items {
				p := &podList.Items[i]
				if n, ok := nodeIdx[p.Spec.NodeName]; ok && p.Status.Phase != corev1.PodSucceeded && p.Status.Phase != corev1.PodFailed {
					if name := mnnvlClaim(p); name != "" {
						owner0[n] = id(name)
					}
				}
			}
			t.cd, t.owner0 = cd, owner0
		}
	}
	// elastic reclaim: t.surplus lists the bound pods of each gang of t.running beyond its PodGroups' MinReplicas
	t.elastic = preempt && b.elastic && !b.preemptQueues && !b.reclaimQueues && !b.reclaimThenPreempt && b.consMax == 0
	rejectedFor := map[string]int{}
	for k, v := range b.rejectedFor {
		rejectedFor[k] = v
	}
	b.mu.Unlock()
	res, err := eng.cycle(t, preempt || len(t.quotas) > 0, large, explain)
	if err != nil {
		return err
	}
	nodeLabels := make(map[string]map[string]string, len(nodeList.Items))
	for i := range nodeList.Items {
		nodeLabels[nodeList.Items[i].Name] = nodeList.Items[i].Labels
	}
	b.mu.Lock()
	if b.rejectedFor == nil {
		b.rejectedFor = map[string]int{}
	}
	for gi, st := range res.status[:len(rows)] { // consecutive Unschedulable cycles; a gated or base-not-scheduled cycle changes nothing
		key := rows[gi].Namespace + "/" + rows[gi].Name
		if st.state == C.GROVE_GANG_REJECTED {
			b.rejectedFor[key]++
		} else if st.state == C.GROVE_GANG_ADMITTED {
			delete(b.rejectedFor, key)
		}
	}
	if len(res.fairShares) > 0 { // the fair shares the pass used (SetOverQuotaWeights)
		b.fairShares = make(map[string][3]uint64, len(t.queueNames))
		for qi, n := range t.queueNames {
			b.fairShares[n] = [3]uint64{uint64(res.fairShares[qi*3]), uint64(res.fairShares[qi*3+1]), uint64(res.fairShares[qi*3+2])}
		}
	}
	for gi, st := range res.status[:len(rows)] { // what an admitted member holds counts against its queue from now on
		if st.state == C.GROVE_GANG_ADMITTED && len(t.queueOf) > 0 && t.queueOf[gi] != C.GROVE_NONE_U32 {
			b.queueOf[rows[gi].Namespace+"/"+rows[gi].Name] = t.queueNames[t.queueOf[gi]]
		}
	}
	queueMsg := queueMessages(t, res, len(rows))
	movedFor := map[int][]string{} // consolidated target row -> the PodGangs moved for it
	for _, m := range res.moves {  // forgotten as running; anchored where this cycle planned it when synced again
		key := moved[m.running]
		st := res.status[t.specOf[m.running]]
		delete(b.running, key)
		delete(b.specOf, key)
		if st.n_pods > 0 {
			if b.moveAnchor == nil {
				b.moveAnchor = map[string]string{}
			}
			b.moveAnchor[key] = nodeNames[res.placements[st.placement_off].node]
		}
		movedFor[int(m.target)] = append(movedFor[int(m.target)], key)
	}
	b.mu.Unlock()
	seen := make([]int, len(t.cliques)) // the r-th entry of a clique binds its r-th PodReference
	for _, pl := range res.placements {
		gi, pgi := cliqueOwner(t, int(pl.clique))
		if gi >= len(rows) { // a moved PodGang: its pods are deleted and it is scheduled anew when synced again
			continue
		}
		ref := rows[gi].Spec.PodGroups[pgi].PodReferences[seen[pl.clique]]
		seen[pl.clique]++
		binding := &corev1.Binding{ObjectMeta: metav1.ObjectMeta{Namespace: ref.Namespace, Name: ref.Name},
			Target: corev1.ObjectReference{Kind: "Node", Name: nodeNames[pl.node]}}
		if err := b.client.SubResource("binding").Create(ctx, &corev1.Pod{ObjectMeta: binding.ObjectMeta}, binding); err != nil {
			return err
		}
	}
	for gi, st := range res.status[:len(rows)] {
		pg := rows[gi]
		switch st.state {
		case C.GROVE_GANG_ADMITTED:
			score := float64(st.score_num) / float64(st.score_den)
			pg.Status.Phase = groveschedulerv1alpha1.PodGangPhaseStarting
			pg.Status.PlacementScore = &score // podgang.go:187-189
			msg := ""
			if st.reserved0&C.GROVE_STATUS_SPREAD_SKEWED != 0 {
				msg = "topology spread (ScheduleAnyway): no domain within the skew had room; placed beyond it"
			}
			if st.reserved0&C.GROVE_STATUS_CONSOLIDATED != 0 {
				msg = "scheduled by moving PodGangs " + strings.Join(movedFor[gi], ", ")
			}
			if m, ok := queueMsg[gi]; ok {
				msg = m
			}
			b.mu.Lock()
			if b.specOf == nil {
				b.specOf = map[string]*groveschedulerv1alpha1.PodGang{}
			}
			b.specOf[pg.Namespace+"/"+pg.Name] = pg.DeepCopy()
			delete(b.moveAnchor, pg.Namespace+"/"+pg.Name)
			b.mu.Unlock()
			meta.SetStatusCondition(&pg.Status.Conditions, metav1.Condition{Type: string(groveschedulerv1alpha1.PodGangConditionTypeScheduled),
				Status: metav1.ConditionTrue, Reason: "Scheduled", Message: msg})
			if _, scaled := pg.Labels[labelBasePodGang]; !scaled && pg.Labels[labelPartOf] != "" {
				b.mu.Lock()
				if b.setOf == nil {
					b.setOf = map[string]string{}
				}
				b.setOf[pg.Namespace+"/"+pg.Name] = pg.Namespace + "/" + pg.Labels[labelPartOf]
				b.mu.Unlock()
			}
		case C.GROVE_GANG_REJECTED:
			why := "no topology domain holds the gang's MinReplicas"
			if res.gangDiag != nil {
				why = explainRejection(t, pg, gi, res.gangDiag[gi], res.cliqueDiag, levels)
			}
			if len(t.spreadOf) > 0 && t.spreadOf[gi] != C.GROVE_NONE_U32 && t.spreadGroups[t.spreadOf[gi]].mode == C.GROVE_SPREAD_HARD {
				why = "topology spread (DoNotSchedule): no domain within the skew had room for this replica"
			}
			if m, ok := queueMsg[gi]; ok {
				why = m
			}
			if st.reserved0&C.GROVE_STATUS_FENCING != 0 && int(st.level) < len(levels) { // the starvation guard's fence held
				key := levels[st.level]
				why = fmt.Sprintf("Unschedulable for %d cycles in a row: %s %s is held for this PodGang; PodGangs ranked after it are kept out of it until it is scheduled",
					rejectedFor[pg.Namespace+"/"+pg.Name]+1, key, nodeLabels[nodeNames[st.domain_node]][key])
			}
			b.setUnschedulable(ctx, pg, why)
			continue
		default: // BASE_REJECTED / GATED_SKIP: waits, like its gated pods do (pod/syncflow.go:319-358)
			continue
		}
		if err := b.client.Status().Update(ctx, pg); err != nil {
			return err
		}
	}
	for _, v := range res.surplusVictims { // a pod beyond MinReplicas: deleted, its PodGang keeps running (podgang.go:80-83)
		b.evictSurplusPod(ctx, int(v.pod), rows[v.preemptor])
	}
	for _, v := range res.victims { // podgang.go:166-170, reason 1
		b.markDisruptionTarget(ctx, int(v.running), rows[v.preemptor])
	}
	for _, m := range res.moves {
		b.markMoved(ctx, moved[m.running], rows[m.target])
	}
	return nil
}

// explainRejection: the Unschedulable message of rejected gang row gi from its grove_diagnose records, as
// GpuBackend::ExplainRejection words it.  levels are the ClusterTopology's label keys, broadest first.
func explainRejection(t *tables, pg *groveschedulerv1alpha1.PodGang, gi int, gd C.grove_gang_diag_t, qd []C.grove_clique_diag_t, levels []string) string {
	g := t.gangs[gi]
	levelName := func(l int) string {
		if l < len(levels) {
			return levels[l]
		}
		return fmt.Sprintf("level %d", l)
	}
	switch gd.verdict {
	case C.GROVE_DIAG_CLIQUE_SHORT:
		q := int(g.clique_off) + int(gd.clique)
		c := qd[q]
		rec := t.cliques[q]
		sc := t.scopes[int(g.scope_off)+int(rec.scope&0x1F)]
		deepest := -1 // the deepest Required level binding the PodGroup: the label a node must carry
		for _, l := range []int{int(g.level), int(sc.level), int(rec.level)} {
			if l != C.GROVE_LEVEL_NONE && l > deepest {
				deepest = l
			}
		}
		label := "topology"
		if deepest >= 0 {
			label = levelName(deepest)
		}
		why := []struct {
			n    C.uint32_t
			what string
		}{{c.unschedulable, "unschedulable"}, {c.selector, "not matching the node selector"}, {c.labels, "without the " + label + " label"},
			{c.cpu, "insufficient cpu"}, {c.mem, "insufficient memory"}, {c.gpu, "insufficient nvidia.com/gpu"}, {c.pods, "too many pods"}}
		parts := []string{}
		nodes := c.nodes_fit
		for _, w := range why {
			nodes += w.n
			if w.n > 0 {
				parts = append(parts, fmt.Sprintf("%d %s", w.n, w.what))
			}
		}
		_, pgi := cliqueOwner(t, q)
		msg := fmt.Sprintf("PodGroup %s: %d/%d nodes fit", pg.Spec.PodGroups[pgi].Name, c.nodes_fit, nodes)
		if len(parts) > 0 {
			msg += " (" + strings.Join(parts, ", ") + ")"
		}
		return msg + fmt.Sprintf("; %d of %d pods fit in the cluster", uint64(c.pods_fit), pg.Spec.PodGroups[pgi].MinReplicas)
	case C.GROVE_DIAG_NO_DOMAIN:
		return fmt.Sprintf("no %s holds every PodGroup's MinReplicas (0 of %d)", levelName(int(gd.level)), gd.domains)
	case C.GROVE_DIAG_NO_JOINT_FIT:
		if gd.level == C.GROVE_LEVEL_NONE {
			return "the cluster holds each PodGroup's MinReplicas alone, but not all of them together"
		}
		return fmt.Sprintf("%d of %d %ss hold each PodGroup's MinReplicas alone, but not all of them together", gd.domains_ok, gd.domains, levelName(int(gd.level)))
	}
	return "no topology domain holds the gang's MinReplicas"
}
