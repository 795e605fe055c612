package gpu

// NOT COMPILED IN THE BUILD IMAGE (see place_cgo.go).  The logic below is what grove_b200/csrc/host/grove_host.cpp
// (`GpuBackend`) does in C++, where it is tested on the CPU (encoding) and on the GPU (cycles): same method names, same
// argument meaning, same error behaviour as the reference's Backend seam.

import (
	"context"
	"fmt"
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
	rejectedFor          map[string]int
	// consolidation (SetConsolidation): off while consMax == 0; specOf: scheduled PodGang -> its spec (restated as a gated row to
	// make it movable); moveAnchor: moved PodGang -> the first node of the placement the cycle planned for it
	consAfter, consMax int
	specOf             map[string]*groveschedulerv1alpha1.PodGang
	moveAnchor         map[string]string
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
	spreadOn := len(b.spread) > 0
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
	for _, pg := range snap {
		wideAny = wideAny || (large && whyNotEncodable(pg, false, false) != "")
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
	rejectedFor := map[string]int{}
	for k, v := range b.rejectedFor {
		rejectedFor[k] = v
	}
	b.mu.Unlock()
	res, err := eng.cycle(t, preempt, large, explain)
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
