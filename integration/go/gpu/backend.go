package gpu

// NOT COMPILED IN THE BUILD IMAGE (see place_cgo.go).  The logic below is what grove_b200/csrc/host/grove_host.cpp
// (`GpuBackend`) does in C++, where it is tested on the CPU (encoding) and on the GPU (cycles): same method names, same
// argument meaning, same error behaviour as the reference's Backend seam.

import (
	"context"
	"fmt"
	"sort"
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
	eng           *engine
	stopLoop chan struct{}
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
	return nil
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
	levels, eng, preempt, large := b.levels, b.eng, b.preempt, b.largePodGangs
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
	for _, pg := range snap {
		if why := whyNotEncodable(pg, large, preempt); why != "" { // large && preempt: within the old limits only
			b.setUnschedulable(ctx, pg, why)
			continue
		}
		b.encodeGang(t, pg, levels, podList.Items) // one grove_gang_t + its cliques / scopes; requests come from the pods
		rows = append(rows, pg)
	}
	res, err := eng.cycle(t, preempt, large)
	if err != nil {
		return err
	}
	seen := make([]int, len(t.cliques)) // the r-th entry of a clique binds its r-th PodReference
	for _, pl := range res.placements {
		gi, pgi := cliqueOwner(t, int(pl.clique))
		ref := rows[gi].Spec.PodGroups[pgi].PodReferences[seen[pl.clique]]
		seen[pl.clique]++
		binding := &corev1.Binding{ObjectMeta: metav1.ObjectMeta{Namespace: ref.Namespace, Name: ref.Name},
			Target: corev1.ObjectReference{Kind: "Node", Name: nodeNames[pl.node]}}
		if err := b.client.SubResource("binding").Create(ctx, &corev1.Pod{ObjectMeta: binding.ObjectMeta}, binding); err != nil {
			return err
		}
	}
	for gi, st := range res.status {
		pg := rows[gi]
		switch st.state {
		case C.GROVE_GANG_ADMITTED:
			score := float64(st.score_num) / float64(st.score_den)
			pg.Status.Phase = groveschedulerv1alpha1.PodGangPhaseStarting
			pg.Status.PlacementScore = &score // podgang.go:187-189
			meta.SetStatusCondition(&pg.Status.Conditions, metav1.Condition{Type: string(groveschedulerv1alpha1.PodGangConditionTypeScheduled),
				Status: metav1.ConditionTrue, Reason: "Scheduled"})
		case C.GROVE_GANG_REJECTED:
			b.setUnschedulable(ctx, pg, "no topology domain holds the gang's MinReplicas")
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
	return nil
}
