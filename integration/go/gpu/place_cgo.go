// Package gpu is the `gpu-scheduler` backend of the Grove operator: the third case of newBackendForProfile
// (operator/internal/scheduler/manager/manager.go:35-52).  It places PodGangs in-process through libgrove_place.so
// (include/grove_place.h of the grove_b200 repository).
//
// NOT COMPILED IN THE BUILD IMAGE OF THAT REPOSITORY (no Go toolchain there): this is the binding a maintainer drops into
// operator/internal/scheduler/gpu/.  Its C side -- every entry point and struct used below -- is compiled, loaded and
// tested (tests/test_abi.py probes every struct offset; the C++ mirror grove_b200/csrc/host/ runs the same call
// sequence on the GPU).
package gpu

/*
#cgo CFLAGS: -I${SRCDIR}/../../../../third_party/grove_b200/include
#cgo LDFLAGS: -L${SRCDIR}/../../../../third_party/grove_b200 -lgrove_place -lcudart
#include "grove_place.h"
*/
import "C"

import (
	"fmt"
	"sync"
)

// engine wraps one grove_engine_t handle.  A handle is not thread-safe (one cycle in flight): every call takes mu.
// SyncPodGang reconciles run concurrently (controller/podgang/register.go:34-36) and only touch the pending set.
type engine struct {
	mu sync.Mutex
	h  *C.grove_engine_t
}

func newEngine(device, nLevels int) (*engine, error) {
	cfg := C.grove_config_t{abi_version: C.GROVE_ABI_VERSION, device: C.int32_t(device), n_levels: C.uint32_t(nLevels)}
	var h *C.grove_engine_t
	if rc := C.grove_engine_create(&cfg, &h); rc != C.GROVE_OK {
		return nil, fmt.Errorf("grove_engine_create: %d (the engine has no CPU fallback)", int(rc))
	}
	return &engine{h: h}, nil
}

func (e *engine) close() { C.grove_engine_destroy(e.h) }

func (e *engine) err(rc C.int32_t) error {
	if rc == C.GROVE_OK {
		return nil
	}
	return fmt.Errorf("grove_place: %d: %s", int(rc), C.GoString(C.grove_last_error(e.h)))
}

// tables is one cycle's input, packed (INTEGRATION.md section 3 says which PodGang field lands where).
type tables struct {
	nodes   []C.grove_node_t
	gangs   []C.grove_gang_t
	cliques []C.grove_clique_t
	counts  []C.grove_clique_count_t // per clique: MinReplicas / replicas, read by grove_submit_gangs_wide (large PodGangs)
	scopes  []C.grove_scope_t
	// reclaim pass (optional): PodGangs this backend scheduled earlier and what they hold per node
	running  []C.grove_running_gang_t
	holdings []C.grove_holding_t
	// topology spread (optional; never together with the reclaim pass): the groups, each gang row's group (GROVE_NONE_U32 =
	// none) and the running replicas
	spreadGroups []C.grove_spread_t
	spreadOf     []C.uint32_t
	spreadSeeds  []C.grove_spread_seed_t
	// fences (optional; ordinary passes only): the gang rows the starvation guard fences (grove_set_fences)
	fences []C.uint32_t
	// bin-packing (optional; ordinary and queue passes only): each gang row's pack level (grove_set_binpack)
	binpack []C.uint8_t
	// ComputeDomain exclusivity (optional; ordinary passes only): each clique row's ComputeDomain (GROVE_CD_NONE: not enrolled)
	// and each node's holder when the pass starts (grove_set_compute_domains)
	cd, owner0 []C.uint32_t
	// queue limits (optional; ordinary passes only): the queues, parents first, each gang row's queue (GROVE_NONE_U32 = none) and
	// the queue names in table order (grove_set_queues)
	queues     []C.grove_queue_t
	queueOf    []C.uint32_t
	// reclaim within queue limits: the queue of each running gang of `running` (GROVE_NONE_U32: none); set only in a pass with
	// preemption and queue members
	runningQueue []C.uint32_t
	// reclaim across queues: each queue's deserved quota, in `queues` order; set only with SetReclaimAcrossQueues
	quotas []C.grove_queue_quota_t
	// reclaim, then preempt: with quotas and runningQueue, both passes in one grove_run_cycle_reclaim_preempt_queues; set only
	// with SetReclaimThenPreempt and preemption
	thenPreempt bool
	// fair-share order: each queue's deserved quota, in `queues` order (grove_set_fair_share); set only with SetFairShareOrder in a
	// pass with queue members and no preemption
	fairShare []C.grove_queue_quota_t
	queueNames []string
	// consolidation (optional; ordinary passes only, never with fences): the target rows, and for each running gang of `running`
	// the gated row that restates it (grove_run_cycle_consolidate)
	targets []C.uint32_t
	specOf  []C.uint32_t
}

type result struct {
	placements []C.grove_placement_t
	status     []C.grove_gang_status_t
	victims    []C.grove_victim_t
	moves      []C.grove_move_t // consolidation: (running gang, target row) per relocated gang
	stats      C.grove_cycle_stats_t
	// explain, after an ordinary cycle with a rejected gang: why each rejected gang did not fit (grove_diagnose)
	gangDiag   []C.grove_gang_diag_t
	cliqueDiag []C.grove_clique_diag_t
}

// cycle runs one scheduling cycle.  All slices are Go memory: the library copies them before each call returns and
// keeps no pointer (cgo pointer-passing rules); outputs are written into Go slices.
func (e *engine) cycle(t *tables, preempt, large, explain bool) (*result, error) {
	e.mu.Lock()
	defer e.mu.Unlock()
	if len(t.nodes) == 0 || len(t.gangs) == 0 {
		return &result{}, nil
	}
	if err := e.err(C.grove_load_nodes(e.h, &t.nodes[0], C.uint32_t(len(t.nodes)))); err != nil {
		return nil, err
	}
	if large {
		if err := e.err(C.grove_submit_gangs_wide(e.h, &t.gangs[0], C.uint32_t(len(t.gangs)), &t.cliques[0], &t.counts[0],
			C.uint32_t(len(t.cliques)), &t.scopes[0], C.uint32_t(len(t.scopes)))); err != nil {
			return nil, err
		}
	} else if err := e.err(C.grove_submit_gangs(e.h, &t.gangs[0], C.uint32_t(len(t.gangs)), &t.cliques[0],
		C.uint32_t(len(t.cliques)), &t.scopes[0], C.uint32_t(len(t.scopes)))); err != nil {
		return nil, err
	}
	if len(t.spreadGroups) > 0 {
		var sp *C.grove_spread_seed_t
		if len(t.spreadSeeds) > 0 {
			sp = &t.spreadSeeds[0]
		}
		if err := e.err(C.grove_set_spread(e.h, &t.spreadGroups[0], C.uint32_t(len(t.spreadGroups)), &t.spreadOf[0],
			C.uint32_t(len(t.spreadOf)), sp, C.uint32_t(len(t.spreadSeeds)))); err != nil {
			return nil, err
		}
	}
	if len(t.fences) > 0 {
		if err := e.err(C.grove_set_fences(e.h, &t.fences[0], C.uint32_t(len(t.fences)))); err != nil {
			return nil, err
		}
	}
	if len(t.binpack) > 0 {
		if err := e.err(C.grove_set_binpack(e.h, &t.binpack[0], C.uint32_t(len(t.binpack)))); err != nil {
			return nil, err
		}
	}
	if len(t.cd) > 0 {
		if err := e.err(C.grove_set_compute_domains(e.h, &t.cd[0], C.uint32_t(len(t.cd)), &t.owner0[0], C.uint32_t(len(t.owner0)))); err != nil {
			return nil, err
		}
	}
	if len(t.queues) > 0 {
		if err := e.err(C.grove_set_queues(e.h, &t.queues[0], C.uint32_t(len(t.queues)), &t.queueOf[0], C.uint32_t(len(t.queueOf)))); err != nil {
			return nil, err
		}
	}
	r := &result{}
	if preempt && len(t.running) > 0 {
		var hp *C.grove_holding_t
		if len(t.holdings) > 0 {
			hp = &t.holdings[0]
		}
		if len(t.runningQueue) > 0 && len(t.quotas) > 0 && t.thenPreempt {
			if err := e.err(C.grove_run_cycle_reclaim_preempt_queues(e.h, &t.quotas[0], C.uint32_t(len(t.quotas)), &t.running[0],
				C.uint32_t(len(t.running)), hp, C.uint32_t(len(t.holdings)), &t.runningQueue[0], &r.stats)); err != nil {
				return nil, err
			}
		} else if len(t.runningQueue) > 0 && len(t.quotas) > 0 {
			if err := e.err(C.grove_run_cycle_reclaim_queues(e.h, &t.quotas[0], C.uint32_t(len(t.quotas)), &t.running[0],
				C.uint32_t(len(t.running)), hp, C.uint32_t(len(t.holdings)), &t.runningQueue[0], &r.stats)); err != nil {
				return nil, err
			}
		} else if len(t.runningQueue) > 0 {
			if err := e.err(C.grove_run_cycle_preempt_queues(e.h, &t.running[0], C.uint32_t(len(t.running)), hp,
				C.uint32_t(len(t.holdings)), &t.runningQueue[0], &r.stats)); err != nil {
				return nil, err
			}
		} else if err := e.err(C.grove_run_cycle_preempt(e.h, &t.running[0], C.uint32_t(len(t.running)), hp,
			C.uint32_t(len(t.holdings)), &r.stats)); err != nil {
			return nil, err
		}
		var n C.uint32_t
		if err := e.err(C.grove_get_victims(e.h, nil, 0, &n)); err != nil {
			return nil, err
		}
		if n > 0 {
			r.victims = make([]C.grove_victim_t, int(n))
			if err := e.err(C.grove_get_victims(e.h, &r.victims[0], n, &n)); err != nil {
				return nil, err
			}
		}
	} else if len(t.targets) > 0 && len(t.running) > 0 {
		var hp *C.grove_holding_t
		if len(t.holdings) > 0 {
			hp = &t.holdings[0]
		}
		if err := e.err(C.grove_run_cycle_consolidate(e.h, &t.targets[0], C.uint32_t(len(t.targets)), &t.specOf[0], &t.running[0],
			C.uint32_t(len(t.running)), hp, C.uint32_t(len(t.holdings)), &r.stats)); err != nil {
			return nil, err
		}
		var n C.uint32_t
		if err := e.err(C.grove_get_moves(e.h, nil, 0, &n)); err != nil {
			return nil, err
		}
		if n > 0 {
			r.moves = make([]C.grove_move_t, int(n))
			if err := e.err(C.grove_get_moves(e.h, &r.moves[0], n, &n)); err != nil {
				return nil, err
			}
		}
	} else if len(t.fairShare) > 0 && len(t.queues) > 0 {
		if err := e.err(C.grove_set_fair_share(e.h, &t.fairShare[0], C.uint32_t(len(t.fairShare)))); err != nil {
			return nil, err
		}
		if err := e.err(C.grove_run_cycle(e.h, &r.stats)); err != nil {
			return nil, err
		}
	} else if err := e.err(C.grove_run_cycle(e.h, &r.stats)); err != nil {
		return nil, err
	}
	r.placements = make([]C.grove_placement_t, int(r.stats.pods_bound)+1)
	var n C.uint32_t
	if err := e.err(C.grove_get_placements(e.h, &r.placements[0], C.uint32_t(len(r.placements)), &n)); err != nil {
		return nil, err
	}
	r.placements = r.placements[:n]
	r.status = make([]C.grove_gang_status_t, len(t.gangs))
	if err := e.err(C.grove_get_gang_status(e.h, &r.status[0], C.uint32_t(len(r.status)))); err != nil {
		return nil, err
	}
	if explain && len(t.running) == 0 { // the running-gang cycles judge gangs against other views: grove_diagnose refuses them
		for _, st := range r.status {
			if st.state != C.GROVE_GANG_REJECTED {
				continue
			}
			gd := make([]C.grove_gang_diag_t, len(t.gangs))
			qd := make([]C.grove_clique_diag_t, len(t.cliques))
			// a failed diagnosis leaves the messages as they were: it never costs the cycle its bindings
			if C.grove_diagnose(e.h, &gd[0], C.uint32_t(len(gd)), &qd[0], C.uint32_t(len(qd))) == C.GROVE_OK {
				r.gangDiag, r.cliqueDiag = gd, qd
			}
			break
		}
	}
	return r, nil
}
