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
}

type result struct {
	placements []C.grove_placement_t
	status     []C.grove_gang_status_t
	victims    []C.grove_victim_t
	stats      C.grove_cycle_stats_t
}

// cycle runs one scheduling cycle.  All slices are Go memory: the library copies them before each call returns and
// keeps no pointer (cgo pointer-passing rules); outputs are written into Go slices.
func (e *engine) cycle(t *tables, preempt, large bool) (*result, error) {
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
	r := &result{}
	if preempt && len(t.running) > 0 {
		var hp *C.grove_holding_t
		if len(t.holdings) > 0 {
			hp = &t.holdings[0]
		}
		if err := e.err(C.grove_run_cycle_preempt(e.h, &t.running[0], C.uint32_t(len(t.running)), hp,
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
	return r, nil
}
