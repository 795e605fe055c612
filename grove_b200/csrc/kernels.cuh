// kernels.cuh -- sm_90a kernels of the gang-placement cycle (umbrella include).
//
//   tables.cuh   k_gather / k_scatter / k_update / k_anchor               table (un)packing
//   fit.cuh      k_fit  K1  node x clique-signature resource-fit bitmap   (Filter; oracle: fit())
//                k_cap8 / k_capsum  per-signature pod capacities and their per-domain sum / max
//   score.cuh    k_score K2 topology-distance score matrix, u8            (Score;  oracle: closeness())
//   admit.cuh    k_eval  K3  one gang against its view: all-or-nothing admission, warp-cooperative packing
//   relax.cuh    k_select / k_apply / k_detect / k_fold    the relaxation that makes the evaluations of all gangs
//                agree with the sequential, priority-ordered pass; k_fin_* / k_emit  outputs
//   reclaim.cuh  k_reclaim_*  reclaim-class views over the running gangs' holdings (grove_run_cycle_reuse_preempt)
//   donor.cuh    k_donor_scan / k_donor_mark  the donor set of a reclaim-across-queues class (grove_run_cycle_reclaim_queues)
//   diagnose.cuh k_diag_*  why each rejected gang did not fit, after the cycle (grove_diagnose)
//   spread.cuh   k_spread_classes / k_spread  allowed level-l_s domains of the topology spread members (grove_set_spread)
//   fence.cuh    k_fence_have / k_fence_pick / k_fence_status  the domain each fencing gang fences (grove_set_fences)
//   consolidate.cuh k_consol_view / k_consol_rank / k_consol_mask  the views of a consolidation try (grove_run_cycle_consolidate)
//   queue.cuh    k_queue_scan / k_queue_gate  the headroom, gate and surplus caps of the queue members (grove_set_queues)
//   fairshare.cuh k_fs_init / k_fs_gather / k_fs_key / k_fs_diff  the turn order of a fair-share cycle (grove_set_fair_share), with
//                cub's segmented scans and stable merge sort
//   binpack.cuh  k_binpack_sum / k_binpack_keys / k_binpack_pick  the fullest domain each bin-packing member is anchored at
//                (grove_set_binpack)
//   imex.cuh     imex_foreign  which nodes another ComputeDomain holds in a gang's view (grove_set_compute_domains; the kImex
//                instantiations of k_eval / k_apply / k_fold)
//
// Semantics are DESIGN.md "Placement semantics"; the reference contract they restate is cited in
// include/grove_place.h.  Integer / compare work only: no tensor cores, no floating point.
#pragma once
#include "common.cuh"
#include "tables.cuh"
#include "fit.cuh"
#include "score.cuh"
#include "admit.cuh"
#include "relax.cuh"
#include "reclaim.cuh"
#include "donor.cuh"
#include "fairshare.cuh"
#include "diagnose.cuh"
#include "spread.cuh"
#include "fence.cuh"
#include "consolidate.cuh"
#include "queue.cuh"
#include "binpack.cuh"
