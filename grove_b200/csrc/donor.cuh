// donor.cuh -- the donor set E(Q) of a class of grove_run_cycle_reclaim_queues (DESIGN.md section 1, "Reclaim across queues").
//
// Built once per call: the (queue X, running gang r) pairs of every queue X with a finite deserved quota, one per standing-or-not
// running gang r whose chain contains X, in victim order (lowest priority first, then the highest running index), with the depth
// of X in r's chain.  Per class only the queue loads and the gone mask change.  k_donor_scan gives every pair the verdicts
// ok_X(r) / over_X(r); k_donor_mark combines them over D(r, Q) = chain(queue(r)) \ chain(Q) into the evictable mask that
// k_reclaim_view reads.  No atomics: every (running gang, depth) byte has exactly one writer, and the result does not depend on
// thread order.
#pragma once
#include "common.cuh"

struct DonorSet {
  const uint32_t* q_off;              // [scanned + 1] first pair of each scanned queue
  const uint32_t* q_id;               // [scanned] its queue index
  const uint2* pr;                    // x = running gang, y = depth of the queue in its chain; victim order within a queue
  const unsigned long long* quota;    // [queue * 3 + resource] deserved, GROVE_QUEUE_UNLIMITED = none
  const long long* load;              // [queue * 3 + resource] the current loads
  const long long* use;               // [running * 3 + resource] what each running gang holds
  const uint32_t* parent;             // [queue] parent, GROVE_NONE_U32 = a root
  const uint32_t* rq;                 // [running] its queue, GROVE_NONE_U32 = none
  const uint8_t* fin;                 // [queue] 1: some resource has a finite quota (the queue is scanned)
  const uint8_t* gone;                // [running] 1: released or evicted
  uint8_t* bits;                      // [running * GROVE_MAX_QUEUE_DEPTH + depth] bit 0 ok, bit 1 over
};

// One CTA per scanned queue X: an inclusive scan, in victim order, of what the standing running gangs of X's subtree hold (three
// signed 64-bit sums at once); a standing pair r gets ok = load_X - P_X(r) >= deserved_X on every resource r holds with a finite
// quota, over = there is such a resource.
__global__ void __launch_bounds__(256) k_donor_scan(DonorSet d) {
  __shared__ long long s_w[8][3];
  const uint32_t X = d.q_id[blockIdx.x], tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  long long load[3], dq[3];
  bool fin[3];
#pragma unroll
  for (uint32_t k = 0; k < 3; ++k) {
    load[k] = d.load[X * 3 + k];
    fin[k] = d.quota[X * 3 + k] != GROVE_QUEUE_UNLIMITED;
    dq[k] = fin[k] ? (long long)d.quota[X * 3 + k] : 0;
  }
  long long c0 = 0, c1 = 0, c2 = 0;   // what the pairs of the earlier chunks hold (the same in every thread)
  for (uint32_t i0 = d.q_off[blockIdx.x], end = d.q_off[blockIdx.x + 1]; i0 < end; i0 += blockDim.x) {
    const uint32_t i = i0 + tid;
    bool in = false;
    uint2 p = make_uint2(0u, 0u);
    long long v0 = 0, v1 = 0, v2 = 0;
    if (i < end) {
      p = d.pr[i];
      in = !d.gone[p.x];
      if (in) { v0 = d.use[p.x * 3 + 0]; v1 = d.use[p.x * 3 + 1]; v2 = d.use[p.x * 3 + 2]; }
    }
    long long x0 = v0, x1 = v1, x2 = v2;   // inclusive warp scan
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const long long t0 = __shfl_up_sync(grove::kFull, x0, s), t1 = __shfl_up_sync(grove::kFull, x1, s);
      const long long t2 = __shfl_up_sync(grove::kFull, x2, s);
      if (lane >= uint32_t(s)) { x0 += t0; x1 += t1; x2 += t2; }
    }
    if (lane == 31) { s_w[warp][0] = x0; s_w[warp][1] = x1; s_w[warp][2] = x2; }
    __syncthreads();
    long long o0 = c0, o1 = c1, o2 = c2;
    for (uint32_t k = 0; k < (blockDim.x >> 5); ++k) {
      if (k < warp) { o0 += s_w[k][0]; o1 += s_w[k][1]; o2 += s_w[k][2]; }
      c0 += s_w[k][0]; c1 += s_w[k][1]; c2 += s_w[k][2];
    }
    if (in) {
      const long long P[3] = {o0 + x0, o1 + x1, o2 + x2}, v[3] = {v0, v1, v2};
      bool ok = true, over = false;
#pragma unroll
      for (uint32_t k = 0; k < 3; ++k)
        if (fin[k] && v[k] > 0) { over = true; ok &= load[k] - P[k] >= dq[k]; }
      d.bits[size_t(p.x) * GROVE_MAX_QUEUE_DEPTH + p.y] = uint8_t(ok) | uint8_t(over) << 1;
    }
    __syncthreads();   // (s_w is rewritten by the next chunk)
  }
}

// One thread per running gang: evict[r] = r is in E(Q).  r stands and has a queue, neither queue(r) nor Q lies in the other's
// chain, and over D(r, Q) every scanned queue says ok and at least one says over (a queue without a finite quota says ok, not over).
__global__ void __launch_bounds__(256) k_donor_mark(DonorSet d, uint32_t Q, uint32_t n_running, uint8_t* evict) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_running) return;
  bool e = false;
  const uint32_t qr = d.rq[r];
  if (!d.gone[r] && qr != GROVE_NONE_U32) {
    bool ok = true, over = false, apart = true;
    uint32_t X = qr;
    for (uint32_t k = 0; X != GROVE_NONE_U32; ++k, X = d.parent[X]) {
      bool shared = false;   // is X in chain(Q)?
      for (uint32_t y = Q; y != GROVE_NONE_U32; y = d.parent[y]) shared |= y == X;
      if (shared) { apart = k > 0 && X != Q; break; }   // queue(r) in chain(Q), or Q in chain(queue(r)): never a donor
      if (d.fin[X]) {
        const uint8_t b = d.bits[size_t(r) * GROVE_MAX_QUEUE_DEPTH + k];
        ok &= (b & 1u) != 0; over |= (b & 2u) != 0;
      }
    }
    e = apart && ok && over;
  }
  evict[r] = uint8_t(e);
}
