// queue.cuh -- queue limits (grove_set_queues; DESIGN.md section 1 "Queue limits"): the headroom each member of a queue with a
// finite limit meets at its turn, and from it the member's gate and the replicas its cliques may take.
#pragma once
#include "common.cuh"

namespace grove {

// The last member a round's bookkeeping has to cover: a member ranked at or beyond the end of the NEXT window is not evaluated
// next round, and k_detect moves the window's end by at most `entry` (relax.cuh k_detect).
__device__ __forceinline__ uint32_t queue_bound(const Tables& tb, const Relax& rx, uint32_t final_pass) {
  return final_pass ? tb.G : min(tb.G, rx.ctl[kHi] + rx.entry);
}

// One CTA per scanned queue: an exclusive scan, in rank order, of U(h) * [h tentatively ADMITTED] over the queue's pairs, three
// signed 64-bit sums at once; pair i gets H_Q = limit - load - (what the members before it hold).  The pairs of ranks at or beyond
// queue_bound are left alone (k_queue_gate does not read them).  In a round's chain after k_apply; before round 1 (every tentative
// state is empty: H_Q = limit - load) and after the cycle (final_pass = 1: every pair, over the final states).
__global__ void __launch_bounds__(256) k_queue_scan(Tables tb, Relax rx, uint32_t final_pass) {
  __shared__ long long s_w[8][3];
  cudaGridDependencySynchronize();   // (launched chained in a round: engine.cu launch_chained)
  if (!final_pass && rx.ctl[kDone]) return;
  const uint32_t q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t bound = queue_bound(tb, rx, final_pass);
  const long long b0 = rx.qu.q_base[q * 3 + 0], b1 = rx.qu.q_base[q * 3 + 1], b2 = rx.qu.q_base[q * 3 + 2];
  long long c0 = 0, c1 = 0, c2 = 0;   // what the pairs of the earlier chunks hold (the same in every thread)
  for (uint32_t i0 = rx.qu.q_off[q], end = rx.qu.q_off[q + 1]; i0 < end; i0 += blockDim.x) {
    const uint32_t i = i0 + tid;
    bool in = false;
    long long v0 = 0, v1 = 0, v2 = 0;
    if (i < end) {
      const uint4 p = rx.qu.pr[i];   // (one load, then the state and the usage side by side)
      in = p.z < bound;
      if (in) {
        const bool adm = rx.tstate[p.x] == GROVE_GANG_ADMITTED;
        const unsigned long long* u = rx.qu.use + size_t(p.y) * 3;
        const long long w0 = (long long)u[0], w1 = (long long)u[1], w2 = (long long)u[2];
        if (adm) { v0 = w0; v1 = w1; v2 = w2; }
      }
    }
    long long x0 = v0, x1 = v1, x2 = v2;   // inclusive warp scan
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const long long t0 = __shfl_up_sync(kFull, x0, d), t1 = __shfl_up_sync(kFull, x1, d), t2 = __shfl_up_sync(kFull, x2, d);
      if (lane >= uint32_t(d)) { x0 += t0; x1 += t1; x2 += t2; }
    }
    if (lane == 31) { s_w[warp][0] = x0; s_w[warp][1] = x1; s_w[warp][2] = x2; }
    __syncthreads();
    long long o0 = c0, o1 = c1, o2 = c2;
    for (uint32_t k = 0; k < (blockDim.x >> 5); ++k) {
      if (k < warp) { o0 += s_w[k][0]; o1 += s_w[k][1]; o2 += s_w[k][2]; }
      c0 += s_w[k][0]; c1 += s_w[k][1]; c2 += s_w[k][2];
    }
    if (in) {
      long long* h = rx.qu.head + size_t(i) * 3;
      h[0] = b0 - (o0 + x0 - v0); h[1] = b1 - (o1 + x1 - v1); h[2] = b2 - (o2 + x2 - v2);
    }
    // pairs are in rank order: once one is out of bound, so are the rest (the barrier also guards s_w)
    if (__syncthreads_or(i < end && !in)) break;
  }
}

// One thread per member ranked below queue_bound: H(g) = the least headroom over its chain (finite limits only), the gate, and
// clique by clique the replicas MinReplicas + s_q its surplus may reach (queue.cuh's arithmetic is DESIGN.md's, step by step).
// mode 0 (before round 1) and 1 (a round's chain): the values go where k_eval reads them; in mode 1 a member of the window whose
// (gate, caps) changed is marked dirty for k_detect (dirty rule (e)).  mode 2 (after the cycle, behind k_fin_status): the status
// flags of the members.
__global__ void __launch_bounds__(256) k_queue_gate(Tables tb, Relax rx, uint32_t mode, grove_gang_status_t* status) {
  cudaGridDependencySynchronize();
  if (mode != 2 && rx.ctl[kDone]) return;
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= rx.qu.n_mem) return;
  const uint32_t g = rx.qu.mem[j], rank = tb.ginfo[g].order;
  const uint32_t hi = rx.ctl[kHi];
  if (rank >= queue_bound(tb, rx, mode == 2)) return;
  const uint4 pr = rx.qu.mem_pair[j];
  const uint32_t fin = rx.qu.mem_fin[j];
  const uint32_t pair[4] = {pr.x, pr.y, pr.z, pr.w};
  const long long kNoLimit = 0x7FFFFFFFFFFFFFFFll;
  long long H[3] = {kNoLimit, kNoLimit, kNoLimit};
  uint32_t fmask = 0;   // resources with a finite limit somewhere in the chain
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k) {
    if (pair[k] == kFull) continue;
#pragma unroll
    for (uint32_t r = 0; r < 3; ++r)
      if ((fin >> (3 * k + r)) & 1u) { H[r] = min(H[r], rx.qu.head[size_t(pair[k]) * 3 + r]); fmask |= 1u << r; }
  }
  const long long R[3] = {rx.qu.rmin[j * 3 + 0], rx.qu.rmin[j * 3 + 1], rx.qu.rmin[j * 3 + 2]};
  bool closed = false;
#pragma unroll
  for (uint32_t r = 0; r < 3; ++r) closed |= ((fmask >> r) & 1u) && R[r] > 0 && R[r] > H[r];
  bool changed = closed != (rx.qu.gate[j] != 0), capped = false;
  if (!closed) {
    const grove_gang_t gg = tb.gangs[g];
    long long rem[3] = {H[0] - R[0], H[1] - R[1], H[2] - R[2]};
    for (uint32_t c = 0; c < gg.n_cliques; ++c) {
      const grove_clique_t q = tb.cliques[gg.clique_off + c];
      const uint32_t extra = uint32_t(q.replicas) - uint32_t(q.min_replicas);
      const long long req[3] = {(long long)q.req_cpu_milli, (long long)q.req_mem_mib, (long long)q.req_gpu};
      long long s = extra;
#pragma unroll
      for (uint32_t r = 0; r < 3; ++r)
        if (((fmask >> r) & 1u) && req[r] > 0) s = rem[r] < 0 ? 0 : min(s, rem[r] / req[r]);
#pragma unroll
      for (uint32_t r = 0; r < 3; ++r) rem[r] -= s * req[r];
      capped |= s < (long long)extra;
      const uint8_t cap = uint8_t(uint32_t(q.min_replicas) + uint32_t(s));
      if (mode != 2 && rx.qu.cap[gg.clique_off + c] != cap) { rx.qu.cap[gg.clique_off + c] = cap; changed = true; }
    }
  }
  if (mode == 2) {
    const uint32_t t = rx.tstate[g];
    if (t == GROVE_GANG_REJECTED && closed) status[g].reserved0 |= GROVE_STATUS_OVER_LIMIT;
    if (t == GROVE_GANG_ADMITTED && capped) status[g].reserved0 |= GROVE_STATUS_SURPLUS_CAPPED;
    return;
  }
  if (changed) {
    rx.qu.gate[j] = uint8_t(closed);
    if (mode == 1 && rank < hi) rx.dirty[g] = 1;   // evaluated with other (gate, caps): again next round
  }
}

}  // namespace grove
