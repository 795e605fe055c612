// overquota.cuh -- the fair shares of a queue tree under over-quota weights (DESIGN.md section 1, "Over-quota weight").
//
// A queue's fair share is its deserved quota plus a slice of the capacity nobody deserves, divided among siblings by their
// over-quota weights and capped by what each asks for (after KAI-Scheduler's proportion plugin, in integers).  Three steps, all
// per resource: the demand of every queue (its starting load plus the requests of the non-gated gangs of its subtree: one thread
// per gang, 64-bit integer atomics, so the sums do not depend on thread order); the capacity (one block over the node table); and
// the division, top-down, one CTA per parent with children and one launch per depth.  Every quantity saturates at kOqClamp =
// 2^62, as the queue tables do.  Tree node ids: the queues 0..NQ-1, NQ = the root.
#pragma once
#include "common.cuh"

constexpr unsigned long long kOqClamp = 1ull << 62;

struct OqTree {
  const uint32_t* parent;              // [queue] parent queue, GROVE_NONE_U32 = top level
  const uint32_t* child_off;           // [node] first child in `child` (NQ + 2 entries)
  const uint32_t* child;               // children of each node, ascending
  const uint32_t* plist;               // the nodes with children, by depth (the root first)
  const unsigned long long* deserved;  // [queue * 3 + r], GROVE_QUEUE_UNLIMITED = none
  const unsigned long long* limit;     // [queue * 3 + r], GROVE_QUEUE_UNLIMITED = none
  const uint32_t* weight;              // [queue * 3 + r] over-quota weight
  unsigned long long* demand;          // [queue * 3 + r] starting load on entry, + the subtree's requests after k_oq_demand
  unsigned long long* pool;            // [node * 3 + r] what a node's children divide (the root's: the capacity)
  unsigned long long* need;            // [queue * 3 + r] scratch of the water-fill
  unsigned long long* fair;            // [queue * 3 + r] the result
};

__device__ __forceinline__ unsigned long long oq_sat(unsigned long long a, unsigned long long b) {
  return a + b >= kOqClamp ? kOqClamp : a + b;   // (a, b <= 2^63: no wrap)
}

// every non-gated gang with a queue adds replicas * request of each of its cliques into every queue of its chain
__global__ void k_oq_demand(OqTree t, const grove_gang_t* __restrict__ gangs, const grove_clique_t* __restrict__ cliques,
                            const uint32_t* __restrict__ gang_queue, uint32_t G) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G || gang_queue[g] == GROVE_NONE_U32 || (gangs[g].flags & GROVE_GANG_GATED)) return;
  const grove_gang_t gg = gangs[g];
  unsigned long long s[3] = {0ull, 0ull, 0ull};
  for (uint32_t c = 0; c < gg.n_cliques; ++c) {
    const grove_clique_t q = cliques[gg.clique_off + c];
    s[0] += (unsigned long long)q.replicas * q.req_cpu_milli;
    s[1] += (unsigned long long)q.replicas * q.req_mem_mib;
    s[2] += (unsigned long long)q.replicas * q.req_gpu;
  }
  for (uint32_t X = gang_queue[g]; X != GROVE_NONE_U32; X = t.parent[X])
    for (int r = 0; r < 3; ++r) if (s[r]) atomicAdd(&t.demand[X * 3 + r], s[r]);
}

// the root's pool += the free cpu, mem, gpu of every schedulable node (one block; the host put the top-level loads there)
__global__ void k_oq_capacity(OqTree t, const uint4* __restrict__ nres, uint32_t n, uint32_t root) {
  __shared__ unsigned long long part[3][32];
  unsigned long long s[3] = {0ull, 0ull, 0ull};
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uint4 x = nres[i];
    if (!(x.w & GROVE_NODE_SCHEDULABLE)) continue;
    s[0] += x.x; s[1] += x.y; s[2] += x.z & 0xFFFFu;
  }
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (int r = 0; r < 3; ++r) {
    for (int o = 16; o; o >>= 1) s[r] += __shfl_down_sync(0xFFFFFFFFu, s[r], o);
    if (!lane) part[r][warp] = s[r];
  }
  __syncthreads();
  if (threadIdx.x) return;
  for (int r = 0; r < 3; ++r) {
    unsigned long long c = 0ull;
    for (uint32_t w = 0; w < (blockDim.x + 31) / 32; ++w) c += part[r][w];
    t.pool[root * 3 + r] = oq_sat(t.pool[root * 3 + r], c >= kOqClamp ? kOqClamp : c);
  }
}

// block-wide sum, saturating at 2^63 (associative for these non-negative terms); every thread gets the result
__device__ __forceinline__ unsigned long long oq_block_sum(unsigned long long v, unsigned long long* red) {
  constexpr unsigned long long kCap = 1ull << 63;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (int o = 16; o; o >>= 1) { const unsigned long long x = __shfl_down_sync(0xFFFFFFFFu, v, o); v = v + x >= kCap ? kCap : v + x; }
  __syncthreads();   // (red is re-used from one call to the next)
  if (!lane) red[warp] = v;
  __syncthreads();
  unsigned long long s = 0ull;
  for (uint32_t w = 0; w < blockDim.x / 32; ++w) s = s + red[w] >= kCap ? kCap : s + red[w];
  return s;
}

// The division at the parents of one depth: blockIdx.x picks the parent in plist[first + blockIdx.x]; per resource, each child
// takes base = min(deserved, demand, limit) -- an unlimited child takes min(demand, limit) and reports GROVE_QUEUE_UNLIMITED --
// and what is left of the pool is water-filled over the children with a weight and some need left, in proportion to their weights
// (floor(R * w / W), 128-bit products), until a round gives nothing; the leftover R < |A| then goes one unit each in (weight desc,
// queue asc) order.  A child's pool for its own children is its fair share (min(demand, limit) when unlimited).
__global__ void __launch_bounds__(256) k_oq_fill(OqTree t, uint32_t first) {
  __shared__ unsigned long long red[8];
  const uint32_t p = t.plist[first + blockIdx.x];
  const uint32_t lo = t.child_off[p], hi = t.child_off[p + 1];
  for (int r = 0; r < 3; ++r) {
    unsigned long long took = 0ull;
    for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      const uint32_t c = t.child[i], k = c * 3 + r;
      const unsigned long long d = t.demand[k] >= kOqClamp ? kOqClamp : t.demand[k], lim = t.limit[k], q = t.deserved[k];
      const unsigned long long want = d < lim ? d : lim;
      if (q == GROVE_QUEUE_UNLIMITED) {
        t.fair[k] = GROVE_QUEUE_UNLIMITED; t.pool[k] = want; t.need[k] = 0ull;
        took = oq_sat(took, want);
      } else {
        const unsigned long long base = q < want ? q : want;
        t.fair[k] = base; t.need[k] = want - base;
        took = oq_sat(took, base);
      }
    }
    const unsigned long long P = t.pool[p * 3 + r], S = oq_block_sum(took, red);
    unsigned long long R = P > S ? P - S : 0ull;
    for (;;) {   // one round: every child of A gets min(need, floor(R * w / W)) of the same R
      unsigned long long w = 0ull;
      for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const uint32_t k = t.child[i] * 3 + r;
        if (t.deserved[k] != GROVE_QUEUE_UNLIMITED && t.need[k] && t.weight[k]) w += t.weight[k];
      }
      const unsigned long long W = oq_block_sum(w, red);
      if (!W || !R) break;
      unsigned long long given = 0ull;
      for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const uint32_t k = t.child[i] * 3 + r;
        if (t.deserved[k] == GROVE_QUEUE_UNLIMITED || !t.need[k] || !t.weight[k]) continue;
        const unsigned long long slice = (unsigned long long)((unsigned __int128)R * t.weight[k] / W);
        const unsigned long long x = slice < t.need[k] ? slice : t.need[k];
        t.fair[k] += x; t.need[k] -= x; given += x;
      }
      const unsigned long long got = oq_block_sum(given, red);
      if (!got) break;
      R -= got;
    }
    // the leftover: R < |A| units, one each to the first R members of A in (weight desc, queue asc) order.  Each thread ranks its
    // own children by a scan over all siblings: O(children^2) per parent, at most 4096^2 / 256 = 64 Ki steps a thread at
    // GROVE_MAX_QUEUES children, and only when a leftover remains
    if (R) {
      for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const uint32_t c = t.child[i], k = c * 3 + r;
        if (t.deserved[k] == GROVE_QUEUE_UNLIMITED || !t.need[k] || !t.weight[k]) continue;
        unsigned long long before = 0ull;
        for (uint32_t j = lo; j < hi && before < R; ++j) {
          const uint32_t c2 = t.child[j], k2 = c2 * 3 + r;
          if (t.deserved[k2] == GROVE_QUEUE_UNLIMITED || !t.need[k2] || !t.weight[k2]) continue;
          before += t.weight[k2] > t.weight[k] || (t.weight[k2] == t.weight[k] && c2 < c);
        }
        if (before < R) t.fair[k] += 1ull;   // (need >= 1: no one is pushed past min(demand, limit))
      }
    }
    __syncthreads();   // every fair[k] of this resource is final before a thread reads another child's need
    for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      const uint32_t k = t.child[i] * 3 + r;
      if (t.deserved[k] != GROVE_QUEUE_UNLIMITED) t.pool[k] = t.fair[k];
    }
  }
}
