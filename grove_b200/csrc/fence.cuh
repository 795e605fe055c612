// fence.cuh -- fences (grove_set_fences; DESIGN.md section 1 "Fences"): the domain each fencing gang keeps the gangs ranked after
// it out of while it is REJECTED, picked once when the cycle starts.
#pragma once
#include "common.cuh"
#include "diagnose.cuh"

namespace grove {

// Cycle start, over the committed table F0: grid = (npad / 256 node tiles, fencing gangs).  For every clique q of fencing gang k
// with MinReplicas m > 0 and every domain D of the gang's Required level l: have[k][q][D] = sum over n in D of min(cap(q, n), m),
// cap the exact capacity of grove_diagnose (0 where K1 fit fails).  The lanes of a warp that share a domain are one
// __match_any_sync segment (sorted order keeps a domain contiguous).  `have` is zeroed by the host.
__global__ void __launch_bounds__(256) k_fence_have(Topo tp, Tables tb, const uint32_t* __restrict__ gang,
                                                    const uint32_t* __restrict__ off, uint32_t* have) {
  const uint32_t gi = gang[blockIdx.y];
  const grove_gang_t g = tb.gangs[gi];
  const uint32_t lane = threadIdx.x & 31, node = blockIdx.x * blockDim.x + threadIdx.x, nd = tp.n_dom[g.level];
  const bool valid = node < tp.n;
  const uint4 r = valid ? tp.nres[node] : make_uint4(0, 0, 0, 0);
  const uint32_t key = valid ? diag_domain(tp, node, g.level) : GROVE_DOM_ABSENT;
  const uint32_t seg = __match_any_sync(kFull, key);
  const bool leader = key != GROVE_DOM_ABSENT && lane == uint32_t(__ffs(seg) - 1);
  for (uint32_t c = 0; c < g.n_cliques; ++c) {
    const uint32_t qi = g.clique_off + c;
    const grove_clique_t q = tb.cliques[qi];
    if (!q.min_replicas) continue;   // (uniform: one gang per CTA row)
    uint32_t cap = 0;
    if (valid) diag_fit(r, q, tb.cinfo[qi].need_depth, cap);
    const uint32_t s = __reduce_add_sync(seg, min(cap, uint32_t(q.min_replicas)));
    if (leader && s) atomicAdd(have + off[blockIdx.y] + size_t(c) * nd + key, s);
  }
}

// One CTA, after k_fence_have: the picks in rank order.  Fencing gang k takes, among the level-l domains that share no node with
// an earlier pick, the one with the least shortfall = sum over its cliques of max(0, m - have); ties by its candidate order at
// level l (descending min(closeness(first node, anchor), l + 1), then ascending rotated index of the first node).  One 64-bit key
// per domain, a block minimum per gang.  Then `list` = the picks sorted by first node (no pick: lo = hi = kFull, last) and `slot`.
__global__ void __launch_bounds__(1024) k_fence_pick(Topo tp, Tables tb, const uint32_t* __restrict__ gang,
                                                     const uint32_t* __restrict__ off, const uint32_t* __restrict__ have, uint32_t n,
                                                     uint4* list, uint32_t* slot) {
  __shared__ unsigned long long s_min[32];
  __shared__ uint32_t s_lo[GROVE_MAX_FENCES], s_hi[GROVE_MAX_FENCES];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t k = 0; k < n; ++k) {
    const uint32_t gi = gang[k];
    const grove_gang_t g = tb.gangs[gi];
    const uint32_t l = g.level, nd = tp.n_dom[l], a = tb.ginfo[gi].anchor;
    const uint4 da = tp.ndom[a];
    const uint32_t ax[GROVE_MAX_LEVELS] = {da.x, da.y, da.z, da.w};
    unsigned long long best = ~0ull;
    for (uint32_t d = tid; d < nd; d += blockDim.x) {
      const uint32_t lo = tp.dom_lo[l][d], hi = tp.dom_hi[l][d];
      bool taken = false;
      for (uint32_t j = 0; j < k; ++j) taken |= s_lo[j] != kFull && lo < s_hi[j] && s_lo[j] < hi;
      if (taken) continue;
      uint32_t short_by = 0;
      for (uint32_t c = 0; c < g.n_cliques; ++c) {
        const uint32_t m = tb.cliques[g.clique_off + c].min_replicas;
        if (!m) continue;
        const uint32_t h = have[off[k] + size_t(c) * nd + d];
        short_by += m > h ? m - h : 0u;
      }
      const uint4 dn = tp.ndom[lo];
      const uint32_t nx[GROVE_MAX_LEVELS] = {dn.x, dn.y, dn.z, dn.w};
      uint32_t close = 0;
#pragma unroll
      for (uint32_t x = 0; x < GROVE_MAX_LEVELS; ++x) close += x < tp.L && nx[x] != GROVE_DOM_ABSENT && nx[x] == ax[x];
      const uint32_t sc = min(close, l + 1u), rot = (lo + tp.n - a) % tp.n;
      best = min(best, (static_cast<unsigned long long>(short_by) << 32) | (uint64_t(7u - sc) << 24) | rot);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) best = min(best, __shfl_xor_sync(kFull, best, o));
    if (lane == 0) s_min[warp] = best;
    __syncthreads();
    if (tid == 0) {
      for (uint32_t w = 1; w < (blockDim.x >> 5); ++w) best = min(best, s_min[w]);
      s_lo[k] = s_hi[k] = kFull;
      if (best != ~0ull) {   // the rotated index names the domain's first node
        const uint32_t lo = (uint32_t(best & 0xFFFFFFu) + a) % tp.n;
        const uint4 dn = tp.ndom[lo];
        const uint32_t d = l == 0 ? dn.x : l == 1 ? dn.y : l == 2 ? dn.z : dn.w;
        s_lo[k] = lo; s_hi[k] = tp.dom_hi[l][d];
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    for (uint32_t k = 0; k < n; ++k) {   // insertion by first node (at most GROVE_MAX_FENCES entries)
      const uint4 e = make_uint4(s_lo[k], s_hi[k], tb.ginfo[gang[k]].order, gang[k]);
      uint32_t j = k;
      for (; j > 0 && list[j - 1].x > e.x; --j) list[j] = list[j - 1];
      list[j] = e;
    }
    for (uint32_t j = 0; j < n; ++j) slot[list[j].w] = j;
  }
}

// After k_fin_status: a REJECTED gang whose fence was active at the end carries GROVE_STATUS_FENCING, its level and the caller
// index of the fenced domain's first node.  A thread per fence.
__global__ void k_fence_status(Tables tb, Relax rx, const uint32_t* __restrict__ perm, grove_gang_status_t* status) {
  const uint32_t j = threadIdx.x;
  if (j >= rx.fc.n) return;
  const uint4 f = rx.fc.list[j];
  if (f.x == kFull || rx.state[f.w] != GROVE_GANG_REJECTED) return;
  grove_gang_status_t& s = status[f.w];
  s.reserved0 |= GROVE_STATUS_FENCING;
  s.level = tb.gangs[f.w].level;
  s.domain_node = perm[f.x];
}

}  // namespace grove
