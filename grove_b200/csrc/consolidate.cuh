// consolidate.cuh -- the device views of grove_run_cycle_consolidate (DESIGN.md section 1, "Consolidation").
//
// The running gangs' holdings are the CSR of reclaim.cuh; its `gone` mask marks the running gangs that cannot move (no spec row)
// or have moved this cycle.  Per target b of priority p: k_consol_view keeps the free table F aside and builds W = F + the
// holdings of the standing movable gangs of priority <= p; k_fence_have (fence.cuh, unchanged) sums the capacities of b's
// cliques per level-l domain once over F and once over W; k_consol_rank picks the domains to try; k_consol_mask turns W into
// the view of one try.
#pragma once
#include "common.cuh"
#include "reclaim.cuh"

namespace grove {

constexpr uint32_t kConsolTries = GROVE_CONSOLIDATE_TRIES;

// real = F (the table as it is), view = F + the standing movable holdings of priority <= p.  One thread per node sums its own
// row (no atomics); k_reclaim_check ruled out a carry between the gpu and pods halves.
__global__ void __launch_bounds__(256) k_consol_view(const uint4* nres, uint4* real, uint4* view, ReclaimCsr c, uint32_t N, int32_t p) {
  const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  uint32_t s0 = 0, s1 = 0, s2 = 0;
  for (uint32_t i = c.off[n]; i < c.off[n + 1]; ++i) {
    const uint4 h = c.ent[i];
    if (!c.gone[h.x] && c.prio[h.x] <= p) { s0 += h.y; s1 += h.z; s2 += h.w; }
  }
  uint4 r = nres[n];
  real[n] = r;
  r.x += s0; r.y += s1; r.z += s2;
  view[n] = r;
}

// One CTA, after k_fence_have over F (haveF) and over W (haveW) for gang `gi` of the loaded tables, of Required level l and
// sorted anchor a.  A level-l domain qualifies when every clique with MinReplicas m > 0 has m in W; the qualifying domains are
// taken in the order of the 64-bit key of k_fence_pick (shortfall over F, then the candidate order at level l), at most
// kConsolTries of them, by repeated block minima.  out[0] = count, then (lo, hi) sorted node ranges.
__global__ void __launch_bounds__(1024) k_consol_rank(Topo tp, Tables tb, uint32_t gi, uint32_t a, const uint32_t* __restrict__ haveF,
                                                      const uint32_t* __restrict__ haveW, uint32_t* out) {
  __shared__ unsigned long long s_min[32];
  __shared__ unsigned long long s_prev;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const grove_gang_t g = tb.gangs[gi];
  const uint32_t l = g.level, nd = tp.n_dom[l];
  const uint4 da = tp.ndom[a];
  const uint32_t ax[GROVE_MAX_LEVELS] = {da.x, da.y, da.z, da.w};
  if (tid == 0) { s_prev = 0; out[0] = 0; }
  __syncthreads();
  for (uint32_t t = 0; t < kConsolTries; ++t) {
    const unsigned long long prev = s_prev;
    unsigned long long best = ~0ull;
    for (uint32_t d = tid; d < nd; d += blockDim.x) {
      uint32_t short_f = 0;
      bool ok = true;
      for (uint32_t c = 0; c < g.n_cliques; ++c) {
        const uint32_t m = tb.cliques[g.clique_off + c].min_replicas;
        if (!m) continue;
        const uint32_t hf = haveF[size_t(c) * nd + d], hw = haveW[size_t(c) * nd + d];
        short_f += m > hf ? m - hf : 0u;
        ok &= hw >= m;
      }
      if (!ok) continue;
      const uint32_t lo = tp.dom_lo[l][d];
      const uint4 dn = tp.ndom[lo];
      const uint32_t nx[GROVE_MAX_LEVELS] = {dn.x, dn.y, dn.z, dn.w};
      uint32_t close = 0;
#pragma unroll
      for (uint32_t x = 0; x < GROVE_MAX_LEVELS; ++x) close += x < tp.L && nx[x] != GROVE_DOM_ABSENT && nx[x] == ax[x];
      const uint32_t sc = min(close, l + 1u), rot = (lo + tp.n - a) % tp.n;
      const unsigned long long key = (static_cast<unsigned long long>(short_f) << 32) | (uint64_t(7u - sc) << 24) | rot;
      if (key > prev) best = min(best, key);   // (keys are distinct and never 0: the rotated index names the domain)
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) best = min(best, __shfl_xor_sync(kFull, best, o));
    if (lane == 0) s_min[warp] = best;
    __syncthreads();
    if (tid == 0) {
      for (uint32_t w = 1; w < (blockDim.x >> 5); ++w) best = min(best, s_min[w]);
      s_prev = best;
      if (best != ~0ull) {
        const uint32_t lo = (uint32_t(best & 0xFFFFFFu) + a) % tp.n;
        const uint4 dn = tp.ndom[lo];
        const uint32_t d = l == 0 ? dn.x : l == 1 ? dn.y : l == 2 ? dn.z : dn.w;
        out[1 + 2 * t] = lo; out[2 + 2 * t] = tp.dom_hi[l][d];
        out[0] = t + 1;
      }
    }
    __syncthreads();
    if (s_prev == ~0ull) break;
  }
}

// The view of one try: nres = view, with every node outside the sorted range [lo, hi) unschedulable.
__global__ void __launch_bounds__(256) k_consol_mask(const uint4* view, uint4* nres, uint32_t N, uint32_t lo, uint32_t hi) {
  const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  uint4 r = view[n];
  if (n < lo || n >= hi) r.w &= ~uint32_t(GROVE_NODE_SCHEDULABLE);
  nres[n] = r;
}

}  // namespace grove
