// binpack.cuh -- bin-packing (grove_set_binpack; DESIGN.md section 1 "Bin-packing"): each member's anchor moves to the first node
// of the fullest domain of its pack level that can hold it, picked once on the table the cycle starts from (F0).
#pragma once
#include <cuda/std/tuple>

#include "common.cuh"

namespace grove {

// Sum of the free resources of the schedulable nodes of one domain, 64-bit
struct BpSum {
  unsigned long long cpu, mem, gpu, pods;
};

// Ranking key of a domain: fewest free GPUs, then CPU, then memory (ties: lowest domain, by the stable sort over domain order)
struct BpKey {
  unsigned long long gpu, cpu, mem;
};

struct BpOff {   // first entry of each level's domains in the sum / key / rank arrays (the levels some member packs at)
  uint32_t o[GROVE_MAX_LEVELS];
};

struct BpKeyDecomposer {   // cub::DeviceRadixSort: most significant field first
  __host__ __device__ ::cuda::std::tuple<unsigned long long&, unsigned long long&, unsigned long long&> operator()(BpKey& k) const {
    return {k.gpu, k.cpu, k.mem};
  }
};

// a[i] of a per-level parameter array by selects: an indexed parameter array would be copied to local memory
template <typename T>
__device__ __forceinline__ T at_level(const T (&a)[GROVE_MAX_LEVELS], uint32_t i) {
  return i == 0 ? a[0] : i == 1 ? a[1] : i == 2 ? a[2] : a[3];
}

// Cycle start, over F0: grid = npad / 256 node tiles.  For every level l in `levels` (a bit per level) and every level-l domain D,
// sum[off[l] + D] += the free resources of D's schedulable nodes.  The lanes of a warp that share a domain are one
// __match_any_sync segment (sorted order keeps a domain contiguous); the 32-bit fields are reduced in 16-bit halves so that a
// warp's sum cannot wrap.  `sum` is zeroed by the host.
__global__ void __launch_bounds__(256) k_binpack_sum(Topo tp, uint32_t levels, BpOff off, BpSum* sum) {
  const uint32_t lane = threadIdx.x & 31, node = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = node < tp.n;
  uint4 r = valid ? tp.nres[node] : make_uint4(0, 0, 0, 0);
  if (!(r.w & GROVE_NODE_SCHEDULABLE)) r = make_uint4(0, 0, 0, 0);
  const uint4 dm = valid ? tp.ndom[node] : make_uint4(kFull, kFull, kFull, kFull);
  const uint32_t key[GROVE_MAX_LEVELS] = {dm.x, dm.y, dm.z, dm.w};
#pragma unroll
  for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) {
    if (!((levels >> l) & 1u)) continue;   // (uniform)
    const uint32_t seg = __match_any_sync(kFull, key[l]);
    const uint32_t c0 = __reduce_add_sync(seg, r.x & 0xFFFFu), c1 = __reduce_add_sync(seg, r.x >> 16);
    const uint32_t m0 = __reduce_add_sync(seg, r.y & 0xFFFFu), m1 = __reduce_add_sync(seg, r.y >> 16);
    const uint32_t gp = __reduce_add_sync(seg, r.z & 0xFFFFu), pd = __reduce_add_sync(seg, r.z >> 16);
    if (key[l] != GROVE_DOM_ABSENT && lane == uint32_t(__ffs(seg) - 1)) {
      BpSum& s = sum[off.o[l] + key[l]];
      const unsigned long long cpu = c0 + (static_cast<unsigned long long>(c1) << 16), mem = m0 + (static_cast<unsigned long long>(m1) << 16);
      if (cpu) atomicAdd(&s.cpu, cpu);
      if (mem) atomicAdd(&s.mem, mem);
      if (gp) atomicAdd(&s.gpu, static_cast<unsigned long long>(gp));
      if (pd) atomicAdd(&s.pods, static_cast<unsigned long long>(pd));
    }
  }
}

// After k_binpack_sum, a thread per domain of one level (n of them): the sort's keys, and the domain index as the value.
__global__ void k_binpack_keys(const BpSum* __restrict__ sum, uint32_t n, BpKey* key, uint32_t* idx) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const BpSum s = sum[i];
  key[i] = BpKey{s.gpu, s.cpu, s.mem};
  idx[i] = i;
}

// After the ranking, a warp per member (mem[k] = gang, pack level b, default sorted anchor): walk the level-b domains in rank order,
// 32 at a time, and take the first that qualifies -- every clique with MinReplicas m > 0 finds m pods in it, and the sums hold the
// aggregate of m x request and m pods.  A clique's pods in D are the capacity tables of the cycle's first build (F0): the unit
// level's bytes, else the per-domain sum.  Exact for "sum >= m": a byte saturates at 255 >= m (a wide submission has no set), so
// a node that saturates meets m alone, and 255 bytes over at most 2^24 nodes do not wrap the 32-bit sum.  Then the member's
// anchor is the first node of the pick, or its default without one, with its ancestor ranges as k_anchor writes them;
// pick[gang] = that first node, or kFull.
__global__ void __launch_bounds__(256) k_binpack_pick(Topo tp, Tables tb, Relax rx, const uint4* __restrict__ mem, uint32_t M,
                                                      const BpSum* __restrict__ sum, const uint32_t* __restrict__ rank,
                                                      BpOff off, GangInfo* ginfo, uint32_t* pick) {
  const uint32_t lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= M) return;   // (a whole warp)
  const uint4 mb = mem[w];
  const uint32_t gi = mb.x, b = mb.y;
  const grove_gang_t g = tb.gangs[gi];
  uint32_t m = 0, sig = 0;
  unsigned long long need_cpu = 0, need_mem = 0, need_gpu = 0, need_pods = 0;
  if (lane < g.n_cliques) {   // (a gang has at most 32 cliques: one per lane)
    const grove_clique_t q = tb.cliques[g.clique_off + lane];
    m = q.min_replicas; sig = tb.cinfo[g.clique_off + lane].sig;
    need_cpu = static_cast<unsigned long long>(m) * q.req_cpu_milli; need_mem = static_cast<unsigned long long>(m) * q.req_mem_mib;
    need_gpu = static_cast<unsigned long long>(m) * q.req_gpu; need_pods = m;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    need_cpu += __shfl_xor_sync(kFull, need_cpu, o); need_mem += __shfl_xor_sync(kFull, need_mem, o);
    need_gpu += __shfl_xor_sync(kFull, need_gpu, o); need_pods += __shfl_xor_sync(kFull, need_pods, o);
  }
  const uint32_t nd = at_level(tp.n_dom, b), o = at_level(off.o, b), unit = at_level(tp.unit, b), col = at_level(tp.cap_off, b);
  const uint32_t* lo_of = at_level(tp.dom_lo, b);
  uint32_t found = kFull;
  for (uint32_t base = 0; base < nd; base += 32) {
    const uint32_t i = base + lane;
    bool ok = i < nd;
    const uint32_t d = ok ? rank[o + i] : 0u;
    if (ok) {
      const BpSum s = sum[o + d];
      ok = s.cpu >= need_cpu && s.mem >= need_mem && s.gpu >= need_gpu && s.pods >= need_pods;
    }
    for (uint32_t c = 0; c < g.n_cliques; ++c) {   // (uniform)
      const uint32_t mc = __shfl_sync(kFull, m, c), sc = __shfl_sync(kFull, sig, c);
      if (!ok || !mc) continue;
      const uint32_t have = unit ? uint32_t(rx.cap8[size_t(sc) * tp.npad + lo_of[d]]) : rx.capsum[size_t(sc) * tp.cap_stride + col + d];
      ok = have >= mc;
    }
    const uint32_t bal = __ballot_sync(kFull, ok);
    if (bal) { found = __shfl_sync(kFull, d, __ffs(bal) - 1); break; }
  }
  const uint32_t a = found != kFull ? lo_of[found] : mb.z;
  if (lane == 0) { ginfo[gi].anchor = a; pick[gi] = found != kFull ? a : kFull; }
  if (lane < GROVE_MAX_LEVELS) {   // k_anchor's ranges, a lane per level
    const uint4 dm = tp.ndom[a];
    const uint32_t dl = lane == 0 ? dm.x : lane == 1 ? dm.y : lane == 2 ? dm.z : dm.w;
    uint32_t lo = a, hi = a;
    if (lane < tp.L && dl != GROVE_DOM_ABSENT) { lo = at_level(tp.dom_lo, lane)[dl]; hi = at_level(tp.dom_hi, lane)[dl]; }
    ginfo[gi].anc_lo[lane] = lo; ginfo[gi].anc_hi[lane] = hi;
  }
}

}  // namespace grove
