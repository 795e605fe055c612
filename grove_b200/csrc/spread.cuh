// spread.cuh -- topology spread (grove_set_spread; DESIGN.md section 1 "Topology spread"): which level-l_s domains each member
// of a spread group may be placed in, at its turn.
#pragma once
#include "common.cuh"

namespace grove {

// Cycle start: per domain of every level, the OR of the selector classes of its schedulable nodes (Spread::dcls, zeroed by the
// host).  A member's eligible domains E_g are those whose mask meets the union of its cliques' class masks.  A thread per node.
__global__ void __launch_bounds__(256) k_spread_classes(Topo tp, Relax rx) {
  const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= tp.n) return;
  const uint32_t w = tp.nres[n].w;
  if (!(w & GROVE_NODE_SCHEDULABLE)) return;
  const uint32_t bit = 1u << ((w >> GROVE_NODE_CLASS_SHIFT) & 0xFu);
  const uint4 d = tp.ndom[n];
  const uint32_t dl[GROVE_MAX_LEVELS] = {d.x, d.y, d.z, d.w};
#pragma unroll
  for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l)
    if (l < tp.L && dl[l] != GROVE_DOM_ABSENT) atomicOr(rx.sp.dcls + rx.sp.dcls_off[l] + dl[l], bit);
}

// The allowed rows of the members, from the tentative results the previous round left (final below the front) and the seeds:
// one CTA per group walks its members in rank order with c(A) in Spread::cnt.  At member g: m = min over E_g of c(A), A is
// allowed iff A is in E_g and c(A) <= m + max_skew - 1; then an admitted g adds one to c(A(g)).  Only the members that rank
// below the window's end are walked (the others are not evaluated this round).  Head of every round's chain in a spread
// cycle; with final_pass = 1, after the cycle, it walks every member and records which SOFT members landed outside their
// allowed domains (Spread::skewed).
__global__ void __launch_bounds__(256) k_spread(Topo tp, Tables tb, Relax rx, uint32_t final_pass) {
  __shared__ uint32_t s_min[8];
  cudaGridDependencySynchronize();   // (launched chained at the head of a round: engine.cu launch_chained)
  if (!final_pass && rx.ctl[kDone]) return;
  const uint32_t s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t info = rx.sp.info[s], l = info & 0xFFu, mode = (info >> 8) & 0xFFu, skew = info >> 16;
  const uint32_t nd = tp.n_dom[l], words = (nd + 31u) >> 5;
  uint32_t* cnt = rx.sp.cnt + rx.sp.cnt_off[s];
  const uint32_t* seed = rx.sp.seed + rx.sp.cnt_off[s];
  const uint32_t* dc = rx.sp.dcls + rx.sp.dcls_off[l];
  for (uint32_t d = tid; d < nd; d += blockDim.x) cnt[d] = seed[d];
  const uint32_t hi = final_pass ? tb.G : rx.ctl[kHi];
  __syncthreads();
  for (uint32_t j = rx.sp.mem_off[s], je = rx.sp.mem_off[s + 1]; j < je; ++j) {
    const uint32_t g = rx.sp.mem[j];
    if (tb.ginfo[g].order >= hi) break;   // members are listed in rank order
    const uint32_t cm = rx.sp.cls[j];
    uint32_t m = kFull;
    for (uint32_t d = tid; d < nd; d += blockDim.x) if (dc[d] & cm) m = min(m, cnt[d]);
#pragma unroll
    for (int o = 16; o; o >>= 1) m = min(m, __shfl_xor_sync(kFull, m, o));
    if (lane == 0) s_min[warp] = m;
    __syncthreads();
    m = kFull;
    for (uint32_t k = 0; k < (blockDim.x >> 5); ++k) m = min(m, s_min[k]);
    const uint32_t thr = m == kFull ? 0u : m + skew - 1u;   // (no eligible domain: no bit is set below)
    uint32_t* row = rx.sp.allowed + rx.sp.row[g];
    for (uint32_t w = tid; w < words; w += blockDim.x) {
      uint32_t bits = 0;
      for (uint32_t b = 0, d = w * 32u; b < 32u && d < nd; ++b, ++d) bits |= uint32_t((dc[d] & cm) && cnt[d] <= thr) << b;
      row[w] = bits;
    }
    __syncthreads();   // every thread is done with c() and s_min before member g counts
    if (tid == 0) {
      const bool adm = rx.tstate[g] == GROVE_GANG_ADMITTED;
      const uint32_t A = adm ? reinterpret_cast<const uint32_t*>(tp.ndom)[size_t(rx.cur_glo[g]) * 4u + l] : GROVE_DOM_ABSENT;
      if (final_pass) rx.sp.skewed[g] = uint8_t(adm && mode == GROVE_SPREAD_SOFT && !((dc[A] & cm) && cnt[A] <= thr));
      if (adm) cnt[A] += 1u;
    }
    __syncthreads();
  }
}

}  // namespace grove
