// imex.cuh -- ComputeDomain exclusivity (grove_set_compute_domains; DESIGN.md section 1 "ComputeDomain exclusivity"): a node's
// GPUs belong to at most one ComputeDomain (CD) at a time, so an enrolled clique's pods land only where no other CD holds the node.
#pragma once
#include "common.cuh"

namespace grove {

constexpr uint32_t kForeignFlag = 1u << 30;   // staged node flag (EvS::begin, kImex): another CD holds the node in the gang's view

// Does a CD other than c hold node n in the view of the gang of rank `rank`?  The committed owner o = owner[n] (owner0, and the CDs
// of the folded gangs), or a live enrolled claim of a lower rank whose gang has another CD (the claim line and the overflow chain
// are read only while the node has enrolled claims, ne = nenr[n]).  A gang's own claims and those of higher ranks do not count.
// The caller loads o and ne (the staged evaluator together with the node's record, in one round trip).
__device__ __forceinline__ bool imex_foreign(const Relax& rx, uint32_t c, uint32_t rank, uint32_t n, uint32_t o, uint32_t ne) {
  if (o != GROVE_CD_NONE && o != c) return true;
  if (!ne) return false;
  auto foreign = [&](uint32_t x) {
    return x != kClaimEmpty && (x & kEnrolled) && (x & kRankBits) < rank && __ldg(rx.im.rank_cd + (x & kRankBits)) != c;
  };
  const uint4* line = rx.claims + size_t(n) * kClaimSlots;
  bool f = false;
#pragma unroll
  for (uint32_t s = 0; s < kClaimSlots; ++s) f |= foreign(__ldg(&line[s].x));
  for (uint32_t i = __ldg(rx.ovf_head + n); i && !f; i = __ldg(rx.ovf_next + i - 1)) f = foreign(__ldg(&rx.ovf_claim[i - 1].x));
  return f;
}
__device__ __forceinline__ bool imex_foreign(const Relax& rx, uint32_t c, uint32_t rank, uint32_t n) {
  return imex_foreign(rx, c, rank, n, __ldg(rx.im.owner + n), __ldg(rx.im.nenr + n));
}

// The tag of the claim of a run of clique `q`'s pods by the gang of rank `rank` (kImex): enrolled cliques' runs carry kEnrolled
__device__ __forceinline__ uint32_t imex_tag(const Relax& rx, uint32_t q, uint32_t rank) {
  return __ldg(rx.im.cd + q) != GROVE_CD_NONE ? rank | kEnrolled : rank;
}

}  // namespace grove
