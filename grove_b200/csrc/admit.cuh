// admit.cuh -- K3: evaluation of one gang against its view of the cluster (warp-cooperative packing).
#pragma once
#include "common.cuh"
#include "imex.cuh"

#ifdef GROVE_INLINE_ALL
#define GROVE_NI __forceinline__
#else
#define GROVE_NI __noinline__
#endif

namespace grove {
// ------------------------------------------------------------------------------------------------
// K3: gang admission.
//
// The cycle's result is the sequential pass (gangs in order rank, each against the state the earlier ones
// left).  The engine reaches it by relaxation: every gang of the window is evaluated against ITS VIEW =
// committed state minus the tentative claims of the gangs that rank before it (relax.cuh), again and again
// until nobody's view changes.  This file is one such evaluation, by ONE WARP:
//   * candidates of the gang's level are taken in score order, 32 at a time: a lane each runs the cheap
//     pre-filter on the per-signature capacity tables (a necessary condition), then the plausible ones are
//     ATTEMPTED ONE AFTER THE OTHER, IN ORDER, the first success is the answer;
//   * an attempt packs scope by scope, clique by clique, with the whole warp: lanes = the 32 nodes of a
//     fit word, capacities from the capacity bytes (nodes nobody claims) or from the node record minus
//     the claims of lower ranks minus the gang's own pods (claimed / touched nodes), prefix sums take the
//     pods in visiting order.  No per-lane stacks, no local memory.
// `extent` = how far along the gang's node visiting order this evaluation may have read node state: only a
// withdrawn claim in front of it can change the result (relax.cuh k_detect).
// ------------------------------------------------------------------------------------------------
struct GangRegs {   // per-gang constants
  uint32_t a, L, n, rank;
  uint32_t anc_lo[GROVE_MAX_LEVELS], anc_hi[GROVE_MAX_LEVELS];
};

struct GangShared {
  uint4 clq[GROVE_MAX_GANG_CLIQUES];       // req_cpu, req_mem, req_gpu, min | replicas << 8 | level << 16 | preferred << 24
  grove_scope_t scopes[GROVE_MAX_GANG_SCOPES];
  uint32_t sig[GROVE_MAX_GANG_CLIQUES];    // fit-bitmap / capacity row of each clique
  uint32_t smask[GROVE_MAX_GANG_CLIQUES];  // class mask | need_depth << 16
  // a wide cycle (kWide) keeps its entry stacks in global memory (Relax::wide_node) and this space for its own state: see wide_own
  uint32_t ent_node[GROVE_MAX_GANG_PODS];
  uint16_t ent_meta[GROVE_MAX_GANG_PODS];  // clique_rel
  uint32_t Hlo[GROVE_MAX_GANG_CLIQUES], Hhi[GROVE_MAX_GANG_CLIQUES];
  uint32_t s_lo[GROVE_MAX_GANG_SCOPES];
  float4 rcp[GROVE_MAX_GANG_CLIQUES];      // 1 / request per resource (0 where nothing is requested)
  int8_t c_got[GROVE_MAX_GANG_CLIQUES];    // level each clique / scope was packed at (-1: the whole cluster)
  int8_t s_got[GROVE_MAX_GANG_SCOPES];
};
// kWide (a gang of up to GROVE_MAX_WIDE_GANG_PODS pods, up to that many replicas per clique): the space of the shared entry
// stack holds Ev::own_word's scratch (int4[32] in ent_node, 16-aligned) and the 16-bit counts, which the packed clq word has no
// room for (min | replicas << 16, uint32_t[32] in ent_meta).  The ordinary instantiations never see these views.
__device__ __forceinline__ int4* wide_own(GangShared& sh) { return reinterpret_cast<int4*>(sh.ent_node); }
__device__ __forceinline__ uint32_t* wide_cnt(GangShared& sh) { return reinterpret_cast<uint32_t*>(sh.ent_meta); }
__device__ __forceinline__ const uint32_t* wide_cnt(const GangShared& sh) { return reinterpret_cast<const uint32_t*>(sh.ent_meta); }
static_assert(sizeof(GangShared::ent_node) >= 32 * sizeof(int4) && offsetof(GangShared, ent_node) % alignof(int4) == 0 &&
              sizeof(GangShared::ent_meta) >= GROVE_MAX_GANG_CLIQUES * 4 && offsetof(GangShared, ent_meta) % 4 == 0, "wide views");

// MinReplicas / replicas of clique cr: the packed word, or (kWide) the 16-bit counts
template <bool kWide>
__device__ __forceinline__ uint32_t clq_min(const GangShared& sh, uint32_t cr) {
  if constexpr (kWide) return wide_cnt(sh)[cr] & 0xFFFFu;
  else return sh.clq[cr].w & 0xFFu;
}
template <bool kWide>
__device__ __forceinline__ uint32_t clq_rep(const GangShared& sh, uint32_t cr) {
  if constexpr (kWide) return wide_cnt(sh)[cr] >> 16;
  else return (sh.clq[cr].w >> 8) & 0xFFu;
}

// Ordered pieces of [lo,hi): descending score, ties by ascending rotated index (n - anchor) mod N.
// from == L: node granularity (ring l = anc_l \ anc_{l+1}, upper part then lower part);
// from <  L: level-`from` domain granularity (the anchor's own domain whole, then the rings).
__device__ __forceinline__ int make_pieces(const GangRegs& g, uint32_t lo, uint32_t hi, uint32_t from,
                                           uint32_t* plo, uint32_t* phi) {
  int k = 0;
  if (g.a < lo || g.a >= hi) { plo[0] = lo; phi[0] = hi; return hi > lo ? 1 : 0; }
  uint32_t prev_lo = g.a, prev_hi = g.a;
  if (from < g.L) {
    prev_lo = max(g.anc_lo[from], lo); prev_hi = min(g.anc_hi[from], hi);
    if (prev_hi > prev_lo) { plo[k] = prev_lo; phi[k] = prev_hi; ++k; }
  }
  for (int l = int(min(from, g.L)) - 1; l >= 0; --l) {
    uint32_t cl = max(g.anc_lo[l], lo), ch = min(g.anc_hi[l], hi);
    if (ch > prev_hi) { plo[k] = prev_hi; phi[k] = ch; ++k; }
    if (prev_lo > cl) { plo[k] = cl; phi[k] = prev_lo; ++k; }
    prev_lo = min(cl, prev_lo); prev_hi = max(ch, prev_hi);
  }
  if (hi > prev_hi) { plo[k] = prev_hi; phi[k] = hi; ++k; }
  if (prev_lo > lo) { plo[k] = lo; phi[k] = prev_lo; ++k; }
  return k;
}

// The same ordered pieces as make_pieces, produced one at a time from a few registers (no per-thread
// arrays: the scalar evaluator runs one attempt per LANE and every local-memory word costs a cache line
// per warp).
struct PieceIt {
  uint32_t lo, hi, prev_lo, prev_hi, first_lo, first_hi;
  int l, stage;  // stage: 0 first piece pending, 1 rings (upper), 2 rings (lower), 3 tail upper, 4 tail lower, 5 done
  bool outside;
  __device__ __forceinline__ void init(const GangRegs& g, uint32_t lo_, uint32_t hi_, uint32_t from) {
    lo = lo_; hi = hi_;
    outside = g.a < lo || g.a >= hi;
    stage = 0; prev_lo = g.a; prev_hi = g.a; first_lo = first_hi = 0;
    l = int(min(from, g.L)) - 1;
    if (!outside && from < g.L) {
      first_lo = max(g.anc_lo[from], lo); first_hi = min(g.anc_hi[from], hi);
      prev_lo = first_lo; prev_hi = first_hi;
    }
  }
  __device__ __forceinline__ bool next(const GangRegs& g, uint32_t& a, uint32_t& b) {
    if (outside) { if (stage == 0 && hi > lo) { stage = 5; a = lo; b = hi; return true; } return false; }
    if (stage == 0) { stage = 1; if (first_hi > first_lo) { a = first_lo; b = first_hi; return true; } }
    while (stage == 1 || stage == 2) {
      if (l < 0) { stage = 3; break; }
      const uint32_t cl = max(g.anc_lo[l], lo), ch = min(g.anc_hi[l], hi);
      if (stage == 1) { stage = 2; if (ch > prev_hi) { a = prev_hi; b = ch; return true; } }
      // stage 2: lower part of ring l, then move one level out
      const uint32_t pl = prev_lo;
      prev_lo = min(cl, prev_lo); prev_hi = max(ch, prev_hi);
      --l; stage = 1;
      if (pl > cl) { a = cl; b = pl; return true; }
    }
    if (stage == 3) { stage = 4; if (hi > prev_hi) { a = prev_hi; b = hi; return true; } }
    if (stage == 4) { stage = 5; if (prev_lo > lo) { a = lo; b = prev_lo; return true; } }
    return false;
  }
};

__device__ __forceinline__ uint32_t cap_from(uint32_t cpu, uint32_t mem, uint32_t gpu, uint32_t pods, const uint4& q) {
  uint32_t c = pods;
  if (q.x) c = min(c, div_small(cpu, q.x));
  if (q.y) c = min(c, div_small(mem, q.y));
  if (q.z) c = min(c, div_small(gpu, q.z));
  return c;
}

// floor(x / d) for the staged evaluator, exact below 256 and >= 256 above (callers never ask for more than 255 pods);
// r = 1.0f / d.  Branch-free so that the three resources -- and the nodes a lane handles -- overlap: the estimate is
// within one of the quotient (relative error of the product < 2^-22, quotients < 257), one signed remainder fixes it.
// kWide (asks of up to GROVE_MAX_WIDE_GANG_PODS pods): exact below 4096 and >= 4096 above.  The clamped estimate is below
// 4097 and the product's relative error below 2^-22, so its absolute error is below 4097 * 2^-22 < 0.001: the truncated
// estimate is still within one of the quotient and the same single fix-up makes it exact.
template <bool kWide = false>
__device__ __forceinline__ uint32_t div_rcp(uint32_t x, uint32_t d, float r) {
  uint32_t q = __float2uint_rz(fminf(__uint2float_rz(x) * r, kWide ? 4096.0f : 256.0f));
  const long long rem = (long long)x - (long long)((unsigned long long)q * d);
  q += uint32_t(rem >= (long long)d) - uint32_t(rem < 0);
  return d ? q : 0xFFFFu;
}
template <bool kWide = false>
__device__ __forceinline__ uint32_t cap_from_rcp(uint32_t cpu, uint32_t mem, uint32_t gpu, uint32_t pods, const uint4& q, const float4& r) {
  return min(min(div_rcp<kWide>(cpu, q.x, r.x), div_rcp<kWide>(mem, q.y, r.y)), min(div_rcp<kWide>(gpu, q.z, r.z), pods));
}

// position of node n in the gang's node visiting order (descending closeness to the anchor, ties by ascending
// rotated index): the anchor's deepest domain from the anchor upwards, then its lower part, then ring by ring
__device__ __forceinline__ uint32_t visit_pos(const GangRegs& g, uint32_t n) {
  uint32_t in_lo = g.a, in_hi = g.a;   // the domain one level deeper than the ring n lies in (empty below the deepest level)
  for (int l = int(g.L) - 1; l >= -1; --l) {
    const uint32_t lo = l >= 0 ? g.anc_lo[l] : 0u, hi = l >= 0 ? g.anc_hi[l] : g.n;
    if (n >= lo && n < hi && hi > lo) {
      const uint32_t inner = in_hi - in_lo;
      if (n >= in_hi) return inner + (n - in_hi);
      return inner + (hi - in_hi) + (n - lo);
    }
    if (hi > lo) { in_lo = min(in_lo, lo); in_hi = max(in_hi, hi); }
  }
  return g.n;
}

// ---- the evaluator: the whole warp packs ONE candidate range ------------------------------------------
// kFence: the nodes of the fences active for the gang (fm0 / fm1, common.cuh fenced) take no pod
// kImex: the nodes another CD holds in the gang's view (imex.cuh imex_foreign) take no pod of its enrolled cliques (enr)
template <bool kPref_, bool kHolds, bool kWide_ = false, bool kFence = false, bool kImex = false>
struct Ev {
  static constexpr bool kPref = kPref_;
  static constexpr bool kWide = kWide_;
  static constexpr bool kStaged = false;
  const Topo& tp; const Relax& rb; GangShared& sh; const GangRegs& g; uint32_t lane;
  uint32_t np;
  uint32_t fm0 = 0, fm1 = 0;   // (kFence) the active fences
  uint32_t enr = 0, icd = GROVE_CD_NONE;   // (kImex) bit cr set for every enrolled clique; the gang's CD
  uint32_t tmask = 0;   // bit (n & 31) set for every node the gang has put a pod on: quick 'untouched' test
  uint32_t ext = 0;     // see the file comment
  uint32_t t_stage = 0, t_pre = 0, t_pack = 0, n_stage = 0;
  // the entry stack: shared memory, or (kWide) the warp's own stack in global memory
  uint32_t* wn = nullptr; uint16_t* wm = nullptr;
  __device__ __forceinline__ uint32_t& en(uint32_t i) const { if constexpr (kWide) return wn[i]; else return sh.ent_node[i]; }
  __device__ __forceinline__ uint16_t& em(uint32_t i) const { if constexpr (kWide) return wm[i]; else return sh.ent_meta[i]; }
  __device__ Ev(const Topo& t, const Relax& r, GangShared& s, const GangRegs& gr, uint32_t ln)
      : tp(t), rb(r), sh(s), g(gr), lane(ln), np(0) {}

  // kWide: what the gang itself has put on each node of the 32-node word at `base` (the lane's node), gathered by the warp in
  // one pass over the entry stack -- np / 32 loads a lane, where a scan per lane and node would cost np.  Warp-collective; the
  // callers skip it for a word whose fit nodes the gang has not touched (tmask & word == 0: every fit lane's usage is zero).
  __device__ __forceinline__ int4 own_word(uint32_t base) const {
    int4* own = wide_own(sh);
    own[lane] = make_int4(0, 0, 0, 0);
    __syncwarp();
    for (uint32_t i = lane; i < np; i += 32) {
      const uint32_t d = wn[i] - base;
      if (d < 32u) {
        const uint4 q = sh.clq[wm[i]];
        int* o = reinterpret_cast<int*>(own + d);
        atomicAdd(o + 0, int(q.x)); atomicAdd(o + 1, int(q.y)); atomicAdd(o + 2, int(q.z)); atomicAdd(o + 3, 1);
      }
    }
    __syncwarp();
    const int4 r = own[lane];
    __syncwarp();
    return r;
  }

  // pods of clique cr that still fit on node n under the gang's view, after what the gang itself put there (kWide: o, from own_word)
  __device__ __forceinline__ uint32_t cap_view(uint32_t cr, uint32_t n, int4 o = int4{}) const {
    if constexpr (kFence) if (fenced(rb.fc, fm0, fm1, n)) return 0u;
    if constexpr (kImex) if (((enr >> cr) & 1u) && imex_foreign(rb, icd, g.rank, n)) return 0u;
    const uint32_t live = (__ldg(rb.nlive + (n >> 2)) >> ((n & 3u) * 8u)) & 0xFFu;
    const bool own = (tmask >> (n & 31u)) & 1u;
    if (!live && !own) {
      const uint32_t c = __ldg(rb.cap8 + size_t(sh.sig[cr]) * tp.npad + n);
      if (c != 255u) return c;   // nobody claims the node and the table is current: the byte is the answer
    }
    const uint4 r = __ldg(tp.nres + n);
    const uint32_t sm = sh.smask[cr];
    if (!(r.w & GROVE_NODE_SCHEDULABLE) || !((sm >> ((r.w >> GROVE_NODE_CLASS_SHIFT) & 0xFu)) & 1u) || ((r.w >> 16) & 0xFu) < (sm >> 16)) return 0u;
    int cpu = int(r.x), mem = int(r.y), gpu = int(r.z & 0xFFFFu), pods = int(r.z >> 16);
    if (live & 0x7Fu) {   // claims: all of them, minus those of the gangs that rank after this one (see EvS::begin)
      const int4 t = __ldg(rb.ctot + n);
      cpu -= t.x; mem -= t.y; gpu -= t.z; pods -= t.w;
      if (__ldg(rb.cmaxr + n) >= g.rank) {
        if (live & 0x3Fu) {
          const uint4* line = rb.claims + size_t(n) * kClaimSlots;
#pragma unroll
          for (uint32_t s = 0; s < kClaimSlots; ++s) {
            const uint4 c = __ldg(line + s);
            if (gives_back<kHolds, kImex>(c.x, g.rank)) { cpu += int(c.y); mem += int(c.z); gpu += int(c.w & 0xFFFFu); pods += int(c.w >> 16); }
          }
        }
        if (live & kHasOvf) {
          for (uint32_t i = __ldg(rb.ovf_head + n); i; i = __ldg(rb.ovf_next + i - 1)) {
            const uint4 c = __ldg(rb.ovf_claim + i - 1);
            if (gives_back<kHolds, kImex>(c.x, g.rank)) { cpu += int(c.y); mem += int(c.z); gpu += int(c.w & 0xFFFFu); pods += int(c.w >> 16); }
          }
        }
      }
    }
    if constexpr (kWide) {
      cpu -= o.x; mem -= o.y; gpu -= o.z; pods -= o.w;
      return cap_from_rcp<true>(uint32_t(max(cpu, 0)), uint32_t(max(mem, 0)), uint32_t(max(gpu, 0)), uint32_t(max(pods, 0)), sh.clq[cr], sh.rcp[cr]);
    } else {
      if (own) {
        for (uint32_t i = 0; i < np; ++i) {
          if (sh.ent_node[i] == n) {
            const uint4 o = sh.clq[sh.ent_meta[i]];
            cpu -= int(o.x); mem -= int(o.y); gpu -= int(o.z); pods -= 1;
          }
        }
      }
      return cap_from(uint32_t(max(cpu, 0)), uint32_t(max(mem, 0)), uint32_t(max(gpu, 0)), uint32_t(max(pods, 0)), sh.clq[cr]);
    }
  }

  __device__ __forceinline__ uint32_t scope_filter(const grove_scope_t&, uint32_t, uint32_t, bool, int) { return kFull; }   // staged evaluator only
  __device__ __forceinline__ void note_read(uint32_t last) { ext = max(ext, visit_pos(g, last) + 1u); }
  __device__ __forceinline__ void begin(uint32_t, uint32_t) { np = 0; tmask = 0; }       // a fresh attempt
  __device__ __forceinline__ void rollback(uint32_t mark) { np = mark; }               // drop the pods placed after mark

  // up to `want` pods of clique cr on fit nodes of [lo,hi) in score order; returns pods placed
  __device__ GROVE_NI uint32_t take(uint32_t cr, uint32_t lo, uint32_t hi, uint32_t want) {
    if (want == 0 || hi <= lo) return 0;
    const uint32_t* Frow = rb.F + size_t(sh.sig[cr]) * tp.words;
    PieceIt pit; pit.init(g, lo, hi, g.L);
    uint32_t placed = 0, last = GROVE_NONE_U32;
    for (uint32_t a, b; placed < want && pit.next(g, a, b);) {
      for (uint32_t base = a & ~31u; base < b && placed < want; base += 32) {
        uint32_t word = __ldg(Frow + (base >> 5));
        if (base < a) word &= kFull << (a - base);
        if (base + 32u > b) word &= (1u << (b - base)) - 1u;
        last = min(base + 31u, b - 1u);
        if (!word) continue;   // no fit node when the tables were built: none now
        const uint32_t n = base + lane;
        int4 o{};
        if constexpr (kWide) if (tmask & word) o = own_word(base);   // (warp-uniform)
        const uint32_t c = ((word >> lane) & 1u) ? cap_view(cr, n, o) : 0u;
        const uint32_t incl = warp_incl_scan(c, lane), excl = incl - c, rem = want - placed;
        const uint32_t t = excl >= rem ? 0u : min(c, rem - excl);
        const uint32_t tincl = warp_incl_scan(t, lane);
        __syncwarp();  // every lane's scan of the entry stack is over before it grows
        if (t) {
          const uint32_t pos = np + tincl - t;
          for (uint32_t j = 0; j < t; ++j) { en(pos + j) = n; em(pos + j) = uint16_t(cr); }
        }
        const uint32_t tb = __ballot_sync(kFull, t != 0);
        const uint32_t tot = __shfl_sync(kFull, tincl, 31);
        tmask |= tb;   // base is 32-aligned: lane == n & 31
        np += tot; placed += tot;
        if (placed >= want && tb) last = base + (31u - __clz(tb));
        __syncwarp();
      }
    }
    if (last != GROVE_NONE_U32) note_read(last);
    return placed;
  }

  __device__ bool fill_min(uint32_t cr, uint32_t lo, uint32_t hi) {
    const uint32_t m = clq_min<kWide>(sh, cr);
    const uint32_t mark = np;
    if (take(cr, lo, hi, m) < m) { rollback(mark); return false; }
    if (lane == 0) { sh.Hlo[cr] = lo; sh.Hhi[cr] = hi; }
    __syncwarp();
    return true;
  }

  // clique whose own Required level is a unit level (one node per domain, e.g. hostname):
  // first node of [lo,hi) in score order that takes all m pods
  __device__ GROVE_NI bool find_unit(uint32_t cr, uint32_t lo, uint32_t hi) {
    const uint32_t m = clq_min<kWide>(sh, cr);
    const uint32_t* Frow = rb.F + size_t(sh.sig[cr]) * tp.words;
    PieceIt pit; pit.init(g, lo, hi, g.L);
    uint32_t last = GROVE_NONE_U32;
    for (uint32_t a, b; pit.next(g, a, b);) {
      for (uint32_t base = a & ~31u; base < b; base += 32) {
        uint32_t word = __ldg(Frow + (base >> 5));
        if (base < a) word &= kFull << (a - base);
        if (base + 32u > b) word &= (1u << (b - base)) - 1u;
        last = min(base + 31u, b - 1u);
        if (!word) continue;
        const uint32_t n = base + lane;
        int4 o{};
        if constexpr (kWide) if (tmask & word) o = own_word(base);   // (warp-uniform)
        const uint32_t c = ((word >> lane) & 1u) ? cap_view(cr, n, o) : 0u;
        const uint32_t okb = __ballot_sync(kFull, c >= m && ((word >> lane) & 1u));
        __syncwarp();
        if (okb) {
          const uint32_t nn = base + (__ffs(okb) - 1);
          for (uint32_t j = lane; j < m; j += 32) { en(np + j) = nn; em(np + j) = uint16_t(cr); }
          if (lane == 0) { sh.Hlo[cr] = nn; sh.Hhi[cr] = nn + 1; }
          tmask |= 1u << (nn & 31u);
          np += m;
          note_read(nn);
          __syncwarp();
          return true;
        }
      }
    }
    if (last != GROVE_NONE_U32) note_read(last);
    return false;
  }
};


// ---- staged evaluator: the candidate range lives in shared memory -------------------------------------------
// For a candidate of at most kStageMax nodes (a rack, a block) the warp first computes the gang's VIEW of every node
// of the range -- committed state minus the claims of lower ranks -- into shared memory (two rounds of independent
// loads), then packs from there: capacities are divisions on the staged record, pods the gang places are subtracted
// from it in place (no entry-stack scans), a failed scope adds them back.  An attempt costs a few thousand cycles
// instead of a chain of dependent L2 look-ups per 32 nodes.
constexpr uint32_t kStageMax = 128;

template <bool kPref_, bool kHolds, bool kWide_ = false, bool kFence = false, bool kImex = false>
struct EvS {
  static constexpr bool kPref = kPref_;
  static constexpr bool kWide = kWide_;
  static constexpr bool kStaged = true;   // node state in shared memory: an attempt costs less than the table look-ups that would skip it
  const Topo& tp; const Relax& rb; GangShared& sh; const GangRegs& g; uint32_t lane;
  int4* view;           // [kStageMax] cpu, mem, gpu, pods the gang may still take.  Signed: the claims of lower ranks may transiently exceed
                        // the committed state (saturating subtraction claim by claim == clamping the sum at zero when it is read)
  uint32_t* vflag;      // [kStageMax] node flags | vdepth << 16
  uint8_t* rk;          // [kStageMax + 256] sub-domain filter scratch: the sub-domain (lane) each staged node belongs to, then
                        // per-sub-domain sum and max (32 words each) of the pods of ONE clique that fit
  uint32_t t_stage = 0, t_pre = 0, t_pack = 0, n_stage = 0;   // GROVE_DEBUG_ADMIT: cycles staging / pre-filtering sub-domains / packing
  uint32_t t_st2 = 0, t_st3 = 0;                              // of the staging: claim lines, overflow chains
  uint32_t vlo = 0, vhi = 0;
  uint32_t np;
  uint32_t fm0 = 0, fm1 = 0;   // (kFence) the active fences: their nodes are staged unschedulable
  uint32_t enr = 0, icd = GROVE_CD_NONE;   // (kImex) the enrolled cliques and the gang's CD: foreign nodes are staged kForeignFlag
  uint32_t tmask = 0;
  uint32_t ext = 0;
  // the entry stack: shared memory, or (kWide) the warp's own stack in global memory
  uint32_t* wn = nullptr; uint16_t* wm = nullptr;
  __device__ __forceinline__ uint32_t& en(uint32_t i) const { if constexpr (kWide) return wn[i]; else return sh.ent_node[i]; }
  __device__ __forceinline__ uint16_t& em(uint32_t i) const { if constexpr (kWide) return wm[i]; else return sh.ent_meta[i]; }
  __device__ EvS(const Topo& t, const Relax& r, GangShared& s, const GangRegs& gr, uint32_t ln, int4* v, uint32_t* vf, uint8_t* cv)
      : tp(t), rb(r), sh(s), g(gr), lane(ln), view(v), vflag(vf), rk(cv), np(0) {}

  // Stage the gang's view of [dl, dh): committed record minus the claims of the ranks before it.  A lane per node, four nodes a
  // lane, ONE L2 round trip for almost every node: the record, the node's claim TOTAL (all ranks) and the highest rank that ever
  // claimed it (relax.cuh ctot / cmaxr).  Gangs enter the window in rank order, so for most evaluations every claim on a node is
  // of a lower rank and the view is record - total.  Only where a HIGHER rank may lean on the node (cmaxr >= rank) are its claim
  // line and overflow chain read, to give those claims back.
  __device__ GROVE_NI void begin(uint32_t dl, uint32_t dh) {
    np = 0; vlo = dl; vhi = dh;
    const long long tb0 = rb.dbg ? clock64() : 0;
    __syncwarp();
    constexpr uint32_t kPer = kStageMax / 32;
    uint4 r[kPer]; int4 t[kPer]; uint32_t live[kPer], mr[kPer];
    uint32_t io[kPer], ine[kPer];   // (kImex) the node's committed owner and enrolled claims, asked for with its record
#pragma unroll
    for (uint32_t k = 0; k < kPer; ++k) {
      const uint32_t n = dl + k * 32u + lane;
      const bool in = n < dh;
      r[k] = in ? __ldg(tp.nres + n) : make_uint4(0, 0, 0, 0);
      t[k] = in ? __ldg(rb.ctot + n) : make_int4(0, 0, 0, 0);
      mr[k] = in ? __ldg(rb.cmaxr + n) : 0u;
      live[k] = in ? (__ldg(rb.nlive + (n >> 2)) >> ((n & 3u) * 8u)) & 0x7Fu : 0u;
      if constexpr (kImex) { io[k] = in && enr ? __ldg(rb.im.owner + n) : GROVE_CD_NONE; ine[k] = in && enr ? __ldg(rb.im.nenr + n) : 0u; }
    }
    const long long tc0 = rb.dbg ? clock64() : 0;
#pragma unroll
    for (uint32_t k = 0; k < kPer; ++k) {
      const uint32_t n = dl + k * 32u + lane;
      int cpu = int(r[k].x) - t[k].x, mem = int(r[k].y) - t[k].y, gpu = int(r[k].z & 0xFFFFu) - t[k].z, pods = int(r[k].z >> 16) - t[k].w;
      if (live[k] && mr[k] >= g.rank) {   // a gang of a higher rank may hold a claim here (invisible to this one), or this gang its hold
        if (live[k] & 0x3Fu) {
          const uint4* line = rb.claims + size_t(n) * kClaimSlots;
          uint4 c[kClaimSlots];
#pragma unroll
          for (uint32_t s = 0; s < kClaimSlots; ++s) c[s] = __ldg(line + s);
#pragma unroll
          for (uint32_t s = 0; s < kClaimSlots; ++s)
            if (gives_back<kHolds, kImex>(c[s].x, g.rank)) { cpu += int(c[s].y); mem += int(c[s].z); gpu += int(c[s].w & 0xFFFFu); pods += int(c[s].w >> 16); }
        }
        if (live[k] & kHasOvf) {
          for (uint32_t i = __ldg(rb.ovf_head + n); i; i = __ldg(rb.ovf_next + i - 1)) {
            const uint4 c = __ldg(rb.ovf_claim + i - 1);
            if (gives_back<kHolds, kImex>(c.x, g.rank)) { cpu += int(c.y); mem += int(c.z); gpu += int(c.w & 0xFFFFu); pods += int(c.w >> 16); }
          }
        }
      }
      view[k * 32u + lane] = make_int4(cpu, mem, gpu, pods);
      uint32_t f = r[k].w;
      if constexpr (kFence) if (n < dh && fenced(rb.fc, fm0, fm1, n)) f &= ~uint32_t(GROVE_NODE_SCHEDULABLE);
      if constexpr (kImex) if (enr && n < dh && imex_foreign(rb, icd, g.rank, n, io[k], ine[k])) f |= kForeignFlag;   // (the CD is the gang's: once per attempt)
      vflag[k * 32u + lane] = f;
    }
    __syncwarp();
    // the whole range has been read: it ends at the furthest position any of its nodes has in the visiting order
    ext = max(ext, (g.a >= dl && g.a < dh) ? dh - dl : visit_pos(g, dh - 1u) + 1u);
    if (rb.dbg) { const long long te = clock64(); t_stage += uint32_t(te - tb0); t_st2 += uint32_t(tc0 - tb0); t_st3 += uint32_t(te - tc0); ++n_stage; }
  }

  __device__ __forceinline__ uint32_t cap(uint32_t cr, uint32_t n) const {
    const int4 v = view[n - vlo];
    const uint32_t f = vflag[n - vlo];
    const uint32_t sm = sh.smask[cr];
    bool usable = (f & GROVE_NODE_SCHEDULABLE) && ((sm >> ((f >> GROVE_NODE_CLASS_SHIFT) & 0xFu)) & 1u) && ((f >> 16) & 0xFu) >= (sm >> 16);
    if constexpr (kImex) usable = usable && !((f & kForeignFlag) && ((enr >> cr) & 1u));
    const uint32_t c = cap_from_rcp<kWide>(uint32_t(max(v.x, 0)), uint32_t(max(v.y, 0)), uint32_t(max(v.z, 0)), uint32_t(max(v.w, 0)), sh.clq[cr], sh.rcp[cr]);
    return usable ? c : 0u;
  }

  // Sub-domain filter on the staged view: which of the (at most 32) level-sl domains [el, eh) -- a lane each -- could take
  // every clique of scope s on its own?  A necessary condition like the table look-ups of scope_plausible, but against what
  // the gang really sees (the tables only know the committed state as of their last build): a candidate whose racks are
  // taken by lower ranks' claims fails here instead of after an attempt per rack.
  __device__ GROVE_NI uint32_t scope_filter(const grove_scope_t& s, uint32_t el, uint32_t eh, bool in, int sl) {
    constexpr uint32_t kPer = kStageMax / 32;
    uint32_t* rsum = reinterpret_cast<uint32_t*>(rk + kStageMax);
    uint32_t* rmax = rsum + 32;
    bool ok = in;
    el = max(el, vlo); eh = min(eh, vhi);
    __syncwarp();
    reinterpret_cast<uint32_t*>(rk)[lane] = kFull;             // a node that lacks the label is in no sub-domain
    __syncwarp();
    if (in) for (uint32_t n = el; n < eh; ++n) rk[n - vlo] = uint8_t(lane);   // (stores: nothing waits on them)
    for (uint32_t i = 0; i < s.n_cliques; ++i) {
      const uint32_t cr = s.first_clique + i;
      const uint32_t w = sh.clq[cr].w;
      const uint32_t m = clq_min<kWide>(sh, cr), ql = (w >> 16) & 0xFFu;
      if (m == 0) continue;
      rsum[lane] = 0; rmax[lane] = 0;
      __syncwarp();
#pragma unroll
      for (uint32_t k = 0; k < kPer; ++k) {
        const uint32_t idx = k * 32u + lane;
        const uint32_t c = vlo + idx < vhi ? cap(cr, vlo + idx) : 0u;
        const uint32_t slot = rk[idx];
        if (c && slot != 0xFFu) { atomicAdd(rsum + slot, c); atomicMax(rmax + slot, c); }
      }
      __syncwarp();
      const bool one_node = ql != GROVE_LEVEL_NONE && int(ql) > sl && tp.unit[ql];   // all m pods on one node
      ok = ok && (one_node ? rmax[lane] >= m : rsum[lane] >= m);
      __syncwarp();
    }
    return __ballot_sync(kFull, ok);
  }

  // give back the pods placed after mark
  __device__ GROVE_NI void rollback(uint32_t mark) {
    __syncwarp();
    for (uint32_t i = mark + lane; i < np; i += 32) {
      const uint4 q = sh.clq[em(i)];
      int* v = reinterpret_cast<int*>(view + (en(i) - vlo));
      if (q.x) atomicAdd(v + 0, int(q.x));
      if (q.y) atomicAdd(v + 1, int(q.y));
      if (q.z) atomicAdd(v + 2, int(q.z));
      atomicAdd(v + 3, 1);
    }
    np = mark;
    __syncwarp();
  }

  __device__ GROVE_NI uint32_t take(uint32_t cr, uint32_t lo, uint32_t hi, uint32_t want) {
    if (want == 0 || hi <= lo) return 0;
    const uint4 q = sh.clq[cr];
    PieceIt pit; pit.init(g, lo, hi, g.L);
    uint32_t placed = 0;
    for (uint32_t a, b; placed < want && pit.next(g, a, b);) {
      for (uint32_t base = a & ~31u; base < b && placed < want; base += 32) {
        const uint32_t n = base + lane;
        const uint32_t c = (n >= a && n < b) ? cap(cr, n) : 0u;
        if (!__any_sync(kFull, c != 0u)) continue;
        const uint32_t incl = warp_incl_scan(c, lane), excl = incl - c, rem = want - placed;
        const uint32_t t = excl >= rem ? 0u : min(c, rem - excl);
        const uint32_t tincl = warp_incl_scan(t, lane);
        if (t) {
          const uint32_t pos = np + tincl - t;
          for (uint32_t j = 0; j < t; ++j) { en(pos + j) = n; em(pos + j) = uint16_t(cr); }
          int4 v = view[n - vlo];
          v.x -= int(t * q.x); v.y -= int(t * q.y); v.z -= int(t * q.z); v.w -= int(t);
          view[n - vlo] = v;
        }
        const uint32_t tot = __shfl_sync(kFull, tincl, 31);
        np += tot; placed += tot;
        __syncwarp();
      }
    }
    return placed;
  }

  __device__ bool fill_min(uint32_t cr, uint32_t lo, uint32_t hi) {
    const uint32_t m = clq_min<kWide>(sh, cr);
    const uint32_t mark = np;
    if (take(cr, lo, hi, m) < m) { rollback(mark); return false; }
    if (lane == 0) { sh.Hlo[cr] = lo; sh.Hhi[cr] = hi; }
    __syncwarp();
    return true;
  }

  __device__ GROVE_NI bool find_unit(uint32_t cr, uint32_t lo, uint32_t hi) {
    const uint32_t m = clq_min<kWide>(sh, cr);
    const uint4 q = sh.clq[cr];
    PieceIt pit; pit.init(g, lo, hi, g.L);
    for (uint32_t a, b; pit.next(g, a, b);) {
      for (uint32_t base = a & ~31u; base < b; base += 32) {
        const uint32_t n = base + lane;
        const bool in = n >= a && n < b;
        const uint32_t c = in ? cap(cr, n) : 0u;
        const uint32_t okb = __ballot_sync(kFull, in && c >= m);
        if (okb) {
          const uint32_t nn = base + (__ffs(okb) - 1);
          for (uint32_t j = lane; j < m; j += 32) { en(np + j) = nn; em(np + j) = uint16_t(cr); }
          if (lane == 0) {
            sh.Hlo[cr] = nn; sh.Hhi[cr] = nn + 1;
            int4 v = view[nn - vlo];
            v.x -= int(m * q.x); v.y -= int(m * q.y); v.z -= int(m * q.z); v.w -= int(m);
            view[nn - vlo] = v;
          }
          np += m;
          __syncwarp();
          return true;
        }
      }
    }
    return false;
  }
};

// ---- candidate pre-filter: a NECESSARY condition for place_in(lo, hi) to succeed ------------------
// (each clique alone must find MinReplicas worth of capacity in a domain it could be packed into, and
// the cliques of a scope must find it inside one common scope domain).  Reads only the small
// per-signature capacity tables.
// kWide: a clique may ask for more than 255 pods, and a capacity byte of 255 is saturated (the node may take any number): such a
// node counts as unbounded, and so does a domain whose capacity maximum is 255 -- its sum under-counts it.
template <bool kWide = false>
__device__ __forceinline__ bool clique_plausible(const Topo& tp, const Relax& rb, const GangShared& sh, uint32_t cr,
                                 uint32_t lo, uint32_t hi, int lvl, uint32_t dE) {
  const uint32_t w = sh.clq[cr].w;
  const uint32_t m = clq_min<kWide>(sh, cr), ql = (w >> 16) & 0xFFu;
  if (m == 0) return true;
  const uint32_t m8 = kWide ? min(m, 255u) : m;   // a single node's byte against the ask
  const size_t row = size_t(sh.sig[cr]);
  const bool tabled = lvl >= 0 && !tp.unit[lvl];
  if (ql != GROVE_LEVEL_NONE && int(ql) > lvl) {
    if (tp.unit[ql]) {  // all m pods on one node
      if (tabled) return __ldg(rb.capmax + row * tp.cap_stride + tp.cap_off[lvl] + dE) >= m8;
      for (uint32_t n = lo; n < hi; ++n) if (__ldg(rb.cap8 + row * tp.npad + n) >= m8) return true;
      return false;
    }
    const uint32_t d0 = __ldg(tp.next_dom[ql] + lo), d1 = __ldg(tp.next_dom[ql] + hi);
    uint32_t any = 0;  // no early exit: the look-ups are independent and overlap
    for (uint32_t d = d0; d < d1; ++d) {
      any |= __ldg(rb.capsum + row * tp.cap_stride + tp.cap_off[ql] + d) >= m;
      if constexpr (kWide) any |= __ldg(rb.capmax + row * tp.cap_stride + tp.cap_off[ql] + d) >= 255u;
    }
    return any != 0;
  }
  if (tabled) {
    if constexpr (kWide) if (__ldg(rb.capmax + row * tp.cap_stride + tp.cap_off[lvl] + dE) >= 255u) return true;
    return __ldg(rb.capsum + row * tp.cap_stride + tp.cap_off[lvl] + dE) >= m;
  }
  uint32_t sum = 0;
  for (uint32_t n = lo; n < hi && sum < m; ++n) {
    const uint32_t c = __ldg(rb.cap8 + row * tp.npad + n);
    sum += (kWide && c == 255u) ? m : c;
  }
  return sum >= m;
}

template <bool kWide = false>
__device__ __forceinline__ bool scope_plausible(const Topo& tp, const Relax& rb, const GangShared& sh, const grove_scope_t& s,
                                uint32_t lo, uint32_t hi, int lvl, uint32_t dE) {
  uint32_t all = 1;
  for (uint32_t i = 0; i < s.n_cliques; ++i) all &= clique_plausible<kWide>(tp, rb, sh, s.first_clique + i, lo, hi, lvl, dE);
  return all != 0;
}

// one scope of a gang inside the candidate [lo, hi) of level lvl
template <bool kWide = false>
__device__ __forceinline__ bool scope_ok(const Topo& tp, const Relax& rb, const GangShared& sh, const grove_scope_t& s,
                                         uint32_t lo, uint32_t hi, int lvl, uint32_t dD) {
  if (s.level != GROVE_LEVEL_NONE && int(s.level) > lvl) {
    const uint32_t d0 = __ldg(tp.next_dom[s.level] + lo), d1 = __ldg(tp.next_dom[s.level] + hi);
    uint32_t any = 0;  // no early exit: children are independent table look-ups
    for (uint32_t d = d0; d < d1; ++d)
      any |= scope_plausible<kWide>(tp, rb, sh, s, __ldg(tp.dom_lo[s.level] + d), __ldg(tp.dom_hi[s.level] + d), int(s.level), d);
    return any != 0;
  }
  return scope_plausible<kWide>(tp, rb, sh, s, lo, hi, lvl, dD);
}

template <bool kWide = false>
__device__ bool gang_plausible(const Topo& tp, const Relax& rb, const GangShared& sh, uint32_t n_scopes,
                               uint32_t lo, uint32_t hi, int lvl, uint32_t dD) {
  for (uint32_t si = 0; si < n_scopes; ++si)
    if (!scope_ok<kWide>(tp, rb, sh, sh.scopes[si], lo, hi, lvl, dD)) return false;
  return true;
}

// Levels a unit (gang / scope / clique) with constraint (req, pref) is tried at inside a parent range of
// level lvl (-1 = whole cluster): `first` down to the returned base.  base = the hard level (Required when
// deeper than the parent's, else the parent range itself); a deeper Preferred level is tried first and
// widened level by level up to base (podgang.go:110-117).  Oracle: level_span().  kPref = false: the submission
// carries no Preferred level anywhere, the walk is the single step `base` (the kernels are instantiated both ways so
// that Required-only workloads run the loop-free code).
template <bool kPref>
__device__ __forceinline__ int level_span(uint32_t req, uint32_t pref, int lvl, int& first) {
  const int base = (req != GROVE_LEVEL_NONE && int(req) > lvl) ? int(req) : lvl;
  first = (kPref && pref != GROVE_LEVEL_NONE && int(pref) > base) ? int(pref) : base;
  return base;
}

template <class Ev>
__device__ GROVE_NI bool place_scope(Ev& ev, const grove_scope_t& s, uint32_t lo, uint32_t hi, int lvl) {
  const Topo& tp = ev.tp;
  const uint32_t mark = ev.np;
  for (uint32_t i = 0; i < s.n_cliques; ++i) {
    const uint32_t cr = s.first_clique + i;
    const uint32_t w = ev.sh.clq[cr].w;
    const uint32_t m = clq_min<Ev::kWide>(ev.sh, cr);
    bool ok = false;
    int first;
    const int base = level_span<Ev::kPref>((w >> 16) & 0xFFu, w >> 24, lvl, first);
    int ql = first;
    do {
      if (ql > lvl) {
        // find_unit scans fit NODES: every fit node is a domain of a Required unit level (the fit row demands the
        // labels down to it), but not of a Preferred one (ragged labels) -- those take the domain walk below
        if (tp.unit[ql] && m >= 1 && ql == base) {
          ok = ev.find_unit(cr, lo, hi);
        } else {
          PieceIt pit; pit.init(ev.g, lo, hi, uint32_t(ql));
          for (uint32_t pa, pb; !ok && pit.next(ev.g, pa, pb);) {
            const uint32_t d0 = __ldg(tp.next_dom[ql] + pa), d1 = __ldg(tp.next_dom[ql] + pb);
            for (uint32_t d = d0; d < d1 && !ok; ++d)
              ok = ev.fill_min(cr, __ldg(tp.dom_lo[ql] + d), __ldg(tp.dom_hi[ql] + d));
          }
        }
      } else {
        ok = ev.fill_min(cr, lo, hi);
      }
      if (ok && ev.lane == 0) ev.sh.c_got[cr] = int8_t(ql);
    } while (Ev::kPref && !ok && --ql >= base);
    if (!ok) { ev.rollback(mark); return false; }
  }
  return true;
}

template <class Ev>
__device__ GROVE_NI bool place_in(Ev& ev, uint32_t n_scopes, uint32_t lo, uint32_t hi, int lvl) {
  const Topo& tp = ev.tp;
  // (staged evaluator) the first / end domain index of every deeper level inside [lo, hi): asked for BEFORE the staging so that
  // the look-ups overlap it -- each scope with a narrower level would otherwise start with one more L2 round trip
  uint32_t pd0[GROVE_MAX_LEVELS], pd1[GROVE_MAX_LEVELS];
#pragma unroll
  for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) {
    pd0[l] = pd1[l] = 0;
    if (Ev::kStaged && int(l) > lvl && l < tp.L) { pd0[l] = __ldg(tp.next_dom[l] + lo); pd1[l] = __ldg(tp.next_dom[l] + hi); }
  }
  ev.begin(lo, hi);
  for (uint32_t si = 0; si < n_scopes; ++si) {
    const grove_scope_t s = ev.sh.scopes[si];
    bool ok = false;
    int first;
    const int base = level_span<Ev::kPref>(s.level, s.preferred1 ? uint32_t(s.preferred1) - 1u : uint32_t(GROVE_LEVEL_NONE), lvl, first);
    int sl = first;
    do {
      bool filtered = false;
      if constexpr (Ev::kStaged) {
        if (sl > lvl) {
          // the staged range holds at most kStageMax nodes: usually all its level-sl domains fit one warp pass.  A lane each:
          // filter them ONCE against the staged view, then attempt the survivors in visiting order (piece by piece, ascending
          // inside a piece -- the order of the general walk below)
          uint32_t d0 = 0, d1 = 0;
#pragma unroll
          for (uint32_t l = 0; l < GROVE_MAX_LEVELS; ++l) if (int(l) == sl) { d0 = pd0[l]; d1 = pd1[l]; }
          if (d1 - d0 <= 32u) {
            filtered = true;
            const long long tp0 = ev.rb.dbg ? clock64() : 0;
            const bool in = d0 + ev.lane < d1;
            uint32_t el = 0, eh = 0;
            if (in) { el = __ldg(tp.dom_lo[sl] + d0 + ev.lane); eh = __ldg(tp.dom_hi[sl] + d0 + ev.lane); }
            const uint32_t plaus = ev.scope_filter(s, el, eh, in, sl);
            const long long tp1 = ev.rb.dbg ? clock64() : 0;
            PieceIt pit; pit.init(ev.g, lo, hi, uint32_t(sl));
            for (uint32_t pa, pb; !ok && plaus && pit.next(ev.g, pa, pb);) {
              uint32_t todo = plaus & __ballot_sync(kFull, in && el >= pa && el < pb);
              while (todo && !ok) {
                const uint32_t src = __ffs(todo) - 1; todo &= todo - 1;
                const uint32_t l0 = __shfl_sync(kFull, el, src), h0 = __shfl_sync(kFull, eh, src);
                ok = place_scope(ev, s, l0, h0, sl);
                if (ok && ev.lane == 0) ev.sh.s_lo[si] = l0;
              }
            }
            if (ev.rb.dbg) { ev.t_pre += uint32_t(tp1 - tp0); ev.t_pack += uint32_t(clock64() - tp1); }
          }
        }
      }
      if (filtered) {
      } else if (sl > lvl) {
        PieceIt pit; pit.init(ev.g, lo, hi, uint32_t(sl));
        for (uint32_t pa, pb; !ok && pit.next(ev.g, pa, pb);) {
          const uint32_t d0 = __ldg(tp.next_dom[sl] + pa), d1 = __ldg(tp.next_dom[sl] + pb);
          // 32 scope domains at a time: a lane each runs the pre-filter (the table-time capacities are an upper
          // bound: a domain that lacks them cannot be packed), the plausible ones are attempted in order
          for (uint32_t db = d0; db < d1 && !ok; db += 32) {
            const uint32_t d = db + ev.lane;
            uint32_t el = 0, eh = 0;
            bool plaus = false;
            const long long tp0 = ev.rb.dbg ? clock64() : 0;
            if (d < d1) {
              el = __ldg(tp.dom_lo[sl] + d); eh = __ldg(tp.dom_hi[sl] + d);
              plaus = scope_plausible<Ev::kWide>(tp, ev.rb, ev.sh, s, el, eh, sl, d);
            }
            uint32_t todo = __ballot_sync(kFull, plaus);
            const long long tp1 = ev.rb.dbg ? clock64() : 0;
            while (todo && !ok) {
              const uint32_t src = __ffs(todo) - 1; todo &= todo - 1;
              const uint32_t l0 = __shfl_sync(kFull, el, src), h0 = __shfl_sync(kFull, eh, src);
              ok = place_scope(ev, s, l0, h0, sl);
              if (ok && ev.lane == 0) ev.sh.s_lo[si] = l0;
            }
            if (ev.rb.dbg) { ev.t_pre += uint32_t(tp1 - tp0); ev.t_pack += uint32_t(clock64() - tp1); }
          }
        }
      } else {
        ok = place_scope(ev, s, lo, hi, lvl);
        if (ok && ev.lane == 0) ev.sh.s_lo[si] = lo;
      }
      if (ok && ev.lane == 0) ev.sh.s_got[si] = int8_t(sl);
    } while (Ev::kPref && !ok && --sl >= base);
    if (!ok) { ev.np = 0; return false; }
  }
  return true;
}

// PlacementScore bookkeeping (oracle: score_unit): a unit that carries a pack constraint asked for `want` = Preferred
// if set else Required and was packed at level `got` (-1: no domain of its own): credit min(got, want) + 1 of want + 1
__device__ __forceinline__ void score_unit(uint32_t req, uint32_t pref, int got, uint32_t& num, uint32_t& den) {
  if (req == GROVE_LEVEL_NONE && pref == GROVE_LEVEL_NONE) return;
  const int want = pref != GROVE_LEVEL_NONE ? int(pref) : int(req);
  den += uint32_t(want) + 1u;
  num += uint32_t(min(got, want) + 1);
}

// The candidate pre-filter per (gang shape, domain): a CTA per 32 domains of one level, FOUR threads per domain (they share the
// gang's scopes: a base gang's scopes are independent chains of table look-ups), the shape's representative gang staged in
// shared memory.  Runs after every capacity-table build; k_eval then reads one bit per candidate.
template <bool kWide>
__global__ void __launch_bounds__(128) k_shape_plaus(Topo tp, Tables tb, Relax rx, const uint32_t* __restrict__ shape_rep) {
  __shared__ GangShared sh;
  __shared__ uint32_t s_bits;
  cudaGridDependencySynchronize();   // (launched chained: engine.cu launch_chained)
  const uint32_t shape = blockIdx.y, l = blockIdx.z;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, slot = threadIdx.x & 3u;
  const uint32_t gi = shape_rep[shape];
  const grove_gang_t gg = tb.gangs[gi];
  // candidate levels of the shape: Preferred (if any) down to Required; the whole cluster needs no table
  int first;
  const int base = level_span<true>(gg.level, gg.preferred, -1, first);
  if (int(l) > first || int(l) < base || l >= tp.L || blockIdx.x * 32u >= tp.n_dom[l]) return;
  for (uint32_t c = threadIdx.x; c < gg.n_cliques; c += blockDim.x) {
    const grove_clique_t q = tb.cliques[gg.clique_off + c];
    sh.clq[c] = make_uint4(q.req_cpu_milli, q.req_mem_mib, q.req_gpu,
                           uint32_t(q.min_replicas) | (uint32_t(q.replicas) << 8) | (uint32_t(q.level) << 16) |
                               (GROVE_CLIQUE_PREFERRED(q.scope) << 24));
    sh.sig[c] = tb.cinfo[gg.clique_off + c].sig;
    if constexpr (kWide) wide_cnt(sh)[c] = rx.ccount[gg.clique_off + c];
  }
  for (uint32_t si = threadIdx.x; si < gg.n_scopes; si += blockDim.x) sh.scopes[si] = tb.scopes[gg.scope_off + si];
  if (threadIdx.x == 0) s_bits = 0;
  __syncthreads();
  const uint32_t j = threadIdx.x >> 2, d = blockIdx.x * 32 + j;   // lanes 4j .. 4j + 3 of a warp share domain d
  bool plaus = d < tp.n_dom[l];
  if (plaus) {
    const uint32_t lo = __ldg(tp.dom_lo[l] + d), hi = __ldg(tp.dom_hi[l] + d);
    for (uint32_t si = slot; si < gg.n_scopes && plaus; si += 4) plaus = scope_ok<kWide>(tp, rx, sh, sh.scopes[si], lo, hi, int(l), d);
  }
  plaus = plaus & bool(__shfl_xor_sync(kFull, uint32_t(plaus), 1));
  plaus = plaus & bool(__shfl_xor_sync(kFull, uint32_t(plaus), 2));
  const uint32_t b = __ballot_sync(kFull, plaus && slot == 0);
  if (lane == 0) {
    uint32_t bits = 0;
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k) bits |= ((b >> (4 * k)) & 1u) << k;
    atomicOr(&s_bits, bits << (warp * 8));
  }
  __syncthreads();
  if (threadIdx.x == 0) const_cast<uint32_t*>(rx.shape_bits)[size_t(shape) * rx.pl_words + ((rx.pl_off[l] + blockIdx.x * 32) >> 5)] = s_bits;
}

// entry i of the round's evaluations: the heavy gangs of the list (from its head), the light ones (from its tail), then the new
// entrants of the window (ranks [kEntryLo, kHi): never evaluated, they need no list entry).  relax.cuh k_detect builds the list.
__device__ __forceinline__ uint32_t eval_list_at(const Relax& rx, const Tables& tb, uint32_t i) {
  const uint32_t nh = rx.ctl[kNHeavy], nl = rx.ctl[kNLight];
  if (i < nh) return rx.eval_list[i];
  if (i - nh < nl) return rx.eval_list[tb.G - 1u - (i - nh)];
  return tb.by_rank[rx.ctl[kEntryLo] + (i - nh - nl)];
}

// K3, one launch per round: CTAs of kEvalWarps warps take work items from a queue (ctl[kEvalNext]), in list order.  First the
// HEAVY gangs (the head of the list: their last evaluation needed many attempts), an item each, evaluated by the whole CTA; then
// the LIGHT ones (the tail of the list and the new entrants: most gangs, answered by their first or second candidate) in groups
// of consecutive entries, a warp each.  Heavy first is longest-first list scheduling: a round lasts as long as its slowest
// evaluation.  A light group holds as many entries as spread the light gangs over every CTA of the grid (at most kEvalWarps):
// a round with a few hundred of them puts one warp on each SM rather than eight on a few.
// A TEAM (the CTA, or one warp) evaluates one gang.  The candidates of the gang's level are pre-filtered 1024 at a time by all
// its warps (a lane each); the plausible ones are then attempted a warp each, and the lowest successful candidate IN ORDER is the
// answer -- exactly what trying them one after the other gives, minus the waiting.  A light evaluation that is still unanswered
// after `max_att` attempts gives up (kEvalDeferred): the gang stays dirty and comes back as a heavy one next round, instead of
// holding the round up.  Writes the "nxt" scratch of the gang.
// Launched as a programmatic dependent of the kernel before it (engine.cu launch_chained): nothing is read before
// cudaGridDependencySynchronize().
constexpr uint32_t kEvalDeferred = 0xFFu;   // nxt_tstate: no result this round
constexpr int kEvalWarps = 8;
// kWide: the instantiation of a wide cycle (16-bit counts; the entry stack of each warp in Relax::wide_node).
// kSpread: the instantiation of a cycle with topology spread members (spread.cuh): a member's candidates are those whose
// level-l_s domain is allowed (HARD, and the first walk of SOFT) or not allowed (the second walk of SOFT).
// kFence: the instantiation of a cycle with fences (fence.cuh): the nodes of an active fence of a gang ranked before the evaluated
// one fail K1 fit in every view it forms (staged attempts, unstaged reads, the record - total fast path).  The capacity tables and
// shape bits come from the committed table and stay upper bounds.
// kQueue: the instantiation of a cycle with queue members (queue.cuh): a member whose gate is closed is REJECTED without evaluation,
// and an admitted member packs each clique's surplus up to the replicas k_queue_gate allows.
// kImex: the instantiation of a cycle with enrolled cliques (imex.cuh): a node another CD holds in the gang's view fails K1 fit for
// the gang's enrolled cliques wherever a view is formed, like a fenced node.  Tables and shape bits stay ownership-blind upper bounds.
template <bool kPref, bool kHolds, bool kWide, bool kSpread = false, bool kFence = false, bool kQueue = false, bool kImex = false>
__global__ void __launch_bounds__(kEvalWarps * 32, 2) k_eval(Topo tp, Tables tb, Relax rx, uint32_t max_att) {
  __shared__ GangShared shs[kEvalWarps];
  __shared__ int4 s_view[kEvalWarps][kStageMax];
  __shared__ uint32_t s_vflag[kEvalWarps][kStageMax];
  __shared__ __align__(16) uint8_t s_rk[kEvalWarps][kStageMax + 256];
  // per team, in the row of its first warp w0: the plausible candidates of the current 1024-candidate chunk, in order; the
  // winning attempt, the extent read, the attempts and the plausible candidates so far
  __shared__ uint32_t s_plaus[kEvalWarps][32];
  __shared__ uint32_t s_win[kEvalWarps], s_ext[kEvalWarps], s_att[kEvalWarps], s_npl[kEvalWarps];
  __shared__ uint32_t s_cl[kEvalWarps][32], s_ch[kEvalWarps][32];   // node ranges of the first chunk's candidates: run c in row w0 + c
  __shared__ uint32_t s_item;
  cudaGridDependencySynchronize();
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (rx.ctl[kDone]) return;
  const uint32_t n_eval = rx.ctl[kNEval], n_heavy = rx.ctl[kNHeavy];
  const uint32_t n_light = n_eval - n_heavy;
  const uint32_t grp = min(uint32_t(kEvalWarps), max(1u, (n_light + gridDim.x - 1u) / gridDim.x));   // light entries per item
  const uint32_t n_items = n_heavy + (n_light + grp - 1u) / grp;
  GangShared& sh = shs[warp];
  uint32_t* wide_node = nullptr; uint16_t* wide_meta = nullptr;
  if constexpr (kWide) {
    const size_t w = size_t(blockIdx.x) * kEvalWarps + warp;
    wide_node = rx.wide_node + w * rx.wide_cap; wide_meta = rx.wide_meta + w * rx.wide_cap;
  }
  for (;;) {
    __syncthreads();   // the previous item's shared state is no longer read
    if (threadIdx.x == 0) s_item = atomicAdd(rx.ctl + kEvalNext, 1u);
    __syncthreads();
    const uint32_t item = s_item;
    if (item >= n_items) break;
    const bool cta = item < n_heavy;                  // CTA-uniform
    const uint32_t ei = cta ? item : n_heavy + (item - n_heavy) * grp + warp;
    if (!cta && (warp >= grp || ei >= n_eval)) continue;
    const uint32_t tw = cta ? uint32_t(kEvalWarps) : 1u;   // warps in the team
    const uint32_t w0 = cta ? 0u : warp;                   // the team's first warp
    const uint32_t wi = cta ? warp : 0u, tt = cta ? threadIdx.x : lane;   // warp / thread within the team
    auto team_sync = [cta]() { if (cta) __syncthreads(); else __syncwarp(); };
    const uint32_t gi = eval_list_at(rx, tb, ei);
    const grove_gang_t gg = tb.gangs[gi];
    const GangInfo info = tb.ginfo[gi];
    // the gang's cliques and scopes (a lane each), the words of the re-evaluation shortcut and the base gang's rank are asked for
    // BEFORE anything looks at them: one L2 round trip for all of them instead of one per question
    const bool has_c = lane < gg.n_cliques, has_s = lane < gg.n_scopes;
    const grove_clique_t q0 = has_c ? tb.cliques[gg.clique_off + lane] : grove_clique_t{};
    const CliqueInfo ci0 = has_c ? tb.cinfo[gg.clique_off + lane] : CliqueInfo{};
    uint32_t cnt0 = 0;
    if constexpr (kWide) cnt0 = has_c ? rx.ccount[gg.clique_off + lane] : 0u;
    const grove_scope_t sc0 = has_s ? tb.scopes[gg.scope_off + lane] : grove_scope_t{};
    const uint32_t round_now = rx.ctl[kRound];
    const uint32_t le = rx.last_eval[gi], fu_word = rx.fail_upto[gi], ext_word = rx.extent[gi];
    uint32_t sp_grp = kFull;
    if constexpr (kSpread) sp_grp = rx.sp.group[gi];
    uint32_t q_slot = kFull;
    if constexpr (kQueue) q_slot = rx.qu.slot[gi];
    // ---- gangs that need no packing
    uint32_t trivial = 0;
    if (gg.flags & GROVE_GANG_GATED) trivial = GROVE_GANG_GATED_SKIP;
    else if (gg.base_gang != GROVE_NONE_U32) {
      // considered at its own turn: the base gang must have been admitted before it (final, or tentatively so far)
      const uint32_t brank = tb.ginfo[gg.base_gang].order;
      uint32_t bs = GROVE_GANG_REJECTED;
      if (brank < info.order) bs = rx.tstate[gg.base_gang];   // final for ranks below the front; 0 (not evaluated yet) counts as not admitted: its first result marks us dirty
      if (bs != GROVE_GANG_ADMITTED) trivial = GROVE_GANG_BASE_REJECTED;
    }
    if constexpr (kQueue) if (!trivial && q_slot != kFull && rx.qu.gate[q_slot]) trivial = GROVE_GANG_REJECTED;   // its queue chain has no room
    if (trivial) {
      if (tt == 0) {
        rx.nxt_tstate[gi] = uint8_t(trivial); rx.nxt_n[gi] = 0; rx.nxt_info[gi] = 0xFFu; rx.nxt_glo[gi] = GROVE_NONE_U32; rx.nxt_extent[gi] = 0;
      }
      for (uint32_t si = tt; si < gg.n_scopes; si += tw * 32) { rx.nxt_sc_lvl[gg.scope_off + si] = 0xFFu; rx.nxt_sc_lo[gg.scope_off + si] = GROVE_NONE_U32; }
      continue;
    }
    GangRegs g;
    g.a = info.anchor; g.L = tp.L; g.n = tp.n; g.rank = info.order;
#pragma unroll
    for (int l = 0; l < GROVE_MAX_LEVELS; ++l) { g.anc_lo[l] = info.anc_lo[l]; g.anc_hi[l] = info.anc_hi[l]; }
    if (has_c) {   // every warp keeps its own copy: attempts run independently (GROVE_MAX_GANG_CLIQUES = 32: a lane each)
      const uint32_t c = lane;
      const grove_clique_t q = q0;
      const CliqueInfo ci = ci0;
      sh.clq[c] = make_uint4(q.req_cpu_milli, q.req_mem_mib, q.req_gpu,
                             uint32_t(q.min_replicas) | (uint32_t(q.replicas) << 8) | (uint32_t(q.level) << 16) |
                                 (GROVE_CLIQUE_PREFERRED(q.scope) << 24));
      sh.rcp[c] = make_float4(q.req_cpu_milli ? 1.0f / float(q.req_cpu_milli) : 0.f, q.req_mem_mib ? 1.0f / float(q.req_mem_mib) : 0.f,
                              q.req_gpu ? 1.0f / float(q.req_gpu) : 0.f, 0.f);
      sh.sig[c] = ci.sig; sh.smask[c] = uint32_t(q.class_mask) | (ci.need_depth << 16);
      sh.Hlo[c] = 0; sh.Hhi[c] = 0; sh.c_got[c] = -1;
      if constexpr (kWide) wide_cnt(sh)[c] = cnt0;
    }
    if (has_s) { sh.scopes[lane] = sc0; sh.s_got[lane] = -1; sh.s_lo[lane] = 0; }
    if (tt == 0) { s_win[w0] = GROVE_NONE_U32; s_ext[w0] = 0; s_att[w0] = 0; s_npl[w0] = 0; }
    team_sync();
    // A candidate that failed in the gang's last evaluation fails again unless a claim was withdrawn inside it since: views only
    // shrink otherwise (claims are added, settled claims move into the committed state).  So a re-evaluation skips the
    // candidates in front of its last answer that no withdrawal touched -- gangs that meet a nearly full cluster would
    // otherwise re-run dozens of failing attempts every round.  (Single candidate level only.)
    Ev<kPref, kHolds, kWide, kFence, kImex> ev(tp, rx, sh, g, lane);                  // candidates of any size, node state from L2
    EvS<kPref, kHolds, kWide, kFence, kImex> evs(tp, rx, sh, g, lane, s_view[warp], s_vflag[warp], s_rk[warp]);         // candidates of <= kStageMax nodes, node state staged in shared memory
    if constexpr (kWide) { ev.wn = evs.wn = wide_node; ev.wm = evs.wm = wide_meta; }
    if constexpr (kFence) {   // the fences active for this gang: a lane per entry (at most 64), fixed for the round (k_apply writes tstate)
      bool a0 = false, a1 = false;
      if (lane < rx.fc.n) { const uint4 f = rx.fc.list[lane]; a0 = f.x != kFull && f.z < g.rank && rx.tstate[f.w] == GROVE_GANG_REJECTED; }
      if (lane + 32u < rx.fc.n) { const uint4 f = rx.fc.list[lane + 32u]; a1 = f.x != kFull && f.z < g.rank && rx.tstate[f.w] == GROVE_GANG_REJECTED; }
      ev.fm0 = evs.fm0 = __ballot_sync(kFull, a0); ev.fm1 = evs.fm1 = __ballot_sync(kFull, a1);
    }
    if constexpr (kImex) {   // the enrolled cliques (a lane each) and the gang's CD, fixed for the cycle
      ev.enr = evs.enr = __ballot_sync(kFull, has_c && __ldg(rx.im.cd + gg.clique_off + lane) != GROVE_CD_NONE);
      ev.icd = evs.icd = __ldg(rx.im.rank_cd + g.rank);
    }
    bool staged = false;  // the winning attempt ran on evs
    bool won = false;     // this warp holds the answer
    bool done = false;    // CTA-uniform
    int g_got = -1; uint32_t g_lo = 0;
    const long long t0 = rx.dbg ? clock64() : 0;
    // candidate levels: the Preferred level first (if any), widened level by level up to the Required one
    // (gl == -1: the whole cluster as a single candidate)
    int gfirst;
    const int gbase = level_span<kPref>(gg.level, gg.preferred, -1, gfirst);
    int gl = gfirst;
    // a spread member: its group's level and mode, its allowed row.  The shortcut over the candidates that failed last time does
    // not hold for it: a candidate that was not allowed then may be now
    uint32_t sp_lvl = 0, sp_mode = 0;
    const uint32_t* sp_bits = nullptr;
    if constexpr (kSpread) {
      if (sp_grp != kFull) { const uint32_t w = rx.sp.info[sp_grp]; sp_lvl = w & 0xFFu; sp_mode = (w >> 8) & 0xFFu; sp_bits = rx.sp.allowed + rx.sp.row[gi]; }
    }
    const uint32_t fu = (!sp_mode && le && gfirst == gbase && gfirst >= 0) ? fu_word : 0u;
    uint32_t k_won = 0;
    bool gave_up = false;
    bool sp_full = false;   // a SOFT member reached its second walk: its extent is the whole visiting order
    for (uint32_t walk = 0;; ++walk) {
    gl = gfirst;
    do {
      if (gl < 0) {
        staged = false;
        if (wi == 0) {
          won = place_in(ev, gg.n_scopes, 0, tp.n, -1);
          if (won) { g_got = -1; g_lo = 0; if (lane == 0) s_win[w0] = 0; }
          if (lane == 0) s_att[w0] += 1;
        }
        team_sync();
        done = s_win[w0] != GROVE_NONE_U32;
      } else {
        // candidate domains of level gl in score order: up to kMaxPieces ranges of domain indices
        uint32_t r0[kMaxPieces], rcnt[kMaxPieces], D = 0;
        {
          uint32_t plo[kMaxPieces], phi[kMaxPieces];
          const int npc = make_pieces(g, 0, tp.n, uint32_t(gl), plo, phi);
          for (int p = 0; p < kMaxPieces; ++p) {
            r0[p] = 0; rcnt[p] = 0;
            if (p < npc) { r0[p] = __ldg(tp.next_dom[gl] + plo[p]); rcnt[p] = __ldg(tp.next_dom[gl] + phi[p]) - r0[p]; D += rcnt[p]; }
          }
        }
        auto cand = [&](uint32_t k, uint32_t& dl, uint32_t& dh) -> uint32_t {   // k-th candidate in order -> its domain
          uint32_t d = 0, rem = k;
#pragma unroll
          for (int p = 0; p < kMaxPieces; ++p) { if (rem < rcnt[p]) { d = r0[p] + rem; break; } rem -= rcnt[p]; }
          dl = __ldg(tp.dom_lo[gl] + d); dh = __ldg(tp.dom_hi[gl] + d);
          return d;
        };
        // candidates are taken in chunks that grow (tw x 32, then up to 1024): most gangs succeed among the first few
        for (uint32_t base = 0, nchunk = tw; base < D && !done && !gave_up; base += nchunk * 32, nchunk = min(32u, nchunk * 4u)) {
          // pre-filter: nchunk runs of 32 candidates, dealt to the team's warps
          for (uint32_t c = wi; c < nchunk; c += tw) {
            const uint32_t k = base + c * 32 + lane;
            bool plaus = false;
            if (k < D) {
              // the candidate's node range is fetched together with its pre-filter bit (the attempt would otherwise pay one more
              // L2 round trip for it); the first chunk's ranges wait in shared memory
              uint32_t dl, dh; const uint32_t d = cand(k, dl, dh);
              if (rx.shape_bits) {   // one bit per (shape, domain), refreshed with the capacity tables
                const uint32_t bit = rx.pl_off[gl] + d;
                plaus = (__ldg(rx.shape_bits + size_t(info.pad) * rx.pl_words + (bit >> 5)) >> (bit & 31u)) & 1u;
              } else {
                plaus = gang_plausible<kWide>(tp, rx, sh, gg.n_scopes, dl, dh, gl, d);
              }
              if (base == 0) { s_cl[w0 + c][lane] = dl; s_ch[w0 + c][lane] = dh; }   // (c < tw in the first chunk)
              if constexpr (kSpread) {
                if (sp_mode && plaus) {   // the level-l_s domain of the candidate's first node: allowed in walk 0, not allowed in walk 1
                  const uint32_t A = __ldg(reinterpret_cast<const uint32_t*>(tp.ndom) + size_t(dl) * 4u + sp_lvl);
                  plaus = ((__ldg(sp_bits + (A >> 5)) >> (A & 31u)) & 1u) == (walk == 0 ? 1u : 0u);
                }
              }
              if (plaus && k < fu) {   // failed last time: worth another attempt only if somebody withdrew a claim in there since
                bool again = false;
                for (uint32_t w = dl >> 5; w <= (dh - 1u) >> 5; ++w) again |= __ldg(rx.rem_round + w) >= le;
                plaus = again;
              }
            }
            const uint32_t b = __ballot_sync(kFull, plaus);
            if (lane == 0) s_plaus[w0][c] = b;
          }
          team_sync();
          uint32_t total = 0;
          for (uint32_t c = 0; c < nchunk; ++c) total += __popc(s_plaus[w0][c]);
          if (tt == 0) s_npl[w0] += total;
          // attempts: tw plausible candidates at a time, in order, a warp each
          for (uint32_t j0 = 0; j0 < total && !done; j0 += tw) {
            if (!cta && max_att && s_att[w0] >= max_att) { gave_up = true; break; }   // team-uniform (read after a barrier)
            const uint32_t j = j0 + wi;
            bool ok = false; uint32_t dl = 0, dh = 0;
            if (j < total) {
              uint32_t rem = j, c = 0;   // the j-th set bit of the bitmap
              for (; c + 1 < nchunk; ++c) { const uint32_t pc = __popc(s_plaus[w0][c]); if (rem < pc) break; rem -= pc; }
              uint32_t w = s_plaus[w0][c];
              for (uint32_t i = 0; i < rem; ++i) w &= w - 1;
              const uint32_t kl = __ffs(w) - 1, k = base + c * 32 + kl;
              if (base == 0) { dl = s_cl[w0 + c][kl]; dh = s_ch[w0 + c][kl]; } else cand(k, dl, dh);
              staged = dh - dl <= kStageMax;
              ok = staged ? place_in(evs, gg.n_scopes, dl, dh, gl) : place_in(ev, gg.n_scopes, dl, dh, gl);
              if (lane == 0) { atomicAdd(&s_att[w0], 1u); if (ok) atomicMin(&s_win[w0], j); }
              if (ok) k_won = k;
            }
            team_sync();
            const uint32_t win = s_win[w0];
            if (win != GROVE_NONE_U32) { done = true; won = ok && win == j; if (won) { g_got = gl; g_lo = dl; } }
          }
          team_sync();   // s_plaus is rewritten by the next chunk
        }
      }
    } while (kPref && !done && !gave_up && --gl >= gbase);
    if (!(kSpread && sp_mode == GROVE_SPREAD_SOFT && walk == 0 && !done && !gave_up)) break;
    sp_full = true;
    }
    // what any of the attempts may have read (attempts past the winner only widen it)
    if (lane == 0) atomicMax(&s_ext[w0], max(max(max(ev.ext, evs.ext), fu ? ext_word : 0u), sp_full ? tp.n : 0u));   // skipped candidates were read by the last evaluation
    team_sync();
    if (tt == 0) rx.last_att[gi] = uint8_t(gave_up ? 255u : min(254u, s_att[w0]));
    if (gave_up) {   // no result this round: k_apply keeps the gang dirty
      if (tt == 0) rx.nxt_tstate[gi] = uint8_t(kEvalDeferred);
      continue;
    }
    if (rx.dbg && tt == 0) {
      const uint32_t cyc = uint32_t(clock64() - t0);
      rx.dbg[gi * 8 + 0] += 1; rx.dbg[gi * 8 + 1] += s_npl[w0]; rx.dbg[gi * 8 + 2] += s_att[w0];
      rx.dbg[gi * 8 + 3] = max(rx.dbg[gi * 8 + 3], cyc); rx.dbg[gi * 8 + 4] = cyc; rx.dbg[gi * 8 + 5] = s_att[w0]; rx.dbg[gi * 8 + 6] = s_npl[w0]; rx.dbg[gi * 8 + 7] = rx.ctl[kRound];
      // warp 0's own phases, summed over the cycle: staging, sub-domain pre-filter, packing, attempts staged
      atomicAdd(rx.dbg + tb.G * 8 + 0, evs.t_stage); atomicAdd(rx.dbg + tb.G * 8 + 1, evs.t_pre); atomicAdd(rx.dbg + tb.G * 8 + 2, evs.t_pack);
      atomicAdd(rx.dbg + tb.G * 8 + 3, evs.n_stage); atomicAdd(rx.dbg + tb.G * 8 + 4, cyc); atomicAdd(rx.dbg + tb.G * 8 + 5, 1u);
      atomicAdd(rx.dbg + tb.G * 8 + 6, evs.t_st2); atomicAdd(rx.dbg + tb.G * 8 + 7, evs.t_st3);
    }
    if (!done) {
      if (tt == 0) {
        rx.last_eval[gi] = round_now; rx.fail_upto[gi] = kFull;   // every candidate failed
        rx.nxt_tstate[gi] = GROVE_GANG_REJECTED; rx.nxt_n[gi] = 0; rx.nxt_info[gi] = 0xFFu; rx.nxt_glo[gi] = GROVE_NONE_U32;
        rx.nxt_extent[gi] = s_ext[w0];
      }
      for (uint32_t si = tt; si < gg.n_scopes; si += tw * 32) { rx.nxt_sc_lvl[gg.scope_off + si] = 0xFFu; rx.nxt_sc_lo[gg.scope_off + si] = GROVE_NONE_U32; }
      continue;
    }
    if (!won) continue;   // warp-uniform: the winner finishes alone
    // surplus beyond MinReplicas (best effort, podgang.go:80-83), inside the domain each clique was packed into
    for (uint32_t cr = 0; cr < gg.n_cliques; ++cr) {
      const uint32_t mn = clq_min<kWide>(sh, cr);
      uint32_t rp = clq_rep<kWide>(sh, cr);
      if constexpr (kQueue) if (q_slot != kFull) rp = rx.qu.cap[gg.clique_off + cr];
      if (rp > mn) { if (staged) evs.take(cr, sh.Hlo[cr], sh.Hhi[cr], rp - mn); else ev.take(cr, sh.Hlo[cr], sh.Hhi[cr], rp - mn); }
    }
    __syncwarp();
    const uint32_t n_ent = staged ? evs.np : ev.np;
    // PlacementScore: levels honoured / levels asked for, over the gang, its scopes and its cliques
    uint32_t num = 0, den = 0;
    if (lane == 0) score_unit(gg.level, gg.preferred, g_got, num, den);
    if (lane < gg.n_scopes) {
      const grove_scope_t s = sh.scopes[lane];
      score_unit(s.level, s.preferred1 ? uint32_t(s.preferred1) - 1u : uint32_t(GROVE_LEVEL_NONE), int(sh.s_got[lane]), num, den);
    }
    if (lane < gg.n_cliques) {
      const uint32_t w = sh.clq[lane].w;
      score_unit((w >> 16) & 0xFFu, w >> 24, int(sh.c_got[lane]), num, den);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { num += __shfl_xor_sync(kFull, num, o); den += __shfl_xor_sync(kFull, den, o); }
    if (den == 0) { num = 1; den = 1; }
    for (uint32_t i = lane; i < n_ent; i += 32) {
      rx.nxt_node[info.pod_off + i] = ev.en(i);   // (ev and evs share the entry stack)
      rx.nxt_meta[info.pod_off + i] = ev.em(i);
    }
    for (uint32_t si = lane; si < gg.n_scopes; si += 32) {
      const bool own = int(sh.s_got[si]) > g_got;   // a scope packed at the gang's own level has no domain of its own
      rx.nxt_sc_lvl[gg.scope_off + si] = own ? uint8_t(sh.s_got[si]) : uint8_t(0xFFu);
      rx.nxt_sc_lo[gg.scope_off + si] = own ? sh.s_lo[si] : GROVE_NONE_U32;
    }
    if (lane == 0) {
      rx.last_eval[gi] = round_now; rx.fail_upto[gi] = g_got >= 0 ? k_won : 0u;
      rx.nxt_tstate[gi] = GROVE_GANG_ADMITTED; rx.nxt_n[gi] = uint16_t(n_ent);
      rx.nxt_info[gi] = (g_got >= 0 ? uint32_t(g_got) : 0xFFu) | (num << 8) | (den << 20);
      rx.nxt_glo[gi] = g_got >= 0 ? g_lo : GROVE_NONE_U32;
      rx.nxt_extent[gi] = max(max(ev.ext, evs.ext), s_ext[w0]);   // the surplus pass above may have read further
    }
  }
}

}  // namespace grove
