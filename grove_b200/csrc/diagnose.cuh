// diagnose.cuh -- why each rejected gang of the last grove_run_cycle did not fit (DESIGN.md section 1, "Diagnosis").
//
// Runs after the cycle, on its outputs, and writes nothing the cycle's getters read.  Gang g is judged against
//   V_g(n) = F_end(n) + sum of the usage of the admitted gangs ranked after g on node n,
// the table the sequential pass evaluated g against.  The usage is kept per node as a list of records (one per bound pod) in
// rank order with suffix sums, so V_g(n) is the committed record plus one binary search.  The predicates and the exact
// capacities are then computed per (rejected gang, clique, node) with plain integer division (no reciprocal, no 255 cap),
// counted per warp and summed per domain of the gang's Required level; a second kernel counts the domains in which every
// clique finds its MinReplicas on its own and writes the verdict.
#pragma once
#include "common.cuh"

namespace grove {

// one rejected gang of a diagnosis batch
struct DiagGang {
  uint32_t gang;        // index in the submission
  uint32_t rank;        // order rank
  uint32_t col_off;     // first column of its domain sums in the batch's scratch: [clique][domain]
  uint32_t ncol;        // level-l domains (1 without a Required level)
  uint16_t n_cliques;
  uint8_t level;        // Required level, GROVE_LEVEL_NONE = the whole cluster is one domain
  uint8_t pad;
};

// the admitted gangs' usage by sorted node: records [off[n], off[n + 1]) of node n, ranks ascending after k_diag_suffix;
// x = cpu, y = mem, z = gpu | pods << 16, w = rank (suffix sums in x..z once built)
struct DiagUse {
  const uint32_t* off;  // [npad + 1]
  const uint4* rec;
};

// pods bound per sorted node
__global__ void __launch_bounds__(256) k_diag_count(const grove_placement_t* __restrict__ out, uint32_t n_out,
                                                    const uint32_t* __restrict__ inv, uint32_t* cnt) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_out) atomicAdd(cnt + inv[out[i].node], 1u);
}

// exclusive scan of cnt[0, n) into off[0, n]; one CTA of 1024 threads, a contiguous chunk each.  cur[] = 0 for the fill.
__global__ void __launch_bounds__(1024) k_diag_scan(const uint32_t* __restrict__ cnt, uint32_t* __restrict__ off,
                                                    uint32_t* __restrict__ cur, uint32_t n) {
  __shared__ uint32_t s_warp[32];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t per = (n + 1023) / 1024, a = min(n, tid * per), z = min(n, a + per);
  uint32_t sum = 0;
  for (uint32_t i = a; i < z; ++i) sum += cnt[i];
  const uint32_t inc = warp_incl_scan(sum, lane);
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) s_warp[lane] = warp_incl_scan(s_warp[lane], lane);
  __syncthreads();
  uint32_t run = inc - sum + (warp ? s_warp[warp - 1] : 0u);
  for (uint32_t i = a; i < z; ++i) { off[i] = run; run += cnt[i]; cur[i] = 0; }
  if (tid == 1023) off[n] = run;
}

// one record per bound pod: what one pod of its clique takes, and its gang's rank
__global__ void __launch_bounds__(256) k_diag_fill(const grove_placement_t* __restrict__ out, uint32_t n_out,
                                                   const uint32_t* __restrict__ inv, Tables tb, const uint32_t* __restrict__ off,
                                                   uint32_t* cur, uint4* __restrict__ rec) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  const grove_placement_t p = out[i];
  const uint32_t n = inv[p.node];
  const grove_clique_t q = tb.cliques[p.clique];
  rec[off[n] + atomicAdd(cur + n, 1u)] =
      make_uint4(q.req_cpu_milli, q.req_mem_mib, uint32_t(q.req_gpu) | (1u << 16), tb.ginfo[tb.cinfo[p.clique].gang].order);
}

// per node: its records by rank (insertion sort: a node holds few pods), then suffix sums from the highest rank down.  A sum
// never exceeds the free table the cycle started from, so gpu | pods << 16 adds without a carry.
__global__ void __launch_bounds__(256) k_diag_suffix(const uint32_t* __restrict__ off, uint4* rec, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t a = off[i], z = off[i + 1];
  for (uint32_t k = a + 1; k < z; ++k) {
    const uint4 v = rec[k];
    uint32_t j = k;
    for (; j > a && rec[j - 1].w > v.w; --j) rec[j] = rec[j - 1];
    rec[j] = v;
  }
  uint32_t s0 = 0, s1 = 0, s2 = 0;
  for (uint32_t k = z; k > a; --k) {
    uint4 v = rec[k - 1];
    s0 += v.x; s1 += v.y; s2 += v.z;
    v.x = s0; v.y = s1; v.z = s2;
    rec[k - 1] = v;
  }
}

// V_g(n): the committed record plus the usage of the admitted gangs ranked after `rank`
__device__ __forceinline__ uint4 diag_view(const uint4* nres, DiagUse u, uint32_t n, uint32_t rank) {
  uint4 r = nres[n];
  uint32_t lo = u.off[n], hi = u.off[n + 1];
  while (lo < hi) {   // first record of a rank after `rank`
    const uint32_t m = (lo + hi) >> 1;
    if (u.rec[m].w > rank) hi = m; else lo = m + 1;
  }
  if (lo < u.off[n + 1]) { const uint4 s = u.rec[lo]; r.x += s.x; r.y += s.y; r.z += s.z; }
  return r;
}

// the level-`level` domain of sorted node n (GROVE_LEVEL_NONE: the whole cluster is domain 0)
__device__ __forceinline__ uint32_t diag_domain(const Topo& tp, uint32_t n, uint32_t level) {
  if (level == GROVE_LEVEL_NONE) return 0;
  const uint4 dm = tp.ndom[n];
  return level == 0 ? dm.x : level == 1 ? dm.y : level == 2 ? dm.z : dm.w;
}

// K1 fit of clique q on a node with record r, exactly (k_diag_fit's predicates and capacity; k_diag_fit keeps its own copy of
// them: written through this function it needs 32 registers instead of 30): 0 = fits, 1..7 = the first predicate it fails (the order of
// grove_clique_diag_t), and the pods that fit (cap, left 0 unless it fits), by integer division with no 255 cap
__device__ __forceinline__ uint32_t diag_fit(const uint4& r, const grove_clique_t& q, uint32_t need_depth, uint32_t& cap) {
  const uint32_t gpu = r.z & 0xFFFFu, pods = r.z >> 16, depth = (r.w >> 16) & 0xFu, cls = (r.w >> GROVE_NODE_CLASS_SHIFT) & 0xFu;
  uint32_t cat;
  if (!(r.w & GROVE_NODE_SCHEDULABLE)) cat = 1;
  else if (!((q.class_mask >> cls) & 1u)) cat = 2;
  else if (depth < need_depth) cat = 3;
  else if (r.x < q.req_cpu_milli) cat = 4;
  else if (r.y < q.req_mem_mib) cat = 5;
  else if (gpu < q.req_gpu) cat = 6;
  else if (pods < 1) cat = 7;
  else {
    cat = 0; cap = pods;
    if (q.req_cpu_milli) cap = min(cap, r.x / q.req_cpu_milli);
    if (q.req_mem_mib) cap = min(cap, r.y / q.req_mem_mib);
    if (q.req_gpu) cap = min(cap, gpu / q.req_gpu);
  }
  return cat;
}

// grid = (npad / 256 node tiles, gangs of the batch).  Per clique of the gang: the node's failure class (0 = fits, 1..7 = the
// first predicate it fails, in the order of grove_clique_diag_t) counted with one ballot per class, the exact capacity summed
// over the warp into pods_fit, and -- for cliques with MinReplicas > 0 -- over the lanes that share the node's level-l domain
// (contiguous in sorted order: one __match_any_sync per node) into that domain's column.
__global__ void __launch_bounds__(256) k_diag_fit(Topo tp, Tables tb, DiagUse use, const DiagGang* __restrict__ dg,
                                                  const uint32_t* __restrict__ minr, unsigned long long* colsum,
                                                  grove_clique_diag_t* cd) {
  const DiagGang d = dg[blockIdx.y];
  const grove_gang_t g = tb.gangs[d.gang];
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t node = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = node < tp.n;
  const uint4 r = valid ? diag_view(tp.nres, use, node, d.rank) : make_uint4(0, 0, 0, 0);
  uint32_t key = GROVE_DOM_ABSENT;
  if (valid) {
    if (d.level == GROVE_LEVEL_NONE) key = 0;
    else { const uint4 dm = tp.ndom[node]; key = d.level == 0 ? dm.x : d.level == 1 ? dm.y : d.level == 2 ? dm.z : dm.w; }
  }
  const uint32_t seg = __match_any_sync(kFull, key);
  const bool leader = key != GROVE_DOM_ABSENT && lane == uint32_t(__ffs(seg) - 1);
  const uint32_t gpu = r.z & 0xFFFFu, pods = r.z >> 16, depth = (r.w >> 16) & 0xFu, cls = (r.w >> GROVE_NODE_CLASS_SHIFT) & 0xFu;
  for (uint32_t c = 0; c < d.n_cliques; ++c) {
    const uint32_t qi = g.clique_off + c;
    const grove_clique_t q = tb.cliques[qi];
    uint32_t cat = 8, cap = 0;   // 8: padding node, counted nowhere
    if (valid) {   // (diag_fit above restates this chain for fence.cuh: a change here goes there too)
      if (!(r.w & GROVE_NODE_SCHEDULABLE)) cat = 1;
      else if (!((q.class_mask >> cls) & 1u)) cat = 2;
      else if (depth < tb.cinfo[qi].need_depth) cat = 3;
      else if (r.x < q.req_cpu_milli) cat = 4;
      else if (r.y < q.req_mem_mib) cat = 5;
      else if (gpu < q.req_gpu) cat = 6;
      else if (pods < 1) cat = 7;
      else {
        cat = 0; cap = pods;
        if (q.req_cpu_milli) cap = min(cap, r.x / q.req_cpu_milli);
        if (q.req_mem_mib) cap = min(cap, r.y / q.req_mem_mib);
        if (q.req_gpu) cap = min(cap, gpu / q.req_gpu);
      }
    }
    uint32_t* cnt = &cd[qi].nodes_fit;
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k) {
      const uint32_t b = __ballot_sync(kFull, cat == k);
      if (lane == 0 && b) atomicAdd(cnt + k, uint32_t(__popc(b)));
    }
    const uint32_t s = __reduce_add_sync(kFull, cap);   // <= 32 * 65535
    if (lane == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(&cd[qi].pods_fit), (unsigned long long)s);
    if ((minr[qi] & 0xFFFFu) && d.ncol) {
      const uint32_t ds = __reduce_add_sync(seg, cap);
      if (leader && ds) atomicAdd(colsum + d.col_off + size_t(c) * d.ncol + key, (unsigned long long)ds);
    }
  }
}

// a CTA per gang of the batch: the domains in which every clique with MinReplicas > 0 has that many pods fitting on its own,
// then the verdict
__global__ void __launch_bounds__(256) k_diag_verdict(Tables tb, const DiagGang* __restrict__ dg, const uint32_t* __restrict__ minr,
                                                      const unsigned long long* __restrict__ colsum,
                                                      const grove_clique_diag_t* __restrict__ cd, grove_gang_diag_t* gd) {
  __shared__ uint32_t s_ok;
  const DiagGang d = dg[blockIdx.x];
  const uint32_t co = tb.gangs[d.gang].clique_off;
  if (threadIdx.x == 0) s_ok = 0;
  __syncthreads();
  uint32_t ok = 0;
  for (uint32_t col = threadIdx.x; col < d.ncol; col += blockDim.x) {
    bool all = true;
    for (uint32_t c = 0; c < d.n_cliques && all; ++c) {
      const uint32_t m = minr[co + c] & 0xFFFFu;
      if (m) all = colsum[d.col_off + size_t(c) * d.ncol + col] >= m;
    }
    ok += all;
  }
  if (ok) atomicAdd(&s_ok, ok);
  __syncthreads();
  if (threadIdx.x) return;
  grove_gang_diag_t o{};
  o.level = d.level;
  o.domains = d.level == GROVE_LEVEL_NONE ? 1u : d.ncol;
  o.domains_ok = s_ok;
  o.verdict = d.level != GROVE_LEVEL_NONE && s_ok == 0 ? GROVE_DIAG_NO_DOMAIN : GROVE_DIAG_NO_JOINT_FIT;
  for (uint32_t c = 0; c < d.n_cliques; ++c)
    if (cd[co + c].pods_fit < (minr[co + c] & 0xFFFFu)) { o.verdict = GROVE_DIAG_CLIQUE_SHORT; o.clique = uint16_t(c); break; }
  gd[d.gang] = o;
}

}  // namespace grove
