// Device-resident reclaim views of the reclaim loop (DESIGN.md section 1, "Reuse with reclaim", "Reclaim across queues").
//
// The running gangs' holdings are uploaded once per call as a per-node CSR over the sorted node order: row n lists every
// (running gang, what it holds on n), running gangs ascending.  A mask marks the running gangs that are gone (released or
// evicted); an evict mask marks the standing running gangs a class may evict (below the class's priority, or the donor set of
// donor.cuh).  A class view is the committed table plus what they hold; one thread per node sums its own row, so no atomics and the
// table does not depend on thread order.
#pragma once
#include "common.cuh"

struct ReclaimCsr {
  const uint32_t* off;   // [N + 1] row offsets, sorted node order
  const uint4* ent;      // x = running gang, y = cpu, z = mem, w = gpu | pods << 16
  const int32_t* prio;   // [running] priority
  const uint8_t* gone;   // [running] 1: released or evicted
};

// Does free plus everything every running gang holds still fit the node record's fields?  *bad = 1 where it does not.
__global__ void __launch_bounds__(256) k_reclaim_check(const uint4* nres, ReclaimCsr c, uint32_t N, uint32_t* bad) {
  const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const uint4 r = nres[n];
  uint64_t v[4] = {r.x, r.y, r.z & 0xFFFFu, r.z >> 16};
  for (uint32_t i = c.off[n]; i < c.off[n + 1]; ++i) {
    const uint4 h = c.ent[i];
    v[0] += h.y; v[1] += h.z; v[2] += h.w & 0xFFFFu; v[3] += h.w >> 16;
  }
  if (v[0] > 0xFFFFFFFFull || v[1] > 0xFFFFFFFFull || v[2] > 0xFFFFu || v[3] > 0xFFFFu) *bad = 1u;
}

// add > 0: real = the committed table as it is (the class's free table), then table += the holdings of the running gangs the
// evict mask marks (the class view: the standing gangs the class may evict).  add == 0: table -= the same sum, with the mask then
// marking those of them still standing (back to the free table once the class's victims are gone).
__global__ void __launch_bounds__(256) k_reclaim_view(uint4* nres, uint4* real, const uint32_t* off, const uint4* ent, const uint8_t* evict,
                                                      uint32_t N, uint32_t add) {
  const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  uint32_t s0 = 0, s1 = 0, s2 = 0;   // (gpu | pods << 16 sums field by field: the check above rules out a carry)
  for (uint32_t i = off[n]; i < off[n + 1]; ++i) {
    const uint4 h = ent[i];
    if (evict[h.x]) { s0 += h.y; s1 += h.z; s2 += h.w; }
  }
  uint4 r = nres[n];
  if (add) real[n] = r;
  if (!(s0 | s1 | s2)) return;
  if (add) { r.x += s0; r.y += s1; r.z += s2; }
  else { r.x -= s0; r.y -= s1; r.z -= s2; }
  nres[n] = r;
}

// The surplus pods of grove_run_cycle_preempt_elastic, uploaded once per call as a per-node CSR over the sorted node order: row n
// lists the pods on n in the caller's order, each as x = running gang, y = cpu, z = mem, w = gpu | 1 << 16 (its pod slot); taken[i]
// marks entry i as taken.  Every pod lies inside its gang's holdings on its node (the entry checks it), so no sum below can
// borrow or carry from one packed field into the next.
struct SurplusCsr {
  const uint32_t* off;   // [N + 1]
  const uint4* ent;
  const uint8_t* taken;
};

// The views of the elastic reclaim loop, as k_reclaim_view's, for the running gangs the evict mask marks.  whole == 0: the
// surplus view, their untaken surplus pods; whole == 1: the whole view, their holdings minus their taken surplus pods.  add > 0:
// real = the table as it is (the pass's free table), then table += the view; add == 0: table -= the same sum.
__global__ void __launch_bounds__(256) k_elastic_view(uint4* nres, uint4* real, const uint32_t* off, const uint4* ent, SurplusCsr s,
                                                      const uint8_t* evict, uint32_t N, uint32_t add, uint32_t whole) {
  const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  uint32_t h0 = 0, h1 = 0, h2 = 0;   // whole: the holdings of the marked gangs
  if (whole)
    for (uint32_t i = off[n]; i < off[n + 1]; ++i) {
      const uint4 h = ent[i];
      if (evict[h.x]) { h0 += h.y; h1 += h.z; h2 += h.w; }
    }
  uint32_t p0 = 0, p1 = 0, p2 = 0;   // their surplus pods: the untaken ones (surplus view) or the taken ones (whole view)
  for (uint32_t i = s.off[n]; i < s.off[n + 1]; ++i) {
    const uint4 p = s.ent[i];
    if (evict[p.x] && (s.taken[i] != 0) == (whole != 0)) { p0 += p.y; p1 += p.z; p2 += p.w; }
  }
  uint32_t s0 = p0, s1 = p1, s2 = p2;
  if (whole) { s0 = h0 - p0; s1 = h1 - p1; s2 = h2 - p2; }
  uint4 r = nres[n];
  if (add) real[n] = r;
  if (!(s0 | s1 | s2)) return;
  if (add) { r.x += s0; r.y += s1; r.z += s2; }
  else { r.x -= s0; r.y -= s1; r.z -= s2; }
  nres[n] = r;
}

// rows idx[i] (sorted node) of a table -> out[i]
__global__ void __launch_bounds__(256) k_reclaim_rows(const uint4* tab, const uint32_t* idx, uint4* out, uint32_t m) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) out[i] = tab[idx[i]];
}

// rec[i] = (sorted node, cpu, mem, gpu | pods << 16) added modulo 2^32 (a negative change comes as its two's complement);
// one record per node
__global__ void __launch_bounds__(256) k_reclaim_patch(uint4* nres, const uint4* rec, uint32_t m) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint4 d = rec[i];
  uint4 r = nres[d.x];
  r.x += d.y; r.y += d.z; r.z += d.w;
  nres[d.x] = r;
}
