// Device-resident reclaim views of grove_run_cycle_reuse_preempt (DESIGN.md section 1, "Reuse with reclaim").
//
// The running gangs' holdings are uploaded once per call as a per-node CSR over the sorted node order: row n lists every
// (running gang, what it holds on n), running gangs ascending.  A mask marks the running gangs that are gone (released or
// evicted).  A class view is the committed table plus the standing holdings of the running gangs below the class's priority;
// one thread per node sums its own row, so no atomics and the table does not depend on thread order.
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

// add > 0: real = the committed table as it is (the class's free table), then table += standing holdings of priority < p (the
// class view).  add == 0: table -= the same sum (back to the free table once the class's victims are marked gone).
__global__ void __launch_bounds__(256) k_reclaim_view(uint4* nres, uint4* real, ReclaimCsr c, uint32_t N, int32_t p, uint32_t add) {
  const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  uint32_t s0 = 0, s1 = 0, s2 = 0;   // (gpu | pods << 16 sums field by field: the check above rules out a carry)
  for (uint32_t i = c.off[n]; i < c.off[n + 1]; ++i) {
    const uint4 h = c.ent[i];
    if (!c.gone[h.x] && c.prio[h.x] < p) { s0 += h.y; s1 += h.z; s2 += h.w; }
  }
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
