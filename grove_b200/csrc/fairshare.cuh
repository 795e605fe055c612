// fairshare.cuh -- the turn order O(R) of a fair-share cycle (DESIGN.md section 1, "Fair-share order").
//
// Given each gang's usage U (what it charges to its queue chain when admitted, 0 otherwise), the order in which gangs take their
// turns is the merge, bottom-up over the queue tree, of every node's children's sequences by head key (share of the child at that
// turn, rank of the head).  A leaf's sequence is its gangs in rank order.  The merge is computed one tree level at a time over all
// gangs at once: the elements of the level's sequences get their child's load at their turn (a segmented exclusive scan of U), the
// key (share, rank), its prefix max along the child's sequence (so that a merge by head becomes a stable sort), and one stable sort
// by (parent, key) forms the parents' sequences.  Shares are compared exactly (128-bit cross products), as the host's share_of
// does.  Tree node ids: the queues 0..NQ-1, NQ = the pseudo-queue of the gangs with no queue (depth 1, share always 0), NQ + 1 =
// the root.
#pragma once
#include "common.cuh"

struct FsKey {
  unsigned long long num, den;   // share = num / den; den 0 = +inf
  uint32_t owner, rank;          // tree node whose sequence the element is in (or joins), rank of the gang
};
struct FsUse { long long v[3]; };

struct FsTree {
  const uint32_t* parent;              // [node] parent node
  const uint8_t* depth;                // [node] 1 for a top-level queue and the pseudo-queue, 0 for the root
  const long long* load0;              // [node * 3 + resource] starting load (own used + descendants')
  const unsigned long long* quota;     // [node * 3 + resource] deserved, GROVE_QUEUE_UNLIMITED = none
  const uint32_t* leaf;                // [gang] its queue, or the pseudo-queue
  const uint32_t* rank;                // [gang] (priority desc, submission index asc)
};

__device__ __forceinline__ bool fs_share_less(unsigned long long an, unsigned long long ad, unsigned long long bn, unsigned long long bd) {
  if (bd == 0) return ad != 0;
  if (ad == 0) return false;
  return (unsigned __int128)an * bd < (unsigned __int128)bn * ad;
}

// (share, rank), the owner not compared
__device__ __forceinline__ bool fs_key_less(const FsKey& a, const FsKey& b) {
  if (fs_share_less(a.num, a.den, b.num, b.den)) return true;
  if (fs_share_less(b.num, b.den, a.num, a.den)) return false;
  return a.rank < b.rank;
}

struct FsSortLess {   // (owner, share, rank)
  __device__ bool operator()(const FsKey& a, const FsKey& b) const { return a.owner != b.owner ? a.owner < b.owner : fs_key_less(a, b); }
};
struct FsMax {
  __device__ FsKey operator()(const FsKey& a, const FsKey& b) const { return fs_key_less(a, b) ? b : a; }
};
struct FsSum {
  __device__ FsUse operator()(const FsUse& a, const FsUse& b) const { return FsUse{{a.v[0] + b.v[0], a.v[1] + b.v[1], a.v[2] + b.v[2]}}; }
};

// every gang in its leaf's sequence (sorted afterwards): key (0, rank), owner = its leaf
__global__ void k_fs_init(FsTree t, uint32_t G, FsKey* keys, uint32_t* vals) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  keys[g] = FsKey{0ull, 1ull, t.leaf[g], t.rank[g]};
  vals[g] = g;
}

// the segment (owner) of each element and its gang's usage, in sequence order: the input of the segmented scan
__global__ void k_fs_gather(uint32_t G, const FsKey* __restrict__ keys, const uint32_t* __restrict__ vals, const FsUse* __restrict__ use,
                            uint32_t* owner, FsUse* use_seq) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  owner[i] = keys[i].owner;
  use_seq[i] = use[vals[i]];
}

// the elements of the depth-d sequences: key (share of their node at their turn, rank), owner = the node's parent.  Every other
// element sits in a leaf of a smaller depth, in rank order, and keeps (0, rank) and its owner.
__global__ void k_fs_key(FsTree t, uint32_t G, uint32_t d, const uint32_t* __restrict__ owner, const uint32_t* __restrict__ vals,
                         const FsUse* __restrict__ before, FsKey* keys) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  const uint32_t o = owner[i], r = t.rank[vals[i]];
  if (t.depth[o] != d) { keys[i] = FsKey{0ull, 1ull, o, r}; return; }
  unsigned long long sn = 0, sd = 1;
  for (int k = 0; k < 3; ++k) {
    const unsigned long long q = t.quota[o * 3 + k];
    if (q == GROVE_QUEUE_UNLIMITED) continue;
    const long long ls = t.load0[o * 3 + k] + before[i].v[k];
    const unsigned long long l = ls > 0 ? (unsigned long long)ls : 0ull;
    unsigned long long xn = l, xd = q;
    if (!q) { xn = l ? 1ull : 0ull; xd = l ? 0ull : 1ull; }
    if (fs_share_less(sn, sd, xn, xd)) { sn = xn; sd = xd; }
  }
  keys[i] = FsKey{sn, sd, t.parent[o], r};
}

// *first = the first position at which the new order differs from the previous one (initialised to G by the caller)
__global__ void k_fs_diff(uint32_t G, const uint32_t* __restrict__ now, const uint32_t* __restrict__ prev, uint32_t* first) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < G && now[i] != prev[i]) atomicMin(first, i);
}
