// fiesta_b200 -- topological skeleton kernels (definition: fb_skel.h, DESIGN.md §3.14).
//
// k_sk_init       : one pass over the box's records: the state byte of every voxel (X0, anchor, in X) and M := -1.
// k_sk_pass       : one thinning pass: every voxel of one subfield that the phase's rule deletes, on X as it stands (no two voxels of
//                   a subfield are 26-neighbours, so the pass reads nothing it writes).  The 26-bit neighbourhood code is built from
//                   the state bytes and tested in registers (fb_sk_simple: a bit-parallel flood fill).  Iterations are queued
//                   FB_SK_BATCH at a time, each counting its deletions into its own counter; iterations after one that deletes
//                   nothing delete nothing, so a batch may overrun the fixpoint.
// (CUB)           : ordered compaction of the thinned set -> idx (box indices in index order); k_sk_map: M[idx[j]] = j.
// The graph of the set, on the compacted voxels only (the box is not read again):
// k_sk_code       : neighbourhood code (26 bits, the centre bit clear) and class (deg != 2: vertex voxel) of every voxel.
// k_sk_union      : union-find on compact ids (fr_union, shared with the frontier clusters) between 26-neighbours of one class;
// k_sk_flatten    : parent := root, the component's smallest compact id, which is also its smallest box index.
// k_sk_attached / k_sk_promote : chain components with no vertex-voxel neighbour are pure cycles; their root becomes a vertex voxel,
//                   and the unions run again.
// (CUB) + k_sk_number : vertex roots and chain roots in index order -> vertex and edge ids.
// k_sk_members    : vertex sizes and coordinate sums, chain sizes and their two end voxels (integer atomics).
// k_sk_orient     : per edge: the attachments at both ends, the orientation, u, v, the voxel count and the vertex degrees.
// Pruning round   : k_sk_prune_edges marks the spurs of rule (a), k_sk_prune_vox every voxel a round removes; k_sk_remove takes them
//                   out of M and X, and a CUB compaction of idx by the state byte keeps the rest in order.
// Final graph     : k_sk_vertices (size, rep, centroid), a CUB scan of the voxel counts, k_sk_walk (one thread per edge walks its
//                   chain from the oriented start, writing the path, the length fold and min_dist), k_sk_labels (M := labels).
//
// Why the result does not depend on the schedule: thinning passes are order-free (above); the union-find roots are the
// components' smallest ids whatever order the unions ran in; everything else is ordered compaction, integer atomics and one
// sequential walk per edge.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include "fb_frontier.cuh"   // fr_find, fr_union
#include "fb_frontier.h"     // fb_fr_centroid
#include "fb_skel.cuh"
#include "fb_skel.h"

#define SK_ID 0x80000000u    // a root's parent word holding its vertex or edge id (compact ids are < 2^31)

__device__ __forceinline__ void sk_coords(const FbNavBox &b, long long i, int &x, int &y, int &z) {
  z = (int)(i % b.n[2]); y = (int)(i / b.n[2] % b.n[1]); x = (int)(i / ((long long)b.n[2] * b.n[1]));
}
__host__ __device__ __forceinline__ long long sk_total(const FbNavBox &b) { return (long long)b.n[0] * b.n[1] * b.n[2]; }

__device__ __forceinline__ bool sk_trav(const FbGeom &g, const uint32_t *cobs, const FbNavBox &b, int x, int y, int z, double r, bool unk) {
  const int v[3] = {b.lo[0] + x, b.lo[1] + y, b.lo[2] + z};
  double d;
  return !fb_seg_blocks(g, cobs, v, r, unk, d);
}
__device__ __forceinline__ bool sk_obst(const FbGeom &g, const uint32_t *cobs, const int *v, int *o) {
  return fb_sk_obstacle(fb_ld_record(&cobs[fb_ii(g, v[0], v[1], v[2])]), o);
}

__global__ void k_sk_init(FbGeom g, const uint32_t *__restrict__ cobs, FbNavBox b, double r, int unk, double max_cos, uint8_t *st,
                          int32_t *M, FbSkCtr *ctr) {
  const long long n = sk_total(b);
  unsigned nt = 0, na = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int x, y, z;
    sk_coords(b, i, x, y, z);
    const bool t = sk_trav(g, cobs, b, x, y, z, r, unk != 0);
    bool a = false;
    int ov[3];
    const int v[3] = {b.lo[0] + x, b.lo[1] + y, b.lo[2] + z};
    if (t && sk_obst(g, cobs, v, ov)) {
      for (int f = 0; f < 6 && !a; ++f) {                                   // the face neighbours inside the box
        int d[3] = {0, 0, 0};
        d[f % 3] = f < 3 ? -1 : 1;
        if (!fb_nav_in_box(b, x + d[0], y + d[1], z + d[2])) continue;
        if (!sk_trav(g, cobs, b, x + d[0], y + d[1], z + d[2], r, unk != 0)) continue;
        const int u[3] = {v[0] + d[0], v[1] + d[1], v[2] + d[2]};
        int ou[3];
        if (sk_obst(g, cobs, u, ou) && fb_sk_anchor_pair(v, ov, u, ou, max_cos)) a = true;
      }
    }
    st[i] = t ? (uint8_t)(FB_SK_TRAV | FB_SK_IN | (a ? FB_SK_ANCHOR : 0u)) : (uint8_t)0;
    M[i] = -1;
    nt += t; na += a;
  }
  nt = __reduce_add_sync(0xffffffffu, nt);
  na = __reduce_add_sync(0xffffffffu, na);
  if ((threadIdx.x & 31) == 0) {
    if (nt) atomicAdd(&ctr->trav, (unsigned long long)nt);
    if (na) atomicAdd(&ctr->anchors, (unsigned long long)na);
  }
}

__device__ __forceinline__ bool sk_in(const FbNavBox &b, const uint8_t *st, int x, int y, int z) {
  return fb_nav_in_box(b, x, y, z) && (st[fb_nav_idx(b, x, y, z)] & FB_SK_IN);
}

__global__ void k_sk_pass(FbNavBox b, int sx, int sy, int sz, int phase, uint8_t *st, unsigned long long *del) {
  const int hx = (b.n[0] - sx + 1) >> 1, hy = (b.n[1] - sy + 1) >> 1, hz = (b.n[2] - sz + 1) >> 1;
  const long long n = (long long)hx * hy * hz;
  unsigned cnt = 0;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int z = 2 * (int)(t % hz) + sz, y = 2 * (int)(t / hz % hy) + sy, x = 2 * (int)(t / ((long long)hz * hy)) + sx;
    const long long i = fb_nav_idx(b, x, y, z);
    const uint8_t c = st[i];
    if (!(c & FB_SK_IN)) continue;
    if (sk_in(b, st, x - 1, y, z) && sk_in(b, st, x + 1, y, z) && sk_in(b, st, x, y - 1, z) && sk_in(b, st, x, y + 1, z) &&
        sk_in(b, st, x, y, z - 1) && sk_in(b, st, x, y, z + 1)) continue;   // interior: never simple (T6 = 0)
    unsigned code = 0;
#pragma unroll
    for (int e = 0; e < 27; ++e) {
      if (e == 13) continue;
      int d[3];
      fb_nav_dir(e, d);
      if (sk_in(b, st, x + d[0], y + d[1], z + d[2])) code |= 1u << e;
    }
    if (fb_sk_deletable(code, (c & FB_SK_ANCHOR) != 0, phase)) { st[i] = (uint8_t)(c & ~FB_SK_IN); ++cnt; }
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(del, (unsigned long long)cnt);
}

struct SkIn {
  const uint8_t *st;
  __device__ bool operator()(uint32_t i) const { return (st[i] & FB_SK_IN) != 0; }
};
struct SkRoot {
  const uint32_t *par;
  const uint8_t *cls;
  uint8_t want;
  __device__ bool operator()(uint32_t j) const { return par[j] == j && cls[j] == want; }
};

__global__ void k_sk_map(const uint32_t *__restrict__ idx, unsigned n, int32_t *M) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) M[idx[j]] = (int32_t)j;
}

// Compact id of neighbour e of the skeleton voxel at box index i (bit e of its code is set, so the neighbour is in the box).
__device__ __forceinline__ unsigned sk_nb(const FbNavBox &b, const int32_t *M, uint32_t i, int e) {
  int x, y, z, d[3];
  sk_coords(b, i, x, y, z);
  fb_nav_dir(e, d);
  return (unsigned)M[fb_nav_idx(b, x + d[0], y + d[1], z + d[2])];
}
// Vertex or edge id of compact voxel j (after k_sk_number).
__device__ __forceinline__ unsigned sk_id(const uint32_t *par, unsigned j) {
  const unsigned p = par[j];
  return ((p & SK_ID) ? p : par[p]) & ~SK_ID;
}

__global__ void k_sk_code(FbNavBox b, const uint32_t *__restrict__ idx, unsigned n, const int32_t *__restrict__ M, uint32_t *code,
                          uint8_t *cls, uint32_t *par, uint8_t *flag) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  int x, y, z;
  sk_coords(b, idx[j], x, y, z);
  unsigned c = 0;
  for (int e = 0; e < 27; ++e) {
    if (e == 13) continue;
    int d[3];
    fb_nav_dir(e, d);
    if (fb_nav_in_box(b, x + d[0], y + d[1], z + d[2]) && M[fb_nav_idx(b, x + d[0], y + d[1], z + d[2])] >= 0) c |= 1u << e;
  }
  code[j] = c;
  cls[j] = __popc(c) != 2;
  par[j] = j;
  flag[j] = 0;
}

__global__ void k_sk_union(FbNavBox b, const uint32_t *__restrict__ idx, unsigned n, const int32_t *__restrict__ M,
                           const uint32_t *__restrict__ code, const uint8_t *__restrict__ cls, uint32_t *par) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  unsigned c = code[j] & ~((2u << 13) - 1);                                  // the 13 neighbours after this voxel in index order
  while (c) {
    const int e = __ffs(c) - 1;
    c &= c - 1;
    const unsigned k = sk_nb(b, M, idx[j], e);
    if (cls[k] == cls[j]) fr_union(par, j, k);
  }
}

__global__ void k_sk_flatten(unsigned n, uint32_t *par) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) par[j] = fr_find(par, j);
}

__global__ void k_sk_attached(FbNavBox b, const uint32_t *__restrict__ idx, unsigned n, const int32_t *__restrict__ M,
                              const uint32_t *__restrict__ code, const uint8_t *__restrict__ cls, const uint32_t *__restrict__ par,
                              uint8_t *flag) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || cls[j]) return;
  unsigned c = code[j];
  while (c) {
    const int e = __ffs(c) - 1;
    c &= c - 1;
    if (cls[sk_nb(b, M, idx[j], e)]) { flag[par[j]] = 1; return; }
  }
}

// A chain root whose component touches no vertex voxel heads a pure cycle: it becomes a vertex voxel.  Every parent word is reset
// for the second labelling.
__global__ void k_sk_promote(unsigned n, uint8_t *cls, uint32_t *par, const uint8_t *__restrict__ flag) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  if (!cls[j] && par[j] == j && !flag[j]) cls[j] = 1;
  par[j] = j;
}

__global__ void k_sk_number(const uint32_t *__restrict__ roots, unsigned k, uint32_t *par) {
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < k) par[roots[t]] = SK_ID | t;
}

__global__ void k_sk_members(FbNavBox b, const uint32_t *__restrict__ idx, unsigned n, const int32_t *__restrict__ M,
                             const uint32_t *__restrict__ code, const uint8_t *__restrict__ cls, const uint32_t *__restrict__ par,
                             uint32_t *vsize, unsigned long long *vsum, uint32_t *esize, uint32_t *end_lo, uint32_t *end_hi) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const unsigned id = sk_id(par, j);
  if (cls[j]) {
    int v[3];
    sk_coords(b, idx[j], v[0], v[1], v[2]);
    atomicAdd(&vsize[id], 1u);
    for (int k = 0; k < 3; ++k) atomicAdd(&vsum[3ull * id + k], (unsigned long long)(b.lo[k] + v[k]));
    return;
  }
  atomicAdd(&esize[id], 1u);
  unsigned c = code[j], chain_nb = 0;
  while (c) {
    const int e = __ffs(c) - 1;
    c &= c - 1;
    chain_nb += cls[sk_nb(b, M, idx[j], e)] == 0;
  }
  if (chain_nb <= 1) { atomicMin(&end_lo[id], j); atomicMax(&end_hi[id], j); }
}

// The vertex-voxel neighbours of chain voxel j in compact-id order (one at a chain's end, two for a 1-voxel chain).
__device__ int sk_attach(const FbNavBox &b, const uint32_t *idx, const int32_t *M, const uint32_t *code, const uint8_t *cls, unsigned j,
                         unsigned *out) {
  unsigned c = code[j];
  int k = 0;
  while (c) {
    const int e = __ffs(c) - 1;
    c &= c - 1;
    const unsigned a = sk_nb(b, M, idx[j], e);
    if (cls[a] && k < 2) out[k++] = a;
  }
  if (k == 2 && out[1] < out[0]) { const unsigned t = out[0]; out[0] = out[1]; out[1] = t; }
  return k;
}
__device__ __forceinline__ bool sk_key_less(unsigned va, uint32_t ia, uint32_t ca, unsigned vb, uint32_t ib, uint32_t cb) {
  if (va != vb) return va < vb;
  if (ia != ib) return ia < ib;
  return ca < cb;
}

__global__ void k_sk_orient(FbNavBox b, const uint32_t *__restrict__ idx, const int32_t *__restrict__ M, const uint32_t *__restrict__ code,
                            const uint8_t *__restrict__ cls, const uint32_t *__restrict__ par, unsigned E,
                            const uint32_t *__restrict__ end_lo, const uint32_t *__restrict__ end_hi, const uint32_t *__restrict__ esize,
                            uint32_t *e_att, uint32_t *e_first, int32_t *o_uv, int64_t *o_nvox, int32_t *o_vdeg, FbSkCtr *ctr) {
  const unsigned e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const unsigned c0 = end_lo[e], c1 = end_hi[e];
  unsigned p, q, a[2];
  if (c0 == c1) {
    sk_attach(b, idx, M, code, cls, c0, a);
    p = a[0]; q = a[1];
  } else {
    sk_attach(b, idx, M, code, cls, c0, a); p = a[0];
    sk_attach(b, idx, M, code, cls, c1, a); q = a[0];
  }
  const unsigned vp = sk_id(par, p), vq = sk_id(par, q);
  const bool fwd = sk_key_less(vp, idx[p], idx[c0], vq, idx[q], idx[c1]);
  e_att[e] = fwd ? p : q;
  e_first[e] = fwd ? c0 : c1;
  o_uv[2ull * e] = (int32_t)(fwd ? vp : vq);
  o_uv[2ull * e + 1] = (int32_t)(fwd ? vq : vp);
  const unsigned long long nv = (unsigned long long)esize[e] + 2;
  o_nvox[e] = (int64_t)nv;
  atomicAdd(&o_vdeg[vp], 1);
  atomicAdd(&o_vdeg[vq], 1);
  atomicAdd(&ctr->path_voxels, nv);
}

// Rule (a): an edge of fewer than min_branch voxels (the leaf counted, the other attachment not) from a leaf to a different vertex
// that is not a leaf.  A leaf is a vertex of one voxel with one neighbour.
__global__ void k_sk_prune_edges(unsigned E, const int32_t *__restrict__ o_uv, const int64_t *__restrict__ o_nvox,
                                 const uint32_t *__restrict__ vsize, const uint32_t *__restrict__ vroot, const uint32_t *__restrict__ code,
                                 long long min_branch, uint8_t *erm, uint8_t *vrm) {
  const unsigned e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const unsigned u = (unsigned)o_uv[2ull * e], v = (unsigned)o_uv[2ull * e + 1];
  if (u == v || o_nvox[e] - 1 >= min_branch) return;
  const bool lu = vsize[u] == 1 && __popc(code[vroot[u]]) == 1, lv = vsize[v] == 1 && __popc(code[vroot[v]]) == 1;
  if (lu == lv) return;
  erm[e] = 1;
  vrm[lu ? u : v] = 1;
}
// Every voxel a round removes: the chains and leaves rule (a) marked, and with min_branch >= 2 (rule (b)) every deg-1 voxel
// whose only neighbour has deg >= 3.
__global__ void k_sk_prune_vox(FbNavBox b, const uint32_t *__restrict__ idx, unsigned n, const int32_t *__restrict__ M,
                               const uint32_t *__restrict__ code, const uint8_t *__restrict__ cls, const uint32_t *__restrict__ par,
                               const uint8_t *__restrict__ erm, const uint8_t *__restrict__ vrm, uint8_t *flag, FbSkCtr *ctr) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const unsigned id = sk_id(par, j), c = code[j];
  bool rm = cls[j] ? vrm[id] != 0 : erm[id] != 0;
  if (!rm && __popc(c) == 1) rm = __popc(code[sk_nb(b, M, idx[j], __ffs(c) - 1)]) >= 3;
  flag[j] = rm;
  if (rm) atomicAdd(&ctr->removed, 1u);
}
__global__ void k_sk_remove(const uint32_t *__restrict__ idx, unsigned n, const uint8_t *__restrict__ flag, int32_t *M, uint8_t *st) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || !flag[j]) return;
  M[idx[j]] = -1;
  st[idx[j]] &= (uint8_t)~FB_SK_IN;
}

__global__ void k_sk_vertices(FbGeom g, FbNavBox b, const uint32_t *__restrict__ idx, unsigned V, const uint32_t *__restrict__ vroot,
                              const uint32_t *__restrict__ vsize, const unsigned long long *__restrict__ vsum, int64_t *o_vsize,
                              int32_t *o_rep, double *o_cen) {
  const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= V) return;
  const unsigned n = vsize[k];
  o_vsize[k] = n;
  int v[3];
  sk_coords(b, idx[vroot[k]], v[0], v[1], v[2]);
  for (int a = 0; a < 3; ++a) {
    o_rep[3ull * k + a] = b.lo[a] + v[a];
    o_cen[3ull * k + a] = fb_fr_centroid((long long)vsum[3ull * k + a], (long long)n, g.res, g.origin[a]);
  }
}

// One thread per edge: the path from the start attachment through the chain to the end attachment.  A chain voxel has exactly two
// neighbours in the set, so the next voxel is the one that is not the previous; the walk ends at the first vertex voxel.
__global__ void k_sk_walk(FbGeom g, const uint32_t *__restrict__ cobs, FbNavBox b, const uint32_t *__restrict__ idx,
                          const int32_t *__restrict__ M, const uint32_t *__restrict__ code, const uint8_t *__restrict__ cls, unsigned E,
                          const uint32_t *__restrict__ e_att, const uint32_t *__restrict__ e_first, const long long *__restrict__ off,
                          double w1, double w2, double w3, int32_t *o_vox, double *o_len, double *o_mind) {
  const unsigned e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const double w[3] = {w1, w2, w3};
  int32_t *out = o_vox + 3 * off[e];
  unsigned prev = e_att[e], cur = e_first[e];
  int pv[3];
  sk_coords(b, idx[prev], pv[0], pv[1], pv[2]);
  for (int a = 0; a < 3; ++a) { pv[a] += b.lo[a]; out[a] = pv[a]; }
  double len = 0.0, mind = fb_get_distance_vox(g, cobs, pv[0], pv[1], pv[2]);
  for (long long s = 1;; ++s) {
    int cv[3];
    sk_coords(b, idx[cur], cv[0], cv[1], cv[2]);
    for (int a = 0; a < 3; ++a) { cv[a] += b.lo[a]; out[3 * s + a] = cv[a]; }
    len = len + fb_nav_weight((cv[0] - pv[0] + 1) * 9 + (cv[1] - pv[1] + 1) * 3 + (cv[2] - pv[2] + 1), w);
    const double d = fb_get_distance_vox(g, cobs, cv[0], cv[1], cv[2]);
    if (d < mind) mind = d;
    if (cls[cur]) break;
    unsigned c = code[cur], next = prev;
    while (c) {
      const int k = __ffs(c) - 1;
      c &= c - 1;
      next = sk_nb(b, M, idx[cur], k);
      if (next != prev) break;
    }
    prev = cur; cur = next;
    for (int a = 0; a < 3; ++a) pv[a] = cv[a];
  }
  o_len[e] = len;
  o_mind[e] = mind;
}

__global__ void k_sk_labels(const uint32_t *__restrict__ idx, unsigned n, const uint8_t *__restrict__ cls, const uint32_t *__restrict__ par,
                            int32_t *M) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int32_t id = (int32_t)sk_id(par, j);
  M[idx[j]] = cls[j] ? id : -2 - id;
}

// ---------------------------------------------------------------- host side
static unsigned sk_blocks(long long n) {
  const long long want = (n + 255) / 256;
  return (unsigned)(want < FB_SMS * 16ll ? want < 1 ? 1 : want : FB_SMS * 16ll);
}
static unsigned sk_grid(unsigned long long n) { return n ? (unsigned)((n + 255) / 256) : 1u; }

#define SK_GROW(buf, n)                                                                                                  \
  do {                                                                                                                 \
    const cudaError_t e_ = (buf).grow((size_t)(n), s);                                                                 \
    if (e_ != cudaSuccess) return alloc_failed(e_, "fiesta_skeleton_compute: cannot allocate %zu elements", (size_t)(n));      \
  } while (0)

template <class Call>
static int sk_cub(FbSkBufs &B, cudaStream_t s, Call call) {
  size_t bytes = 0;
  CK(call((void *)nullptr, bytes));
  SK_GROW(B.tmp, bytes ? bytes : 16);
  bytes = B.tmp.cap;
  CK(call((void *)B.tmp.p, bytes));
  return FIESTA_OK;
}
static int sk_read_ctr(FbSkBufs &B, cudaStream_t s) {
  CK(cudaMemcpyAsync(B.h_ctr, B.ctr, sizeof(FbSkCtr), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return FIESTA_OK;
}

struct SkRun {                     // one compute: its arguments, stream and counts
  const FbGeom &g;
  const uint32_t *cobs;
  FbNavBox b;
  FbSkBufs &B;
  cudaStream_t s;
  int launches = 0;
  int cur = 0;                     // which idx buffer holds the current set
  unsigned n = 0, V = 0, E = 0;
  unsigned long long deleted = 0;  // voxels thinning deleted
};

// Thinning phase `phase`, FB_SK_BATCH iterations at a time; *iters := the iterations up to and including the first that deletes
// nothing.
static int sk_thin(SkRun &R, int phase, int64_t *iters) {
  FbSkBufs &B = R.B;
  const cudaStream_t s = R.s;
  const long long nv = sk_total(R.b);
  *iters = 0;
  for (;;) {
    CK(cudaMemsetAsync(B.ctr->del, 0, sizeof(B.ctr->del), s));
    for (int it = 0; it < FB_SK_BATCH; ++it)
      for (int p = 0; p < 8; ++p)
        k_sk_pass<<<sk_blocks((nv + 7) / 8), 256, 0, s>>>(R.b, p >> 2, (p >> 1) & 1, p & 1, phase, B.st, &B.ctr->del[it]);
    CK(cudaGetLastError());
    R.launches += 8 * FB_SK_BATCH;
    int rc;
    if ((rc = sk_read_ctr(B, s))) return rc;
    for (int it = 0; it < FB_SK_BATCH; ++it) {
      R.deleted += B.h_ctr->del[it];
      if (B.h_ctr->del[it] == 0) { *iters += it + 1; return FIESTA_OK; }
    }
    *iters += FB_SK_BATCH;
  }
}

// The graph of the current set (R.n voxels in B.idx[R.cur], mapped by M): classes, vertex and edge ids, sizes, orientation.
static int sk_graph(SkRun &R) {
  FbSkBufs &B = R.B;
  const cudaStream_t s = R.s;
  const unsigned n = R.n;
  const uint32_t *idx = B.idx[R.cur];
  const thrust::counting_iterator<uint32_t> it(0);
  int rc;
  k_sk_code<<<sk_grid(n), 256, 0, s>>>(R.b, idx, n, B.M, B.code, B.cls, B.par, B.flag);
  k_sk_union<<<sk_grid(n), 256, 0, s>>>(R.b, idx, n, B.M, B.code, B.cls, B.par);
  k_sk_flatten<<<sk_grid(n), 256, 0, s>>>(n, B.par);
  k_sk_attached<<<sk_grid(n), 256, 0, s>>>(R.b, idx, n, B.M, B.code, B.cls, B.par, B.flag);
  k_sk_promote<<<sk_grid(n), 256, 0, s>>>(n, B.cls, B.par, B.flag);
  k_sk_union<<<sk_grid(n), 256, 0, s>>>(R.b, idx, n, B.M, B.code, B.cls, B.par);
  k_sk_flatten<<<sk_grid(n), 256, 0, s>>>(n, B.par);
  CK(cudaGetLastError());
  for (int c = 0; c < 2; ++c) {
    uint32_t *out = c ? B.eroot.p : B.vroot.p;
    if ((rc = sk_cub(B, s, [&](void *t, size_t &nb) {
           return cub::DeviceSelect::If(t, nb, it, out, &B.ctr->sel[c], (int)n, SkRoot{B.par, B.cls, (uint8_t)(1 - c)}, s);
         }))) return rc;
  }
  R.launches += 9;
  if ((rc = sk_read_ctr(B, s))) return rc;
  R.V = B.h_ctr->sel[0];
  R.E = B.h_ctr->sel[1];
  const unsigned V = R.V, E = R.E;
  k_sk_number<<<sk_grid(V), 256, 0, s>>>(B.vroot, V, B.par);
  k_sk_number<<<sk_grid(E), 256, 0, s>>>(B.eroot, E, B.par);
  CK(cudaMemsetAsync(B.vsize, 0, (size_t)V * 4, s));
  CK(cudaMemsetAsync(B.vsum, 0, (size_t)V * 24, s));
  CK(cudaMemsetAsync(B.o_vdeg, 0, (size_t)V * 4, s));
  CK(cudaMemsetAsync(B.esize, 0, (size_t)E * 4, s));
  CK(cudaMemsetAsync(B.end_lo, 0xff, (size_t)E * 4, s));
  CK(cudaMemsetAsync(B.end_hi, 0, (size_t)E * 4, s));
  CK(cudaMemsetAsync(&B.ctr->path_voxels, 0, sizeof(unsigned long long), s));
  k_sk_members<<<sk_grid(n), 256, 0, s>>>(R.b, idx, n, B.M, B.code, B.cls, B.par, B.vsize, B.vsum, B.esize, B.end_lo, B.end_hi);
  k_sk_orient<<<sk_grid(E), 256, 0, s>>>(R.b, idx, B.M, B.code, B.cls, B.par, E, B.end_lo, B.end_hi, B.esize, B.e_att, B.e_first, B.o_uv,
                                         B.o_nvox, B.o_vdeg, B.ctr);
  CK(cudaGetLastError());
  R.launches += 4;
  return FIESTA_OK;
}

// One pruning round on the graph sk_graph left: removes what the round removes; *removed := how many.
static int sk_prune(SkRun &R, long long min_branch, unsigned *removed) {
  FbSkBufs &B = R.B;
  const cudaStream_t s = R.s;
  const unsigned n = R.n;
  int rc;
  CK(cudaMemsetAsync(B.erm, 0, R.E ? R.E : 1, s));
  CK(cudaMemsetAsync(B.vrm, 0, R.V ? R.V : 1, s));
  CK(cudaMemsetAsync(&B.ctr->removed, 0, sizeof(unsigned), s));
  k_sk_prune_edges<<<sk_grid(R.E), 256, 0, s>>>(R.E, B.o_uv, B.o_nvox, B.vsize, B.vroot, B.code, min_branch, B.erm, B.vrm);
  k_sk_prune_vox<<<sk_grid(n), 256, 0, s>>>(R.b, B.idx[R.cur], n, B.M, B.code, B.cls, B.par, B.erm, B.vrm, B.flag, B.ctr);
  k_sk_remove<<<sk_grid(n), 256, 0, s>>>(B.idx[R.cur], n, B.flag, B.M, B.st);
  CK(cudaGetLastError());
  R.launches += 3;
  if ((rc = sk_read_ctr(B, s))) return rc;
  *removed = B.h_ctr->removed;
  if (*removed == 0) return FIESTA_OK;
  if ((rc = sk_cub(B, s, [&](void *t, size_t &nb) {
         return cub::DeviceSelect::If(t, nb, B.idx[R.cur].p, B.idx[1 - R.cur].p, &B.ctr->sel[2], (int)n, SkIn{B.st}, s);
       }))) return rc;
  R.cur = 1 - R.cur;
  R.n = n - *removed;
  k_sk_map<<<sk_grid(R.n), 256, 0, s>>>(B.idx[R.cur], R.n, B.M);
  CK(cudaGetLastError());
  R.launches += 2;
  return FIESTA_OK;
}

// The outputs of the final graph: vertex arrays, edge paths, labels.
static int sk_outputs(SkRun &R, unsigned long long path_voxels) {
  FbSkBufs &B = R.B;
  const cudaStream_t s = R.s;
  int rc;
  SK_GROW(B.o_vox, 3 * (path_voxels ? path_voxels : 1));
  k_sk_vertices<<<sk_grid(R.V), 256, 0, s>>>(R.g, R.b, B.idx[R.cur], R.V, B.vroot, B.vsize, B.vsum, B.o_vsize, B.o_rep, B.o_cen);
  CK(cudaGetLastError());
  R.launches += 1;
  if (R.E) {
    const int64_t *nv = B.o_nvox.p;
    long long *off = B.off.p;
    const unsigned E = R.E;
    if ((rc = sk_cub(B, s, [&](void *t, size_t &nb) { return cub::DeviceScan::ExclusiveSum(t, nb, nv, off, (int)E, s); }))) return rc;
    const double res = R.g.res;
    k_sk_walk<<<sk_grid(E), 256, 0, s>>>(R.g, R.cobs, R.b, B.idx[R.cur], B.M, B.code, B.cls, E, B.e_att, B.e_first, B.off,
                                         res * sqrt(1.0), res * sqrt(2.0), res * sqrt(3.0), B.o_vox, B.o_len, B.o_mind);
    CK(cudaGetLastError());
    R.launches += 2;
  }
  k_sk_labels<<<sk_grid(R.n), 256, 0, s>>>(B.idx[R.cur], R.n, B.cls, B.par, B.M);
  CK(cudaGetLastError());
  R.launches += 1;
  return FIESTA_OK;
}

static int skeleton_compute(SkRun &R, fiesta_skeleton *f, double r, int flags, double max_cos, long long min_branch,
                            fiesta_skeleton_stats &st) {
  FbSkBufs &B = R.B;
  const cudaStream_t s = R.s;
  const long long nv = sk_total(R.b);
  const thrust::counting_iterator<uint32_t> it(0);
  int rc;
  SK_GROW(B.st, nv);
  SK_GROW(B.M, nv);
  CK(cudaMemsetAsync(B.ctr, 0, sizeof(FbSkCtr), s));
  k_sk_init<<<sk_blocks(nv), 256, 0, s>>>(R.g, R.cobs, R.b, r, flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS, max_cos, B.st, B.M, B.ctr);
  CK(cudaGetLastError());
  R.launches += 1;
  CK(cudaEventRecord(f->ev[1], s));
  for (int phase = 1; phase <= 2; ++phase)
    if ((rc = sk_thin(R, phase, &st.iterations[phase - 1]))) return rc;
  CK(cudaEventRecord(f->ev[2], s));
  st.traversable = (int64_t)B.h_ctr->trav;
  st.anchors = (int64_t)B.h_ctr->anchors;
  R.n = (unsigned)(B.h_ctr->trav - R.deleted);
  if (R.n == 0) {                                                           // no skeleton: every label is -1 already
    st.prune_rounds = min_branch > 1;                                       // one round, on the empty set, removes nothing
    return FIESTA_OK;
  }
  // the thinned set, compacted in index order
  SK_GROW(B.idx[0], R.n);
  if ((rc = sk_cub(B, s, [&](void *t, size_t &nb) {
         return cub::DeviceSelect::If(t, nb, it, B.idx[0].p, &B.ctr->n, (int)nv, SkIn{B.st}, s);
       }))) return rc;
  R.launches += 1;
  const size_t n = R.n;
  SK_GROW(B.idx[1], n); SK_GROW(B.code, n); SK_GROW(B.par, n); SK_GROW(B.cls, n); SK_GROW(B.flag, n);
  SK_GROW(B.vroot, n); SK_GROW(B.eroot, n); SK_GROW(B.vsize, n); SK_GROW(B.esize, n); SK_GROW(B.end_lo, n); SK_GROW(B.end_hi, n);
  SK_GROW(B.e_att, n); SK_GROW(B.e_first, n); SK_GROW(B.vsum, 3 * n); SK_GROW(B.vrm, n); SK_GROW(B.erm, n); SK_GROW(B.off, n);
  SK_GROW(B.o_vsize, n); SK_GROW(B.o_nvox, n); SK_GROW(B.o_rep, 3 * n); SK_GROW(B.o_vdeg, n); SK_GROW(B.o_uv, 2 * n);
  SK_GROW(B.o_cen, 3 * n); SK_GROW(B.o_len, n); SK_GROW(B.o_mind, n);
  R.cur = 0;
  k_sk_map<<<sk_grid(n), 256, 0, s>>>(B.idx[0], R.n, B.M);
  CK(cudaGetLastError());
  R.launches += 1;
  const unsigned n0 = R.n;
  for (;;) {
    if ((rc = sk_graph(R))) return rc;
    if (min_branch <= 1) break;
    unsigned removed = 0;
    ++st.prune_rounds;
    if ((rc = sk_prune(R, min_branch, &removed))) return rc;
    if (removed == 0) break;
  }
  st.pruned_voxels = (int64_t)(n0 - R.n);
  if ((rc = sk_read_ctr(B, s))) return rc;
  const unsigned long long pv = B.h_ctr->path_voxels;
  if ((rc = sk_outputs(R, pv))) return rc;
  st.skeleton_voxels = R.n;
  st.vertices = R.V;
  st.edges = R.E;
  st.edge_voxels = (int64_t)pv;
  return FIESTA_OK;
}

// ---------------------------------------------------------------- entry points (include/fiesta_b200.h)
void fiesta_skeleton_destroy(fiesta_skeleton *f) { handle_destroy(f); }
int fiesta_skeleton_create(fiesta_map *m, fiesta_skeleton **out) {
  if (!m || !out) { fb_set_error("fiesta_skeleton_create: null argument"); return FIESTA_ERR_INVALID; }
  *out = nullptr;
  FbHandle<fiesta_skeleton> f;
  int r;
  if ((r = handle_new(m, f))) return r;
  if (!f) { fb_set_error("out of host memory"); return FIESTA_ERR_INVALID; }
  for (cudaEvent_t &e : f->ev) CK(cudaEventCreate(&e));
  CK(f->B.ctr.alloc(1));
  CK(f->B.h_ctr.alloc(1));
  *out = f.release();
  return FIESTA_OK;
}
int fiesta_skeleton_compute(fiesta_skeleton *f, const int box_lo[3], const int box_hi[3], double clearance, int flags, double max_cos,
                            int64_t min_branch, fiesta_skeleton_stats *stats) {
  const char *fn = "fiesta_skeleton_compute";
  if (!f || !box_lo || !box_hi) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  if (!clearance_flags_ok(fn, clearance, flags)) return FIESTA_ERR_INVALID;
  if (!(max_cos >= -1.0 && max_cos < 1.0)) { fb_set_error("%s: max_cos must be finite and in [-1, 1)", fn); return FIESTA_ERR_INVALID; }
  if (min_branch < 0) { fb_set_error("%s: min_branch must be >= 0", fn); return FIESTA_ERR_INVALID; }
  fiesta_map *m = f->m;
  FbNavBox b{};
  if (!box_arg(fn, m->g, box_lo, box_hi, &b)) return FIESTA_ERR_INVALID;
  CK(cudaSetDevice(m->device));
  f->valid = false;
  CK(cudaEventRecord(f->ev[0], m->stream));
  fiesta_skeleton_stats st{};
  st.box_voxels = sk_total(b);
  SkRun R{m->g, m->cobs, b, f->B, m->stream};
  const int r = skeleton_compute(R, f, clearance, flags, max_cos, (long long)min_branch, st);
  m->st.kernel_launches += R.launches;
  if (r != FIESTA_OK) return r;
  CK(cudaEventRecord(f->ev[3], m->stream));
  CK(cudaStreamSynchronize(m->stream));
  CK(cudaEventElapsedTime(&st.ms_compute, f->ev[0], f->ev[3]));
  CK(cudaEventElapsedTime(&st.ms_init, f->ev[0], f->ev[1]));
  CK(cudaEventElapsedTime(&st.ms_thin, f->ev[1], f->ev[2]));
  CK(cudaEventElapsedTime(&st.ms_graph, f->ev[2], f->ev[3]));
  f->st = st;
  f->box = b;
  f->valid = true;
  if (stats) *stats = f->st;
  return FIESTA_OK;
}
static bool sk_read_ok(const fiesta_skeleton *f, const char *fn, int64_t cap, bool buffers) {
  if (!f || cap < 0 || (cap > 0 && !buffers)) { fb_set_error("%s: null buffer or negative capacity", fn); return false; }
  if (!f->valid) { fb_set_error("%s: no skeleton has been computed", fn); return false; }
  return true;
}
int fiesta_skeleton_vertices(const fiesta_skeleton *f, int64_t cap, int64_t *size, int32_t *rep_xyz, double *centroid_xyz, int32_t *degree) {
  if (!sk_read_ok(f, "fiesta_skeleton_vertices", cap, size && rep_xyz && centroid_xyz && degree)) return FIESTA_ERR_INVALID;
  const size_t n = (size_t)(cap < f->st.vertices ? cap : f->st.vertices);
  if (n == 0) return FIESTA_OK;
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  CK(cudaMemcpyAsync(size, f->B.o_vsize, n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(rep_xyz, f->B.o_rep, n * 12, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(centroid_xyz, f->B.o_cen, n * 24, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(degree, f->B.o_vdeg, n * 4, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
int fiesta_skeleton_edges(const fiesta_skeleton *f, int64_t cap, int32_t *uv, int64_t *n_vox, double *length, double *min_dist) {
  if (!sk_read_ok(f, "fiesta_skeleton_edges", cap, uv && n_vox && length && min_dist)) return FIESTA_ERR_INVALID;
  const size_t n = (size_t)(cap < f->st.edges ? cap : f->st.edges);
  if (n == 0) return FIESTA_OK;
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  CK(cudaMemcpyAsync(uv, f->B.o_uv, n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(n_vox, f->B.o_nvox, n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(length, f->B.o_len, n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(min_dist, f->B.o_mind, n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
int fiesta_skeleton_edge_voxels(const fiesta_skeleton *f, int64_t cap, int32_t *vox_xyz) {
  if (!sk_read_ok(f, "fiesta_skeleton_edge_voxels", cap, vox_xyz != nullptr)) return FIESTA_ERR_INVALID;
  const size_t n = (size_t)(cap < f->st.edge_voxels ? cap : f->st.edge_voxels);
  if (n == 0) return FIESTA_OK;
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  CK(cudaMemcpyAsync(vox_xyz, f->B.o_vox, n * 12, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
int fiesta_skeleton_export(const fiesta_skeleton *f, uint8_t *mask, int32_t *label) {
  if (!f) { fb_set_error("fiesta_skeleton_export: null argument"); return FIESTA_ERR_INVALID; }
  if (!f->valid) { fb_set_error("fiesta_skeleton_export: no skeleton has been computed"); return FIESTA_ERR_INVALID; }
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  if (mask) CK(cudaMemcpyAsync(mask, f->B.st, (size_t)f->st.box_voxels, cudaMemcpyDeviceToHost, m->stream));
  if (label) CK(cudaMemcpyAsync(label, f->B.M, (size_t)f->st.box_voxels * 4, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
