// fiesta_b200 -- frontier extraction kernels (definition: fb_frontier.h, DESIGN.md §3.6).
//
// k_fr_tile     : one CTA per 8^3 box tile.  Evaluates fb_fr_is_frontier for its voxels, joins the tile's frontier voxels into
//                 26-connected components with union-find in shared memory, and writes each voxel's parent word P: the box
//                 index of its tile component's smallest voxel, FR_NONE for voxels that are not frontier voxels.
// k_fr_merge    : every frontier voxel near a tile boundary unions with its frontier neighbours in other tiles (lock-free union
//                 by index on P: the larger root is hooked under the smaller with atomicMin; retried on contention).
// k_fr_flatten  : P := root; counts the roots (the clusters before the size filter).
// (CUB)         : ordered compaction of the roots -> pre-filter cluster ids in index order.
// k_fr_number   : each root's slot of P takes FR_ID | its id, so any member finds its id in two loads.
// k_fr_stats    : sizes, coordinate sums and bounding boxes by id, with warp-aggregated integer atomics (no fp atomics).
// (CUB)         : ordered compaction of the clusters of at least min_size voxels -> kept ids.
// k_fr_clusters : per kept cluster: the id map and the outputs (size, rep, bbox, centroid).
// k_fr_label    : the box-shaped label array.
// (CUB)         : the kept members in index order, then a stable radix sort by label; k_fr_members writes their xyz.
//
// Why the result does not depend on the schedule: parent words only ever decrease and always point at a smaller index of the
// same component, so after the merge each component is one tree whose root is its smallest index, whatever order the unions ran
// in.  Everything after that is ordered compaction, integer atomics and a stable sort, and the centroid is one fp64 expression.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include "fb_frontier.cuh"
#include "fb_frontier.h"

#define FR_THREADS 512          // one thread per voxel of an 8^3 tile
#define FR_NONE 0xffffffffu     // not a frontier voxel
#define FR_ID 0x80000000u       // a root's slot of P holding its cluster id (box indices are < 2^31)

__device__ __forceinline__ void fr_coords(const FbNavBox &b, long long i, int &x, int &y, int &z) {
  z = (int)(i % b.n[2]); y = (int)(i / b.n[2] % b.n[1]); x = (int)(i / ((long long)b.n[2] * b.n[1]));
}
__host__ __device__ __forceinline__ long long fr_total(const FbNavBox &b) { return (long long)b.n[0] * b.n[1] * b.n[2]; }

// ---- union-find by index in shared memory (one tile, local indices); the global-memory form is fr_find / fr_union (fb_frontier.cuh)
__device__ __forceinline__ unsigned fr_find_s(volatile unsigned *s, unsigned x) {
  unsigned p;
  while ((p = s[x]) != x) x = p;
  return x;
}
__device__ void fr_union_s(unsigned *s, unsigned a, unsigned b) {
  for (;;) {
    a = fr_find_s(s, a); b = fr_find_s(s, b);
    if (a == b) return;
    if (a > b) { const unsigned t = a; a = b; b = t; }
    const unsigned old = atomicMin(&s[b], a);   // hook the larger root under the smaller
    if (old == b) return;
    b = old;                                      // b was hooked meanwhile: join a with what it was hooked to
  }
}
__global__ void __launch_bounds__(FR_THREADS) k_fr_tile(FbGeom g, const uint32_t *__restrict__ cobs, const double *__restrict__ occ,
                                                        double l_occ, double r, FbNavBox b, int tn1, int tn2, uint32_t *P, FbFrCtr *ctr) {
  __shared__ unsigned s[FR_THREADS];
  const int tid = threadIdx.x, lx = tid >> 6, ly = (tid >> 3) & 7, lz = tid & 7;
  const unsigned tile = blockIdx.x;
  const int tz = (int)(tile % (unsigned)tn2), ty = (int)(tile / (unsigned)tn2 % (unsigned)tn1), tx = (int)(tile / (unsigned)(tn2 * tn1));
  const int x = tx * FB_TILE + lx, y = ty * FB_TILE + ly, z = tz * FB_TILE + lz;
  const bool in = fb_nav_in_box(b, x, y, z);
  bool f = false;
  if (in) {
    const int v[3] = {b.lo[0] + x, b.lo[1] + y, b.lo[2] + z};
    f = fb_fr_is_frontier(g, cobs, occ, l_occ, v, r);
  }
  s[tid] = f ? (unsigned)tid : FR_NONE;
  const unsigned cnt = __reduce_add_sync(0xffffffffu, f ? 1u : 0u);
  if ((tid & 31) == 0 && cnt) atomicAdd(&ctr->frontier, (unsigned long long)cnt);
  __syncthreads();
  if (f) {
    // the 13 neighbours after this voxel in index order ((dx, dy, dz) > 0 lexicographically): each pair is joined once
    for (int k = 14; k < 27; ++k) {
      int d[3];
      fb_nav_dir(k, d);
      const int nx = lx + d[0], ny = ly + d[1], nz = lz + d[2];
      if (nx < 0 || nx >= FB_TILE || ny < 0 || ny >= FB_TILE || nz < 0 || nz >= FB_TILE) continue;
      const unsigned j = (unsigned)((nx * FB_TILE + ny) * FB_TILE + nz);
      if (((volatile unsigned *)s)[j] != FR_NONE) fr_union_s(s, (unsigned)tid, j);   // FR_NONE entries never change
    }
  }
  __syncthreads();
  if (!in) return;
  unsigned p = FR_NONE;
  if (f) {
    const unsigned root = fr_find_s(s, (unsigned)tid);   // local index order is box index order inside a tile
    p = (unsigned)fb_nav_idx(b, tx * FB_TILE + (int)(root >> 6), ty * FB_TILE + (int)((root >> 3) & 7), tz * FB_TILE + (int)(root & 7));
  }
  P[fb_nav_idx(b, x, y, z)] = p;
}

__global__ void k_fr_merge(FbNavBox b, uint32_t *P) {
  const long long n = fr_total(b);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (__ldcg(&P[i]) == FR_NONE) continue;                                // stays so: only frontier voxels' words change
    int x, y, z;
    fr_coords(b, i, x, y, z);
    const int lx = x & 7, ly = y & 7, lz = z & 7;
    if (lx > 0 && lx < 7 && ly > 0 && ly < 7 && lz > 0 && lz < 7) continue;   // every neighbour is in the same tile
    for (int k = 14; k < 27; ++k) {                                       // faces, edges and corners of the tile alike
      int d[3];
      fb_nav_dir(k, d);
      const int nx = x + d[0], ny = y + d[1], nz = z + d[2];
      if (!fb_nav_in_box(b, nx, ny, nz)) continue;
      if ((nx >> 3) == (x >> 3) && (ny >> 3) == (y >> 3) && (nz >> 3) == (z >> 3)) continue;   // joined by k_fr_tile
      const long long j = fb_nav_idx(b, nx, ny, nz);
      if (__ldcg(&P[j]) != FR_NONE) fr_union(P, (unsigned)i, (unsigned)j);
    }
  }
}

__global__ void k_fr_flatten(FbNavBox b, uint32_t *P, FbFrCtr *ctr) {
  const long long n = fr_total(b);
  unsigned roots = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (__ldcg(&P[i]) == FR_NONE) continue;
    const unsigned root = fr_find(P, (unsigned)i);
    P[i] = root;
    roots += root == (unsigned)i;
  }
  roots = __reduce_add_sync(0xffffffffu, roots);
  if ((threadIdx.x & 31) == 0 && roots) atomicAdd(&ctr->roots, (unsigned long long)roots);
}

struct FrIsRoot {
  const uint32_t *P;
  __device__ bool operator()(uint32_t i) const { return P[i] == i; }
};
struct FrKeep {
  const uint32_t *size;
  unsigned min_size;
  __device__ bool operator()(uint32_t k) const { return size[k] >= min_size; }
};
struct FrKept {
  const int32_t *L;
  __device__ bool operator()(uint32_t i) const { return L[i] >= 0; }
};

__global__ void k_fr_number(const uint32_t *__restrict__ roots, unsigned n, uint32_t *P) {
  const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) P[roots[k]] = FR_ID | k;
}
// Pre-filter cluster id of a frontier voxel whose parent word is p (after k_fr_number).
__device__ __forceinline__ unsigned fr_cluster(const uint32_t *P, unsigned p) { return ((p & FR_ID) ? p : P[p]) & ~FR_ID; }

// Sizes, grid-coordinate sums and bounding boxes by pre-filter id.  The loop runs whole warps together so that lanes of one
// cluster combine their values (__match_any_sync, then one atomic per cluster and warp).  A warp holds at most 32 voxels of
// coordinate <= 2046, so the per-warp sums fit 32 bits.
__global__ void k_fr_stats(FbNavBox b, const uint32_t *__restrict__ P, uint32_t *size, unsigned long long *sum, int32_t *box, unsigned C) {
  const long long n = fr_total(b);
  const int lane = threadIdx.x & 31;
  for (long long base = (long long)blockIdx.x * blockDim.x + threadIdx.x - lane; base < n; base += (long long)gridDim.x * blockDim.x) {
    const long long i = base + lane;
    unsigned id = FR_NONE;
    int v[3] = {0, 0, 0};
    if (i < n) {
      const unsigned p = P[i];
      if (p != FR_NONE) {
        id = fr_cluster(P, p);
        fr_coords(b, i, v[0], v[1], v[2]);
        for (int k = 0; k < 3; ++k) v[k] += b.lo[k];
      }
    }
    const unsigned grp = __match_any_sync(0xffffffffu, id);
    if (id == FR_NONE) continue;
    const bool leader = lane == __ffs(grp) - 1;
    if (leader) atomicAdd(&size[id], (unsigned)__popc(grp));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const unsigned s = __reduce_add_sync(grp, (unsigned)v[k]);
      const int lo = __reduce_min_sync(grp, v[k]), hi = __reduce_max_sync(grp, v[k]);
      if (leader) {
        atomicAdd(&sum[3ull * id + k], (unsigned long long)s);
        atomicMin(&box[3ull * id + k], lo);
        atomicMax(&box[3ull * (C + id) + k], hi);
      }
    }
  }
}

__global__ void k_fr_clusters(FbGeom g, FbNavBox b, const uint32_t *__restrict__ kept,
                              const uint32_t *__restrict__ roots, const uint32_t *__restrict__ size, const unsigned long long *__restrict__ sum,
                              const int32_t *__restrict__ box, unsigned C, int32_t *newid, int64_t *o_size, int32_t *o_i32, double *o_cen,
                              FbFrCtr *ctr) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= __ldcg(&ctr->sel[1])) return;                                 // the number of kept clusters
  const unsigned k = kept[j];
  newid[k] = (int32_t)j;
  const unsigned n = size[k];
  o_size[j] = n;
  int rv[3];
  fr_coords(b, roots[k], rv[0], rv[1], rv[2]);
  for (int a = 0; a < 3; ++a) {
    o_i32[3ull * j + a] = b.lo[a] + rv[a];                               // rep
    o_i32[3ull * (C + j) + a] = box[3ull * k + a];                       // bbox lo
    o_i32[3ull * (2 * C + j) + a] = box[3ull * (C + k) + a];             // bbox hi
    o_cen[3ull * j + a] = fb_fr_centroid((long long)sum[3ull * k + a], (long long)n, g.res, g.origin[a]);
  }
  atomicAdd(&ctr->kept_voxels, (unsigned long long)n);
}

__global__ void k_fr_label(FbNavBox b, const uint32_t *__restrict__ P, const int32_t *__restrict__ newid, int32_t *L) {
  const long long n = fr_total(b);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned p = P[i];
    L[i] = p == FR_NONE ? -1 : newid[fr_cluster(P, p)];
  }
}

__global__ void k_fr_keys(const uint32_t *__restrict__ idx, const int32_t *__restrict__ L, unsigned n, uint32_t *key) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) key[j] = (uint32_t)L[idx[j]];
}

__global__ void k_fr_members(FbNavBox b, const uint32_t *__restrict__ idx, unsigned n, int32_t *xyz) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  int v[3];
  fr_coords(b, idx[j], v[0], v[1], v[2]);
  for (int a = 0; a < 3; ++a) xyz[3ull * j + a] = b.lo[a] + v[a];
}

// ---------------------------------------------------------------- host side
static unsigned fr_blocks(long long n) {
  const long long want = (n + 255) / 256;
  return (unsigned)(want < FB_SMS * 16ll ? want < 1 ? 1 : want : FB_SMS * 16ll);
}
static unsigned fr_grid(unsigned long long n) { return (unsigned)((n + 255) / 256); }

#define FR_GROW(buf, n)                                                                                                  \
  do {                                                                                                                 \
    const cudaError_t e_ = (buf).grow((size_t)(n), s);                                                                 \
    if (e_ != cudaSuccess) return alloc_failed(e_, "fiesta_frontiers_compute: cannot allocate %zu elements", (size_t)(n));     \
  } while (0)

// One CUB call with temporary storage from B.tmp (grown as needed).
template <class Call>
static int fr_cub(FbFrBufs &B, cudaStream_t s, Call call) {
  size_t bytes = 0;
  CK(call((void *)nullptr, bytes));
  FR_GROW(B.tmp, bytes ? bytes : 16);
  bytes = B.tmp.cap;
  CK(call((void *)B.tmp.p, bytes));
  return FIESTA_OK;
}

static int fr_read_ctr(FbFrBufs &B, cudaStream_t s) {
  CK(cudaMemcpyAsync(B.h_ctr, B.ctr, sizeof(FbFrCtr), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return FIESTA_OK;
}

static int frontier_compute(const FbGeom &g, const uint32_t *cobs, const double *occ, double l_occ, const FbNavBox &b, double r,
                            long long min_size, FbFrBufs &B, cudaStream_t s, int *launches) {
  const long long nv = fr_total(b);
  const int tn[3] = {(b.n[0] + FB_TILE - 1) / FB_TILE, (b.n[1] + FB_TILE - 1) / FB_TILE, (b.n[2] + FB_TILE - 1) / FB_TILE};
  const unsigned nt = (unsigned)(tn[0] * tn[1] * tn[2]);
  const thrust::counting_iterator<uint32_t> it(0);
  int rc;
  FR_GROW(B.P, nv);
  FR_GROW(B.L, nv);
  uint32_t *P = B.P;
  CK(cudaMemsetAsync(B.ctr, 0, sizeof(FbFrCtr), s));
  k_fr_tile<<<nt, FR_THREADS, 0, s>>>(g, cobs, occ, l_occ, r, b, tn[1], tn[2], P, B.ctr);
  k_fr_merge<<<fr_blocks(nv), 256, 0, s>>>(b, P);
  k_fr_flatten<<<fr_blocks(nv), 256, 0, s>>>(b, P, B.ctr);
  CK(cudaGetLastError());
  *launches += 3;
  if ((rc = fr_read_ctr(B, s))) return rc;
  const unsigned C = (unsigned)B.h_ctr->roots;
  if (C == 0) {                                                           // no frontier voxel: every label is -1
    CK(cudaMemsetAsync(B.L, 0xff, (size_t)nv * 4, s));
    return FIESTA_OK;
  }
  FR_GROW(B.roots, C); FR_GROW(B.size, C); FR_GROW(B.kept, C); FR_GROW(B.newid, C);
  FR_GROW(B.sum, 3ull * C); FR_GROW(B.box, 6ull * C);
  FR_GROW(B.o_size, C); FR_GROW(B.o_i32, 9ull * C); FR_GROW(B.o_cen, 3ull * C);
  B.C = C;
  // clusters in index order of their roots
  if ((rc = fr_cub(B, s, [&](void *t, size_t &n) {
         return cub::DeviceSelect::If(t, n, it, B.roots.p, &B.ctr->sel[0], (int)nv, FrIsRoot{P}, s);
       }))) return rc;
  k_fr_number<<<fr_grid(C), 256, 0, s>>>(B.roots, C, P);
  CK(cudaMemsetAsync(B.size, 0, (size_t)C * 4, s));
  CK(cudaMemsetAsync(B.sum, 0, (size_t)C * 24, s));
  CK(cudaMemsetAsync(B.box, 0x7f, (size_t)C * 12, s));                 // lo: 0x7f7f7f7f, above every coordinate
  CK(cudaMemsetAsync(B.box + 3ull * C, 0x80, (size_t)C * 12, s));      // hi: 0x80808080, below every coordinate
  CK(cudaMemsetAsync(B.newid, 0xff, (size_t)C * 4, s));                // dropped clusters: -1
  k_fr_stats<<<fr_blocks(nv), 256, 0, s>>>(b, P, B.size, B.sum, B.box, C);
  CK(cudaGetLastError());
  // the size filter, keeping index order
  const unsigned ms = min_size > 0xffffffffll ? 0xffffffffu : (unsigned)min_size;
  if ((rc = fr_cub(B, s, [&](void *t, size_t &n) {
         return cub::DeviceSelect::If(t, n, it, B.kept.p, &B.ctr->sel[1], (int)C, FrKeep{B.size, ms}, s);
       }))) return rc;
  k_fr_clusters<<<fr_grid(C), 256, 0, s>>>(g, b, B.kept, B.roots, B.size, B.sum, B.box, C, B.newid, B.o_size, B.o_i32, B.o_cen, B.ctr);
  k_fr_label<<<fr_blocks(nv), 256, 0, s>>>(b, P, B.newid, B.L);
  CK(cudaGetLastError());
  *launches += 6;
  if ((rc = fr_read_ctr(B, s))) return rc;
  const unsigned K = B.h_ctr->sel[1];
  const unsigned long long M = B.h_ctr->kept_voxels;
  if (M == 0) return FIESTA_OK;
  // the member list: kept frontier voxels in index order, stably sorted by label
  for (int k = 0; k < 2; ++k) { FR_GROW(B.mkey[k], M); FR_GROW(B.mval[k], M); }
  FR_GROW(B.m_xyz, 3 * M);
  if ((rc = fr_cub(B, s, [&](void *t, size_t &n) {
         return cub::DeviceSelect::If(t, n, it, B.mval[0].p, &B.ctr->sel[2], (int)nv, FrKept{B.L}, s);
       }))) return rc;
  k_fr_keys<<<fr_grid(M), 256, 0, s>>>(B.mval[0], B.L, (unsigned)M, B.mkey[0]);
  int bits = 1;
  while (bits < 32 && (1ull << bits) < K) ++bits;
  if ((rc = fr_cub(B, s, [&](void *t, size_t &n) {
         return cub::DeviceRadixSort::SortPairs(t, n, B.mkey[0].p, B.mkey[1].p, B.mval[0].p, B.mval[1].p, (int)M, 0, bits, s);
       }))) return rc;
  k_fr_members<<<fr_grid(M), 256, 0, s>>>(b, B.mval[1], (unsigned)M, B.m_xyz);
  CK(cudaGetLastError());
  *launches += 5;
  return FIESTA_OK;
}

// ---------------------------------------------------------------- entry points (include/fiesta_b200.h)
void fiesta_frontiers_destroy(fiesta_frontiers *f) { handle_destroy(f); }
int fiesta_frontiers_create(fiesta_map *m, fiesta_frontiers **out) {
  if (!m || !out) { fb_set_error("fiesta_frontiers_create: null argument"); return FIESTA_ERR_INVALID; }
  *out = nullptr;
  FbHandle<fiesta_frontiers> f;
  int r;
  if ((r = handle_new(m, f))) return r;
  if (!f) { fb_set_error("out of host memory"); return FIESTA_ERR_INVALID; }
  for (cudaEvent_t &e : f->ev) CK(cudaEventCreate(&e));
  CK(f->B.ctr.alloc(1));
  CK(f->B.h_ctr.alloc(1));
  *out = f.release();
  return FIESTA_OK;
}
int fiesta_frontiers_compute(fiesta_frontiers *f, const int box_lo[3], const int box_hi[3], double clearance, int64_t min_cluster_size,
                             fiesta_frontier_stats *stats) {
  const char *fn = "fiesta_frontiers_compute";
  if (!f || !box_lo || !box_hi) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  if (!clearance_flags_ok(fn, clearance, 0)) return FIESTA_ERR_INVALID;
  if (min_cluster_size < 1) { fb_set_error("%s: min_cluster_size must be >= 1", fn); return FIESTA_ERR_INVALID; }
  fiesta_map *m = f->m;
  FbNavBox b{};
  if (!box_arg(fn, m->g, box_lo, box_hi, &b)) return FIESTA_ERR_INVALID;
  CK(cudaSetDevice(m->device));
  f->valid = false;
  int launches = 0;
  CK(cudaEventRecord(f->ev[0], m->stream));
  const int r = frontier_compute(m->g, m->cobs, m->occ, m->l_occ, b, clearance, (long long)min_cluster_size, f->B, m->stream, &launches);
  m->st.kernel_launches += launches;
  if (r != FIESTA_OK) return r;
  CK(cudaEventRecord(f->ev[1], m->stream));
  CK(cudaStreamSynchronize(m->stream));
  const FbFrCtr &c = *f->B.h_ctr;
  f->st = fiesta_frontier_stats{};
  f->st.box_voxels = (int64_t)b.n[0] * b.n[1] * b.n[2];
  f->st.frontier_voxels = (int64_t)c.frontier;
  f->st.clusters = (int64_t)c.roots;
  f->st.kept_clusters = (int64_t)c.sel[1];
  f->st.kept_voxels = (int64_t)c.kept_voxels;
  CK(cudaEventElapsedTime(&f->st.ms_compute, f->ev[0], f->ev[1]));
  f->box = b;
  f->valid = true;
  if (stats) *stats = f->st;
  return FIESTA_OK;
}
int fiesta_frontiers_clusters(const fiesta_frontiers *f, int64_t cap, int64_t *size, int32_t *rep_xyz, int32_t *bbox_lo_xyz,
                              int32_t *bbox_hi_xyz, double *centroid_xyz) {
  const char *fn = "fiesta_frontiers_clusters";
  if (!f || cap < 0 || (cap > 0 && !(size && rep_xyz && bbox_lo_xyz && bbox_hi_xyz && centroid_xyz))) {
    fb_set_error("%s: null buffer or negative capacity", fn);
    return FIESTA_ERR_INVALID;
  }
  if (!f->valid) { fb_set_error("%s: no frontiers have been computed", fn); return FIESTA_ERR_INVALID; }
  const size_t n = (size_t)(cap < f->st.kept_clusters ? cap : f->st.kept_clusters), C = f->B.C;
  if (n == 0) return FIESTA_OK;
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  CK(cudaMemcpyAsync(size, f->B.o_size, n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(rep_xyz, f->B.o_i32, n * 12, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(bbox_lo_xyz, f->B.o_i32 + 3 * C, n * 12, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(bbox_hi_xyz, f->B.o_i32 + 6 * C, n * 12, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(centroid_xyz, f->B.o_cen, n * 24, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
int fiesta_frontiers_voxels(const fiesta_frontiers *f, int64_t cap, int32_t *vox_xyz) {
  const char *fn = "fiesta_frontiers_voxels";
  if (!f || cap < 0 || (cap > 0 && !vox_xyz)) { fb_set_error("%s: null buffer or negative capacity", fn); return FIESTA_ERR_INVALID; }
  if (!f->valid) { fb_set_error("%s: no frontiers have been computed", fn); return FIESTA_ERR_INVALID; }
  const size_t n = (size_t)(cap < f->st.kept_voxels ? cap : f->st.kept_voxels);
  if (n == 0) return FIESTA_OK;
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  CK(cudaMemcpyAsync(vox_xyz, f->B.m_xyz, n * 12, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
int fiesta_frontiers_export(const fiesta_frontiers *f, int32_t *labels) {
  if (!f || !labels) { fb_set_error("fiesta_frontiers_export: null argument"); return FIESTA_ERR_INVALID; }
  if (!f->valid) { fb_set_error("fiesta_frontiers_export: no frontiers have been computed"); return FIESTA_ERR_INVALID; }
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  CK(cudaMemcpyAsync(labels, f->B.L, (size_t)f->st.box_voxels * 4, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
