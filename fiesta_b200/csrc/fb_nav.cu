// fiesta_b200 -- cost-to-go field kernels (definition: fb_nav.h, DESIGN.md §3.5).
//
// k_nav_init   : D := -1 on blocked box voxels (fb_seg_blocks, the segment-clearance predicate), +inf elsewhere.
// k_nav_goals  : D := 0 on each goal voxel that is in the box and traversable; every tile holding the goal or one of its 26
//                neighbours is queued for generation 0.
// k_nav_relax  : persistent cooperative kernel over a work list of 8^3 box tiles, one grid barrier per generation.  A tile and a
//                1-voxel halo (10^3 costs) are staged in shared memory and relaxed to a local fixpoint; improved voxels are
//                written back, and every neighbour tile that holds a neighbour of an improved boundary voxel is queued for the
//                next generation (generation stamps de-duplicate the list).  The kernel stops on an empty list.
// k_nav_count  : blocked and reached voxels of the finished field.
// k_nav_path   : one thread per start applies fb_nav_path.
//
// Why the result is exact without fp64 atomics: every value ever stored is fl(D(u) + w) of a stored value, i.e. the left fold
// of some path from a goal, and values only decrease.  A tile writes only its own voxels, and an aligned 64-bit load or store
// does not tear, so a halo value read mid-generation is the cost of some path: a valid upper bound.  A decrease of a boundary
// voxel -- a goal placed by k_nav_goals included -- always queues every tile holding one of its 26 neighbours, so when the list is empty no voxel can improve; fl-addition is
// monotone, so that fixpoint is the least one, the same bits a sequential Dijkstra gives, whatever the tile schedule.
#include <cooperative_groups.h>
#include "fb_common.cuh"
#include "fb_segment.h"

namespace cg = cooperative_groups;

#define NAV_THREADS 512        // one thread per voxel of an 8^3 tile
#define NAV_H (FB_TILE + 2)    // staged tile + 1-voxel halo per axis
#define NAV_NONE 0xffffffffu

__global__ void k_nav_init(FbGeom g, const uint32_t *__restrict__ cobs, FbNavArgs a, double r, int unknown_blocks) {
  const long long n = (long long)a.b.n[0] * a.b.n[1] * a.b.n[2];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % a.b.n[2]), y = (int)(i / a.b.n[2] % a.b.n[1]), x = (int)(i / ((long long)a.b.n[2] * a.b.n[1]));
    const int v[3] = {a.b.lo[0] + x, a.b.lo[1] + y, a.b.lo[2] + z};
    double d;
    a.D[i] = fb_seg_blocks(g, cobs, v, r, unknown_blocks != 0, d) ? FB_NAV_BLOCKED : (double)INFINITY;
  }
}

__global__ void k_nav_goals(FbGeom g, FbNavArgs a, const double *__restrict__ goals, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int v[3];
  if (!fb_nav_locate(g, a.b, goals + 3 * i, v)) return;
  const long long ii = fb_nav_idx(a.b, v[0], v[1], v[2]);
  if (!(a.D[ii] >= 0.0)) return;                                          // blocked goal
  a.D[ii] = 0.0;
  atomicAdd(&a.ctr->goals_placed, 1ull);
  // A goal is a decrease like any other: queue every tile that holds it or one of its 26 neighbours (the rule of k_nav_relax).
  // Its own tile alone would miss a neighbour tile that only the goal voxel itself touches.
  const int tc[3] = {v[0] >> 3, v[1] >> 3, v[2] >> 3};
  for (int ox = ((v[0] & 7) == 0 ? -1 : 0); ox <= ((v[0] & 7) == FB_TILE - 1 ? 1 : 0); ++ox)
    for (int oy = ((v[1] & 7) == 0 ? -1 : 0); oy <= ((v[1] & 7) == FB_TILE - 1 ? 1 : 0); ++oy)
      for (int oz = ((v[2] & 7) == 0 ? -1 : 0); oz <= ((v[2] & 7) == FB_TILE - 1 ? 1 : 0); ++oz) {
        const int nx = tc[0] + ox, ny = tc[1] + oy, nz = tc[2] + oz;
        if (nx < 0 || nx >= a.tn[0] || ny < 0 || ny >= a.tn[1] || nz < 0 || nz >= a.tn[2]) continue;
        const unsigned t = (unsigned)((nx * a.tn[1] + ny) * a.tn[2] + nz);
        if (atomicExch(&a.stamp[t], 1u) != 1u) a.list[0][atomicAdd(&a.ctr->n[0], 1u)] = t;   // generation 0 has stamp 1
      }
}

__global__ void __launch_bounds__(NAV_THREADS, 2) k_nav_relax(FbNavArgs a) {
  __shared__ double sD[NAV_H * NAV_H * NAV_H];
  __shared__ unsigned s_tile, s_q;
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lx = tid >> 6, ly = (tid >> 3) & 7, lz = tid & 7;
  const int c = ((lx + 1) * NAV_H + ly + 1) * NAV_H + lz + 1;
  const double w1 = a.w[0], w2 = a.w[1], w3 = a.w[2];
  unsigned long long visits = 0;
  unsigned gen = 0;
  // Three list counters rotate: generation g reads n[g % 3], appends to n[(g + 1) % 3] and clears n[(g + 2) % 3], which every
  // block read at the start of generation g - 1, before the barrier that ended it.  The fetch counters rotate the same way.
  for (;; ++gen) {
    const unsigned cur = gen % 3u, nxt = (gen + 1u) % 3u;
    const unsigned nwork = __ldcg(&a.ctr->n[cur]);
    if (nwork == 0) break;
    if (blockIdx.x == 0 && tid == 0) { a.ctr->n[(gen + 2u) % 3u] = 0; a.ctr->next[(gen + 2u) % 3u] = 0; }
    const uint32_t *list = (gen & 1u) ? a.list[1] : a.list[0];
    uint32_t *out = (gen & 1u) ? a.list[0] : a.list[1];
    const unsigned stamp_next = gen + 2u;
    for (;;) {
      if (tid == 0) {
        const unsigned w = atomicAdd(&a.ctr->next[cur], 1u);
        s_tile = w < nwork ? __ldcg(&list[w]) : NAV_NONE;
        s_q = 0;
      }
      __syncthreads();
      const unsigned tile = s_tile;
      if (tile == NAV_NONE) break;
      if (tid == 0) ++visits;
      const int tz = (int)(tile % (unsigned)a.tn[2]), ty = (int)(tile / (unsigned)a.tn[2] % (unsigned)a.tn[1]),
                tx = (int)(tile / (unsigned)(a.tn[2] * a.tn[1]));
      const int x0 = tx * FB_TILE - 1, y0 = ty * FB_TILE - 1, z0 = tz * FB_TILE - 1;
      for (int i = tid; i < NAV_H * NAV_H * NAV_H; i += NAV_THREADS) {
        const int x = x0 + i / (NAV_H * NAV_H), y = y0 + i / NAV_H % NAV_H, z = z0 + i % NAV_H;
        sD[i] = fb_nav_in_box(a.b, x, y, z) ? __ldcg(&a.D[fb_nav_idx(a.b, x, y, z)]) : FB_NAV_BLOCKED;
      }
      __syncthreads();
      // allowed moves into this voxel: bit k (fb_nav_dir order) when the box spanned by the voxel and its neighbour k is
      // traversable; nb bit e = voxel + e traversable, e over the 3x3x3 neighbourhood in the same order
      unsigned nb = 0, allowed = 0;
#pragma unroll
      for (int e = 0; e < 27; ++e) nb |= (sD[c + ((e / 9 - 1) * NAV_H + (e / 3 % 3 - 1)) * NAV_H + (e % 3 - 1)] >= 0.0 ? 1u : 0u) << e;
      if (nb & (1u << 13)) {
#pragma unroll
        for (int k = 0; k < 27; ++k) {
          if (k == 13) continue;
          const int dx = k / 9 - 1, dy = k / 3 % 3 - 1, dz = k % 3 - 1;
          unsigned need = 0;
#pragma unroll
          for (int ex = (dx < 0 ? -1 : 0); ex <= (dx > 0 ? 1 : 0); ++ex)
#pragma unroll
            for (int ey = (dy < 0 ? -1 : 0); ey <= (dy > 0 ? 1 : 0); ++ey)
#pragma unroll
              for (int ez = (dz < 0 ? -1 : 0); ez <= (dz > 0 ? 1 : 0); ++ez) need |= 1u << ((ex + 1) * 9 + (ey + 1) * 3 + ez + 1);
          if ((nb & need) == need) allowed |= 1u << k;
        }
      }
      const double orig = sD[c];
      double my = orig;
      for (;;) {                                                          // local fixpoint of the tile
        double best = my;
#pragma unroll
        for (int k = 0; k < 27; ++k) {
          if (k == 13) continue;
          const int dx = k / 9 - 1, dy = k / 3 % 3 - 1, dz = k % 3 - 1, nz = (dx != 0) + (dy != 0) + (dz != 0);
          if (allowed & (1u << k)) {
            const double cand = sD[c + (dx * NAV_H + dy) * NAV_H + dz] + (nz == 1 ? w1 : nz == 2 ? w2 : w3);
            if (cand < best) best = cand;
          }
        }
        const bool ch = best < my;
        if (ch) { my = best; sD[c] = best; }
        if (!__syncthreads_or(ch)) break;
      }
      if (my < orig) {
        const int x = tx * FB_TILE + lx, y = ty * FB_TILE + ly, z = tz * FB_TILE + lz;
        __stcg(&a.D[fb_nav_idx(a.b, x, y, z)], my);
        // neighbour tiles that hold a neighbour of this voxel: on each axis, the tile itself plus the one across a tile face
        unsigned q = 0;
        for (int ox = (lx == 0 ? -1 : 0); ox <= (lx == FB_TILE - 1 ? 1 : 0); ++ox)
          for (int oy = (ly == 0 ? -1 : 0); oy <= (ly == FB_TILE - 1 ? 1 : 0); ++oy)
            for (int oz = (lz == 0 ? -1 : 0); oz <= (lz == FB_TILE - 1 ? 1 : 0); ++oz) q |= 1u << ((ox + 1) * 9 + (oy + 1) * 3 + oz + 1);
        q &= ~(1u << 13);
        if (q) atomicOr(&s_q, q);
      }
      __syncthreads();
      if (tid < 27 && ((s_q >> tid) & 1u)) {
        const int nx = tx + tid / 9 - 1, ny = ty + tid / 3 % 3 - 1, nz = tz + tid % 3 - 1;
        if (nx >= 0 && nx < a.tn[0] && ny >= 0 && ny < a.tn[1] && nz >= 0 && nz < a.tn[2]) {
          const unsigned t = (unsigned)((nx * a.tn[1] + ny) * a.tn[2] + nz);
          if (atomicExch(&a.stamp[t], stamp_next) != stamp_next) out[atomicAdd(&a.ctr->n[nxt], 1u)] = t;
        }
      }
      __syncthreads();                                                    // s_tile and s_q are rewritten for the next tile
    }
    grid.sync();
  }
  if (tid == 0) {
    if (visits) atomicAdd(&a.ctr->tile_visits, visits);
    if (blockIdx.x == 0) a.ctr->generations = gen;
  }
}

__global__ void k_nav_count(FbNavArgs a) {
  const long long n = (long long)a.b.n[0] * a.b.n[1] * a.b.n[2];
  unsigned blocked = 0, reached = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double d = a.D[i];
    blocked += d < 0.0;
    reached += d >= 0.0 && d < (double)INFINITY;
  }
  blocked = __reduce_add_sync(0xffffffffu, blocked);
  reached = __reduce_add_sync(0xffffffffu, reached);
  if ((threadIdx.x & 31) == 0) {
    if (blocked) atomicAdd(&a.ctr->blocked, (unsigned long long)blocked);
    if (reached) atomicAdd(&a.ctr->reached, (unsigned long long)reached);
  }
}

__global__ void k_nav_path(FbGeom g, FbNavBox b, const double *__restrict__ D, double w1, double w2, double w3, const double *__restrict__ starts,
                           long long n, int max_len, int32_t *status, int32_t *len, double *cost, int32_t *vox) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double *p = starts + 3 * i;
  const double w[3] = {w1, w2, w3};
  int v[3];
  if (!fb_pos_in_map(g, p) || !fb_nav_locate(g, b, p, v)) {               // NaN fails fb_nav_locate
    status[i] = FB_NAV_INVALID_START; len[i] = 0; cost[i] = nan("");
    return;
  }
  status[i] = fb_nav_path(b, D, w, v, max_len, vox + 3 * (long long)max_len * i, &len[i], &cost[i]);
}

// ---------------------------------------------------------------- host side
static unsigned nav_blocks(long long n) {
  const long long want = (n + 255) / 256;
  return (unsigned)(want < FB_SMS * 16ll ? want : FB_SMS * 16ll);
}

int fb_nav_relax_blocks(int device) {
  int per_sm = 0, sms = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_nav_relax, NAV_THREADS, 0) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return 0;
  return per_sm * sms;                                                    // every block co-resident: required by grid.sync()
}

cudaError_t fb_nav_compute(const FbGeom &g, const uint32_t *cobs, const FbNavArgs &a, const double *goals, long long n_goals, double r,
                           int unknown_blocks, int nblocks, cudaStream_t s) {
  const long long n = (long long)a.b.n[0] * a.b.n[1] * a.b.n[2];
  k_nav_init<<<nav_blocks(n), 256, 0, s>>>(g, cobs, a, r, unknown_blocks);
  if (n_goals > 0) k_nav_goals<<<(unsigned)((n_goals + 127) / 128), 128, 0, s>>>(g, a, goals, n_goals);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  void *args[] = {(void *)&a};
  if ((e = cudaLaunchCooperativeKernel((void *)k_nav_relax, dim3(nblocks), dim3(NAV_THREADS), args, 0, s)) != cudaSuccess) return e;
  k_nav_count<<<nav_blocks(n), 256, 0, s>>>(a);
  return cudaGetLastError();
}

cudaError_t fb_nav_paths(const FbGeom &g, const FbNavBox &b, const double *D, const double *w, const double *starts, long long n, int max_len,
                         int32_t *status, int32_t *len, double *cost, int32_t *vox, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  k_nav_path<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(g, b, D, w[0], w[1], w[2], starts, n, max_len, status, len, cost, vox);
  return cudaGetLastError();
}
