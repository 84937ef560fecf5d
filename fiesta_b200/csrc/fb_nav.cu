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
#include "fb_nav.cuh"
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

// ---------------------------------------------------------------- field update (DESIGN.md §3.11)
// k_navu_scan     : the new traversability of every box voxel against the field's sign (the old one) into the scratch byte
//                   (FB_NAVU_NEWT, FB_NAVU_CHG); counts the changes and queues for the withdrawal wave every tile holding a
//                   26-neighbour of a newly blocked voxel (only those voxels can lose a move).
// k_navu_withdraw : the withdrawal wave, persistent and cooperative with k_nav_relax's work list, stamps and rotating counters.  A
//                   tile stages old costs and scratch bytes with a 1-voxel halo, and withdraws (FB_NAVU_WD) each candidate none of
//                   whose tight supports is still kept through a still-allowed move, to a local fixpoint; the tiles across the
//                   faces of a newly withdrawn boundary voxel are queued.  Withdrawals only accumulate and the support relation is
//                   acyclic, so from all-kept every schedule ends at the unique solution.  The field itself is only read.
// k_navu_apply    : the start state of the re-relaxation (-1 newly blocked, +inf withdrawn and newly free, everything else as it
//                   was) and generation 0's tile list: the tile of a withdrawn voxel, every tile holding a newly free voxel or
//                   one of its 26 neighbours (a newly placed goal is always newly free, so its tiles are among them).
// k_navu_goals    : D := 0 on the stored goals that are traversable, as k_nav_goals does.
// Then k_nav_relax and k_nav_count run unchanged.

// Allowed moves into the centre voxel from the traversability of its 3x3x3 neighbourhood: fb_nav_move_bits without bit 13, unrolled
// as in k_nav_relax.
static __device__ __forceinline__ unsigned navu_allowed(unsigned nb) {
  unsigned allowed = 0;
  if (!(nb & (1u << 13))) return 0;
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
  return allowed;
}

// Queue every tile that holds box voxel v or one of its 26 neighbours (own) or only those across its faces (!own) with `stamp`.
static __device__ void navu_queue(const FbNavArgs &a, int x, int y, int z, bool own, unsigned stamp, uint32_t *list, unsigned *n) {
  const int v[3] = {x, y, z};
  for (int ox = ((v[0] & 7) == 0 ? -1 : 0); ox <= ((v[0] & 7) == FB_TILE - 1 ? 1 : 0); ++ox)
    for (int oy = ((v[1] & 7) == 0 ? -1 : 0); oy <= ((v[1] & 7) == FB_TILE - 1 ? 1 : 0); ++oy)
      for (int oz = ((v[2] & 7) == 0 ? -1 : 0); oz <= ((v[2] & 7) == FB_TILE - 1 ? 1 : 0); ++oz) {
        if (!own && ox == 0 && oy == 0 && oz == 0) continue;
        const int nx = (v[0] >> 3) + ox, ny = (v[1] >> 3) + oy, nz = (v[2] >> 3) + oz;
        if (nx < 0 || nx >= a.tn[0] || ny < 0 || ny >= a.tn[1] || nz < 0 || nz >= a.tn[2]) continue;
        const unsigned t = (unsigned)((nx * a.tn[1] + ny) * a.tn[2] + nz);
        // the plain read spares the atomic on tiles already queued (a stamp, once set, stays for the rest of the kernel)
        if (__ldcg(&a.stamp[t]) != stamp && atomicExch(&a.stamp[t], stamp) != stamp) list[atomicAdd(n, 1u)] = t;
      }
}

__global__ void k_navu_scan(FbGeom g, const uint32_t *__restrict__ cobs, FbNavArgs w, uint8_t *__restrict__ flags, FbNavUCtr *u,
                            double r, int unknown_blocks) {
  const long long n = (long long)w.b.n[0] * w.b.n[1] * w.b.n[2];
  unsigned nblk = 0, nfree = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % w.b.n[2]), y = (int)(i / w.b.n[2] % w.b.n[1]), x = (int)(i / ((long long)w.b.n[2] * w.b.n[1]));
    const int v[3] = {w.b.lo[0] + x, w.b.lo[1] + y, w.b.lo[2] + z};
    double d;
    const bool newt = !fb_seg_blocks(g, cobs, v, r, unknown_blocks != 0, d), oldt = w.D[i] >= 0.0;
    flags[i] = (uint8_t)((newt ? FB_NAVU_NEWT : 0u) | (newt != oldt ? FB_NAVU_CHG : 0u));
    if (oldt && !newt) {
      ++nblk;
      navu_queue(w, x, y, z, true, 1u, w.list[0], &w.ctr->n[0]);          // generation 0 has stamp 1
    }
    nfree += newt && !oldt;
  }
  nblk = __reduce_add_sync(0xffffffffu, nblk);
  nfree = __reduce_add_sync(0xffffffffu, nfree);
  if ((threadIdx.x & 31) == 0) {
    if (nblk) atomicAdd(&u->became_blocked, (unsigned long long)nblk);
    if (nfree) atomicAdd(&u->became_free, (unsigned long long)nfree);
  }
}

__global__ void __launch_bounds__(NAV_THREADS, 2) k_navu_withdraw(FbNavArgs a, uint8_t *flags) {
  __shared__ double sD[NAV_H * NAV_H * NAV_H];
  __shared__ uint8_t sF[NAV_H * NAV_H * NAV_H];
  __shared__ unsigned s_tile, s_q;
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lx = tid >> 6, ly = (tid >> 3) & 7, lz = tid & 7;
  const int c = ((lx + 1) * NAV_H + ly + 1) * NAV_H + lz + 1;
  unsigned long long visits = 0;
  unsigned gen = 0;
  for (;; ++gen) {                                                        // the generation loop of k_nav_relax
    const unsigned cur = gen % 3u, nxt = (gen + 1u) % 3u;
    const unsigned nwork = __ldcg(&a.ctr->n[cur]);
    if (nwork == 0) break;
    if (blockIdx.x == 0 && tid == 0) { a.ctr->n[(gen + 2u) % 3u] = 0; a.ctr->next[(gen + 2u) % 3u] = 0; }
    const uint32_t *list = (gen & 1u) ? a.list[1] : a.list[0];
    uint32_t *out = (gen & 1u) ? a.list[0] : a.list[1];
    const unsigned stamp_next = gen + 2u;
    for (;;) {
      if (tid == 0) {
        const unsigned k = atomicAdd(&a.ctr->next[cur], 1u);
        s_tile = k < nwork ? __ldcg(&list[k]) : NAV_NONE;
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
        const bool in = fb_nav_in_box(a.b, x, y, z);
        const long long ii = in ? fb_nav_idx(a.b, x, y, z) : 0;
        sD[i] = in ? __ldcg(&a.D[ii]) : FB_NAV_BLOCKED;
        sF[i] = in ? __ldcg(&flags[ii]) : (uint8_t)0;
      }
      __syncthreads();
      // candidates: still traversable, finite non-zero old cost, not yet withdrawn; sup = tight supports still allowed now
      const double dv = sD[c];
      const uint8_t f0 = sF[c];
      bool cand = (f0 & FB_NAVU_NEWT) && !(f0 & FB_NAVU_WD) && dv > 0.0 && dv < (double)INFINITY;
      unsigned sup = 0;
      if (cand) {
        unsigned nb = 0;
#pragma unroll
        for (int e = 0; e < 27; ++e) nb |= (sD[c + ((e / 9 - 1) * NAV_H + (e / 3 % 3 - 1)) * NAV_H + (e % 3 - 1)] >= 0.0 ? 1u : 0u) << e;
        const unsigned old_bits = navu_allowed(nb);
        for (unsigned m = old_bits; m; m &= m - 1u) {                      // the moves allowed before, one set bit at a time
          const int k = __ffs(m) - 1, dx = k / 9 - 1, dy = k / 3 % 3 - 1, dz = k % 3 - 1, nz = (dx != 0) + (dy != 0) + (dz != 0);
          if (fb_nav_is_support(true, sD[c + (dx * NAV_H + dy) * NAV_H + dz], nz == 1 ? a.w[0] : nz == 2 ? a.w[1] : a.w[2], dv)) sup |= 1u << k;
        }
        nb = 0;
#pragma unroll
        for (int e = 0; e < 27; ++e) nb |= ((sF[c + ((e / 9 - 1) * NAV_H + (e / 3 % 3 - 1)) * NAV_H + (e % 3 - 1)] & FB_NAVU_NEWT) ? 1u : 0u) << e;
        sup &= navu_allowed(nb);
      }
      for (;;) {                                                          // local fixpoint: withdrawals only accumulate
        bool ch = false;
        if (cand) {
          bool kept = false;
          for (unsigned m = sup; m && !kept; m &= m - 1u) {                 // the supports, one set bit at a time
            const int k = __ffs(m) - 1;
            kept = !(sF[c + ((k / 9 - 1) * NAV_H + (k / 3 % 3 - 1)) * NAV_H + (k % 3 - 1)] & FB_NAVU_WD);
          }
          if (!kept) { sF[c] = (uint8_t)(f0 | FB_NAVU_WD); cand = false; ch = true; }
        }
        if (!__syncthreads_or(ch)) break;
      }
      if ((sF[c] & FB_NAVU_WD) && !(f0 & FB_NAVU_WD)) {
        const int x = tx * FB_TILE + lx, y = ty * FB_TILE + ly, z = tz * FB_TILE + lz;
        __stcg(&flags[fb_nav_idx(a.b, x, y, z)], sF[c]);
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
      __syncthreads();
    }
    grid.sync();
  }
  if (tid == 0) {
    if (visits) atomicAdd(&a.ctr->tile_visits, visits);
    if (blockIdx.x == 0) a.ctr->generations = gen;
  }
}

__global__ void k_navu_apply(FbNavArgs a, const uint8_t *__restrict__ flags, FbNavUCtr *u) {
  const long long n = (long long)a.b.n[0] * a.b.n[1] * a.b.n[2];
  unsigned wd = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned f = flags[i];
    if (!(f & FB_NAVU_NEWT)) {
      if (f & FB_NAVU_CHG) a.D[i] = FB_NAV_BLOCKED;
      continue;
    }
    if (!(f & (FB_NAVU_CHG | FB_NAVU_WD))) continue;                     // kept, or unreached before and after
    a.D[i] = (double)INFINITY;
    wd += (f & FB_NAVU_CHG) == 0;
    const int z = (int)(i % a.b.n[2]), y = (int)(i / a.b.n[2] % a.b.n[1]), x = (int)(i / ((long long)a.b.n[2] * a.b.n[1]));
    if (f & FB_NAVU_CHG) {
      navu_queue(a, x, y, z, true, 1u, a.list[0], &a.ctr->n[0]);        // a freed voxel can allow a move between two others
    } else {
      const unsigned t = (unsigned)(((x >> 3) * a.tn[1] + (y >> 3)) * a.tn[2] + (z >> 3));
      if (__ldcg(&a.stamp[t]) != 1u && atomicExch(&a.stamp[t], 1u) != 1u) a.list[0][atomicAdd(&a.ctr->n[0], 1u)] = t;
    }
  }
  wd = __reduce_add_sync(0xffffffffu, wd);
  if ((threadIdx.x & 31) == 0 && wd) atomicAdd(&u->withdrawn, (unsigned long long)wd);
}

__global__ void k_navu_goals(FbGeom g, FbNavArgs a, const uint8_t *__restrict__ flags, FbNavUCtr *u, const double *__restrict__ goals,
                             long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int v[3];
  if (!fb_nav_locate(g, a.b, goals + 3 * i, v)) return;
  const long long ii = fb_nav_idx(a.b, v[0], v[1], v[2]);
  if (!(a.D[ii] >= 0.0)) return;                                          // blocked goal
  a.D[ii] = 0.0;
  atomicAdd(&a.ctr->goals_placed, 1ull);
  if (flags[ii] & FB_NAVU_CHG) atomicAdd(&u->goals_new, 1ull);           // newly free: its tiles are queued by k_navu_apply
}

// ---------------------------------------------------------------- host side
static unsigned nav_blocks(long long n) {
  const long long want = (n + 255) / 256;
  return (unsigned)(want < FB_SMS * 16ll ? want : FB_SMS * 16ll);
}

static int nav_relax_blocks(int device) {
  int per_sm = 0, sms = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_nav_relax, NAV_THREADS, 0) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return 0;
  return per_sm * sms;                                                    // every block co-resident: required by grid.sync()
}

static int nav_withdraw_blocks(int device) {
  int per_sm = 0, sms = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_navu_withdraw, NAV_THREADS, 0) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return 0;
  return per_sm * sms;
}

// The whole compute on stream s: 3 launches, 4 with goals.  Expects the stamps and a.ctr zeroed.
static cudaError_t nav_compute_launch(const FbGeom &g, const uint32_t *cobs, const FbNavArgs &a, const double *goals, long long n_goals,
                                      double r, int unknown_blocks, int nblocks, cudaStream_t s) {
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

// The whole update on stream s: 5 launches, 6 with goals.  a.D holds the old field; a.ctr and u are cleared here.
static cudaError_t nav_update_launch(const FbGeom &g, const uint32_t *cobs, const FbNavArgs &a, uint8_t *flags, FbNavUCtr *u,
                                     const double *goals, long long n_goals, double r, int unknown_blocks, int nblocks, int wblocks,
                                     cudaStream_t s) {
  const long long n = (long long)a.b.n[0] * a.b.n[1] * a.b.n[2];
  const size_t nt = (size_t)a.tn[0] * a.tn[1] * a.tn[2];
  FbNavArgs w = a;                                                        // the wave: same lists and stamps, its own counters
  w.ctr = &u->wave;
  cudaError_t e;
  if ((e = cudaMemsetAsync(u, 0, sizeof(FbNavUCtr), s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(a.stamp, 0, nt * 4, s)) != cudaSuccess) return e;
  k_navu_scan<<<nav_blocks(n), 256, 0, s>>>(g, cobs, w, flags, u, r, unknown_blocks);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  void *wargs[] = {(void *)&w, (void *)&flags};
  if ((e = cudaLaunchCooperativeKernel((void *)k_navu_withdraw, dim3(wblocks), dim3(NAV_THREADS), wargs, 0, s)) != cudaSuccess) return e;
  // old costs are read until here; the re-relaxation starts from clean stamps and counters, as in fiesta_nav_compute
  if ((e = cudaMemsetAsync(a.stamp, 0, nt * 4, s)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(a.ctr, 0, sizeof(FbNavCtr), s)) != cudaSuccess) return e;
  k_navu_apply<<<nav_blocks(n), 256, 0, s>>>(a, flags, u);
  if (n_goals > 0) k_navu_goals<<<(unsigned)((n_goals + 127) / 128), 128, 0, s>>>(g, a, flags, u, goals, n_goals);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if ((e = cudaMemcpyAsync(&u->seed_tiles, &a.ctr->n[0], 4, cudaMemcpyDeviceToDevice, s)) != cudaSuccess) return e;
  void *args[] = {(void *)&a};
  if ((e = cudaLaunchCooperativeKernel((void *)k_nav_relax, dim3(nblocks), dim3(NAV_THREADS), args, 0, s)) != cudaSuccess) return e;
  k_nav_count<<<nav_blocks(n), 256, 0, s>>>(a);
  return cudaGetLastError();
}

// ---------------------------------------------------------------- entry points (include/fiesta_b200.h)
void fiesta_nav_destroy(fiesta_nav_field *f) { handle_destroy(f); }
int fiesta_nav_create(fiesta_map *m, fiesta_nav_field **out) {
  if (!m || !out) { fb_set_error("fiesta_nav_create: null argument"); return FIESTA_ERR_INVALID; }
  *out = nullptr;
  FbHandle<fiesta_nav_field> f;
  int r;
  if ((r = handle_new(m, f))) return r;
  if (!f) { fb_set_error("out of host memory"); return FIESTA_ERR_INVALID; }
  f->blocks = nav_relax_blocks(m->device);
  f->mblocks = fb_navm_relax_blocks(m->device);
  f->wblocks = nav_withdraw_blocks(m->device);
  if (f->blocks <= 0 || f->mblocks <= 0 || f->wblocks <= 0) { fb_set_error("fiesta_nav_create: the relaxation kernel does not fit on this device"); return FIESTA_ERR_CUDA; }
  for (cudaEvent_t &e : f->ev) CK(cudaEventCreate(&e));
  CK(f->ctr.alloc(1));
  CK(f->h_ctr.alloc(1));
  CK(f->m_ctr.alloc(1));
  CK(f->m_tot.alloc(1));
  CK(f->h_mtot.alloc(1));
  CK(f->u_ctr.alloc(1));
  CK(f->h_uctr.alloc(1));
  for (int k = 0; k < 3; ++k) f->w[k] = m->g.res * sqrt((double)(k + 1));
  *out = f.release();
  return FIESTA_OK;
}
int fiesta_nav_compute(fiesta_nav_field *f, const int box_lo[3], const int box_hi[3], const double *goals_xyz, int64_t n_goals,
                       double clearance, int flags, fiesta_nav_stats *stats) {
  const char *fn = "fiesta_nav_compute";
  if (!f || !box_lo || !box_hi) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  if (!count_buffers_ok(fn, n_goals, goals_xyz != nullptr) || !clearance_flags_ok(fn, clearance, flags)) return FIESTA_ERR_INVALID;
  fiesta_map *m = f->m;
  const FbGeom &g = m->g;
  FbNavArgs a{};
  if (!box_arg(fn, g, box_lo, box_hi, &a.b)) return FIESTA_ERR_INVALID;
  for (int k = 0; k < 3; ++k) {
    a.tn[k] = (a.b.n[k] + FB_TILE - 1) / FB_TILE;
    a.w[k] = f->w[k];
  }
  const size_t nv = (size_t)a.b.n[0] * a.b.n[1] * a.b.n[2], nt = (size_t)a.tn[0] * a.tn[1] * a.tn[2];
  CK(cudaSetDevice(m->device));
  f->valid = false;
  cudaError_t e = f->D.grow(nv, m->stream);
  for (FbDevBuf<uint32_t> *b : {&f->stamp, &f->list[0], &f->list[1]})
    if (e == cudaSuccess) e = b->grow(nt, m->stream);
  if (e == cudaSuccess && n_goals > 0) e = f->d_goals.grow((size_t)n_goals * 3, m->stream);
  if (e != cudaSuccess) return alloc_failed(e, "%s: cannot allocate the field of %zu voxels", fn, nv);
  a.D = f->D; a.stamp = f->stamp; a.list[0] = f->list[0]; a.list[1] = f->list[1]; a.ctr = f->ctr;
  if (n_goals > 0) CK(cudaMemcpyAsync(f->d_goals, goals_xyz, (size_t)n_goals * 24, cudaMemcpyHostToDevice, m->stream));
  CK(cudaMemsetAsync(f->stamp, 0, nt * 4, m->stream));
  CK(cudaMemsetAsync(f->ctr, 0, sizeof(FbNavCtr), m->stream));
  CK(cudaEventRecord(f->ev[0], m->stream));
  CK(nav_compute_launch(g, m->cobs, a, f->d_goals, n_goals, clearance, flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS, f->blocks, m->stream));
  m->st.kernel_launches += n_goals > 0 ? 4 : 3;
  CK(cudaEventRecord(f->ev[1], m->stream));
  CK(cudaMemcpyAsync(f->h_ctr, f->ctr, sizeof(FbNavCtr), cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  f->box = a.b;
  f->valid = true;
  f->n_goals = n_goals;
  f->clearance = clearance;
  f->flags = flags;
  if (stats) {
    const FbNavCtr &c = *f->h_ctr;
    *stats = fiesta_nav_stats{};
    stats->box_voxels = (int64_t)nv;
    stats->blocked = (int64_t)c.blocked;
    stats->reached = (int64_t)c.reached;
    stats->goals_placed = (int64_t)c.goals_placed;
    stats->generations = (int64_t)c.generations;
    stats->tile_visits = (int64_t)c.tile_visits;
    CK(cudaEventElapsedTime(&stats->ms_compute, f->ev[0], f->ev[1]));
  }
  return FIESTA_OK;
}
int fiesta_nav_update(fiesta_nav_field *f, fiesta_nav_update_stats *stats) {
  const char *fn = "fiesta_nav_update";
  if (!f) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  if (!f->valid) { fb_set_error("%s: no field has been computed", fn); return FIESTA_ERR_INVALID; }
  fiesta_map *m = f->m;
  FbNavArgs a{};
  a.b = f->box;
  for (int k = 0; k < 3; ++k) {
    a.tn[k] = (a.b.n[k] + FB_TILE - 1) / FB_TILE;
    a.w[k] = f->w[k];
  }
  const size_t nv = (size_t)a.b.n[0] * a.b.n[1] * a.b.n[2];
  CK(cudaSetDevice(m->device));
  if (cudaError_t e = f->u_flags.grow(nv, m->stream))                    // before anything is written: the field stays valid
    return alloc_failed(e, "%s: cannot allocate the scratch of %zu voxels", fn, nv);
  a.D = f->D; a.stamp = f->stamp; a.list[0] = f->list[0]; a.list[1] = f->list[1]; a.ctr = f->ctr;
  f->valid = false;                                                       // until the update has finished
  CK(cudaEventRecord(f->ev[0], m->stream));
  CK(nav_update_launch(m->g, m->cobs, a, f->u_flags, f->u_ctr, f->d_goals, f->n_goals, f->clearance, f->flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS,
                       f->blocks, f->wblocks, m->stream));
  m->st.kernel_launches += f->n_goals > 0 ? 6 : 5;
  CK(cudaEventRecord(f->ev[1], m->stream));
  CK(cudaMemcpyAsync(f->h_ctr, f->ctr, sizeof(FbNavCtr), cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(f->h_uctr, f->u_ctr, sizeof(FbNavUCtr), cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  f->valid = true;
  if (stats) {
    const FbNavCtr &c = *f->h_ctr;
    const FbNavUCtr &u = *f->h_uctr;
    *stats = fiesta_nav_update_stats{};
    stats->box_voxels = (int64_t)nv;
    stats->became_blocked = (int64_t)u.became_blocked;
    stats->became_free = (int64_t)u.became_free;
    stats->withdrawn = (int64_t)u.withdrawn;
    stats->goals_placed = (int64_t)c.goals_placed;
    stats->goals_new = (int64_t)u.goals_new;
    stats->seed_tiles = (int64_t)u.seed_tiles;
    stats->withdraw_generations = (int64_t)u.wave.generations;
    stats->generations = (int64_t)c.generations;
    stats->tile_visits = (int64_t)c.tile_visits;
    stats->blocked = (int64_t)c.blocked;
    stats->reached = (int64_t)c.reached;
    CK(cudaEventElapsedTime(&stats->ms_compute, f->ev[0], f->ev[1]));
  }
  return FIESTA_OK;
}
int fiesta_nav_export(const fiesta_nav_field *f, double *out) {
  if (!f || !out) { fb_set_error("fiesta_nav_export: null argument"); return FIESTA_ERR_INVALID; }
  if (!f->valid) { fb_set_error("fiesta_nav_export: no field has been computed"); return FIESTA_ERR_INVALID; }
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  CK(cudaMemcpyAsync(out, f->D, (size_t)f->box.n[0] * f->box.n[1] * f->box.n[2] * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
int fiesta_nav_paths(fiesta_nav_field *f, const double *starts_xyz, int64_t n, int32_t max_len, int32_t *status, int32_t *len, double *cost,
                     int32_t *vox_xyz) {
  const char *fn = "fiesta_nav_paths";
  if (!f || n < 0 || max_len < 1 || (n > 0 && !(starts_xyz && status && len && cost && vox_xyz))) {
    fb_set_error("%s: null buffer, negative count or max_len < 1", fn);
    return FIESTA_ERR_INVALID;
  }
  if (!f->valid) { fb_set_error("%s: no field has been computed", fn); return FIESTA_ERR_INVALID; }
  if (n == 0) return FIESTA_OK;
  fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  const size_t nv = (size_t)n * max_len * 3;
  cudaError_t e = f->d_pd.grow((size_t)n * 4, m->stream);
  if (e == cudaSuccess) e = f->d_pi.grow((size_t)n * 2 + nv, m->stream);
  if (e != cudaSuccess) return alloc_failed(e, "%s: cannot allocate %lld paths of %d voxels", fn, (long long)n, (int)max_len);
  double *d_starts = f->d_pd, *d_cost = d_starts + 3 * n;
  int32_t *d_st = f->d_pi, *d_len = d_st + n, *d_vox = d_len + n;
  CK(cudaMemcpyAsync(d_starts, starts_xyz, (size_t)n * 24, cudaMemcpyHostToDevice, m->stream));
  CK(cudaMemsetAsync(d_vox, 0xff, nv * 4, m->stream));                    // -1 past each path's end
  k_nav_path<<<(unsigned)((n + 127) / 128), 128, 0, m->stream>>>(m->g, f->box, f->D, f->w[0], f->w[1], f->w[2], d_starts, n, max_len, d_st,
                                                                 d_len, d_cost, d_vox);
  CK(cudaGetLastError());
  m->st.kernel_launches++;
  CK(cudaMemcpyAsync(status, d_st, (size_t)n * 4, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(len, d_len, (size_t)n * 4, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(cost, d_cost, (size_t)n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(vox_xyz, d_vox, nv * 4, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
