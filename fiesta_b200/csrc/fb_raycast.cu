// fiesta_b200 -- per-frame ray casting into the hit/miss counters.
//
// Replaces Fiesta::RaycastMultithread + RaycastProcess (FIESTA include/Fiesta.h:194-303), Raycast()
// (FIESTA src/raycast.cpp:56-158) and the counter half of ESDFMap::SetOccupancy
// (FIESTA src/ESDFMap.cpp:401-437) with results identical to the reference's SERIAL mode
// (ray_cast_num_thread = 0, the only deterministic one).
//
// The serial loop is order dependent: a ray's back-to-front free-space marking stops at the first voxel an EARLIER
// ray already stamped this frame (set_free_, Fiesta.h:265-273), and a ray is skipped when an earlier point ended in the
// same voxel (set_occ_, Fiesta.h:227-230).  The device pipeline reproduces that exactly:
//   k_ray_endpoints : per point: transform, length gating, endpoint SetOccupancy (one 64-bit atomicAdd on
//                     {hit:32|total:32}), and "lowest point index wins" ownership of the endpoint voxel (atomicMax on a
//                     tagged stamp) == the set_occ_ dedupe.
//   k_ray_trace     : per surviving ray (one thread each; the DDA's tMax += tDelta recurrence is sequential fp64 and
//                     must round exactly like the reference): Amanatides-Woo traversal with the reference's quirks
//                     (direction from integer voxel deltas, tie order z>y>x, corner-based distance cut); every pushed voxel
//                     is classified (count / skip / stop / stamp-only) and stored in the ray's row.
//   k_ray_resolve   : persistent cooperative kernel, event driven, one WARP per walking ray.  Every voxel holds a claim
//                     word {ray, position in that ray's list}; a claim is VALID while position < the claiming ray's current
//                     reach.  A ray walks its list from the far end 32 voxels at a time, stops at the first voxel validly
//                     claimed by a LOWER ray index and claims (atomicCAS) what it passes.  Claims are updated in place, so
//                     higher rays see what lower rays did; a ray that displaces a higher ray's claim records the position
//                     (atomicMin).  Round 1 walks every ray (contiguous index blocks per warp); afterwards a ray walks again
//                     only if it was displaced (resuming at that position) or the claim that stopped it became invalid
//                     (resuming there) -- otherwise its walk would give the same result.  One grid barrier per round.  A
//                     ray only depends on lower indices, so by induction the only state in which no ray has to walk is the
//                     serial result.  A last pass adds the counts.
// All fp64 arithmetic is written in the reference's operation order and the library is compiled with -fmad=false.
#include <cooperative_groups.h>
#include "fb_common.cuh"

namespace cg = cooperative_groups;

__device__ __forceinline__ double fb_norm3(double ax, double ay, double az, const double *b) {
  const double x = ax - b[0], y = ay - b[1], z = az - b[2];
  return sqrt((x * x + y * y) + z * z);                       // Eigen squaredNorm order, then sqrt
}

// ESDFMap::SetOccupancy(Vector3d,int) index part (ESDFMap.cpp:401-421): returns false when pos is outside the map.
// ref_idx = the reference's linear index (may alias when pos lies exactly on the map's upper face).
__device__ __forceinline__ bool fb_pos_to_vox(const FbGeom &g, double px, double py, double pz, int &vx, int &vy, int &vz) {
  if (px < g.min_range[0] || py < g.min_range[1] || pz < g.min_range[2]) return false;   // PosInMap, ESDFMap.cpp:46-61
  if (px > g.max_range[0] || py > g.max_range[1] || pz > g.max_range[2]) return false;
  vx = (int)floor((px - g.origin[0]) / g.res);                                            // Pos2Vox, ESDFMap.cpp:74-77
  vy = (int)floor((py - g.origin[1]) / g.res);
  vz = (int)floor((pz - g.origin[2]) / g.res);
  return true;
}

// Resolve the voxel a SetOccupancy call addresses.  Returns the list/stamp element: class + device index.
// The reference indexes set_free_/set_occ_ with the LINEAR index, which aliases for an out-of-grid coordinate; aliasing
// is reproduced while the linear index stays inside the array and treated as "not in map" beyond it.
__device__ __forceinline__ bool fb_resolve_vox(const FbGeom &g, int vx, int vy, int vz, long long &ii, bool &in_range) {
  in_range = fb_in_range(g, vx, vy, vz);
  if (fb_in_grid(g, vx, vy, vz)) { ii = fb_ii(g, vx, vy, vz); return true; }
  const long long ri = (long long)vx * g.gyz + (long long)vy * g.gz + vz;                 // Vox2Idx, ESDFMap.cpp:91
  if (ri < 0 || ri >= g.total) return false;
  const int ax = (int)(ri / g.gyz), ay = (int)(ri % g.gyz / g.gz), az = (int)(ri % g.gz); // Idx2Vox, ESDFMap.cpp:113-115
  ii = fb_ii(g, ax, ay, az);
  in_range = false;                                           // VoxInRange is evaluated on the coordinates, not the alias
  return true;
}

// Point -> world endpoint with the reference's gating (Fiesta.h:200-215).  Returns 0 = skipped, 1 = hit, 2 = clipped miss.
__device__ __forceinline__ int fb_endpoint(const FbRayArgs &a, long long i, double &px, double &py, double &pz) {
  const float fx = a.xyz[3 * i], fy = a.xyz[3 * i + 1], fz = a.xyz[3 * i + 2];
  if (isnan(fx) || isnan(fy) || isnan(fz)) return 0;
  const double x = (double)fx, y = (double)fy, z = (double)fz;
  double w[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) w[r] = ((a.T[4 * r] * x + a.T[4 * r + 1] * y) + a.T[4 * r + 2] * z) + a.T[4 * r + 3] * 1.0;
  px = w[0] / w[3]; py = w[1] / w[3]; pz = w[2] / w[3];
  const double len = fb_norm3(px, py, pz, a.org);
  if (len < a.min_len) return 0;
  if (len > a.max_len) {
    px = (px - a.org[0]) / len * a.max_len + a.org[0];
    py = (py - a.org[1]) / len * a.max_len + a.org[1];
    pz = (pz - a.org[2]) / len * a.max_len + a.org[2];
    return 2;
  }
  return 1;
}

// sub = 0 for the endpoint observation of point i, 1 + t for the free-space observation at back-walk position t: the serial
// reference makes them in exactly this order (Fiesta.h:213-215, then :239-276).
__device__ __forceinline__ void fb_count(const FbGeom &g, const FbRayArgs &a, long long ii, unsigned occ, unsigned long long i, unsigned sub) {
  FbTouch t = {a.cnt, a.touch_flag, a.touch_list, a.touch_epoch, a.ctr, a.tkey, a.key_hi};
  fb_touch(g, t, (unsigned)ii, occ, a.key_base + (i << 11) + sub);
}

// ---------------------------------------------------------------- endpoints
__global__ void k_ray_endpoints(FbGeom g, FbRayArgs a) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  double px, py, pz;
  const int kind = fb_endpoint(a, i, px, py, pz);
  int len = -1;                                               // -1: no ray (skipped point)
  if (kind) {
    len = 0;
    int vx, vy, vz;
    if (fb_pos_to_vox(g, px, py, pz, vx, vy, vz)) {
      long long ii; bool in_range;
      if (fb_resolve_vox(g, vx, vy, vz, ii, in_range)) {
        if (in_range) fb_count(g, a, ii, kind == 1 ? 1u : 0u, (unsigned long long)i, 0u);
        // set_occ_ ownership: lowest point index wins (Fiesta.h:227-230)
        atomicMax(&a.stamp[1][ii], (a.owner_tag << FB_RAY_BITS) | (FB_RAY_MASK - (unsigned)i));
      }
    }
  }
  a.ray_len[i] = len;
}

#define FB_RAY_CLEAN 0xffffffffu   // ray_dirty: no lower ray has displaced this one since its last walk

// ---------------------------------------------------------------- DDA
struct FbDda {
  int c[3], e[3], step[3];
  double tmax[3], tdelta[3], maxd;
};

__device__ __forceinline__ double fb_intbound(double s, double ds) {   // raycast.cpp:10-23
  if (ds < 0) { s = -s; ds = -ds; }
  s = fmod(fmod(s, 1.0) + 1.0, 1.0);
  return (1 - s) / ds;
}

__device__ __forceinline__ bool fb_dda_init(FbDda &d, const double *start, double ex, double ey, double ez) {
  const double end[3] = {ex, ey, ez};
  double dd[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) { d.c[k] = (int)floor(start[k]); d.e[k] = (int)floor(end[k]); dd[k] = end[k] - start[k]; }
  d.maxd = (dd[0] * dd[0] + dd[1] * dd[1]) + dd[2] * dd[2];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double delta = (double)(d.e[k] - d.c[k]);
    d.step[k] = (delta == 0.0) ? 0 : (delta < 0.0 ? -1 : 1);
    d.tmax[k] = fb_intbound(start[k], delta);
    d.tdelta[k] = ((double)d.step[k]) / delta;
  }
  return d.step[0] != 0 || d.step[1] != 0 || d.step[2] != 0;
}

// Walks the reference loop (raycast.cpp:116-157).  emit(x,y,z) is called for every voxel Raycast() would push.
// Returns the number of pushed voxels, or -1 (reference throws, > 1500 voxels) or -2 (reference never returns: it has
// overshot the end voxel and left the box for good -- see oracle/esdf_oracle.c for the same guard).
template <typename F>
__device__ __forceinline__ int fb_dda_walk(FbDda d, const FbRayArgs &a, F emit) {
  int n = 0;
  for (;;) {
    if (d.c[0] >= a.bmin[0] && d.c[0] < a.bmax[0] && d.c[1] >= a.bmin[1] && d.c[1] < a.bmax[1] && d.c[2] >= a.bmin[2] && d.c[2] < a.bmax[2]) {
      emit(d.c[0], d.c[1], d.c[2], n);
      ++n;
      const double x = d.c[0] - a.start[0], y = d.c[1] - a.start[1], z = d.c[2] - a.start[2];
      if ((x * x + y * y) + z * z > d.maxd) return n;
      if (n > 1500) return -1;
    }
    if (d.c[0] == d.e[0] && d.c[1] == d.e[1] && d.c[2] == d.e[2]) break;
    bool overshot = false, gone = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if ((d.step[k] > 0 && d.c[k] > d.e[k]) || (d.step[k] < 0 && d.c[k] < d.e[k]) || (d.step[k] == 0 && d.c[k] != d.e[k])) overshot = true;
      if ((d.step[k] >= 0 && !(d.c[k] < a.bmax[k])) || (d.step[k] <= 0 && !(d.c[k] >= a.bmin[k]))) gone = true;
    }
    if (overshot && gone) return -2;
    if (d.tmax[0] < d.tmax[1]) {
      if (d.tmax[0] < d.tmax[2]) { d.c[0] += d.step[0]; d.tmax[0] += d.tdelta[0]; } else { d.c[2] += d.step[2]; d.tmax[2] += d.tdelta[2]; }
    } else {
      if (d.tmax[1] < d.tmax[2]) { d.c[1] += d.step[1]; d.tmax[1] += d.tdelta[1]; } else { d.c[2] += d.step[2]; d.tmax[2] += d.tdelta[2]; }
    }
  }
  return n;
}

// One thread per point: ownership check (set_occ_ dedupe), then the DDA; every pushed voxel is classified and stored in
// the ray's row in forward order.  The walk back-to-front in k_ray_resolve reads row[L-1-t].
__global__ void k_ray_trace(FbGeom g, FbRayArgs a) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  if (a.ray_len[i] < 0) return;                               // point skipped by the gating in k_ray_endpoints
  double px, py, pz;
  fb_endpoint(a, i, px, py, pz);
  {
    int vx, vy, vz;
    if (fb_pos_to_vox(g, px, py, pz, vx, vy, vz)) {
      long long ii; bool in_range;
      if (fb_resolve_vox(g, vx, vy, vz, ii, in_range)) {
        const unsigned own = __ldcg(&a.stamp[1][ii]);
        if ((own & FB_RAY_MASK) != (FB_RAY_MASK - (unsigned)i)) { a.ray_len[i] = -1; return; }   // an earlier point owns this voxel
      }
    }
  }
  FbDda d;
  const bool moving = fb_dda_init(d, a.start, px / g.res, py / g.res, pz / g.res);
  uint32_t *row = a.ray_list + i * a.cap;
  int n = 0;
  if (moving)
    n = fb_dda_walk(d, a, [&](int x, int y, int z, int j) {
      if (j >= a.cap) return;
      const double cx = (x + 0.5) * g.res, cy = (y + 0.5) * g.res, cz = (z + 0.5) * g.res;   // Fiesta.h:240
      const double l = fb_norm3(cx, cy, cz, a.org);
      unsigned e;
      if (l < a.min_len) e = FB_CLS_STOP << 30;
      else if (l > a.max_len) e = FB_CLS_SKIP << 30;
      else if (a.lattice_ok) {                                // host-verified: map voxel = DDA voxel - offset, always in map
        const int vx = x - a.lattice_off[0], vy = y - a.lattice_off[1], vz = z - a.lattice_off[2];
        e = ((fb_in_range(g, vx, vy, vz) ? FB_CLS_COUNT : FB_CLS_STAMP) << 30) | (unsigned)fb_ii(g, vx, vy, vz);
      } else {
        int vx, vy, vz; long long ii; bool in_range;
        if (fb_pos_to_vox(g, cx, cy, cz, vx, vy, vz) && fb_resolve_vox(g, vx, vy, vz, ii, in_range))
          e = ((in_range ? FB_CLS_COUNT : FB_CLS_STAMP) << 30) | (unsigned)ii;
        else e = FB_CLS_SKIP << 30;                           // SetOccupancy returned -10000 (Fiesta.h:253)
      }
      row[j] = e;
    });
  atomicAdd(&a.ctr->rays_cast, 1u);
  if (n < 0) { atomicAdd(&a.ctr->rays_dropped, 1u); if (n == -1) atomicExch(&a.ctr->ray_error, 1u); n = 0; }
  int L = n > 0 ? n - 1 : 0;                                  // `for (i = output.size() - 2; ...)`: the last voxel is skipped
  if (L > a.cap) { L = 0; atomicExch(&a.ctr->ray_error, 2u); atomicAdd(&a.ctr->rays_dropped, 1u); }
  a.ray_len[i] = L;
  a.ray_reach[i] = L;                                         // optimistic: claims made while walking count as valid
  a.ray_dirty[i] = FB_RAY_CLEAN;
  if (L) atomicAdd(&a.ctr->ray_voxels, (unsigned long long)L);
}

// ---------------------------------------------------------------- stamp resolution + counting
// One warp per ray.  reach[i] = index at which the back-walk stops (L if it runs off the list) | FB_REACH_BLOCKED when it
// stopped at a voxel stamped by an earlier ray (that voxel is still counted, Fiesta.h:248-268).
#define FB_REACH_BLOCKED 0x40000000

// Is the voxel whose claim word is `seen` validly claimed by a ray with a lower index than `i`?
__device__ __forceinline__ bool fb_claim_blocks(const FbRayArgs &a, unsigned seen, unsigned i) {
  if ((seen >> FB_CLAIM_FRAME_SHIFT) != a.frame_tag) return false;                       // claim of an older frame
  const unsigned j = (seen >> FB_POS_BITS) & FB_RAY_MASK, tj = seen & FB_POS_MASK;
  return j < i && (int)tj < (__ldcg(&a.ray_reach[j]) & ~FB_REACH_BLOCKED);               // set_free_[idx] == tt by an EARLIER ray
}

// One warp walks ray i from the far end: stops at the first voxel validly claimed by a lower ray (or at the
// min_ray_length class), claims what it passes and marks every higher ray it displaces dirty.  Returns the new reach.
__device__ __forceinline__ int fb_walk_ray(const FbRayArgs &a, unsigned i, unsigned lane, int start) {
  uint32_t *claims = a.stamp[0];
  const unsigned fr = a.frame_tag << FB_CLAIM_FRAME_SHIFT;
  const int L = a.ray_len[i];
  const uint32_t *row = a.ray_list + (long long)i * a.cap;
  int result = L;
  // Everything before `start` is still claimed by this ray (a displacement there would have lowered `start`), so the walk
  // resumes at the 32-aligned chunk holding it.  Two-deep software pipeline: the list entries of chunk c+2 and the claim
  // words of chunk c+1 are in flight while chunk c is resolved (a stale claim word is caught by the CAS / the next check).
  int t0 = start & ~31;
  unsigned e = (FB_CLS_SKIP << 30), e1 = (FB_CLS_SKIP << 30), seen = 0;
  if (t0 + (int)lane < L) e = __ldcg(&row[L - 1 - (t0 + (int)lane)]);
  if (t0 + 32 + (int)lane < L) e1 = __ldcg(&row[L - 1 - (t0 + 32 + (int)lane)]);
  if ((e >> 30) == FB_CLS_COUNT || (e >> 30) == FB_CLS_STAMP) seen = __ldcg(&claims[e & FB_LIST_IDX_MASK]);
  for (; t0 < L; t0 += 32) {
    const int t = t0 + (int)lane;
    unsigned e2 = (FB_CLS_SKIP << 30), seen1 = 0;
    if (t + 64 < L) e2 = __ldcg(&row[L - 1 - (t + 64)]);
    if ((e1 >> 30) == FB_CLS_COUNT || (e1 >> 30) == FB_CLS_STAMP) seen1 = __ldcg(&claims[e1 & FB_LIST_IDX_MASK]);
    const unsigned cls = e >> 30, ii = e & FB_LIST_IDX_MASK;
    const bool normal = cls == FB_CLS_COUNT || cls == FB_CLS_STAMP;
    const unsigned mine = fr | (i << FB_POS_BITS) | (unsigned)t;
    int st = 0;                           // 0 = passable & already mine, 1 = passable & must be claimed, 2 = blocked
    if (normal && seen != mine) st = fb_claim_blocks(a, seen, i) ? 2 : 1;
    const unsigned m = __ballot_sync(0xffffffffu, st == 2 || cls == FB_CLS_STOP);
    const int first = m ? (__ffs(m) - 1) : 32;
    while (st == 1 && (int)lane < first) {                    // claim; a failed CAS means someone else wrote: look again
      const unsigned old = atomicCAS(&claims[ii], seen, mine);
      if (old == seen) {
        st = 0;
        if ((old >> FB_CLAIM_FRAME_SHIFT) == a.frame_tag) {   // displaced a (higher) ray: it has to walk again from there
          const unsigned k = (old >> FB_POS_BITS) & FB_RAY_MASK;
          if (k != i) { __threadfence(); atomicMin(&a.ray_dirty[k], old & FB_POS_MASK); }
        }
        break;
      }
      seen = old;
      if (seen == mine) { st = 0; break; }
      if (fb_claim_blocks(a, seen, i)) { st = 2; break; }
    }
    const unsigned m2 = __ballot_sync(0xffffffffu, st == 2 || cls == FB_CLS_STOP);
    if (m2) {
      const int f2 = __ffs(m2) - 1;
      const bool by_stamp = __shfl_sync(0xffffffffu, st == 2 ? 1 : 0, f2) != 0;
      result = (t0 + f2) | (by_stamp ? FB_REACH_BLOCKED : 0);
      break;
    }
    e = e1; e1 = e2; seen = seen1;
  }
  return result;
}

#define RR_THREADS 1024
#define RR_WARPS (RR_THREADS / 32)
__global__ void __launch_bounds__(RR_THREADS, 1) k_ray_resolve(FbGeom g, FbRayArgs a) {
  cg::grid_group grid = cg::this_grid();
  const unsigned lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
  const unsigned gw = blockIdx.x * RR_WARPS + wib, nwarps = gridDim.x * RR_WARPS;
  const unsigned gt = blockIdx.x * RR_THREADS + threadIdx.x;
  const uint32_t *claims = a.stamp[0];

  // Event-driven rounds, one grid barrier each.  Round 1 walks every ray.  In a later round each lane looks at one ray and
  // decides whether it has to walk again: a lower ray displaced it from a voxel (dirty position), or the claim that stopped
  // it is no longer valid; the warp then walks those rays from the position in question.  A ray whose claims are intact
  // and whose blocker is still valid would walk to exactly the same result, so skipping it is exact.  Checks run
  // concurrently with the walks of other warps and may see stale state -- but only walks change state, so the first round
  // without any walk has seen the final state everywhere, and that is where the loop ends.
  unsigned round = 0;
  for (;;) {
    ++round;
    unsigned long long t_a = 0;
    if (a.dbg && gt == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_a));
    unsigned *work_n = &a.ctr->ray_work[round % 3u];
    if (round == 1u) {
      // Contiguous index blocks per warp: neighbouring rays (which share most voxels) are resolved in serial order by one
      // warp, so far fewer optimistic claims have to be taken back in the later rounds.
      const long long per = (a.n + nwarps - 1) / nwarps;
      const long long hi = min((long long)(gw + 1) * per, a.n);
      unsigned walked = 0;
      for (long long i = (long long)gw * per; i < hi; ++i) {
        if (a.ray_len[i] <= 0) continue;
        const int result = fb_walk_ray(a, (unsigned)i, lane, 0);
        if (lane == 0) a.ray_reach[i] = result;
        ++walked;
      }
      if (lane == 0 && walked) atomicAdd(work_n, walked);
    } else {
      // ray of (warp, lane) = gw + lane * nwarps: the rays a lower ray displaces are its index neighbours, which land in
      // different warps and are walked concurrently
      for (long long base = 0; base < a.n; base += (long long)nwarps * 32) {
        const long long i = base + (long long)lane * nwarps + gw;
        bool need = false;
        int start = 0;
        if (i < a.n) {
          const int L = a.ray_len[i];
          if (L > 0) {
            unsigned dp = a.ray_dirty[i];                     // lowest position a lower ray displaced this one from
            if (dp != FB_RAY_CLEAN) dp = atomicExch(&a.ray_dirty[i], FB_RAY_CLEAN);   // (a concurrent mark must not get lost)
            const int rr = a.ray_reach[i], rpos = rr & ~FB_REACH_BLOCKED;
            if (dp < (unsigned)rpos) { need = true; start = (int)dp; }   // (a displaced claim beyond the reach was stale anyway)
            else if (rr & FB_REACH_BLOCKED) {
              const unsigned e = __ldcg(&a.ray_list[i * a.cap + (L - 1 - rpos)]);
              need = !fb_claim_blocks(a, __ldcg(&claims[e & FB_LIST_IDX_MASK]), (unsigned)i);
              start = rpos;
            }
          }
        }
        unsigned bal = __ballot_sync(0xffffffffu, need);
        if (lane == 0 && bal) atomicAdd(work_n, (unsigned)__popc(bal));
        while (bal) {
          const int src = __ffs(bal) - 1;
          bal &= bal - 1u;
          const unsigned wi = (unsigned)__shfl_sync(0xffffffffu, (int)i, src);
          const int ws = __shfl_sync(0xffffffffu, start, src);
          const int result = fb_walk_ray(a, wi, lane, ws);
          if (lane == 0) a.ray_reach[wi] = result;
        }
      }
    }
    grid.sync();
    const unsigned nw = __ldcg(work_n);
    if (blockIdx.x == 0 && threadIdx.x == 0) a.ctr->ray_work[(round + 2u) % 3u] = 0u;   // next used two barriers from now
    if (a.dbg && gt == 0 && round < 300u) {
      unsigned long long t_c; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_c));
      a.dbg[3 * round] = nw; a.dbg[3 * round + 1] = 0; a.dbg[3 * round + 2] = t_c - t_a;
    }
    if (nw == 0u || round >= a.max_rounds) break;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.ctr->ray_rounds = round;
    if (round >= a.max_rounds) a.ctr->ray_error = 3u;
  }
  unsigned long long t_d = 0;
  if (a.dbg && gt == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_d));
  // ---- counts: SetOccupancy(tmp, 0) for every visited voxel, including the one that stopped the walk (Fiesta.h:248-268)
  for (long long i = gw; i < a.n; i += nwarps) {
    const int L = a.ray_len[i];
    if (L <= 0) continue;
    const int rr = a.ray_reach[i];
    const int R = (rr & ~FB_REACH_BLOCKED) + ((rr & FB_REACH_BLOCKED) ? 1 : 0);
    const uint32_t *row = a.ray_list + (long long)i * a.cap;
    for (int t0 = 0; t0 < R; t0 += 128) {                     // four independent list loads in flight per lane
      unsigned e[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { const int t = t0 + 32 * u + (int)lane; e[u] = t < R ? __ldcg(&row[L - 1 - t]) : (FB_CLS_SKIP << 30); }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if ((e[u] >> 30) == FB_CLS_COUNT) fb_count(g, a, e[u] & FB_LIST_IDX_MASK, 0u, (unsigned long long)i, 1u + (unsigned)(t0 + 32 * u + (int)lane));
    }
  }
  if (a.dbg) {
    grid.sync();
    if (gt == 0) { unsigned long long t_e; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_e)); a.dbg[0] = t_e - t_d; }
  }
}

int fb_ray_resolve_blocks(int device) {
  int per_sm = 0, sms = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_ray_resolve, RR_THREADS, 0) != cudaSuccess) return 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  return per_sm * sms;
}

cudaError_t fb_ray_frame(const FbGeom &g, const FbRayArgs &a, int nblocks_resolve, cudaStream_t s, int *launches) {
  if (a.n <= 0) return cudaSuccess;
  const unsigned blocks = (unsigned)((a.n + 127) / 128);
  k_ray_endpoints<<<blocks, 128, 0, s>>>(g, a);
  k_ray_trace<<<blocks, 128, 0, s>>>(g, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  int nb = nblocks_resolve;
  if (nb < 1) nb = 1;
  void *args[] = {(void *)&g, (void *)&a};
  e = cudaLaunchCooperativeKernel((void *)k_ray_resolve, dim3(nb), dim3(RR_THREADS), args, 0, s);
  if (launches) *launches += 3;
  return e;
}
