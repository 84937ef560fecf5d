// fiesta_b200 -- incremental ESDF update kernels (replaces ESDFMap::UpdateESDF, FIESTA src/ESDFMap.cpp:273-398).
//
// E1 insert seeds   (ESDFMap.cpp:278-291)  k_seed_inserts : record := {0, self}, activate the tiles within reach.
// E2 delete         (ESDFMap.cpp:292-337)  k_delete_scan  : the per-obstacle doubly linked lists (ESDFMap.cpp:24-42) are
//                   gone; dependants of deleted obstacles are found by ONE streaming scan of the closest-obstacle array
//                   (128-bit loads) against the L2-resident Exist() bitmap, reset, and their tiles activated; the pull
//                   relaxation below re-seeds them from valid neighbours.
// E3 wavefront      (ESDFMap.cpp:338-392)  k_wavefront    : persistent cooperative kernel over a device work-list of
//                   active 8^3 tiles.  Each tile (+2-voxel halo, because dirs_ contains the +-2 axis steps,
//                   parameters.h:66-68; 4 in z to keep TMA's 16-byte start alignment) is staged into shared memory with ONE TMA box
//                   load (cp.async.bulk.tensor.3d;
//                   out-of-grid voxels are zero-filled = "never observed" = barrier), relaxed to a local fixpoint with the
//                   reference's 24-neighbourhood, strict-improvement rule and unknown-voxel barriers, written to a staging
//                   grid if it changed, and after a grid-wide barrier committed and its neighbours activated for the next
//                   generation.  Reads inside a generation only see the previous generation (Jacobi), so the result is
//                   deterministic and independent of the tile schedule.
// Frontier semantics: the reference only touches voxels a wave actually reaches -- an observed voxel whose distance is
// still +10000 stays so until a popped neighbour pushes to it (ESDFMap.cpp:375-391) or it is popped itself and pulls
// (:349-367).  Bit 31 of a record (FB_FRESH) marks "changed in the previous generation / local iteration" = "is in the
// update queue": a voxel takes candidates from FRESH neighbours (their push) and, when FRESH itself, from all neighbours
// (its own pull; skipped where it provably finds nothing, see `pulls` below).  Nothing else is relaxed, so unreached voxels
// stay unreached exactly like in the reference.
// Tie-break: the reference keeps the first arrival in FIFO order (ESDFMap.cpp:357,382); a parallel wave has no such
// order, so exact distance ties go to the smallest packed obstacle coordinate (x, then y, then z).
#include <cooperative_groups.h>
#include <stdio.h>
#include "fb_common.cuh"

namespace cg = cooperative_groups;

__device__ __forceinline__ unsigned ld_cg_u32(const unsigned *p) { return __ldcg(p); }

// Queue tile t for the generation identified by `stamp` (dedupe through tile_flag).
// `tyz` = tiles per x column; tiles outside this map's x-slab belong to another rank and are never queued here.
__device__ __forceinline__ void fb_activate(const FbEsdfArgs &a, unsigned t, unsigned stamp, int which, bool work = true, unsigned tyz = 0) {
  if (tyz) { const int txc = (int)(t / tyz); if (txc < a.tile_x_lo || txc >= a.tile_x_hi) return; }
  if (work) a.nb_flag[t] = stamp;
  if (atomicExch(&a.tile_flag[t], stamp) != stamp) {
    unsigned slot = atomicAdd(&a.ctr->n_list[which], 1u);
    a.list[which][slot] = t;
  }
}

// ---------------------------------------------------------------- E1
__global__ void k_seed_inserts(FbGeom g, FbEsdfArgs a, const uint32_t *ins, unsigned n) {
  unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned ii = ins[i];
  if (!(a.occ[ii] > a.l_occ)) return;                       // `if (Exist(idx))`, ESDFMap.cpp:282
  int z = ii % g.pz, y = (ii / g.pz) % g.gy, x = ii / (g.pz * g.gy);
  a.cobs[ii] = fb_pack(x, y, z) | FB_FRESH;                 // closest_obstacle_ = self, distance_ = 0, update_queue_.push
  const unsigned stamp = a.ctr->gen_stamp;
  int tx0 = max(x - 2, 0) >> 3, tx1 = min(x + 2, g.gx - 1) >> 3;
  int ty0 = max(y - 2, 0) >> 3, ty1 = min(y + 2, g.gy - 1) >> 3;
  int tz0 = max(z - 2, 0) >> 3, tz1 = min(z + 2, g.gz - 1) >> 3;
  for (int tx = tx0; tx <= tx1; ++tx)
    for (int ty = ty0; ty <= ty1; ++ty)
      for (int tz = tz0; tz <= tz1; ++tz) fb_activate(a, (unsigned)((tx * g.ty + ty) * g.tz + tz), stamp, 0, true, (unsigned)(g.ty * g.tz));
}

// ---------------------------------------------------------------- E2
// One thread handles 4 consecutive voxels (one 128-bit load).  ptotal is a multiple of 4 because pz is.
__global__ void k_delete_scan(FbGeom g, FbEsdfArgs a) {
  const long long nvec = g.ptotal >> 2;
  const unsigned stamp = a.ctr->gen_stamp;
  unsigned local_reset = 0;
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (long long)gridDim.x * blockDim.x) {
    uint4 q = reinterpret_cast<const uint4 *>(a.cobs)[v];
    uint32_t c[4] = {q.x, q.y, q.z, q.w};
    bool any = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if ((c[k] & FB_CODE_MASK) >= 2u) {
        int ox, oy, oz;
        fb_unpack(c[k], ox, oy, oz);
        long long oi = fb_ii(g, ox, oy, oz);
        if (!((__ldg(&a.occbits[oi >> 5]) >> (oi & 31)) & 1u)) { c[k] = FB_INF | FB_FRESH; any = true; ++local_reset; }  // !Exist(cobs)
      }
    }
    if (any) {
      reinterpret_cast<uint4 *>(a.cobs)[v] = make_uint4(c[0], c[1], c[2], c[3]);
      long long ii = v << 2;                                // the 4 voxels share (x, y) and lie in at most 1 tile (z % 4 == 0)
      int z = (int)(ii % g.pz), y = (int)((ii / g.pz) % g.gy), x = (int)(ii / ((long long)g.pz * g.gy));
      fb_activate(a, (unsigned)(((x >> 3) * g.ty + (y >> 3)) * g.tz + (z >> 3)), stamp, 0, true, (unsigned)(g.ty * g.tz));
    }
  }
  if (local_reset) atomicAdd(&a.ctr->voxels_reset, (unsigned long long)local_reset);
}

// ---------------------------------------------------------------- E3
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "FB_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra FB_DONE_%=;\n"
      "bra FB_WAIT_%=;\n"
      "FB_DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
// TMA: one 12x12x16 (x,y,z; z fastest) u32 box -> shared memory, completion signalled on `bar`.
// The innermost start coordinate must be a multiple of 4 elements (16 bytes) or the instruction faults.
__device__ __forceinline__ void tma_load_box(void *dst, const CUtensorMap *tmap, int cz, int cy, int cx, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
          smem_u32(dst)),
      "l"((unsigned long long)tmap), "r"(cz), "r"(cy), "r"(cx), "r"(smem_u32(bar))
      : "memory");
}

#define WF_THREADS 256     // a thread owns 2 voxels (x and x+4) of the tile; four CTAs = four independent tile pipelines per SM

#ifndef WF_GROUP
#define WF_GROUP 2          // lanes that share the evaluation of one listed voxel (1, 2, 4 or 8)
#endif
#ifndef WF_CTAS
#define WF_CTAS 4           // resident CTAs per SM the register budget is sized for
#endif
__global__ void __launch_bounds__(WF_THREADS, WF_CTAS)
k_wavefront(const __grid_constant__ CUtensorMap tmap, FbGeom g, FbEsdfArgs a) {
  // buf[0], buf[1]: TMA landing buffers (tile k in buf[k&1], tile k+1 prefetched into the other); a tile is relaxed in place
  __shared__ __align__(128) uint32_t buf[2][FB_BOX_WORDS];
  __shared__ __align__(8) uint64_t mbar[2];
  __shared__ int s_bbox[6];
  __shared__ unsigned s_next[6];            // {work index, tile id, 1 = needs a full visit, tile x, y, z} of the prefetched item
  __shared__ uint32_t s_inner[FB_BOX * FB_BOX];   // per z-row: bits that belong to the halo (all of them for a halo row)
  // per z-row bit masks of the FRESH flags (bit = box z index): a voxel finds out with 13 loads which of its 24 neighbours
  // are in the queue.  fm_halo keeps the (constant) halo bits, fm additionally the interior voxels changed last iteration.
  __shared__ uint32_t fm[FB_BOX * FB_BOX], fm_halo[FB_BOX * FB_BOX];
  // active list of one local iteration: voxel (lx<<6|ly<<3|lz), candidate mask (bit k = direction kd[k]), result
  __shared__ unsigned short listV[FB_TILE * FB_TILE * FB_TILE];
  __shared__ uint32_t listF[FB_TILE * FB_TILE * FB_TILE], res[FB_TILE * FB_TILE * FB_TILE];
  __shared__ unsigned s_cnt[2];
  __shared__ int s_koff[24];
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x;
  const int ly = (tid >> 3) & 7, lz = tid & 7;
  int lxh[2], sh[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    lxh[h] = (tid >> 6) + 4 * h;
    sh[h] = (lxh[h] + FB_HALO) * (FB_BOX * FB_BOXZ) + (ly + FB_HALO) * FB_BOXZ + (lz + FB_ZPAD);
  }
  // dirs_ (parameters.h:55-68) grouped by z-row so that the queue bits of all 24 neighbours come out of 13 mask words:
  // same row dz = -2,-1,+1,+2 | rows x-1, x+1, y-1, y+1 with dz = -1,0,+1 | the four xy diagonals | x-2, x+2, y-2, y+2
  constexpr int kd[24][3] = {{0, 0, -2}, {0, 0, -1}, {0, 0, 1}, {0, 0, 2},
                             {-1, 0, -1}, {-1, 0, 0}, {-1, 0, 1}, {1, 0, -1}, {1, 0, 0}, {1, 0, 1},
                             {0, -1, -1}, {0, -1, 0}, {0, -1, 1}, {0, 1, -1}, {0, 1, 0}, {0, 1, 1},
                             {-1, -1, 0}, {-1, 1, 0}, {1, -1, 0}, {1, 1, 0},
                             {-2, 0, 0}, {2, 0, 0}, {0, -2, 0}, {0, 2, 0}};
#pragma unroll
  for (int k = 0; k < 24; ++k)
    if (tid == k) s_koff[k] = kd[k][0] * (FB_BOX * FB_BOXZ) + kd[k][1] * FB_BOXZ + kd[k][2];

  if (tid < FB_BOX * FB_BOX) {
    const int rx = tid / FB_BOX, ry = tid % FB_BOX;
    const bool inner = rx >= FB_HALO && rx < FB_HALO + FB_TILE && ry >= FB_HALO && ry < FB_HALO + FB_TILE;
    s_inner[tid] = inner ? ~(0xffu << FB_ZPAD) : 0xffffffffu;
  }
  if (tid == 0) { mbar_init(&mbar[0], 1); mbar_init(&mbar[1], 1); }
  __syncthreads();
  unsigned parity[2] = {0u, 0u};
  unsigned cur = 0, gen = 0;
  unsigned long long my_visits = 0;
  const unsigned stamp0 = a.ctr->gen_stamp;   // stamp of generation 0 (seeded by k_seed_inserts / k_delete_scan)

  for (;;) {
    const unsigned nwork = ld_cg_u32(&a.ctr->n_list[cur]);
    if (nwork == 0) break;
    unsigned long long t_a = 0;
    if (a.dbg && blockIdx.x == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_a));
    const unsigned par = gen & 1u;
    if (blockIdx.x == 0 && tid == 0) {                        // counters of the other parity were last read two barriers ago
      a.ctr->n_changed[par ^ 1u] = 0; a.ctr->next_work[par ^ 1u] = 0; a.ctr->next_work[2u + (par ^ 1u)] = 0;
    }
    const unsigned stamp_cur = stamp0 + gen;

    // Fetch the next work item (dynamic distribution) and, if it needs a full visit, start its TMA load into buf[slot].
    auto fetch = [&](int slot) {
      const unsigned w = atomicAdd(&a.ctr->next_work[par], 1u);
      unsigned tile = 0, full = 0;
      int tzc = 0, tyc = 0, txc = 0;
      if (w < nwork) {
        tile = ld_cg_u32(&a.list[cur][w]);
        full = ld_cg_u32(&a.nb_flag[tile]) == stamp_cur ? 1u : 0u;
        tzc = tile % g.tz; tyc = (tile / g.tz) % g.ty; txc = tile / (g.tz * g.ty);
        if (full) {
          mbar_expect_tx(&mbar[slot], FB_BOX_WORDS * 4);
          tma_load_box(buf[slot], &tmap, tzc * FB_TILE - FB_ZPAD, tyc * FB_TILE - FB_HALO, txc * FB_TILE - FB_HALO, &mbar[slot]);
        }
      }
      s_next[0] = w; s_next[1] = tile; s_next[2] = full; s_next[3] = (unsigned)txc; s_next[4] = (unsigned)tyc; s_next[5] = (unsigned)tzc;
    };

    // ---------------- phase 1: relax every active tile against the previous generation
    int slot = 0;
    if (tid == 0) fetch(0);
    __syncthreads();
    for (;;) {
      const unsigned w = s_next[0], tile = s_next[1], full = s_next[2];
      const int txc = (int)s_next[3], tyc = (int)s_next[4], tzc = (int)s_next[5];   // (three divisions by run-time values, done once)
      __syncthreads();
      if (w >= nwork) break;
      if (tid == 0) {
        fetch(slot ^ 1);                                      // prefetch: overlaps the next tile's load with this tile's relaxation
        s_bbox[0] = s_bbox[2] = s_bbox[4] = 8; s_bbox[1] = s_bbox[3] = s_bbox[5] = -1;
        ++my_visits;
      }
      const int x0 = txc * FB_TILE, y0 = tyc * FB_TILE, z0 = tzc * FB_TILE;
      const int vy = y0 + ly, vz = z0 + lz;
      if (!full) {
        // Queued only by itself: nothing within reach changed since its local fixpoint, so its FRESH voxels would pull the
        // same values again.  Just retire the flags (through the staging grid, so that neighbours relaxing in this very
        // generation still see them).
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int vx = x0 + lxh[h];
          if (fb_in_grid(g, vx, vy, vz)) { const long long ii = fb_ii(g, vx, vy, vz); a.cobs_b[ii] = __ldcg(&a.cobs[ii]) & FB_CODE_MASK; }
        }
        if (tid == 0) {
          const unsigned sl = atomicAdd(&a.ctr->n_changed[par], 1u);
          a.changed[par][sl] = tile;
          a.changed_bbox[par][sl] = 0u;
        }
        __syncthreads();
        slot ^= 1;                                            // the prefetched item (if any) landed in the other buffer
        continue;
      }
      mbar_wait(&mbar[slot], parity[slot]);
      parity[slot] ^= 1u;
      uint32_t *V = buf[slot];
      // FRESH mask of every z-row of the box: a warp reads 32 consecutive words (two rows, conflict free) and votes
      for (int w0 = (tid >> 5) * 32; w0 < FB_BOX_WORDS; w0 += WF_THREADS) {
        const uint32_t bal = __ballot_sync(0xffffffffu, (V[w0 + (tid & 31)] >> 31) != 0u);
        if ((tid & 31) < 2) {
          const int row = (w0 >> 4) + (tid & 31);
          const uint32_t mk = (bal >> (16 * (tid & 31))) & 0xffffu;
          fm[row] = mk;
          fm_halo[row] = mk & s_inner[row];
        }
      }
      if (tid == 0) { s_cnt[0] = 0; s_cnt[1] = 0; }
      uint32_t orig[2], mine[2], nmask[2];
      bool updatable[2], pulls[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int vx = x0 + lxh[h];
        orig[h] = V[sh[h]];
        // A voxel relaxes iff it has been observed (unknown voxels are barriers: distance_ = -10000 is never > tmp,
        // ESDFMap.cpp:382) and lies inside the update box (only in-box voxels are ever queued, ESDFMap.cpp:351,378).
        updatable[h] = (orig[h] & FB_CODE_MASK) != FB_UNKNOWN && fb_in_range(g, vx, vy, vz);
        // While every relaxation of this map has covered the whole grid, every value a neighbour holds was offered to this
        // voxel when it was set (the neighbour was in the queue then) and records only improve -- so the pull of a queued
        // voxel (ESDFMap.cpp:349-367) can only find something new if its own record was (re)set to "no obstacle": first
        // observation, local-map reset or a deleted obstacle.  Once a relaxation ran under a smaller box, VoxInRange(new_pos)
        // (:351) withheld pushes to the voxels outside it, so that does not hold any more and every queued voxel pulls
        // (a.pull_all, sticky per map).
        pulls[h] = a.pull_all || (orig[h] & FB_CODE_MASK) == FB_INF;
        nmask[h] = 0xffffffu;
        if (!g.box_is_full) {                                 // VoxInRange(new_pos), ESDFMap.cpp:351
          nmask[h] = 0;
#pragma unroll
          for (int k = 0; k < 24; ++k)
            if (fb_in_range(g, vx + kd[k][0], vy + kd[k][1], vz + kd[k][2])) nmask[h] |= 1u << k;
        }
      }
      __syncthreads();
      // Local Jacobi iterations.  (A) every thread derives, for its two voxels, the set of neighbours whose value it has to
      // look at -- the ones in the queue (their push, ESDFMap.cpp:375-391) or all of them when the voxel itself pulls --
      // and lists the voxel if that set is not empty; (B) the listed voxels are evaluated by WF_GROUP lanes each (every
      // lane its share of the directions, only the set bits), which turns the sparse, clustered activity of a wave front into dense work for
      // all warps; (C) the improvements are applied and become the queue of the next iteration.
      for (int it = 0;; ++it) {
        const int par2 = it & 1;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t F = 0;
          if (updatable[h]) {
            const int r = (lxh[h] + FB_HALO) * FB_BOX + (ly + FB_HALO), zb = lz + FB_ZPAD;
            const uint32_t m0 = fm[r];
            F = ((m0 >> (zb - 2)) & 3u) | (((m0 >> (zb + 1)) & 3u) << 2) |
                (((fm[r - FB_BOX] >> (zb - 1)) & 7u) << 4) | (((fm[r + FB_BOX] >> (zb - 1)) & 7u) << 7) |
                (((fm[r - 1] >> (zb - 1)) & 7u) << 10) | (((fm[r + 1] >> (zb - 1)) & 7u) << 13) |
                (((fm[r - FB_BOX - 1] >> zb) & 1u) << 16) | (((fm[r - FB_BOX + 1] >> zb) & 1u) << 17) |
                (((fm[r + FB_BOX - 1] >> zb) & 1u) << 18) | (((fm[r + FB_BOX + 1] >> zb) & 1u) << 19) |
                (((fm[r - 2 * FB_BOX] >> zb) & 1u) << 20) | (((fm[r + 2 * FB_BOX] >> zb) & 1u) << 21) |
                (((fm[r - 2] >> zb) & 1u) << 22) | (((fm[r + 2] >> zb) & 1u) << 23);
            if (pulls[h] && ((m0 >> zb) & 1u)) F = 0xffffffu;
            F &= nmask[h];
          }
          const uint32_t bal = __ballot_sync(0xffffffffu, F != 0u);
          if (bal) {
            const int lane = tid & 31;
            unsigned base = 0;
            if (lane == 0) base = atomicAdd(&s_cnt[par2], (unsigned)__popc(bal));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (F) {
              const unsigned pos = base + (unsigned)__popc(bal & ((1u << lane) - 1u));
              listV[pos] = (unsigned short)((lxh[h] << 6) | (ly << 3) | lz);
              listF[pos] = F;
            }
          }
        }
        __syncthreads();
        const int n = (int)s_cnt[par2];
        if (n == 0) break;
        if (tid < FB_BOX * FB_BOX) fm[tid] = fm_halo[tid];
        if (tid == 0) s_cnt[par2 ^ 1] = 0;
        int anych = 0;
        {
          constexpr int GE = 32 / WF_GROUP;                   // listed voxels per warp pass
          constexpr uint32_t slice0 = WF_GROUP == 1 ? 0xffffffu : WF_GROUP == 2 ? 0x555555u : WF_GROUP == 4 ? 0x111111u : 0x010101u;
          const int lane = tid & 31, sub = lane % WF_GROUP;
          for (int e0 = (tid >> 5) * GE; e0 < n; e0 += (WF_THREADS / 32) * GE) {
            const int e = e0 + lane / WF_GROUP;
            const bool valid = e < n;
            uint32_t self = 0, best = 0, m = 0;
            unsigned bestd = 0xffffffffu;
            int sidx = 0, vx = 0, wy = 0, wz = 0;
            if (valid) {
              const int v = listV[e];
              const int lx = v >> 6, ly2 = (v >> 3) & 7, lz2 = v & 7;
              sidx = (lx + FB_HALO) * (FB_BOX * FB_BOXZ) + (ly2 + FB_HALO) * FB_BOXZ + (lz2 + FB_ZPAD);
              vx = x0 + lx; wy = y0 + ly2; wz = z0 + lz2;
              self = V[sidx] & FB_CODE_MASK;
              best = self;
              if (best >= 2u) { int ox, oy, oz; fb_unpack(best, ox, oy, oz); ox -= vx; oy -= wy; oz -= wz; bestd = (unsigned)(ox * ox + oy * oy + oz * oz); }
              m = listF[e] & (slice0 << sub);
            }
            while (m) {
              const int k = __ffs(m) - 1;
              m &= m - 1u;
              const uint32_t c = V[sidx + s_koff[k]] & FB_CODE_MASK;
              if (c >= 2u && c != best) {                     // the neighbour has a closest obstacle (ESDFMap.cpp:353)
                int ox, oy, oz; fb_unpack(c, ox, oy, oz); ox -= vx; oy -= wy; oz -= wz;
                const unsigned d = (unsigned)(ox * ox + oy * oy + oz * oz);
                if (d < bestd || (d == bestd && c < best)) { bestd = d; best = c; }   // strict improvement; ties -> smallest coordinate
              }
            }
#pragma unroll
            for (int off = 1; off < WF_GROUP; off <<= 1) {
              const unsigned od = __shfl_xor_sync(0xffffffffu, bestd, off);
              const uint32_t oc = __shfl_xor_sync(0xffffffffu, best, off);
              if (od < bestd || (od == bestd && oc < best)) { bestd = od; best = oc; }
            }
            if (valid && sub == 0) {
              const bool ch = best != self;
              res[e] = ch ? best : 0u;
              anych |= ch ? 1 : 0;
            }
          }
        }
        const int any = __syncthreads_or(anych);
        if (!any) break;
        for (int e = tid; e < n; e += WF_THREADS) {
          const uint32_t rr = res[e];
          if (rr) {
            const int v = listV[e];
            const int lx = v >> 6, ly2 = (v >> 3) & 7, lz2 = v & 7;
            V[(lx + FB_HALO) * (FB_BOX * FB_BOXZ) + (ly2 + FB_HALO) * FB_BOXZ + (lz2 + FB_ZPAD)] = rr;
            atomicOr(&fm[(lx + FB_HALO) * FB_BOX + (ly2 + FB_HALO)], 1u << (lz2 + FB_ZPAD));
          }
        }
        __syncthreads();
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) mine[h] = V[sh[h]] & FB_CODE_MASK;
      int nch = 0;
      bool diff = false;
      uint32_t outw[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const bool changed = mine[h] != (orig[h] & FB_CODE_MASK);   // changed during this generation -> FRESH for the next one
        outw[h] = mine[h] | (changed ? FB_FRESH : 0u);
        if (changed) {
          ++nch;
          atomicMin(&s_bbox[0], lxh[h]); atomicMax(&s_bbox[1], lxh[h]);
          atomicMin(&s_bbox[2], ly); atomicMax(&s_bbox[3], ly);
          atomicMin(&s_bbox[4], lz); atomicMax(&s_bbox[5], lz);
        }
        diff = diff || outw[h] != orig[h];
      }
      const int nchanged = __syncthreads_count(nch > 0) ;      // threads with a change (exact voxel count accumulated below)
      const int dirty = __syncthreads_or(diff);               // also true when only stale FRESH flags must be retired
      if (dirty) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int vx = x0 + lxh[h];
          if (fb_in_grid(g, vx, vy, vz)) a.cobs_b[fb_ii(g, vx, vy, vz)] = outw[h];   // stage the whole tile interior
        }
      }
      {
        const unsigned c2 = __reduce_add_sync(0xffffffffu, (unsigned)nch);     // exact number of changed voxels, per warp
        if ((tid & 31) == 0 && c2) atomicAdd(&a.ctr->voxels_changed, (unsigned long long)c2);
      }
      if (tid == 0 && dirty) {
        const unsigned sl = atomicAdd(&a.ctr->n_changed[par], 1u);
        a.changed[par][sl] = tile;
        a.changed_bbox[par][sl] = nchanged ? ((unsigned)s_bbox[0] | ((unsigned)s_bbox[1] << 3) | ((unsigned)s_bbox[2] << 6) |
                                              ((unsigned)s_bbox[3] << 9) | ((unsigned)s_bbox[4] << 12) | ((unsigned)s_bbox[5] << 15) | (1u << 18))
                                           : 0u;
      }
      // generic-proxy accesses to buf[slot] must be ordered before the async-proxy (TMA) write of a later prefetch into it
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      slot ^= 1;
    }
    grid.sync();

    unsigned long long t_b = 0;
    if (a.dbg && blockIdx.x == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_b));
    // ---------------- phase 2: commit changed tiles, activate their neighbours for the next generation
    if (blockIdx.x == 0 && tid == 0) a.ctr->n_list[cur] = 0;    // consumed; becomes the append target two phases from now
    const unsigned nchg = ld_cg_u32(&a.ctr->n_changed[par]);
    const unsigned stamp = stamp0 + gen + 1u;
    // (uniform items -- one 8^3 copy + <= 19 activations -- so a static stride needs no counter and no block barrier, and the
    // warps of a CTA run ahead of each other through the dependent loads)
    for (unsigned w = blockIdx.x; w < nchg; w += gridDim.x) {
      const unsigned tile = ld_cg_u32(&a.changed[par][w]);
      const unsigned bb = ld_cg_u32(&a.changed_bbox[par][w]);
      const int tzc = tile % g.tz, tyc = (tile / g.tz) % g.ty, txc = tile / (g.tz * g.ty);
      const int vy = tyc * FB_TILE + ly, vz = tzc * FB_TILE + lz;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int vx = txc * FB_TILE + lxh[h];
        if (fb_in_grid(g, vx, vy, vz)) {
          const long long ii = fb_ii(g, vx, vy, vz);
          a.cobs[ii] = __ldcg(&a.cobs_b[ii]);
        }
      }
      if (tid < 27 && (bb >> 18)) {                            // some record changed: its new value must reach the neighbours
        const int ox = tid / 9 - 1, oy = (tid / 3) % 3 - 1, oz = tid % 3 - 1;
        const int nz = (ox != 0) + (oy != 0) + (oz != 0);
        if (nz == 0) fb_activate(a, tile, stamp, (int)(cur ^ 1u), false);   // revisit once more, only to retire the FRESH flags
        if (nz == 1 || nz == 2) {                              // no 3-D corner directions in dirs_
          const int mnx = bb & 7, mxx = (bb >> 3) & 7, mny = (bb >> 6) & 7, mxy = (bb >> 9) & 7, mnz = (bb >> 12) & 7, mxz = (bb >> 15) & 7;
          bool need = true;
          if (ox < 0) need = need && (mnx < 2); if (ox > 0) need = need && (mxx > 5);
          if (oy < 0) need = need && (mny < 2); if (oy > 0) need = need && (mxy > 5);
          if (oz < 0) need = need && (mnz < 2); if (oz > 0) need = need && (mxz > 5);
          const int nx = txc + ox, ny = tyc + oy, nzc = tzc + oz;
          if (need && nx >= 0 && nx < g.tx && ny >= 0 && ny < g.ty && nzc >= 0 && nzc < g.tz)
            fb_activate(a, (unsigned)((nx * g.ty + ny) * g.tz + nzc), stamp, (int)(cur ^ 1u), true, (unsigned)(g.ty * g.tz));
        }
      }
    }
    grid.sync();
    if (a.dbg && blockIdx.x == 0 && tid == 0 && gen < 256u) {
      unsigned long long t_c; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_c));
      a.dbg[4 * gen] = nwork; a.dbg[4 * gen + 1] = nchg; a.dbg[4 * gen + 2] = t_b - t_a; a.dbg[4 * gen + 3] = t_c - t_b;
    }
    cur ^= 1u;
    ++gen;
  }
  if (tid == 0) {
    if (my_visits) atomicAdd(&a.ctr->tile_visits, my_visits);
    if (blockIdx.x == 0) { a.ctr->generations = gen; a.ctr->gen_stamp = stamp0 + gen + 1u; }
  }
}

// ---------------------------------------------------------------- x-slab sharding: ghost layers
// Received ghost layers (2 x-layers below and above the slab, as sent by the neighbouring ranks) are compared with the local
// copy; a voxel whose record differs is overwritten, marked FRESH (it pushes into this slab in the next generation) and the
// own tiles within reach are queued.
__global__ void k_halo_ingest(FbGeom g, FbEsdfArgs a, const uint32_t *recv, int x_first, int nlayers, int own_tile_x, unsigned *nchanged) {
  const long long per = (long long)g.gy * g.pz;
  const unsigned stamp = a.ctr->gen_stamp;
  unsigned local = 0;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < per * nlayers; k += (long long)gridDim.x * blockDim.x) {
    const int x = x_first + (int)(k / per);
    const long long r = k % per;
    const int y = (int)(r / g.pz), z = (int)(r % g.pz);
    if (z >= g.gz) continue;
    const long long ii = fb_ii(g, x, y, z);
    const uint32_t nw = recv[k] & FB_CODE_MASK, old = a.cobs[ii] & FB_CODE_MASK;
    if (nw != old) {
      a.cobs[ii] = nw | FB_FRESH;
      ++local;
      const int ty0 = max(y - 2, 0) >> 3, ty1 = min(y + 2, g.gy - 1) >> 3, tz0 = max(z - 2, 0) >> 3, tz1 = min(z + 2, g.gz - 1) >> 3;
      for (int ty = ty0; ty <= ty1; ++ty)
        for (int tz = tz0; tz <= tz1; ++tz) fb_activate(a, (unsigned)((own_tile_x * g.ty + ty) * g.tz + tz), stamp, 0, true, (unsigned)(g.ty * g.tz));
    }
  }
  if (local) atomicAdd(nchanged, local);
}
__global__ void k_halo_retire(FbGeom g, uint32_t *cobs, int x_first, int nlayers) {
  const long long per = (long long)g.gy * g.pz;
  uint32_t *p = cobs + (long long)x_first * per;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < per * nlayers; k += (long long)gridDim.x * blockDim.x) p[k] &= FB_CODE_MASK;
}
cudaError_t fb_esdf_halo_ingest(const FbGeom &g, const FbEsdfArgs &a, const uint32_t *recv, int x_first, int nlayers, int own_tile_x, unsigned *d_nchanged, cudaStream_t s) {
  if (nlayers <= 0) return cudaSuccess;
  k_halo_ingest<<<FB_SMS * 4, 256, 0, s>>>(g, a, recv, x_first, nlayers, own_tile_x, d_nchanged);
  return cudaGetLastError();
}
cudaError_t fb_esdf_halo_retire(const FbGeom &g, uint32_t *cobs, int x_first, int nlayers, cudaStream_t s) {
  if (nlayers <= 0) return cudaSuccess;
  k_halo_retire<<<FB_SMS * 4, 256, 0, s>>>(g, cobs, x_first, nlayers);
  return cudaGetLastError();
}

// ---------------------------------------------------------------- host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

cudaError_t fb_esdf_make_tensor_map(CUtensorMap *out, const FbGeom &g, uint32_t *cobs, char *err, int errlen) {
  void *fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || fn == nullptr) { snprintf(err, errlen, "cuTensorMapEncodeTiled entry point unavailable"); return e != cudaSuccess ? e : cudaErrorUnknown; }
  cuuint64_t dims[3] = {(cuuint64_t)g.gz, (cuuint64_t)g.gy, (cuuint64_t)g.gx};
  cuuint64_t strides[2] = {(cuuint64_t)g.pz * 4ull, (cuuint64_t)g.pz * (cuuint64_t)g.gy * 4ull};
  cuuint32_t box[3] = {FB_BOXZ, FB_BOX, FB_BOX};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = ((PFN_encodeTiled)fn)(out, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, cobs, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return cudaErrorInvalidValue; }
  return cudaSuccess;
}

cudaError_t fb_esdf_seed_inserts(const FbGeom &g, const FbEsdfArgs &a, const uint32_t *ins, unsigned n, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  k_seed_inserts<<<(n + 255) / 256, 256, 0, s>>>(g, a, ins, n);
  return cudaGetLastError();
}

cudaError_t fb_esdf_delete_scan(const FbGeom &g, const FbEsdfArgs &a, cudaStream_t s) {
  long long nvec = g.ptotal >> 2;
  long long blocks = (nvec + 255) / 256;
  if (blocks > FB_SMS * 16) blocks = FB_SMS * 16;                   // grid-stride, a multiple of the SM count
  k_delete_scan<<<(unsigned)blocks, 256, 0, s>>>(g, a);
  return cudaGetLastError();
}

int fb_esdf_wavefront_blocks(int device) {
  int per_sm = 0, sms = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_wavefront, WF_THREADS, 0) != cudaSuccess) return 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  return per_sm * sms;                                        // every block co-resident: required by grid.sync()
}

cudaError_t fb_esdf_wavefront(const FbGeom &g, const FbEsdfArgs &a, const CUtensorMap &tmap, int nblocks, cudaStream_t s) {
  void *args[] = {(void *)&tmap, (void *)&g, (void *)&a};
  return cudaLaunchCooperativeKernel((void *)k_wavefront, dim3(nblocks), dim3(WF_THREADS), args, 0, s);
}
