// fiesta_b200 -- ORDER-EXACT mode, E2 (second half) + E3: the re-seeding of the delete loop and the FIFO relaxation loop of
// UpdateESDF (FIESTA src/ESDFMap.cpp:301-334, 338-392) as ONE persistent kernel, k_x_relax: every FIFO generation,
// every round of its behaviour fixpoint and the ordered hand-over to the next generation run on the device, separated by
// grid barriers; the host launches it once per UpdateESDF and reads one control block back.
// (CPU model of exactly this formulation, checked against the sequential reference: oracle/exact_model.c.)
//
//  * A FIFO generation is one list E of voxels in queue order.  Element i, direction k acts at the timestamp 32*i + k
//    (its pull at 32*i + 24).  MB[v] is the packed word {queue position, behaviour, code} of the live entry at voxel v.
//  * state(v, T): what voxel v holds at time T = the snapshot, or the lexicographic minimum (distance, timestamp) over the
//    offers with timestamp < T of the <= 25 elements that can write v which beat the snapshot -- exactly what a sequence
//    of strict `>` tests in timestamp order leaves behind (x_gather / x_state_nb).  BIG generations cache, per target voxel,
//    a summary {first improving timestamp, best timestamp, best code, snapshot code}, computed once per pass by whoever
//    stamps the target first (x_claim_summaries); a query gathers only if first < T <= best.
//  * An element's behaviour (stale / pulled code / pushes code, :345-373) depends only on states at its own pop time, i.e.
//    on the words at the 129 offsets a+b (a,b in {0} u dirs_) around it.  Round 1 evaluates every element against the guess
//    "everybody pushes its snapshot code"; a flip lists every LATER element it can touch for the next round (all 129 offsets
//    if pushing is involved, else only the 24 neighbours: just the offer to its own voxel changed).  SMALL generations
//    evaluate from a per-warp shared-memory stage filled by one round of loads (x_stage); the later rounds of BIG
//    generations first refresh the summaries of last round's flips' targets, then evaluate through them.  Element i is right once all
//    earlier ones are, so the fixpoint -- reached by a round without flips, which has only read final words -- is the
//    sequential execution.  In BIG generations, once a list is short, the rest of the fixpoint runs without rounds from a
//    work queue (x_async), followed by one summary refresh.
//  * Hand-over: element i owns slot k iff the final state of its k-th target carries the timestamp 32*i + k; the owned slots in
//    timestamp order (per-element masks, exclusive scan over CTA-contiguous ranges) are the next generation; old words are
//    retired by compare-and-swap (a generation-parity bit tells old from new).
//  * Before it, k_x_reseed re-seeds the dependants of the deleted obstacles (:308-321) in four stages (see there) and appends
//    the re-seeded ones, in list-walk order, to the insert seeds in E[0]; k_x_relax reads generation 0's length from
//    ctl->nE0.
#include <stdio.h>
#include "fb_common.cuh"
#include "fb_exact.h"
#include "fb_divmagic.h"

#define XT 1024                       // threads per CTA, one CTA per SM
#define XW (XT / 32)
#define XNONE 0xffffffffu
#define X_DEAD 0ull
#define X_PULL 1ull
#define X_PUSH 2ull
#define XMB_NONE 0xffffffffffffffffull
#define X_NOFF 129
#define X_MAX_ROUNDS 4000000u
#define XGB 8                         // writer words loaded per batch by a gather (24 / XGB batches)
// trace layout (FIESTA_DEBUG_X): fb_exact.h.  Phase categories 14 and 15 hold summed work / flip list lengths, and the
// dependants final after the classification / summed closure list lengths, instead of times.
#define XDBG_PHASE FB_XDBG_PHASE
#define XDBG_ROUNDS FB_XDBG_ROUNDS
#define XDBG_WMAX FB_XDBG_WMAX

static __constant__ int x_dirs[24][3] = {
    {-1, 0, 0}, {1, 0, 0}, {0, -1, 0}, {0, 1, 0}, {0, 0, -1}, {0, 0, 1},
    {-1, -1, 0}, {1, 1, 0}, {0, -1, -1}, {0, 1, 1}, {-1, 0, -1}, {1, 0, 1},
    {-1, 1, 0}, {1, -1, 0}, {0, -1, 1}, {0, 1, -1}, {1, 0, -1}, {-1, 0, 1},
    {-2, 0, 0}, {2, 0, 0}, {0, -2, 0}, {0, 2, 0}, {0, 0, -2}, {0, 0, 2}};
static __constant__ int x_off_c[X_NOFF];     // the distinct sums a+b, packed (dx+4) | (dy+4)<<4 | (dz+4)<<8 (filled by fb_xrelax_init)

// Index arithmetic was a third of this kernel's instruction stream (ncu source view): 64-bit linear
// indices, six-compare box tests and divisions by the run-time pitch.  The forms below are exact for every grid the library
// accepts (< 2^30 voxels): 32-bit indices, unsigned grid tests, multiply-high divisions with host-made constants.
__device__ __forceinline__ unsigned x_vi(const FbGeom &g, int x, int y, int z) { return (unsigned)((x * g.gy + y) * g.pz + z); }
__device__ __forceinline__ bool x_in_grid(const FbGeom &g, int x, int y, int z) {
  return (unsigned)x < (unsigned)g.gx && (unsigned)y < (unsigned)g.gy && (unsigned)z < (unsigned)g.gz;
}
// VoxInRange (ESDFMap.cpp:63-72); fb_xrelax_launch makes min_vec / max_vec of the kernel's copy an unreachable box when the
// update box is empty.  Compared with the bounds as they are, which stay kernel parameters: the extents max - min of an
// unsigned test are loop-invariant values that the compiler keeps in registers, and at k_x_relax's 64-register limit they
// spill inside the per-element loops.
__device__ __forceinline__ bool x_in_range(const FbGeom &g, int x, int y, int z) {
  return x >= g.min_vec[0] && x <= g.max_vec[0] && y >= g.min_vec[1] && y <= g.max_vec[1] && z >= g.min_vec[2] && z <= g.max_vec[2];
}
// dirs_[j][k] for a compile-time j (unrolled loops): folded into immediates, unlike a read of the constant-memory table
__device__ __forceinline__ int x_dc(int j, int k) {
  const int D[24][3] = {{-1, 0, 0}, {1, 0, 0}, {0, -1, 0}, {0, 1, 0}, {0, 0, -1}, {0, 0, 1}, {-1, -1, 0}, {1, 1, 0}, {0, -1, -1}, {0, 1, 1}, {-1, 0, -1}, {1, 0, 1},
                        {-1, 1, 0}, {1, -1, 0}, {0, -1, 1}, {0, 1, -1}, {1, 0, -1}, {-1, 0, 1}, {-2, 0, 0}, {2, 0, 0}, {0, -2, 0}, {0, 2, 0}, {0, 0, -2}, {0, 0, 2}};
  return D[j][k];
}
// word of the j-th writer of the in-grid voxel v = (x,y,z), i.e. of the entry at (x,y,z) - dirs_[j]: only the components the
// direction moves need a bounds test, and the linear index is v minus a per-direction constant
__device__ __forceinline__ unsigned long long x_writer_word(const FbGeom &g, const unsigned long long *MB, unsigned v, int x, int y, int z, int j, bool inr) {
  const int dx = x_dc(j, 0), dy = x_dc(j, 1), dz = x_dc(j, 2);
  const bool ok = inr && (dx == 0 || (unsigned)(x - dx) < (unsigned)g.gx) && (dy == 0 || (unsigned)(y - dy) < (unsigned)g.gy) &&
                  (dz == 0 || (unsigned)(z - dz) < (unsigned)g.gz);
  return ok ? __ldcg(&MB[v - (unsigned)((dx * g.gy + dy) * g.pz + dz)]) : XMB_NONE;
}

struct XShared {
  int off[X_NOFF];                    // copy of x_off_c (lane-varying index: shared memory, not the constant cache)
  int dir[32];                        // dirs_ packed the same way; entry 24 = (0,0,0)
  unsigned char slot[25 * 24];        // index in off[] of (target t) - dirs_[k]: where the k-th writer of an element's target t sits
  unsigned char self[32];             // index in off[] of target t itself (entry 24 = 0)
  unsigned red[XW], red2[XW];
  unsigned base, total;
  // thread 0's alone: the grid barrier's arrival target and k_x_relax's totals.  They stay live across the whole generation
  // loop, which runs at the 64-register limit, so they are kept here rather than in registers that would spill.
  unsigned bar_target;
  unsigned generations, rounds, dense_rounds;
  unsigned long long changed;
  unsigned qdone;                     // the work queue of the current asynchronous phase is done (copy of ctl->qdone)
};

__device__ __forceinline__ unsigned x_d2(int x, int y, int z, uint32_t c) {
  int ox, oy, oz; fb_unpack(c, ox, oy, oz); ox -= x; oy -= y; oz -= z;
  return (unsigned)(ox * ox + oy * oy + oz * oz);
}
__device__ __forceinline__ unsigned x_dist_of(int x, int y, int z, uint32_t c) { return c < 2u ? 0xffffffffu : x_d2(x, y, z, c); }
// packed word: {generation parity:1 | unused:3 | queue position:27 | behaviour:2 | code:31}; all ones = no live entry here
__device__ __forceinline__ unsigned long long x_mb(unsigned par, unsigned i, unsigned long long kind, uint32_t code) {
  return ((unsigned long long)(par & 1u) << 63) | ((unsigned long long)i << 33) | (kind << 31) | (unsigned long long)(code & FB_CODE_MASK);
}
__device__ __forceinline__ unsigned x_mb_idx(unsigned long long w) { return (unsigned)(w >> 33) & 0x7ffffffu; }
__device__ __forceinline__ unsigned x_mb_par(unsigned long long w) { return (unsigned)(w >> 63); }
__device__ __forceinline__ unsigned long long x_mb_kind(unsigned long long w) { return (w >> 31) & 3ull; }
__device__ __forceinline__ uint32_t x_mb_code(unsigned long long w) { return (uint32_t)(w & FB_CODE_MASK); }

struct XState { unsigned d; uint32_t c; unsigned ts; };
// Per-warp stage of one element's neighbourhood: the words at the 129 offsets and the records of its 25 targets.
struct XNb { unsigned long long w[X_NOFF + 3]; uint32_t c[28]; };

// Everything the kernel reads is written by other SMs between barriers: all loads bypass L1 (ld.global.cg).
// State of voxel (x,y,z) as seen at time T (exclusive); *first = earliest timestamp of an offer that beats the snapshot.
template <bool WANT_FIRST>
__device__ __forceinline__ XState x_gather(const FbGeom &g, const uint32_t *cobs, const unsigned long long *MB, int x, int y, int z, unsigned T,
                                           unsigned &first, uint32_t &snap) {
  XState s;
  const unsigned v = x_vi(g, x, y, z);
  // All loads are issued before anything is decided (the round trip to L2 is what a query costs): the snapshot, the own
  // word and the first half of the writers' words together, then the second half.
  const bool inr = x_in_range(g, x, y, z);                    // pushes only go to voxels inside the update box (:378)
  unsigned long long w[XGB];
  const uint32_t snap_raw = __ldcg(&cobs[v]);
  const unsigned long long wown = __ldcg(&MB[v]);
#pragma unroll
  for (int j = 0; j < XGB; ++j) w[j] = x_writer_word(g, MB, v, x, y, z, j, inr);
  snap = snap_raw & FB_CODE_MASK;
  s.c = snap; s.d = (snap_raw & FB_DINF) ? 0xffffffffu : x_dist_of(x, y, z, s.c); s.ts = XNONE;   // FB_DINF: distance_ forced to +infinity_ (:256-259)
  first = XNONE;
  const unsigned d0 = s.d;
  if (s.c == FB_UNKNOWN) return s;                             // never observed: distance_ = -10000 is never > tmp (:382)
#pragma unroll
  for (int h = 0; h < 24 / XGB; ++h) {
    if (h >= 1) {
#pragma unroll
      for (int j = 0; j < XGB; ++j) w[j] = x_writer_word(g, MB, v, x, y, z, XGB * h + j, inr);
    }
#pragma unroll
    for (int j = 0; j < XGB; ++j) {
      const unsigned long long ww = w[j];
      if (ww == XMB_NONE || x_mb_kind(ww) != X_PUSH) continue;
      const unsigned ts = x_mb_idx(ww) * 32u + (unsigned)(XGB * h + j);
      const uint32_t c = x_mb_code(ww);
      const unsigned d = x_d2(x, y, z, c);
      if (d < d0) {
        if (WANT_FIRST && ts < first) first = ts;
        if (ts < T && (d < s.d || (d == s.d && ts < s.ts))) { s.d = d; s.c = c; s.ts = ts; }
      }
    }
  }
  if (wown != XMB_NONE && x_mb_kind(wown) == X_PULL) {         // the entry's own pull is not range-checked (:349-367)
    const unsigned ts = x_mb_idx(wown) * 32u + 24u;
    const uint32_t c = x_mb_code(wown);
    const unsigned d = x_d2(x, y, z, c);
    if (d < d0) {
      if (WANT_FIRST && ts < first) first = ts;
      if (ts < T && (d < s.d || (d == s.d && ts < s.ts))) { s.d = d; s.c = c; s.ts = ts; }
    }
  }
  return s;
}
// summary of a target: {first, best timestamp, best code, snapshot code}
__device__ __forceinline__ void x_summarize(const FbGeom &g, const uint32_t *cobs, const unsigned long long *MB, uint4 *SUM, int x, int y, int z) {
  unsigned first; uint32_t snap;
  const XState f = x_gather<true>(g, cobs, MB, x, y, z, XNONE, first, snap);
  SUM[x_vi(g, x, y, z)] = make_uint4(first, f.ts, f.c, snap);
}
template <bool USE_SUM>
__device__ __forceinline__ XState x_state(const FbGeom &g, const uint32_t *cobs, const unsigned long long *MB, const uint4 *SUM, int x, int y, int z,
                                          unsigned T, uint32_t &snap) {
  unsigned first;
  if (USE_SUM) {
    const uint4 u = __ldcg(&SUM[x_vi(g, x, y, z)]);
    snap = u.w;
    XState s;
    if (u.x == XNONE || T <= u.x) { s.c = u.w; s.d = x_dist_of(x, y, z, s.c); s.ts = XNONE; return s; }
    if (T > u.y) { s.c = u.z; s.d = x_dist_of(x, y, z, s.c); s.ts = u.y; return s; }
  }
  return x_gather<false>(g, cobs, MB, x, y, z, T, first, snap);  // first < T <= best: gather
}

// ---- grid barrier (all CTAs are co-resident: cooperative launch, one CTA per SM) ---------------------------------------
__device__ __forceinline__ unsigned x_ld_acquire(const unsigned *p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void x_gsync(unsigned *bar, unsigned &target) {
  // bar.sync orders the CTA's writes before thread 0's release; the release / acquire pair at gpu scope is cumulative, and
  // every load of shared data in this kernel bypasses L1 (ld.global.cg), so no further fences are needed.
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(bar), "r"(1u) : "memory");
    while (x_ld_acquire(bar) < target) { }
  }
  __syncthreads();
}

struct XArgs {
  FbGeom g;
  uint32_t *cobs;
  unsigned long long *MB, *LS;
  uint4 *SUM;
  uint32_t *SUMg;
  uint32_t *E[2];
  uint32_t *emask;
  uint32_t *W[3], *F[3];
  uint32_t *wstamp;
  uint32_t *slotc;          // SMALL mode: winner codes, [small_max][32]
  FbXCtl *ctl;
  unsigned small_max, dense_min;
  // E2 (delete loop): dependants of deleted obstacles in the order of the reference's list walk
  const uint32_t *deps; unsigned ndep;
  uint32_t *ord;            // per voxel: position in deps, or XNONE
  uint32_t *nc;             // per dependant: re-seeded code (k_x_reseed: or X_PAR | parent dependant)
  uint32_t *M;              // per dependant: k_x_reseed's mask of earlier dependant neighbours | X_STATIC | X_VALID
  const uint32_t *occbits;
  unsigned long long ls_deps;   // link time of dependant 0 (InsertIntoList order, :333)
  unsigned long long *dbg;  // optional per-generation trace {nE, rounds, ns} (FIESTA_DEBUG_X)
  unsigned div_pz_m, div_pz_s, div_gy_m, div_gy_s;   // n / d = umulhi(n, m) >> s for n < 2^31 (fb_div_make, fb_divmagic.h); m == 0: d == 1
};
// voxel index -> coordinates: two divisions by run-time constants, as multiply-high + shift
__device__ __forceinline__ unsigned x_div(unsigned n, unsigned m, unsigned s) { return m ? (__umulhi(n, m) >> s) : n; }
__device__ __forceinline__ void x_coords(const XArgs &a, uint32_t ii, int &x, int &y, int &z) {
  const unsigned xy = x_div(ii, a.div_pz_m, a.div_pz_s);
  z = (int)(ii - xy * (unsigned)a.g.pz);
  const unsigned xx = x_div(xy, a.div_gy_m, a.div_gy_s);
  y = (int)(xy - xx * (unsigned)a.g.gy);
  x = (int)xx;
}

__device__ __forceinline__ void x_unpack_off(int o, int &dx, int &dy, int &dz) { dx = (o & 15) - 4; dy = ((o >> 4) & 15) - 4; dz = ((o >> 8) & 15) - 4; }

// Summaries of the targets of element i (one warp; lane k = target k): whoever first stamps a target for this summary pass
// (`sclock`, unique per pass) computes it, so every target is summarised exactly once without a target list.
__device__ __forceinline__ void x_claim_summaries(const XArgs &a, const XShared &sh, unsigned lane, int x, int y, int z, unsigned sclock) {
  if (lane >= 25u) return;
  int dx, dy, dz; x_unpack_off(sh.dir[lane], dx, dy, dz);
  const int nx = x + dx, ny = y + dy, nz = z + dz;
  if (!x_in_grid(a.g, nx, ny, nz) || !(lane == 24u || x_in_range(a.g, nx, ny, nz))) return;
  const unsigned n = x_vi(a.g, nx, ny, nz);
  if (__ldcg(&a.SUMg[n]) != sclock && atomicExch(&a.SUMg[n], sclock) != sclock) x_summarize(a.g, a.cobs, a.MB, a.SUM, nx, ny, nz);
}

// After element i (at x,y,z) flipped: bring the summaries of its <= 25 targets up to date (one warp; lane k = target k).
// The offer of (i, k) carries the timestamp 32*i + k whatever its code, so a summary has to be recomputed only if that
// timestamp is its `first` or `best` (the old offer defined it) or if the element's new offer would become one of them;
// otherwise neither removing the old offer nor adding the new one changes {first, best}.
__device__ __forceinline__ void x_refresh_summaries(const XArgs &a, const XShared &sh, unsigned lane, unsigned i, uint32_t p, int x, int y, int z) {
  unsigned long long w = 0;
  if (lane == 0) w = __ldcg(&a.MB[p]);
  w = __shfl_sync(0xffffffffu, w, 0);
  if (lane >= 25u) return;
  int dx, dy, dz; x_unpack_off(sh.dir[lane], dx, dy, dz);
  const int nx = x + dx, ny = y + dy, nz = z + dz;
  if (!x_in_grid(a.g, nx, ny, nz) || !(lane == 24u || x_in_range(a.g, nx, ny, nz))) return;
  const uint4 u = __ldcg(&a.SUM[x_vi(a.g, nx, ny, nz)]);
  if (u.w == FB_UNKNOWN) return;                               // never observed: accepts nothing, its summary never changes
  const unsigned ts = i * 32u + lane;
  bool redo = u.x == ts || u.y == ts;
  if (!redo) {
    const unsigned long long kind = x_mb_kind(w);
    const uint32_t c = x_mb_code(w);
    if (((kind == X_PUSH && lane < 24u) || (kind == X_PULL && lane == 24u)) && c >= 2u) {
      // the snapshot distance is not in the summary (a voxel whose distance was forced to infinity keeps its code): an offer
      // that does not beat the current best cannot matter, one that does is checked against the snapshot by the recomputation
      const unsigned d = x_d2(nx, ny, nz, c);
      if (u.y == XNONE) redo = true;                           // no accepted offer so far: the new one may be the first
      else { const unsigned bd = x_d2(nx, ny, nz, u.z); redo = ts < u.x || d < bd || (d == bd && ts < u.y); }
    }
  }
  if (redo) x_summarize(a.g, a.cobs, a.MB, a.SUM, nx, ny, nz);
}

// Lists, for the next round, the later elements among the first `nof` offsets around (x,y,z) (deduplicated by the per-entry
// round stamp).  One warp; every stage issues its loads / atomics for all of a lane's <= 5 offsets before the next stage looks
// at the results, so the whole search costs four round trips instead of four per offset, and ends with ONE append.
__device__ __forceinline__ void x_list_affected(const XArgs &a, const XShared &sh, unsigned lane, unsigned i, int x, int y, int z, unsigned nof,
                                                unsigned wclock, unsigned out) {
  const FbGeom &g = a.g;
  unsigned long long w[5];
#pragma unroll
  for (int t = 0; t < 5; ++t) {
    const unsigned o = lane + 32u * (unsigned)t;
    w[t] = XMB_NONE;
    if (o < nof) {
      int dx, dy, dz; x_unpack_off(sh.off[o], dx, dy, dz);
      const int nx = x + dx, ny = y + dy, nz = z + dz;
      if (x_in_grid(g, nx, ny, nz)) w[t] = __ldcg(&a.MB[x_vi(g, nx, ny, nz)]);
    }
  }
  unsigned j[5], st[5];
#pragma unroll
  for (int t = 0; t < 5; ++t) {
    j[t] = w[t] != XMB_NONE ? x_mb_idx(w[t]) : 0u;
    st[t] = (w[t] != XMB_NONE && j[t] > i) ? __ldcg(&a.wstamp[j[t]]) : wclock;      // wclock = nothing to do
  }
  unsigned pm = 0;
#pragma unroll
  for (int t = 0; t < 5; ++t)
    if (st[t] != wclock && atomicExch(&a.wstamp[j[t]], wclock) != wclock) pm |= 1u << t;
  const unsigned cnt = (unsigned)__popc(pm);
  unsigned incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += v; }
  const unsigned total = __shfl_sync(0xffffffffu, incl, 31);
  if (total == 0u) return;
  unsigned base = 0;
  if (lane == 0) base = atomicAdd(&a.ctl->nW[out], total);
  base = __shfl_sync(0xffffffffu, base, 0) + incl - cnt;
#pragma unroll
  for (int t = 0; t < 5; ++t) if ((pm >> t) & 1u) a.W[out][base++] = j[t];
}

// Behaviour of element i (one warp; lanes 0..23 = neighbour k at pop time, lane 24 = the element itself).  Returns the new word.
template <bool USE_SUM>
__device__ __forceinline__ unsigned long long x_eval(const XArgs &a, const XShared &sh, unsigned lane, unsigned par, unsigned i, uint32_t p, int x, int y, int z) {
  const FbGeom &g = a.g;
  const unsigned T0 = i * 32u;
  int qx = x, qy = y, qz = z;
  bool valid = lane == 24;
  if (lane < 24) {
    int dx, dy, dz; x_unpack_off(sh.dir[lane], dx, dy, dz);
    qx += dx; qy += dy; qz += dz;
    valid = x_in_range(g, qx, qy, qz) && x_in_grid(g, qx, qy, qz);
  }
  XState st; st.d = 0xffffffffu; st.c = 0; st.ts = XNONE;
  uint32_t snap = 0;
  if (valid) st = x_state<USE_SUM>(g, a.cobs, a.MB, a.SUM, qx, qy, qz, T0, snap);
  const unsigned sd = __shfl_sync(0xffffffffu, st.d, 24);
  const uint32_t sc = __shfl_sync(0xffffffffu, st.c, 24);
  const uint32_t c0 = __shfl_sync(0xffffffffu, snap, 24);
  if (sd != x_dist_of(x, y, z, c0)) return x_mb(par, i, X_DEAD, 0);   // `xx.distance_ != distance_buffer_[idx]`: stale (:345)
  unsigned long long key = ~0ull;                              // pull phase (:349-367) = lexicographic minimum (tmp, k) below the own distance
  if (lane < 24 && valid && st.c >= 2u) {
    const unsigned t = x_d2(x, y, z, st.c);
    if (t < sd) key = ((unsigned long long)t << 8) | lane;
  }
  unsigned long long best = key;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o); best = other < best ? other : best; }
  if (best == ~0ull) return x_mb(par, i, X_PUSH, sc);
  return x_mb(par, i, X_PULL, __shfl_sync(0xffffffffu, st.c, (int)(best & 0xffu)));
}

// ---- gathering evaluation through a per-warp stage ------------------------------------------------------------------------
// One round of loads brings the words at all 129 offsets and the records of the 25 targets into shared memory; the 25 state
// queries, the search for the elements a flip can touch and (SMALL generations) the slot masks then read the stage.  Every
// dependent access to HBM costs a microsecond here (random accesses into GB-sized arrays), so this is what a round costs.
__device__ __forceinline__ void x_stage(const XArgs &a, const XShared &sh, XNb &nb, unsigned lane, int x, int y, int z) {
  const FbGeom &g = a.g;
  unsigned long long w[5];
#pragma unroll
  for (int t = 0; t < 5; ++t) {
    const unsigned o = lane + 32u * (unsigned)t;
    w[t] = XMB_NONE;
    if (o < X_NOFF) {
      int dx, dy, dz; x_unpack_off(sh.off[o], dx, dy, dz);
      const int nx = x + dx, ny = y + dy, nz = z + dz;
      if (x_in_grid(g, nx, ny, nz)) w[t] = __ldcg(&a.MB[x_vi(g, nx, ny, nz)]);
    }
  }
  uint32_t c = 0;
  if (lane < 25u) {
    int dx, dy, dz; x_unpack_off(sh.dir[lane], dx, dy, dz);
    const int nx = x + dx, ny = y + dy, nz = z + dz;
    if (x_in_grid(g, nx, ny, nz)) c = __ldcg(&a.cobs[x_vi(g, nx, ny, nz)]);
  }
  __syncwarp();                                                // the previous element's readers are done
#pragma unroll
  for (int t = 0; t < 5; ++t) { const unsigned o = lane + 32u * (unsigned)t; if (o < X_NOFF) nb.w[o] = w[t]; }
  if (lane < 25u) nb.c[lane] = c;
  __syncwarp();
}
// state of target `lane` (of the staged element at x,y,z) at time T; (qx,qy,qz) = the target's coordinates
__device__ __forceinline__ XState x_state_nb(const FbGeom &g, const XShared &sh, const XNb &nb, unsigned lane, int qx, int qy, int qz, unsigned T, uint32_t &snap) {
  XState s;
  const uint32_t raw = nb.c[lane];
  snap = raw & FB_CODE_MASK;
  s.c = snap; s.d = (raw & FB_DINF) ? 0xffffffffu : x_dist_of(qx, qy, qz, snap); s.ts = XNONE;
  const unsigned d0 = s.d;
  if (snap == FB_UNKNOWN) return s;                            // never observed: accepts nothing (:382)
  if (x_in_range(g, qx, qy, qz)) {                            // pushes only go to voxels inside the update box (:378)
#pragma unroll 8
    for (int k = 0; k < 24; ++k) {
      const unsigned long long ww = nb.w[sh.slot[lane * 24u + (unsigned)k]];
      if (ww == XMB_NONE || x_mb_kind(ww) != X_PUSH) continue;
      const unsigned ts = x_mb_idx(ww) * 32u + (unsigned)k;
      const uint32_t c = x_mb_code(ww);
      const unsigned d = x_d2(qx, qy, qz, c);
      if (d < d0 && ts < T && (d < s.d || (d == s.d && ts < s.ts))) { s.d = d; s.c = c; s.ts = ts; }
    }
  }
  const unsigned long long wown = nb.w[sh.self[lane]];         // the entry's own pull is not range-checked (:349-367)
  if (wown != XMB_NONE && x_mb_kind(wown) == X_PULL) {
    const unsigned ts = x_mb_idx(wown) * 32u + 24u;
    const uint32_t c = x_mb_code(wown);
    const unsigned d = x_d2(qx, qy, qz, c);
    if (d < d0 && ts < T && (d < s.d || (d == s.d && ts < s.ts))) { s.d = d; s.c = c; s.ts = ts; }
  }
  return s;
}
// behaviour of the staged element i (the same reduction as x_eval)
__device__ __forceinline__ unsigned long long x_eval_nb(const XArgs &a, const XShared &sh, const XNb &nb, unsigned lane, unsigned par, unsigned i, int x, int y, int z) {
  const FbGeom &g = a.g;
  const unsigned T0 = i * 32u;
  int qx = x, qy = y, qz = z;
  bool valid = lane == 24;
  if (lane < 24) {
    int dx, dy, dz; x_unpack_off(sh.dir[lane], dx, dy, dz);
    qx += dx; qy += dy; qz += dz;
    valid = x_in_range(g, qx, qy, qz) && x_in_grid(g, qx, qy, qz);
  }
  XState st; st.d = 0xffffffffu; st.c = 0; st.ts = XNONE;
  uint32_t snap = 0;
  if (valid) st = x_state_nb(g, sh, nb, lane, qx, qy, qz, T0, snap);
  const unsigned sd = __shfl_sync(0xffffffffu, st.d, 24);
  const uint32_t sc = __shfl_sync(0xffffffffu, st.c, 24);
  const uint32_t c0 = __shfl_sync(0xffffffffu, snap, 24);
  if (sd != x_dist_of(x, y, z, c0)) return x_mb(par, i, X_DEAD, 0);   // stale (:345)
  unsigned long long key = ~0ull;                              // pull phase (:349-367)
  if (lane < 24 && valid && st.c >= 2u) {
    const unsigned t = x_d2(x, y, z, st.c);
    if (t < sd) key = ((unsigned long long)t << 8) | lane;
  }
  unsigned long long best = key;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o); best = other < best ? other : best; }
  if (best == ~0ull) return x_mb(par, i, X_PUSH, sc);
  return x_mb(par, i, X_PULL, __shfl_sync(0xffffffffu, st.c, (int)(best & 0xffu)));
}
// x_list_affected with the words taken from the stage (no reload)
__device__ __forceinline__ void x_list_affected_nb(const XArgs &a, const XNb &nb, unsigned lane, unsigned i, unsigned nof, unsigned wclock, unsigned out) {
  unsigned j[5], st[5];
#pragma unroll
  for (int t = 0; t < 5; ++t) {
    const unsigned o = lane + 32u * (unsigned)t;
    const unsigned long long w = o < nof ? nb.w[o] : XMB_NONE;
    j[t] = w != XMB_NONE ? x_mb_idx(w) : 0u;
    st[t] = (w != XMB_NONE && j[t] > i) ? __ldcg(&a.wstamp[j[t]]) : wclock;
  }
  unsigned pm = 0;
#pragma unroll
  for (int t = 0; t < 5; ++t)
    if (st[t] != wclock && atomicExch(&a.wstamp[j[t]], wclock) != wclock) pm |= 1u << t;
  const unsigned cnt = (unsigned)__popc(pm);
  unsigned incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += v; }
  const unsigned total = __shfl_sync(0xffffffffu, incl, 31);
  if (total == 0u) return;
  unsigned base = 0;
  if (lane == 0) base = atomicAdd(&a.ctl->nW[out], total);
  base = __shfl_sync(0xffffffffu, base, 0) + incl - cnt;
#pragma unroll
  for (int t = 0; t < 5; ++t) if ((pm >> t) & 1u) a.W[out][base++] = j[t];
}

// Exclusive scan of one count per thread over the CTA (two block barriers); returns the CTA total in `total`.
__device__ __forceinline__ unsigned x_block_scan(XShared &sh, unsigned c, unsigned lane, unsigned wid, unsigned &total) {
  unsigned incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += t; }
  __syncthreads();                                             // earlier readers of sh.red are done
  if (lane == 31) sh.red[wid] = incl;
  __syncthreads();
  const unsigned v = sh.red[lane]; unsigned s = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, s, o); if ((int)lane >= o) s += t; }
  total = __shfl_sync(0xffffffffu, s, 31);
  return __shfl_sync(0xffffffffu, s - v, (int)wid) + incl - c;
}

// ---- asynchronous schedule of the short work lists ------------------------------------------------------------------------
// Rounds are a scheduling device: element i's behaviour depends only on the words of earlier elements, so the fixpoint is
// unique and every fair schedule that re-evaluates an element after each change of its inputs reaches it (by induction on
// i).  x_async runs such a schedule without grid barriers: every warp pops an element from a work queue, evaluates it from
// its stage exactly as a round does, and on a flip pushes the later elements it can touch.
//  * Element state, in wstamp with the phase's base A (stamps of earlier rounds and phases are all below A): RUNNING = A,
//    MARKED = A + 1 (queued, or dirty while running), IDLE = anything below A.  A lister does atomicMax(MARKED) and pushes
//    iff the element was IDLE; a running element that gets marked is dirty, and its worker evaluates it again before
//    setting it IDLE (compare-and-swap RUNNING -> A - 1).  Hence an element is queued at most once and evaluated by one warp
//    at a time.
//  * No missed update.  The flipping warp stores its word, then fence.sc, then reads the state of each element it lists;
//    a worker swaps the state to RUNNING, then fence.sc, then stages.  Of two such store-fence-load sequences at least one
//    load sees the other's store.  So either the lister sees RUNNING / IDLE and marks the element (a worker will evaluate
//    it again, after a swap that comes later), or the lister sees MARKED and the swap that follows it sees the flip.
//    After the last flip of each input some evaluation sees it; an element whose inputs stop changing stops changing.
//  * Ring: a buffer with one slot per element of the generation (at most nE elements are queued at once); pushes and pops
//    reserve consecutive indices, slot = index mod nE.  A full slot carries bit 31 (work lists leave elements < 2^27 in the
//    buffer, pops leave 0): a pusher waits for the slot to be free, a popper takes whatever element is in its slot (items
//    may swap between poppers of one slot, which is harmless: each is taken once).  A pusher never waits forever: with
//    at most nE distinct queued elements, every full slot has a reserved popper that has not taken an item yet.
//  * Termination: qtail's high half counts the outstanding items (incremented with the push that creates one,
//    decremented when its evaluation is over, after its own pushes) plus one token per warp until the warp has pushed its
//    share of the seed list.  Zero is final (nothing runs that could push); whoever reaches it sets qdone.
//  * Every wait is bounded (X_Q_WAIT_NS of no progress): the kernel then sets ctl->err = 3 and qdone, and every warp leaves.
#define X_Q_FULL 0x80000000u
#define X_Q_WAIT_NS 2000000000ull
__device__ __forceinline__ unsigned x_ld_relaxed(const unsigned *p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long x_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void x_q_abort(const XArgs &a) {
  atomicCAS(&a.ctl->err, 0u, 3u);
  atomicExch(&a.ctl->qdone, 1u);
}
// qtail += delta (one lane); sets qdone when the outstanding count reaches zero, and the CTA's copy with it, so that the
// warp that ends the phase (often the only one left working) leaves at once instead of at its next poll of the global
// flag.  Returns the old push count.
__device__ __forceinline__ unsigned x_q_count(const XArgs &a, XShared &sh, unsigned long long delta) {
  const unsigned long long old = atomicAdd(&a.ctl->qtail, delta);
  if ((unsigned)((old + delta) >> 32) == 0u) { atomicExch(&a.ctl->qdone, 1u); sh.qdone = 1u; }
  return (unsigned)old;
}
// (qdone cannot be set while the pusher's own item is outstanding, unless the phase was abandoned: then it leaves at once)
__device__ __forceinline__ void x_q_put(const XArgs &a, XShared &sh, uint32_t *ring, unsigned cap, unsigned idx, unsigned e) {
  unsigned *slot = &ring[idx % cap];
  const volatile unsigned *done = &sh.qdone;
  unsigned cur = x_ld_relaxed(slot);
  const unsigned long long t0 = x_globaltimer();
  for (unsigned it = 0;; ++it) {
    if (!(cur & X_Q_FULL)) {
      const unsigned o = atomicCAS(slot, cur, e | X_Q_FULL);
      if (o == cur) return;
      cur = o;
      continue;
    }
    if (*done) return;
    if ((it & 15u) == 15u) {
      if (x_ld_acquire(&a.ctl->qdone)) { sh.qdone = 1u; return; }
      if (x_globaltimer() - t0 > X_Q_WAIT_NS) { x_q_abort(a); sh.qdone = 1u; return; }
    }
    __nanosleep(64);
    cur = x_ld_relaxed(slot);
  }
}
// One lane: the next element from the queue, or XNONE once the phase is over.  `h` keeps the reserved pop index between calls.
template <bool DBG>
__device__ __forceinline__ unsigned x_q_take(const XArgs &a, XShared &sh, uint32_t *ring, unsigned cap, unsigned &h) {
  if (h == XNONE) h = atomicAdd(&a.ctl->qhead, 1u);
  unsigned *slot = &ring[h % cap];
  const volatile unsigned *done = &sh.qdone;
  const long long c0 = DBG ? clock64() : 0;
  unsigned long long t0 = 0;
  unsigned ns = 32;
  for (unsigned it = 0;; ++it) {
    if (x_ld_relaxed(slot) & X_Q_FULL) {
      const unsigned v = atomicExch(slot, 0u);
      if (v & X_Q_FULL) { h = XNONE; if (DBG) atomicAdd(&a.dbg[FB_XDBG_Q + 3], (unsigned long long)(clock64() - c0)); return v & ~X_Q_FULL; }
    }
    if (*done) break;
    if ((it & 15u) == 15u) {                                   // the global flag is polled by few warps at a time
      if (x_ld_acquire(&a.ctl->qdone)) { sh.qdone = 1u; break; }
      const unsigned long long t = x_globaltimer();
      if (t0 == 0) t0 = t;
      else if (t - t0 > X_Q_WAIT_NS) { x_q_abort(a); sh.qdone = 1u; break; }
    }
    __nanosleep(ns);
    ns = ns < 256u ? 2u * ns : 256u;
  }
  if (DBG) atomicAdd(&a.dbg[FB_XDBG_Q + 3], (unsigned long long)(clock64() - c0));
  return XNONE;
}
// Marks the later elements among the first `nof` staged offsets of element i and pushes those that were IDLE (one warp,
// after the flip's word was stored and fenced).
__device__ __forceinline__ unsigned x_q_list(const XArgs &a, XShared &sh, const XNb &nb, uint32_t *ring, unsigned cap, unsigned lane, unsigned i, unsigned nof, unsigned A) {
  unsigned j[5], st[5];
#pragma unroll
  for (int t = 0; t < 5; ++t) {
    const unsigned o = lane + 32u * (unsigned)t;
    const unsigned long long w = o < nof ? nb.w[o] : XMB_NONE;
    j[t] = w != XMB_NONE ? x_mb_idx(w) : 0u;
    st[t] = (w != XMB_NONE && j[t] > i) ? x_ld_relaxed(&a.wstamp[j[t]]) : A + 1u;   // A + 1 = already marked or not a candidate
  }
  unsigned pm = 0;
#pragma unroll
  for (int t = 0; t < 5; ++t)
    if (st[t] != A + 1u && atomicMax(&a.wstamp[j[t]], A + 1u) < A) pm |= 1u << t;
  const unsigned cnt = (unsigned)__popc(pm);
  unsigned incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += v; }
  const unsigned total = __shfl_sync(0xffffffffu, incl, 31);
  if (total == 0u) return 0u;
  unsigned base = 0;
  if (lane == 0) base = x_q_count(a, sh, (unsigned long long)total * 0x100000001ull);
  base = __shfl_sync(0xffffffffu, base, 0) + incl - cnt;
#pragma unroll
  for (int t = 0; t < 5; ++t) if ((pm >> t) & 1u) x_q_put(a, sh, ring, cap, base++, j[t]);
  return total;
}
// One element of an asynchronous phase, taken from the queue: evaluated from its stage, its word stored on a flip and
// recorded in F[fout], and the later elements it can touch listed; evaluated again while a lister marked it dirty meanwhile.
template <bool DBG>
__device__ __forceinline__ void x_q_run(const XArgs &a, XShared &sh, XNb &stg, unsigned lane, const uint32_t *E, unsigned nE, uint32_t *ring,
                                        unsigned gen, unsigned A, unsigned fout, unsigned i) {
  const uint32_t p = __ldcg(&E[i]);
  int x, y, z; x_coords(a, p, x, y, z);
  for (;;) {
    if (DBG && lane == 0) atomicAdd(&a.dbg[FB_XDBG_Q + 0], 1ull);
    if (lane == 0) atomicExch(&a.wstamp[i], A);                // RUNNING (from MARKED: queued, or dirty)
    __syncwarp();
    __threadfence();
    x_stage(a, sh, stg, lane, x, y, z);
    const unsigned long long old = stg.w[0], nw2 = x_eval_nb(a, sh, stg, lane, gen, i, x, y, z);
    if (nw2 != old) {                                          // flip
      if (lane == 0) {
        a.MB[p] = nw2;
        const unsigned f = atomicAdd(&a.ctl->nF[fout], 1u);
        if (f < (unsigned)a.g.ptotal) a.F[fout][f] = i;
      }
      __syncwarp();
      __threadfence();
      const unsigned np = x_q_list(a, sh, stg, ring, nE, lane, i, (x_mb_kind(old) == X_PUSH || x_mb_kind(nw2) == X_PUSH) ? (unsigned)X_NOFF : 25u, A);
      if (DBG && lane == 0 && np) atomicAdd(&a.dbg[FB_XDBG_Q + 2], (unsigned long long)np);
    }
    unsigned again = 0;
    if (lane == 0) again = atomicCAS(&a.wstamp[i], A, A - 1u) != A ? 1u : 0u;   // IDLE, unless marked dirty meanwhile
    if (!__shfl_sync(0xffffffffu, again, 0)) break;
    if (DBG && lane == 0) atomicAdd(&a.dbg[FB_XDBG_Q + 1], 1ull);
  }
}
// The asynchronous phase of one BIG generation (all warps of the grid): the nw elements of the work list `wl` seed the
// queue, `ring` (nE slots) holds it; every flip is recorded in F[fout] for the summary refresh that follows.
template <bool DBG>
__device__ void x_async(const XArgs &a, XShared &sh, XNb &stg, unsigned lane, unsigned gwarp, unsigned gwarps, const uint32_t *E, unsigned nE,
                        const uint32_t *wl, unsigned nw, uint32_t *ring, unsigned gen, unsigned A, unsigned fout) {
  // seeds: this warp's chunks of 32, then its token
  for (unsigned q0 = gwarp * 32u; q0 < nw; q0 += gwarps * 32u) {
    const unsigned q = q0 + lane;
    const unsigned e = q < nw ? __ldcg(&wl[q]) : 0u;
    const bool push = q < nw && atomicMax(&a.wstamp[e], A + 1u) < A;
    const unsigned pm = __ballot_sync(0xffffffffu, push), cnt = (unsigned)__popc(pm);
    if (cnt == 0u) continue;
    unsigned base = 0;
    if (lane == 0) base = x_q_count(a, sh, (unsigned long long)cnt * 0x100000001ull);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (push) x_q_put(a, sh, ring, nE, base + (unsigned)__popc(pm & ((1u << lane) - 1u)), e);
    if (DBG && lane == 0) atomicAdd(&a.dbg[FB_XDBG_Q + 2], (unsigned long long)cnt);
  }
  if (lane == 0) x_q_count(a, sh, 0ull - (1ull << 32));
  unsigned h = XNONE;
  for (;;) {
    unsigned i = 0;
    if (lane == 0) i = x_q_take<DBG>(a, sh, ring, nE, h);
    i = __shfl_sync(0xffffffffu, i, 0);
    if (i == XNONE) break;
    x_q_run<DBG>(a, sh, stg, lane, E, nE, ring, gen, A, fout, i);
    if (lane == 0) x_q_count(a, sh, 0ull - (1ull << 32));
  }
}
extern __shared__ __align__(16) unsigned char x_dyn_smem[];

// ---- E2, second half: re-seeding of the dependants of the deleted obstacles (:301-334) ----------------------------------
// The reference walks the dependants in list order and gives dependant i the closest obstacle of the FIRST neighbour, in
// dirs_ order and inside the update box, whose closest obstacle exists (:308-321); earlier dependants show their new value,
// later ones are skipped.  So i's final code is INF or a code copied, through a chain of earlier dependants, from a
// non-dependant neighbour that passed the Exist test (a static source).  It follows that
//  * validity is monotone: i ends valid iff it has a static source or an earlier dependant neighbour that ends valid.  This
//    is an OR closure over a DAG (o -> i only for o < i): each dependant turns valid at most once;
//  * once validity is known, i's source is local: its first direction, in dirs_ order, whose neighbour is a static source
//    or a valid earlier dependant (its parent);
//  * parents have smaller indices, so pointer jumping resolves every code in ceil(log2(longest chain)) + 1 passes.
// By induction on i this is the sequential rule, whatever the dependant order.  k_x_reseed runs it in four stages separated
// by grid barriers (CPU model checked against the sequential rule: scripts/reseed_model.c):
//  A classify  one thread per dependant walks its neighbours up to the first static source: nc[i] = its code, or INF;
//              M[i] = the mask of the earlier dependant neighbours before it | X_STATIC | X_VALID if there is one.  An empty
//              mask is final.
//  B closure   round 1: every dependant with no static source and a non-empty mask becomes X_VALID if a masked neighbour
//              is (pull); each later round: every dependant made valid in the round before marks its later dependant
//              neighbours that have no static source (push, atomicOr: each enters a list once).  Until a round lists none.
//  C choose    a valid dependant with a non-empty mask takes its first masked valid neighbour as parent: nc[i] = X_PAR | o.
//  D resolve   nc[i] = nc[parent] over the dependants still holding a parent, until none does.  In place: a concurrent
//              write only moves a parent further up its chain, and a 32-bit word never tears.
// ctl->reseed_rounds = the rounds of B plus the passes of D.
#define X_STATIC 0x20000000u
#define X_VALID 0x40000000u
#define X_PAR 0x80000000u                // codes use 31 bits (FB_CODE_MASK)
#define X_LAP(cat) do { if (DBG && gtid == 0) { const long long t_now = clock64(); a.dbg[XDBG_PHASE + 2 * (cat)] += (unsigned long long)(t_now - t_ph); a.dbg[XDBG_PHASE + 2 * (cat) + 1] += 1ull; t_ph = t_now; } } while (0)

// The dependant at the in-grid, in-box voxel x + dirs_[k] (XNONE: none, or outside the grid or the box) for the directions
// k = K0..K0+7 set in `want`: all loads of a chunk are issued before any is looked at.
template <int K0>
__device__ __forceinline__ void x_dep_nb(const XArgs &a, int x, int y, int z, unsigned want, unsigned (&nv)[8], unsigned (&o)[8]) {
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const int nx = x + x_dc(K0 + t, 0), ny = y + x_dc(K0 + t, 1), nz = z + x_dc(K0 + t, 2);
    nv[t] = ((want >> (K0 + t)) & 1u) && x_in_grid(a.g, nx, ny, nz) && x_in_range(a.g, nx, ny, nz) ? x_vi(a.g, nx, ny, nz) : XNONE;
    o[t] = nv[t] != XNONE ? __ldcg(&a.ord[nv[t]]) : XNONE;
  }
}
// first masked direction of chunk K0 whose dependant is valid (24: none)
template <int K0>
__device__ __forceinline__ unsigned x_first_valid(const XArgs &a, int x, int y, int z, unsigned mask, unsigned &par) {
  unsigned nv[8], o[8], m[8];
  x_dep_nb<K0>(a, x, y, z, mask, nv, o);                     // a masked direction holds an earlier dependant
#pragma unroll
  for (int t = 0; t < 8; ++t) m[t] = o[t] != XNONE ? __ldcg(&a.M[o[t]]) : 0u;
#pragma unroll
  for (int t = 0; t < 8; ++t) if (m[t] & X_VALID) { par = o[t]; return (unsigned)(K0 + t); }
  return 24u;
}
// A for dependant i: directions K0..K0+7 (until `done`)
template <int K0>
__device__ __forceinline__ void x_classify(const XArgs &a, unsigned i, int x, int y, int z, unsigned &mask, uint32_t &sc, bool &done) {
  unsigned nv[8], o[8];
  uint32_t c[8];
  x_dep_nb<K0>(a, x, y, z, 0xffffffu, nv, o);
#pragma unroll
  for (int t = 0; t < 8; ++t) c[t] = (nv[t] != XNONE && o[t] == XNONE) ? __ldcg(&a.cobs[nv[t]]) & FB_CODE_MASK : 0u;
  unsigned e[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    e[t] = 0u;
    if (c[t] >= 2u) { int ox, oy, oz; fb_unpack(c[t], ox, oy, oz); const unsigned oi = x_vi(a.g, ox, oy, oz); e[t] = (__ldg(&a.occbits[oi >> 5]) >> (oi & 31)) & 1u; }
  }
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    if (done || nv[t] == XNONE) continue;
    if (o[t] != XNONE) { if (o[t] < i) mask |= 1u << (K0 + t); }
    else if (e[t]) { sc = c[t]; done = true; }                // Exist(closest obstacle) (:312), then `break` (:319)
  }
}
// B, push (if `act`): the later dependants without a static source next to the newly valid dependant o at (x,y,z), directions
// K0..K0+7, turn valid and are listed in W[out].  Called by whole warps (the appends are warp-aggregated).
template <int K0>
__device__ __forceinline__ void x_mark_later(const XArgs &a, bool act, unsigned o, int x, int y, int z, unsigned out) {
  unsigned j[8], m[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const int nx = x + x_dc(K0 + t, 0), ny = y + x_dc(K0 + t, 1), nz = z + x_dc(K0 + t, 2);
    j[t] = act && x_in_grid(a.g, nx, ny, nz) ? __ldcg(&a.ord[x_vi(a.g, nx, ny, nz)]) : XNONE;
  }
#pragma unroll
  for (int t = 0; t < 8; ++t) m[t] = (j[t] != XNONE && j[t] > o) ? __ldcg(&a.M[j[t]]) : X_VALID;
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const bool push = !(m[t] & (X_STATIC | X_VALID)) && !(atomicOr(&a.M[j[t]], X_VALID) & X_VALID);
    const unsigned slot = fb_warp_append(&a.ctl->nW[out], push);
    if (push) a.W[out][slot] = j[t];
  }
}

template <bool DBG>
__global__ void __launch_bounds__(XT, 1) k_x_reseed(const XArgs a) {
  __shared__ XShared sh;
  FbXCtl *ctl = a.ctl;
  const unsigned tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5, G = gridDim.x, b = blockIdx.x;
  const unsigned gtid = b * XT + tid, gthreads = G * XT;
  unsigned bar_target = 0;
  long long t_ph = DBG ? clock64() : 0;
  // A: classify; the dependants with a non-empty mask and no static source are the list of B's first round (W[1])
  for (unsigned i0 = 0; i0 < a.ndep; i0 += gthreads) {
    const unsigned i = i0 + gtid;
    unsigned mask = 0;
    uint32_t sc = FB_INF;
    bool done = true;
    if (i < a.ndep) {
      int x, y, z; x_coords(a, __ldcg(&a.deps[i]), x, y, z);
      done = false;
      x_classify<0>(a, i, x, y, z, mask, sc, done);
      if (!done) x_classify<8>(a, i, x, y, z, mask, sc, done);
      if (!done) x_classify<16>(a, i, x, y, z, mask, sc, done);
      a.nc[i] = sc;
      a.M[i] = mask | (done ? X_STATIC | X_VALID : 0u);
    }
    const bool pull = !done && mask;
    const unsigned slot = fb_warp_append(&ctl->nW[1], pull);
    if (pull) a.W[1][slot] = i;
    if (DBG) { const unsigned f = __popc(__ballot_sync(0xffffffffu, i < a.ndep && !mask)); if ((threadIdx.x & 31u) == 0 && f) atomicAdd(&a.dbg[XDBG_PHASE + 2 * 15], (unsigned long long)f); }
  }
  x_gsync(&ctl->rbar, bar_target);
  X_LAP(12);
  // B: closure rounds over the lists W[r % 3] (the list counters rotate as in k_x_relax's rounds)
  unsigned r = 1, rounds = 0;
  for (;; ++r) {
    const unsigned in = r % 3u, out = (r + 1u) % 3u, zz = (r + 2u) % 3u;
    const unsigned nw = __ldcg(&ctl->nW[in]);
    if (gtid == 0) ctl->nW[zz] = 0;
    if (nw == 0u) break;
    ++rounds;
    if (DBG && gtid == 0) a.dbg[XDBG_PHASE + 2 * 15 + 1] += nw;
    for (unsigned q0 = 0; q0 < nw; q0 += gthreads) {          // (every warp runs the same iterations: its appends are collective)
      const unsigned q = q0 + gtid;
      const bool act = q < nw;
      const unsigned i = act ? __ldcg(&a.W[in][q]) : 0u;
      int x = 0, y = 0, z = 0;
      if (act) x_coords(a, __ldcg(&a.deps[i]), x, y, z);
      if (r == 1u) {                                           // pull: a masked neighbour is valid
        unsigned k = 24u, par;
        if (act) {
          const unsigned mask = __ldcg(&a.M[i]);
          k = x_first_valid<0>(a, x, y, z, mask, par);
          if (k == 24u) k = x_first_valid<8>(a, x, y, z, mask, par);
          if (k == 24u) k = x_first_valid<16>(a, x, y, z, mask, par);
          if (k != 24u) a.M[i] = mask | X_VALID;               // nobody else writes M[i] in this round
        }
        const unsigned slot = fb_warp_append(&ctl->nW[out], k != 24u);
        if (k != 24u) a.W[out][slot] = i;
      } else {                                                 // push; later dependants see this one only inside the box
        const bool push = act && x_in_range(a.g, x, y, z);
        x_mark_later<0>(a, push, i, x, y, z, out);
        x_mark_later<8>(a, push, i, x, y, z, out);
        x_mark_later<16>(a, push, i, x, y, z, out);
      }
    }
    x_gsync(&ctl->rbar, bar_target);
    X_LAP(20);
  }
  // C: choose the parents; the dependants that took one are the list of D's first pass
  {
    const unsigned out = (r + 1u) % 3u;
    for (unsigned i0 = 0; i0 < a.ndep; i0 += gthreads) {
      const unsigned i = i0 + gtid;
      const unsigned m = i < a.ndep ? __ldcg(&a.M[i]) : 0u;
      unsigned k = 24u, par = 0;
      if ((m & X_VALID) && (m & 0xffffffu)) {
        int x, y, z; x_coords(a, __ldcg(&a.deps[i]), x, y, z);
        k = x_first_valid<0>(a, x, y, z, m, par);
        if (k == 24u) k = x_first_valid<8>(a, x, y, z, m, par);
        if (k == 24u) k = x_first_valid<16>(a, x, y, z, m, par);
        if (k != 24u) a.nc[i] = X_PAR | par;                   // else the static code stays
      }
      const unsigned slot = fb_warp_append(&ctl->nW[out], k != 24u);
      if (k != 24u) a.W[out][slot] = i;
    }
    x_gsync(&ctl->rbar, bar_target);
    X_LAP(21);
  }
  // D: resolve by pointer jumping
  unsigned passes = 0;
  for (++r;; ++r) {
    const unsigned in = r % 3u, out = (r + 1u) % 3u, zz = (r + 2u) % 3u;
    const unsigned nw = __ldcg(&ctl->nW[in]);
    if (gtid == 0) ctl->nW[zz] = 0;
    if (nw == 0u) break;
    ++passes;
    for (unsigned q0 = 0; q0 < nw; q0 += gthreads) {
      const unsigned q = q0 + gtid;
      bool again = false;
      unsigned i = 0;
      if (q < nw) {
        i = __ldcg(&a.W[in][q]);
        const uint32_t c = __ldcg(&a.nc[__ldcg(&a.nc[i]) & ~X_PAR]);
        a.nc[i] = c;
        again = (c & X_PAR) != 0u;
      }
      const unsigned slot = fb_warp_append(&ctl->nW[out], again);
      if (again) a.W[out][slot] = i;
    }
    x_gsync(&ctl->rbar, bar_target);
    X_LAP(22);
  }
  // Hand-over: the re-seeded dependants, in list-walk order, follow the insert seeds in E[0] (:329-333): per-CTA counts over
  // CTA-contiguous ranges, then an exclusive scan
  const unsigned per = (a.ndep + G - 1u) / G;
  const unsigned lo = min(a.ndep, b * per), hi = min(a.ndep, lo + per);
  unsigned mine = 0;
  for (unsigned i = lo + tid; i < hi; i += XT) mine += __ldcg(&a.nc[i]) >= 2u ? 1u : 0u;
  unsigned tot;
  x_block_scan(sh, mine, lane, wid, tot);
  if (tid == 0) ctl->partial[b] = tot;
  const unsigned nE = __ldcg(&ctl->nE0);                       // the insert seeds
  x_gsync(&ctl->rbar, bar_target);
  if (wid == 0) {
    unsigned before = 0, all = 0;
    for (unsigned k = lane; k < G; k += 32u) { const unsigned c = __ldcg(&ctl->partial[k]); all += c; if (k < b) before += c; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { before += __shfl_xor_sync(0xffffffffu, before, o); all += __shfl_xor_sync(0xffffffffu, all, o); }
    if (lane == 0) { sh.base = before; sh.total = all; }
  }
  __syncthreads();
  unsigned run = nE + sh.base;
  for (unsigned i0 = lo; i0 < hi; i0 += XT) {
    const unsigned i = i0 + tid;
    uint32_t c = FB_INF, v = 0;
    if (i < hi) {
      c = __ldcg(&a.nc[i]); v = __ldcg(&a.deps[i]);
      a.cobs[v] = c;
      a.LS[v] = a.ls_deps + i;                                 // InsertIntoList(new_obs_idx, obs_idx) (:333)
    }
    unsigned ctot;
    const unsigned pos = x_block_scan(sh, (i < hi && c >= 2u) ? 1u : 0u, lane, wid, ctot);
    if (i < hi && c >= 2u) a.E[0][run + pos] = v;              // `if (distance < infinity_) update_queue_.push` (:329-331)
    run += ctot;
  }
  if (gtid == 0) {                                             // (every CTA has read nE0 and the list counters)
    ctl->nE0 = nE + sh.total;
    ctl->reseed_rounds = rounds + passes;
    ctl->nW[0] = ctl->nW[1] = ctl->nW[2] = 0;
  }
  X_LAP(13);
}

// DBG: the FIESTA_DEBUG_X trace (a.dbg != nullptr).  The production instance carries none of its clocks and counters, which
// would otherwise stay live across the generation loop and the queue phases (spills at the 64-register limit).
template <bool DBG>
__global__ void __launch_bounds__(XT, 1) k_x_relax(const XArgs a) {
  __shared__ XShared sh;
  const FbGeom &g = a.g;
  FbXCtl *ctl = a.ctl;
  const unsigned tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
  const unsigned G = gridDim.x, b = blockIdx.x;
  const unsigned gtid = b * XT + tid, gthreads = G * XT;
  const unsigned gwarp = gtid >> 5, gwarps = gthreads >> 5;
  for (unsigned k = tid; k < X_NOFF; k += XT) sh.off[k] = x_off_c[k];
  if (tid < 32) sh.self[tid] = 0;
  if (tid == 0) { sh.qdone = 0u; sh.bar_target = 0u; }
  if (gtid == 0) a.ctl->qtail = (unsigned long long)gwarps << 32;   // one seeding token per warp (x_async)
  if (tid < 32) sh.dir[tid] = tid < 24 ? ((x_dirs[tid][0] + 4) | ((x_dirs[tid][1] + 4) << 4) | ((x_dirs[tid][2] + 4) << 8)) : (4 | (4 << 4) | (4 << 8));
  __syncthreads();
  for (unsigned q = tid; q < 25u * 24u + 25u; q += XT) {         // where target t's k-th writer (and t itself) sits among the 129 offsets
    const unsigned t = q < 600u ? q / 24u : q - 600u, k = q < 600u ? q % 24u : 24u;
    int tx, ty, tz, kx = 0, ky = 0, kz = 0; x_unpack_off(sh.dir[t], tx, ty, tz);
    if (k < 24u) x_unpack_off(sh.dir[k], kx, ky, kz);
    const int code = (tx - kx + 4) | ((ty - ky + 4) << 4) | ((tz - kz + 4) << 8);
    unsigned found = 0;
    for (unsigned o = 0; o < X_NOFF; ++o) if (sh.off[o] == code) found = o;
    if (q < 600u) sh.slot[q] = (unsigned char)found; else sh.self[t] = (unsigned char)found;
  }
  __syncthreads();
  XNb &stg = reinterpret_cast<XNb *>(x_dyn_smem)[wid];

  // grid-uniform state (every CTA computes the same values)
  unsigned nE = ctl->nE0;
  int cur = 0;
  unsigned gen = ctl->gen_id, wclock = ctl->wclock;
  unsigned long long tclock = ctl->tclock;
  if (tid == 0) { sh.generations = 0; sh.rounds = 0; sh.dense_rounds = 0; sh.changed = 0; }
  if (DBG) {                                                 // cost of an empty grid barrier
    const long long t0 = clock64();
    for (int q = 0; q < 32; ++q) x_gsync(&ctl->bar, sh.bar_target);
    if (gtid == 0) a.dbg[XDBG_PHASE + 2 * 11] = (unsigned long long)(clock64() - t0) / 32ull;
  }
  long long t_ph = DBG ? clock64() : 0;
  bool big = nE > a.small_max;

  // generation 0: words.  Initial guess of the fixpoint: every entry pushes its snapshot code.
  // (Tried and dropped, both bit-exact: a silent start for the re-seeded dependants -- same number of rounds; resolving a
  // generation window by window in queue order -- the dependency chains of the sweep after a delete are short and local, so
  // windows only serialise work that the whole-generation rounds do concurrently: 2983 rounds instead of 919.)
  ++gen;
  unsigned sclock = ctl->sclock;
  for (unsigned i = gtid; i < nE; i += gthreads) {
    const uint32_t v = __ldcg(&a.E[0][i]);
    a.MB[v] = x_mb(gen, i, X_PUSH, __ldcg(&a.cobs[v]) & FB_CODE_MASK);
  }
  x_gsync(&ctl->bar, sh.bar_target);

  while (nE) {
    const long long t_gen = DBG ? clock64() : 0;
    X_LAP(10);
    if (tid == 0) ++sh.generations;
    const uint32_t *E = a.E[cur];
    // ---- behaviour fixpoint
    unsigned rounds = 0;
    bool aborted = false;
    if (big) {
      ++sclock;
      for (unsigned i = gwarp; i < nE; i += gwarps) { int x, y, z; x_coords(a, __ldcg(&E[i]), x, y, z); x_claim_summaries(a, sh, lane, x, y, z, sclock); }
      x_gsync(&ctl->bar, sh.bar_target);
      X_LAP(0);
    }
    for (unsigned r = 1;; ++r) {
      const unsigned in = r % 3u, out = (r + 1u) % 3u, zz = (r + 2u) % 3u;
      const unsigned nw = r == 1u ? nE : __ldcg(&ctl->nW[in]);
      const unsigned nf = (big && r > 1u) ? __ldcg(&ctl->nF[in]) : 0u;
      if (gtid == 0) { ctl->nW[zz] = 0; ctl->nF[zz] = 0; }
      if (r > 1u && nw == 0u && nf == 0u) break;
      if (r > X_MAX_ROUNDS) { if (gtid == 0) ctl->err = 2u; break; }   // cannot happen (element i is final after i+1 rounds at the latest); never spin forever on the GPU
      if (DBG && gtid == 0) { a.dbg[XDBG_PHASE + 2 * 14] += nw; a.dbg[XDBG_PHASE + 2 * 14 + 1] += nf; }
      if (big && r > 1u && nw <= a.dense_min) {
        // the rest of the fixpoint from the work queue, with W[out] as its ring; then the summaries of the targets of every
        // flip since the last refresh: last round's (F[in]) and the queue's (F[out]).  A summary's offer timestamps 32*i+k
        // are fixed, so the refresh rule needs only the final word and the summary's first / best, however often the element
        // flipped in between.
        ++rounds; wclock += 3u;
        const unsigned A = wclock - 1u;                        // RUNNING; MARKED = wclock; the stamps of the next rounds are above
        x_async<DBG>(a, sh, stg, lane, gwarp, gwarps, E, nE, a.W[in], nw, a.W[out], gen, A, out);
        x_gsync(&ctl->bar, sh.bar_target);
        X_LAP(16);
        if (tid == 0) sh.qdone = 0u;
        if (gtid == 0) { ctl->qtail = (unsigned long long)gwarps << 32; ctl->qhead = 0u; ctl->qdone = 0u; }
        if (__ldcg(&ctl->err)) { aborted = true; break; }
        const unsigned nfa = __ldcg(&ctl->nF[out]);
        if (nfa > (unsigned)g.ptotal) {                        // flip list overflowed: summarise every target again
          ++sclock;
          for (unsigned i = gwarp; i < nE; i += gwarps) { int x, y, z; x_coords(a, __ldcg(&E[i]), x, y, z); x_claim_summaries(a, sh, lane, x, y, z, sclock); }
        } else {
          for (unsigned q = gwarp; q < nf + nfa; q += gwarps) {
            const unsigned i = q < nf ? __ldcg(&a.F[in][q]) : __ldcg(&a.F[out][q - nf]);
            const uint32_t p = __ldcg(&E[i]);
            int x, y, z; x_coords(a, p, x, y, z);
            x_refresh_summaries(a, sh, lane, i, p, x, y, z);
          }
        }
        x_gsync(&ctl->bar, sh.bar_target);
        X_LAP(18);
        break;
      }
      ++rounds; ++wclock;
      const bool dense = big && r > 1u;                        // (shorter lists went to the queue): through the summaries
      if (dense) {                                             // bring the summaries up to date first, then evaluate through them
        if (tid == 0) ++sh.dense_rounds;
        if (nf < nE / 4u) {                                    // few flips: only the targets of last round's flips
          for (unsigned q = gwarp; q < nf; q += gwarps) {
            const unsigned i = __ldcg(&a.F[in][q]);
            const uint32_t p = __ldcg(&E[i]);
            int x, y, z; x_coords(a, p, x, y, z);
            x_refresh_summaries(a, sh, lane, i, p, x, y, z);
          }
        } else {
          ++sclock;
          for (unsigned i = gwarp; i < nE; i += gwarps) { int x, y, z; x_coords(a, __ldcg(&E[i]), x, y, z); x_claim_summaries(a, sh, lane, x, y, z, sclock); }
        }
        x_gsync(&ctl->bar, sh.bar_target);
      }
      const uint32_t *wl = a.W[in];
      const long long t_w0 = DBG ? clock64() : 0;
      for (unsigned q = gwarp; q < nw; q += gwarps) {
        const unsigned i = r == 1u ? q : __ldcg(&wl[q]);
        const uint32_t p = __ldcg(&E[i]);
        int x, y, z; x_coords(a, p, x, y, z);
        if (!big) {                                            // gathering evaluation: everything from one staged round of loads
          x_stage(a, sh, stg, lane, x, y, z);
          const unsigned long long old = stg.w[0], nw2 = x_eval_nb(a, sh, stg, lane, gen, i, x, y, z);
          if (nw2 == old) continue;
          if (lane == 0) a.MB[p] = nw2;                        // flip
          x_list_affected_nb(a, stg, lane, i, (x_mb_kind(old) == X_PUSH || x_mb_kind(nw2) == X_PUSH) ? (unsigned)X_NOFF : 25u, wclock, out);
          continue;
        }
        unsigned long long old = 0;
        if (lane == 0) old = __ldcg(&a.MB[p]);
        const unsigned long long nb = x_eval<true>(a, sh, lane, gen, i, p, x, y, z);
        old = __shfl_sync(0xffffffffu, old, 0);
        if (nb == old) continue;
        if (lane == 0) {                                       // flip
          a.MB[p] = nb;
          a.F[out][atomicAdd(&ctl->nF[out], 1u)] = i;
        }
        // later elements whose inputs this element can touch: a pushing element offers to its 24 neighbours, which the elements
        // within the 129 offsets a+b read; a flip between "stale" and "pulls" (or of the pulled code) only changes the
        // element's offer to its own voxel, which only its 24 neighbours read (the table starts with 0 and dirs_)
        x_list_affected(a, sh, lane, i, x, y, z, (x_mb_kind(old) == X_PUSH || x_mb_kind(nb) == X_PUSH) ? (unsigned)X_NOFF : 25u, wclock, out);
      }
      if (DBG) { __syncthreads(); if (tid == 0) atomicMax(&a.dbg[XDBG_WMAX + ((sh.rounds + rounds) & 4095u)], (unsigned long long)(clock64() - t_w0)); }
      x_gsync(&ctl->bar, sh.bar_target);
      X_LAP(big ? (r == 1u ? 1 : 3) : (r == 1u ? 6 : 7));
      if (DBG && gtid == 0) {
        if (sh.generations <= 2u && rounds <= 512u) a.dbg[XDBG_ROUNDS + (sh.generations - 1u) * 512u + (rounds - 1u)] = nw;
        // the round's longest CTA work time and list length, summed per category: the rest of the category's time is barrier
        // and waiting for the slowest CTA
        const unsigned cat = big ? (r == 1u ? 1u : 3u) : (r == 1u ? 6u : 7u);
        unsigned long long *wm = &a.dbg[XDBG_WMAX + ((sh.rounds + rounds) & 4095u)];
        a.dbg[FB_XDBG_WORK + 2 * cat] += __ldcg(wm); a.dbg[FB_XDBG_WORK + 2 * cat + 1] += nw; *wm = 0;
        if (cat == 7u) a.dbg[FB_XDBG_NWH + 32u + (nw ? 32u - __clz(nw) : 0u)] += 1ull;
      }
    }
    if (tid == 0) sh.rounds += rounds;
    if (rounds > X_MAX_ROUNDS || aborted) break;

    // ---- commit: per-element masks of owned slots, winner counts per CTA (CTA-contiguous ranges keep the order)
    const unsigned per = (nE + G - 1u) / G;
    const unsigned lo = min(nE, b * per), hi = min(nE, lo + per);
    unsigned wcount = 0, wlive = 0;
    for (unsigned i = lo + wid; i < hi; i += XW) {
      const uint32_t p = __ldcg(&E[i]);
      int x, y, z; x_coords(a, p, x, y, z);
      unsigned long long w = 0;
      if (!big) { x_stage(a, sh, stg, lane, x, y, z); w = stg.w[0]; }
      else { if (lane == 0) w = __ldcg(&a.MB[p]); w = __shfl_sync(0xffffffffu, w, 0); }
      const unsigned long long kind = x_mb_kind(w);
      bool win = false;
      if ((kind == X_PUSH && lane < 24) || (kind == X_PULL && lane == 24)) {
        int dx, dy, dz; x_unpack_off(sh.dir[lane], dx, dy, dz);
        const int nx = x + dx, ny = y + dy, nz = z + dz;
        if (x_in_grid(g, nx, ny, nz) && (lane == 24 || x_in_range(g, nx, ny, nz))) {
          const unsigned ts = i * 32u + lane;
          if (big) win = __ldcg(&a.SUM[x_vi(g, nx, ny, nz)]).y == ts;
          else {
            uint32_t snap;
            const XState f = x_state_nb(g, sh, stg, lane, nx, ny, nz, XNONE, snap);
            win = f.ts == ts;
            if (win) a.slotc[ts] = f.c;
          }
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, win);
      if (lane == 0) { a.emask[i] = m; wcount += __popc(m); wlive += kind != X_DEAD ? 1u : 0u; }
    }
    // (the words of this generation are retired in the apply phase: SMALL-mode commits still gather from them here)
    if (lane == 0) { sh.red[wid] = wcount; sh.red2[wid] = wlive; }
    __syncthreads();
    if (wid == 0) {
      unsigned c = sh.red[lane], l = sh.red2[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { c += __shfl_xor_sync(0xffffffffu, c, o); l += __shfl_xor_sync(0xffffffffu, l, o); }
      if (lane == 0) { ctl->partial[b] = c; if (l) atomicAdd(&ctl->expansions, (unsigned long long)l); }   // `times++` (:347)
    }
    if (gtid == 0) { ctl->nW[0] = ctl->nW[1] = ctl->nW[2] = 0; ctl->nF[0] = ctl->nF[1] = ctl->nF[2] = 0; }
    x_gsync(&ctl->bar, sh.bar_target);
    X_LAP(big ? 4 : 8);

    // ---- apply: exclusive scan of the counts -> queue positions of the next generation; words + targets of the new entries
    if (wid == 0) {
      unsigned before = 0, all = 0;
      for (unsigned k = lane; k < G; k += 32u) { const unsigned c = __ldcg(&ctl->partial[k]); all += c; if (k < b) before += c; }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { before += __shfl_xor_sync(0xffffffffu, before, o); all += __shfl_xor_sync(0xffffffffu, all, o); }
      if (lane == 0) { sh.base = before; sh.total = all; }
    }
    __syncthreads();
    const unsigned n2 = sh.total;
    const bool big2 = n2 > a.small_max;
    uint32_t *En = a.E[cur ^ 1];
    unsigned run = sh.base;                                    // queue position of the first winner of the current chunk
    for (unsigned i0 = lo; i0 < hi; i0 += XT) {
      const unsigned i = i0 + tid;
      const uint32_t m = i < hi ? __ldcg(&a.emask[i]) : 0u;
      if (i < hi) {                                            // retire the old entry's word unless a new entry already replaced it
        const uint32_t p = __ldcg(&E[i]);
        const unsigned long long w = __ldcg(&a.MB[p]);
        if (w != XMB_NONE && x_mb_par(w) == (gen & 1u)) atomicCAS(&a.MB[p], w, XMB_NONE);
      }
      unsigned ctot;
      unsigned r = run + x_block_scan(sh, (unsigned)__popc(m), lane, wid, ctot);
      if (m) {                                                 // this thread's element owns slots: records, link times, words of the new entries
        const uint32_t p = __ldcg(&E[i]);
        int x, y, z; x_coords(a, p, x, y, z);
        uint32_t me = m;
        while (me) {
          const int k = __ffs(me) - 1; me &= me - 1u;
          int dx, dy, dz; x_unpack_off(sh.dir[k], dx, dy, dz);
          const uint32_t v = (uint32_t)x_vi(g, x + dx, y + dy, z + dz);
          const unsigned ts = i * 32u + (unsigned)k;
          const uint32_t code = big ? __ldcg(&a.SUM[v]).z : __ldcg(&a.slotc[ts]);
          a.cobs[v] = code;
          a.LS[v] = tclock + ts;                               // every accepted write relinks the voxel at its list's front (:24-42)
          En[r] = v;
          a.MB[v] = x_mb(gen + 1u, r, X_PUSH, code);
          ++r;
        }
      }
      run += ctot;
    }
    if (DBG && gtid == 0 && sh.generations <= FB_XDBG_GENS) { a.dbg[3 * (sh.generations - 1u)] = nE; a.dbg[3 * (sh.generations - 1u) + 1] = rounds; a.dbg[3 * (sh.generations - 1u) + 2] = (unsigned long long)(clock64() - t_gen); }
    tclock += (unsigned long long)nE * 32ull + 1ull;
    if (tid == 0) sh.changed += n2;
    if (n2 >= (1u << 27)) { if (gtid == 0) ctl->err = 1u; break; }
    const bool was_big = big;
    nE = n2; cur ^= 1; big = big2; ++gen;
    x_gsync(&ctl->bar, sh.bar_target);
    X_LAP(was_big ? 5 : 9);
  }
  if (gtid == 0) {
    ctl->gen_id = gen; ctl->wclock = wclock; ctl->tclock = tclock; ctl->sclock = sclock;
    ctl->generations = sh.generations; ctl->rounds = sh.rounds; ctl->dense_rounds = sh.dense_rounds; ctl->voxels_changed = sh.changed;
  }
}

static bool g_off_ready = false;
cudaError_t fb_xrelax_init() {
  if (g_off_ready) return cudaSuccess;
  static const int D[24][3] = {
      {-1, 0, 0}, {1, 0, 0}, {0, -1, 0}, {0, 1, 0}, {0, 0, -1}, {0, 0, 1},
      {-1, -1, 0}, {1, 1, 0}, {0, -1, -1}, {0, 1, 1}, {-1, 0, -1}, {1, 0, 1},
      {-1, 1, 0}, {1, -1, 0}, {0, -1, 1}, {0, 1, -1}, {1, 0, -1}, {-1, 0, 1},
      {-2, 0, 0}, {2, 0, 0}, {0, -2, 0}, {0, 2, 0}, {0, 0, -2}, {0, 0, 2}};
  int off[1024], n = 0;
  for (int p = -1; p < 24; ++p)
    for (int q = -1; q < 24; ++q) {
      int o[3];
      for (int k = 0; k < 3; ++k) o[k] = (p < 0 ? 0 : D[p][k]) + (q < 0 ? 0 : D[q][k]);
      const int code = (o[0] + 4) | ((o[1] + 4) << 4) | ((o[2] + 4) << 8);
      bool dup = false;
      for (int j = 0; j < n; ++j) dup = dup || off[j] == code;
      if (!dup) off[n++] = code;
    }
  if (n != X_NOFF) return cudaErrorUnknown;
  cudaError_t e = cudaMemcpyToSymbol(x_off_c, off, sizeof(int) * X_NOFF);
  if (e == cudaSuccess) g_off_ready = true;
  return e;
}

int fb_xrelax_blocks(int device) {
  int per_sm = 0, sms = 0;
  for (const void *k : {(const void *)k_x_relax<false>, (const void *)k_x_relax<true>})
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, XT, sizeof(XNb) * XW) != cudaSuccess || per_sm < 1) return -1;
  for (const void *k : {(const void *)k_x_reseed<false>, (const void *)k_x_reseed<true>})
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, XT, 0) != cudaSuccess || per_sm < 1) return -1;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return -1;
  return sms;                                                  // one CTA per SM: the barrier is cheapest with few arrivals
}

cudaError_t fb_xrelax_launch(FbExact *X, const FbGeom &g, uint32_t *cobs, const uint32_t *deps, unsigned ndep, uint32_t *ord, uint32_t *nc, uint32_t *M,
                             const uint32_t *occbits, unsigned long long ls_deps, unsigned long long *dbg, cudaStream_t s) {
  XArgs a;
  a.deps = deps; a.ndep = ndep; a.ord = ord; a.nc = nc; a.M = M; a.occbits = occbits; a.ls_deps = ls_deps;
  fb_div_make((unsigned)g.pz, a.div_pz_m, a.div_pz_s);
  fb_div_make((unsigned)g.gy, a.div_gy_m, a.div_gy_s);
  a.g = g;
  if (a.g.max_vec[0] < a.g.min_vec[0] || a.g.max_vec[1] < a.g.min_vec[1] || a.g.max_vec[2] < a.g.min_vec[2])
    for (int k = 0; k < 3; ++k) a.g.min_vec[k] = a.g.max_vec[k] = 0x3fffffff;      // empty update box: VoxInRange is false everywhere (x_in_range)
  a.cobs = cobs; a.MB = X->MB; a.LS = X->LS; a.SUM = X->SUM; a.SUMg = X->SUMg;
  a.E[0] = X->E[0]; a.E[1] = X->E[1]; a.emask = X->emask;
  for (int k = 0; k < 3; ++k) { a.W[k] = X->W[k]; a.F[k] = X->F[k]; }
  a.wstamp = X->wstamp; a.slotc = X->slotc; a.ctl = X->d_ctl; a.small_max = X->small_max; a.dense_min = X->dense_min; a.dbg = dbg;
  void *args[] = {(void *)&a};
  if (ndep) {
    const cudaError_t e = cudaLaunchCooperativeKernel(dbg ? (void *)k_x_reseed<true> : (void *)k_x_reseed<false>, dim3(X->relax_blocks), dim3(XT), args, 0, s);
    if (e != cudaSuccess) return e;
  }
  return cudaLaunchCooperativeKernel(dbg ? (void *)k_x_relax<true> : (void *)k_x_relax<false>, dim3(X->relax_blocks), dim3(XT), args, sizeof(XNb) * XW, s);
}
