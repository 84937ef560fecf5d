// fiesta_b200 -- cost matrices between many points through free space (definition: fb_nav.h, DESIGN.md §3.9).
//
// k_navm_trav   : M := bit 13 on the traversable box voxels (fb_seg_blocks, as k_nav_init), 0 elsewhere.
// k_navm_mask   : M := fb_nav_move_bits of each traversable voxel, from bit 13 of its 26 neighbours' words.
// k_navm_locate : status and box index of each source and target.
// k_navm_fill   : D := +inf on the channels of a pass.
// k_navm_place  : D_c := 0 on source c's voxel; the tiles k_nav_goals would queue for it are queued in channel c.
// k_navm_relax  : k_nav_relax over (channel, tile) work items, all channels of a pass in one list, one grid barrier per
//                 generation.  Moves come from M, so a channel's field only holds +inf and reached costs.  A channel retires, and
//                 its work items are dropped, once every status-0 target reads D_c <= m_c(g - 1), the least value written in channel
//                 c in the previous generation (proof: DESIGN.md §3.9).
// k_navm_gather : cost rows of a pass: D_c at the status-0 targets, NaN at the others; or NaN rows for the sources not placed.
//
// Exactness is k_nav_relax's argument per channel: every stored value is the left fold of a path from the source, values only
// decrease, a decrease of a boundary voxel queues every tile that holds one of its neighbours, and the least fixpoint does not
// depend on the schedule.  Retirement only drops work whose writes could not reach a target any more.
#include <cooperative_groups.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "fb_nav.cuh"
#include "fb_segment.h"

namespace cg = cooperative_groups;

#define NAVM_THREADS 512       // one thread per voxel of an 8^3 tile
#define NAVM_H (FB_TILE + 2)   // staged tile + 1-voxel halo per axis
#define NAVM_NONE 0xffffffffu
#define NAVM_TRAV (1u << 13)

__device__ __forceinline__ void navm_coords(const FbNavBox &b, long long i, int &x, int &y, int &z) {
  z = (int)(i % b.n[2]); y = (int)(i / b.n[2] % b.n[1]); x = (int)(i / ((long long)b.n[2] * b.n[1]));
}

__global__ void k_navm_trav(FbGeom g, const uint32_t *__restrict__ cobs, FbNavBox b, double r, int unknown_blocks, uint32_t *M) {
  const long long n = (long long)b.n[0] * b.n[1] * b.n[2];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int x, y, z;
    navm_coords(b, i, x, y, z);
    const int v[3] = {b.lo[0] + x, b.lo[1] + y, b.lo[2] + z};
    double d;
    M[i] = fb_seg_blocks(g, cobs, v, r, unknown_blocks != 0, d) ? 0u : NAVM_TRAV;
  }
}

// In place: a thread rewrites only its own word and keeps its bit 13, the only bit any thread reads, and an aligned 32-bit access
// does not tear, so every read sees the bit k_navm_trav wrote.
__global__ void k_navm_mask(FbNavBox b, uint32_t *M) {
  const long long n = (long long)b.n[0] * b.n[1] * b.n[2];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (!(M[i] & NAVM_TRAV)) continue;
    int x, y, z;
    navm_coords(b, i, x, y, z);
    unsigned nb = 0;
    for (int e = 0; e < 27; ++e) {
      int d[3];
      fb_nav_dir(e, d);
      if (fb_nav_in_box(b, x + d[0], y + d[1], z + d[2]) && (M[fb_nav_idx(b, x + d[0], y + d[1], z + d[2])] & NAVM_TRAV)) nb |= 1u << e;
    }
    M[i] = fb_nav_move_bits(nb);
  }
}

__global__ void k_navm_locate(FbGeom g, FbNavBox b, const uint32_t *__restrict__ M, const double *__restrict__ pts, long long n,
                              int32_t *status, long long *idx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int v[3];
  if (!fb_pos_in_map(g, pts + 3 * i) || !fb_nav_locate(g, b, pts + 3 * i, v)) {   // NaN fails fb_nav_locate
    status[i] = FB_NAVM_OUTSIDE; idx[i] = -1;
    return;
  }
  const long long ii = fb_nav_idx(b, v[0], v[1], v[2]);
  const bool ok = (M[ii] & NAVM_TRAV) != 0;
  status[i] = ok ? FB_NAVM_PLACED : FB_NAVM_BLOCKED;
  idx[i] = ok ? ii : -1;
}

__global__ void k_navm_fill(double *D, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) D[i] = (double)INFINITY;
}

__global__ void k_navm_place(FbNavMArgs a, const long long *__restrict__ src_idx) {
  const int c = threadIdx.x;
  if (c >= a.nch) return;
  FbNavMCtr *ctr = a.ctr;
  const long long ii = src_idx[c];
  int v[3];
  navm_coords(a.b, ii, v[0], v[1], v[2]);
  a.D[(long long)c * a.nv + ii] = 0.0;
  // placement is a write of 0 in "generation -1" (slot 2); generations 0 and 1 start from +inf
  ctr->mmin[c][0] = ctr->mmin[c][1] = 0x7ff0000000000000ull;
  ctr->mmin[c][2] = 0ull;
  // the tiles k_nav_goals queues: the voxel's own tile and those across every tile face, edge or corner it lies on
  const int tc[3] = {v[0] >> 3, v[1] >> 3, v[2] >> 3};
  for (int ox = ((v[0] & 7) == 0 ? -1 : 0); ox <= ((v[0] & 7) == FB_TILE - 1 ? 1 : 0); ++ox)
    for (int oy = ((v[1] & 7) == 0 ? -1 : 0); oy <= ((v[1] & 7) == FB_TILE - 1 ? 1 : 0); ++oy)
      for (int oz = ((v[2] & 7) == 0 ? -1 : 0); oz <= ((v[2] & 7) == FB_TILE - 1 ? 1 : 0); ++oz) {
        const int nx = tc[0] + ox, ny = tc[1] + oy, nz = tc[2] + oz;
        if (nx < 0 || nx >= a.tn[0] || ny < 0 || ny >= a.tn[1] || nz < 0 || nz >= a.tn[2]) continue;
        const unsigned item = (unsigned)c * a.nt + (unsigned)((nx * a.tn[1] + ny) * a.tn[2] + nz);
        a.stamp[item] = 1u;                                                 // generation 0 has stamp 1; one thread per channel
        a.list[0][atomicAdd(&ctr->n[0], 1u)] = item;
        ++ctr->queued[c][0];
      }
}

// Block 0, at the start of generation g: retire every channel whose status-0 targets all read D_c <= m_c(g - 1).  m_c(g - 1) is
// complete (the barrier that ended g - 1 is behind), and D only decreases, so a later read is as good.  Also clears the per-channel
// slots that generation g + 1 writes (m) and counts into (queued) -- both last read at the start of generation g - 1.
__device__ void navm_retire(const FbNavMArgs &a, unsigned gen, unsigned *s_open) {
  const int tid = threadIdx.x;
  FbNavMCtr *ctr = a.ctr;
  const unsigned prev = (gen + 2u) % 3u;
  if (tid < a.nch) s_open[tid] = __ldcg(&ctr->retired[tid]);
  __syncthreads();
  for (int i = tid; i < a.nch * a.n_tgt; i += NAVM_THREADS) {
    const int c = i / a.n_tgt;
    if (s_open[c] & 1u) continue;
    const double m = __longlong_as_double((long long)__ldcg(&ctr->mmin[c][prev]));
    if (!(__ldcg(&a.D[(long long)c * a.nv + a.tgt[i - c * a.n_tgt]]) <= m)) s_open[c] = 2u;
  }
  __syncthreads();
  if (tid < a.nch) {
    if (s_open[tid] == 0u) {
      ctr->retired[tid] = 1u;
      if (__ldcg(&ctr->queued[tid][gen % 3u]) != 0u) atomicAdd(&a.tot->retired_early, 1ull);   // work was left in its list
    }
    ctr->mmin[tid][(gen + 1u) % 3u] = 0x7ff0000000000000ull;
    ctr->queued[tid][(gen + 2u) % 3u] = 0u;
  }
}

__global__ void __launch_bounds__(NAVM_THREADS, 2) k_navm_relax(FbNavMArgs a) {
  __shared__ double sD[NAVM_H * NAVM_H * NAVM_H];
  __shared__ unsigned s_item, s_q, s_open[FB_NAVM_CH];
  __shared__ unsigned long long s_min;
  cg::grid_group grid = cg::this_grid();
  FbNavMCtr *ctr = a.ctr;
  const int tid = threadIdx.x, lx = tid >> 6, ly = (tid >> 3) & 7, lz = tid & 7;
  const int c = ((lx + 1) * NAVM_H + ly + 1) * NAVM_H + lz + 1;
  const double w1 = a.w[0], w2 = a.w[1], w3 = a.w[2];
  unsigned long long visits = 0;
  unsigned gen = 0;
  for (;; ++gen) {                                                      // counters rotate as in k_nav_relax
    const unsigned cur = gen % 3u, nxt = (gen + 1u) % 3u;
    const unsigned nwork = __ldcg(&ctr->n[cur]);
    if (nwork == 0) break;
    if (blockIdx.x == 0) {
      if (tid == 0) { ctr->n[(gen + 2u) % 3u] = 0; ctr->next[(gen + 2u) % 3u] = 0; }
      navm_retire(a, gen, s_open);
    }
    const uint32_t *list = (gen & 1u) ? a.list[1] : a.list[0];
    uint32_t *out = (gen & 1u) ? a.list[0] : a.list[1];
    const unsigned stamp_next = gen + 2u;
    for (;;) {
      if (tid == 0) {
        unsigned item;
        for (;;) {                                                      // items of retired channels are dropped
          const unsigned w = atomicAdd(&ctr->next[cur], 1u);
          item = w < nwork ? __ldcg(&list[w]) : NAVM_NONE;
          if (item == NAVM_NONE || !__ldcg(&ctr->retired[item / a.nt])) break;
        }
        s_item = item;
        s_q = 0;
        s_min = ~0ull;
      }
      __syncthreads();
      const unsigned item = s_item;
      if (item == NAVM_NONE) break;
      if (tid == 0) ++visits;
      const unsigned ch = item / a.nt, tile = item - ch * a.nt;
      double *D = a.D + (long long)ch * a.nv;
      const int tz = (int)(tile % (unsigned)a.tn[2]), ty = (int)(tile / (unsigned)a.tn[2] % (unsigned)a.tn[1]),
                tx = (int)(tile / (unsigned)(a.tn[2] * a.tn[1]));
      const int x0 = tx * FB_TILE - 1, y0 = ty * FB_TILE - 1, z0 = tz * FB_TILE - 1;
      for (int i = tid; i < NAVM_H * NAVM_H * NAVM_H; i += NAVM_THREADS) {
        const int x = x0 + i / (NAVM_H * NAVM_H), y = y0 + i / NAVM_H % NAVM_H, z = z0 + i % NAVM_H;
        sD[i] = fb_nav_in_box(a.b, x, y, z) ? __ldcg(&D[fb_nav_idx(a.b, x, y, z)]) : (double)INFINITY;   // never read through a move
      }
      const int x = tx * FB_TILE + lx, y = ty * FB_TILE + ly, z = tz * FB_TILE + lz;
      const bool in = fb_nav_in_box(a.b, x, y, z);
      const unsigned allowed = in ? __ldg(&a.M[fb_nav_idx(a.b, x, y, z)]) : 0u;
      __syncthreads();
      const double orig = sD[c];
      double my = orig;
      for (;;) {                                                        // local fixpoint of the tile
        double best = my;
#pragma unroll
        for (int k = 0; k < 27; ++k) {
          if (k == 13) continue;
          const int dx = k / 9 - 1, dy = k / 3 % 3 - 1, dz = k % 3 - 1, nz = (dx != 0) + (dy != 0) + (dz != 0);
          if (allowed & (1u << k)) {
            const double cand = sD[c + (dx * NAVM_H + dy) * NAVM_H + dz] + (nz == 1 ? w1 : nz == 2 ? w2 : w3);
            if (cand < best) best = cand;
          }
        }
        const bool chg = best < my;
        if (chg) { my = best; sD[c] = best; }
        if (!__syncthreads_or(chg)) break;
      }
      const bool improved = my < orig;
      if (improved) {
        __stcg(&D[fb_nav_idx(a.b, x, y, z)], my);
        unsigned q = 0;
        for (int ox = (lx == 0 ? -1 : 0); ox <= (lx == FB_TILE - 1 ? 1 : 0); ++ox)
          for (int oy = (ly == 0 ? -1 : 0); oy <= (ly == FB_TILE - 1 ? 1 : 0); ++oy)
            for (int oz = (lz == 0 ? -1 : 0); oz <= (lz == FB_TILE - 1 ? 1 : 0); ++oz) q |= 1u << ((ox + 1) * 9 + (oy + 1) * 3 + oz + 1);
        q &= ~(1u << 13);
        if (q) atomicOr(&s_q, q);
      }
      // m_c(gen): non-negative doubles order like their bit patterns
      unsigned long long bits = improved ? (unsigned long long)__double_as_longlong(my) : ~0ull;
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const unsigned long long ob = __shfl_xor_sync(0xffffffffu, bits, o);
        bits = ob < bits ? ob : bits;
      }
      if ((tid & 31) == 0 && bits != ~0ull) atomicMin(&s_min, bits);
      __syncthreads();
      if (tid < 27 && ((s_q >> tid) & 1u)) {
        const int nx = tx + tid / 9 - 1, ny = ty + tid / 3 % 3 - 1, nz = tz + tid % 3 - 1;
        if (nx >= 0 && nx < a.tn[0] && ny >= 0 && ny < a.tn[1] && nz >= 0 && nz < a.tn[2]) {
          const unsigned t = ch * a.nt + (unsigned)((nx * a.tn[1] + ny) * a.tn[2] + nz);
          if (atomicExch(&a.stamp[t], stamp_next) != stamp_next) {
            out[atomicAdd(&ctr->n[nxt], 1u)] = t;
            atomicAdd(&ctr->queued[ch][nxt], 1u);
          }
        }
      }
      if (tid == 32 && s_min != ~0ull) atomicMin(&ctr->mmin[ch][cur], s_min);
      __syncthreads();                                                  // s_item, s_q and s_min are rewritten for the next item
    }
    grid.sync();
  }
  if (tid == 0) {
    if (visits) atomicAdd(&a.tot->tile_visits, visits);
    if (blockIdx.x == 0) atomicAdd(&a.tot->generations, (unsigned long long)gen);
  }
}

__global__ void k_navm_gather(const double *__restrict__ D, long long nv, const int32_t *__restrict__ rows, long long n_rows,
                              const long long *__restrict__ tgt_idx, long long n_tgt, double *cost) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows * n_tgt) return;
  const long long c = i / n_tgt, j = i - c * n_tgt, t = tgt_idx[j];
  cost[(long long)rows[c] * n_tgt + j] = D && t >= 0 ? D[c * nv + t] : nan("");
}

// ---------------------------------------------------------------- host side
static unsigned navm_blocks(long long n) {
  const long long want = (n + 255) / 256;
  return (unsigned)(want < FB_SMS * 16ll ? want : FB_SMS * 16ll);
}

int fb_navm_relax_blocks(int device) {
  int per_sm = 0, sms = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_navm_relax, NAVM_THREADS, 0) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return 0;
  return per_sm * sms;                                                  // every block co-resident: required by grid.sync()
}

// 2 launches, 3 with points
static cudaError_t navm_locate(const FbGeom &g, const uint32_t *cobs, const FbNavBox &b, double r, int unknown_blocks, uint32_t *M,
                               const double *pts, long long n, int32_t *status, long long *idx, cudaStream_t s) {
  const long long nv = (long long)b.n[0] * b.n[1] * b.n[2];
  k_navm_trav<<<navm_blocks(nv), 256, 0, s>>>(g, cobs, b, r, unknown_blocks, M);
  k_navm_mask<<<navm_blocks(nv), 256, 0, s>>>(b, M);
  if (n > 0) k_navm_locate<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(g, b, M, pts, n, status, idx);
  return cudaGetLastError();
}

// One pass, 3 launches: a.nch channels, sources src_idx[0 .. nch); expects ctr zeroed and stamp zeroed on the pass's items.
static cudaError_t navm_pass(const FbNavMArgs &a, const long long *src_idx, int nblocks, cudaStream_t s) {
  k_navm_fill<<<navm_blocks(a.nch * a.nv), 256, 0, s>>>(a.D, a.nch * a.nv);
  k_navm_place<<<1, FB_NAVM_CH, 0, s>>>(a, src_idx);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  void *args[] = {(void *)&a};
  return cudaLaunchCooperativeKernel((void *)k_navm_relax, dim3(nblocks), dim3(NAVM_THREADS), args, 0, s);
}

static cudaError_t navm_gather(const double *D, long long nv, const int32_t *rows, long long n_rows, const long long *tgt_idx,
                               long long n_tgt, double *cost, cudaStream_t s) {
  const long long n = n_rows * n_tgt;
  if (n <= 0) return cudaSuccess;
  k_navm_gather<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(D, nv, rows, n_rows, tgt_idx, n_tgt, cost);
  return cudaGetLastError();
}

// ---------------------------------------------------------------- entry point (include/fiesta_b200.h)
int fiesta_nav_matrix(fiesta_nav_field *f, const int box_lo[3], const int box_hi[3], const double *sources_xyz, int64_t n_src,
                      const double *targets_xyz, int64_t n_tgt, double clearance, int flags, int32_t *src_status, int32_t *tgt_status,
                      double *cost, fiesta_nav_matrix_stats *stats) {
  const char *fn = "fiesta_nav_matrix";
  if (!f || !box_lo || !box_hi) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  if (n_src < 0 || n_tgt < 0 || (n_src > 0 && !(sources_xyz && src_status)) || (n_tgt > 0 && !(targets_xyz && tgt_status)) ||
      (n_src > 0 && n_tgt > 0 && !cost)) {
    fb_set_error("%s: negative count or null buffer", fn);
    return FIESTA_ERR_INVALID;
  }
  if (!clearance_flags_ok(fn, clearance, flags)) return FIESTA_ERR_INVALID;
  fiesta_map *m = f->m;
  FbNavMArgs a{};
  if (!box_arg(fn, m->g, box_lo, box_hi, &a.b)) return FIESTA_ERR_INVALID;
  for (int k = 0; k < 3; ++k) {
    a.tn[k] = (a.b.n[k] + FB_TILE - 1) / FB_TILE;
    a.w[k] = f->w[k];
  }
  if (n_src > 0 && n_tgt > 0 && n_src >= ((1ll << 31) + n_tgt - 1) / n_tgt) {
    fb_set_error("%s: n_src * n_tgt must be below 2^31", fn);
    return FIESTA_ERR_LIMIT;
  }
  const long long nv = (long long)a.b.n[0] * a.b.n[1] * a.b.n[2], nt = (long long)a.tn[0] * a.tn[1] * a.tn[2], np = n_src + n_tgt;
  a.nv = nv;
  a.nt = (unsigned)nt;
  cudaStream_t s = m->stream;
  CK(cudaSetDevice(m->device));
  // (1) move masks, statuses and box indices of every point; the statuses and indices come back for the host to plan the passes
  cudaError_t e = f->M.grow((size_t)nv, s);
  if (e == cudaSuccess && np > 0) e = f->m_pts.grow((size_t)np * 3, s);
  if (e == cudaSuccess && np > 0) e = f->m_st.grow((size_t)np, s);
  if (e == cudaSuccess && np > 0) e = f->m_idx.grow((size_t)np, s);
  if (e != cudaSuccess) return alloc_failed(e, "%s: cannot allocate the move masks of %lld voxels", fn, nv);
  CK(cudaEventRecord(f->ev[0], s));
  if (n_src > 0) CK(cudaMemcpyAsync(f->m_pts, sources_xyz, (size_t)n_src * 24, cudaMemcpyHostToDevice, s));
  if (n_tgt > 0) CK(cudaMemcpyAsync(f->m_pts + 3 * n_src, targets_xyz, (size_t)n_tgt * 24, cudaMemcpyHostToDevice, s));
  CK(navm_locate(m->g, m->cobs, a.b, clearance, flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS, f->M, f->m_pts, np, f->m_st, f->m_idx, s));
  m->st.kernel_launches += np > 0 ? 3 : 2;
  std::vector<int32_t> st((size_t)np);
  std::vector<long long> idx((size_t)np);
  if (np > 0) {
    CK(cudaMemcpyAsync(st.data(), f->m_st, (size_t)np * 4, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(idx.data(), f->m_idx, (size_t)np * 8, cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  // rows: the placed sources in index order (channel k of the passes is placed source k), then the others (NaN rows)
  std::vector<int32_t> rows;
  std::vector<long long> src, tgt;
  long long n_ps = 0;
  for (long long i = 0; i < n_src; ++i) n_ps += st[i] == FB_NAVM_PLACED;
  if (n_tgt > 0) {                                                         // then n_src < 2^31
    for (long long i = 0; i < n_src; ++i)
      if (st[i] == FB_NAVM_PLACED) { rows.push_back((int32_t)i); src.push_back(idx[i]); }
    for (long long i = 0; i < n_src; ++i)
      if (st[i] != FB_NAVM_PLACED) rows.push_back((int32_t)i);
  }
  for (long long j = n_src; j < np; ++j)
    if (st[j] == FB_NAVM_PLACED) tgt.push_back(idx[j]);
  const long long n_pt = (long long)tgt.size();
  // (2) passes of C channels: C = min(32, sources left, max(1, floor(2^32 B / (8 B x box voxels))))
  const long long per_pass = std::max(1ll, std::min((long long)FB_NAVM_CH, (1ll << 32) / (8 * nv)));
  const long long C = std::min(per_pass, n_ps);
  const bool work = n_ps > 0 && n_pt > 0;
  if (work && C * nt >= (long long)0xffffffffu) {
    fb_set_error("%s: the box has too many tiles", fn);
    return FIESTA_ERR_LIMIT;
  }
  e = cudaSuccess;
  if (n_src > 0 && n_tgt > 0) e = f->m_cost.grow((size_t)(n_src * n_tgt), s);
  if (e == cudaSuccess && n_src > 0 && n_tgt > 0) e = f->m_rows.grow((size_t)n_src, s);
  if (work) {
    if (e == cudaSuccess) e = f->MD.grow((size_t)(C * nv), s);
    for (FbDevBuf<uint32_t> *b : {&f->m_stamp, &f->m_list[0], &f->m_list[1]})
      if (e == cudaSuccess) e = b->grow((size_t)(C * nt), s);
    if (e == cudaSuccess) e = f->m_src.grow((size_t)n_ps, s);
    if (e == cudaSuccess) e = f->m_tgt.grow((size_t)n_pt, s);
  }
  if (e != cudaSuccess)
    return alloc_failed(e, "%s: cannot allocate %lld fields of %lld voxels and the %lld x %lld matrix", fn, C, nv, (long long)n_src, (long long)n_tgt);
  if (n_src > 0 && n_tgt > 0) CK(cudaMemcpyAsync(f->m_rows, rows.data(), (size_t)n_src * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(f->m_tot, 0, sizeof(FbNavMTot), s));
  long long passes = 0;
  if (work) {
    CK(cudaMemcpyAsync(f->m_src, src.data(), (size_t)n_ps * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(f->m_tgt, tgt.data(), (size_t)n_pt * 8, cudaMemcpyHostToDevice, s));
    a.D = f->MD; a.M = f->M; a.stamp = f->m_stamp; a.list[0] = f->m_list[0]; a.list[1] = f->m_list[1];
    a.ctr = f->m_ctr; a.tot = f->m_tot; a.tgt = f->m_tgt; a.n_tgt = (int)n_pt;
    for (long long p0 = 0; p0 < n_ps; p0 += C, ++passes) {
      a.nch = (int)std::min(C, n_ps - p0);
      CK(cudaMemsetAsync(f->m_stamp, 0, (size_t)(a.nch * nt) * 4, s));
      CK(cudaMemsetAsync(f->m_ctr, 0, sizeof(FbNavMCtr), s));
      CK(navm_pass(a, f->m_src + p0, f->mblocks, s));
      CK(navm_gather(f->MD, nv, f->m_rows + p0, a.nch, f->m_idx + n_src, n_tgt, f->m_cost, s));
      m->st.kernel_launches += 4;
    }
  }
  // NaN rows: every source when no target is placed, else the sources not placed
  const long long nan_from = work ? n_ps : 0;
  if (n_src > nan_from && n_tgt > 0) {
    CK(navm_gather(nullptr, nv, f->m_rows + nan_from, n_src - nan_from, f->m_idx + n_src, n_tgt, f->m_cost, s));
    m->st.kernel_launches++;
  }
  CK(cudaEventRecord(f->ev[1], s));
  if (n_src > 0 && n_tgt > 0) CK(cudaMemcpyAsync(cost, f->m_cost, (size_t)(n_src * n_tgt) * 8, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(f->h_mtot, f->m_tot, sizeof(FbNavMTot), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (n_src > 0) memcpy(src_status, st.data(), (size_t)n_src * 4);
  if (n_tgt > 0) memcpy(tgt_status, st.data() + n_src, (size_t)n_tgt * 4);
  if (stats) {
    const FbNavMTot &t = *f->h_mtot;
    *stats = fiesta_nav_matrix_stats{};
    stats->sources_placed = n_ps;
    stats->targets_placed = n_pt;
    stats->passes = passes;
    stats->generations = (int64_t)t.generations;
    stats->tile_visits = (int64_t)t.tile_visits;
    stats->sources_retired_early = (int64_t)t.retired_early;
    CK(cudaEventElapsedTime(&stats->ms_compute, f->ev[0], f->ev[1]));
  }
  return FIESTA_OK;
}
