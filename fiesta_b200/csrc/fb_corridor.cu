// fiesta_b200 -- safe flight corridor kernels (definition: fb_corridor.h, DESIGN.md §3.8).
//
// k_corr_mask      : one warp per z-row word of the limit box: lane l evaluates fb_seg_blocks at z = 32 * word + l; a ballot is
//                    the word.  One streaming pass over the records; the predicate is evaluated once per box voxel.
// k_corr_transpose : one warp per y-row word, gathered from the z-row bits (L2-resident), so that the layers of the +-z faces read
//                    whole words too.
// k_corr_inflate   : one warp per independent seed; k_corr_chain: one warp per path, running the chain sequentially (the boxes of
//                    a path depend on each other).  Both run the rule of fb_corr_inflate / fb_corr_chain on every lane with the
//                    same values; only the accessor's steps are spread over the lanes: a box test is a warp-strided loop over mask
//                    words with edge masks that issues CORR_BATCH loads per lane before testing any (the layer tests of one box
//                    are a dependent chain, so latency is the cost) and leaves at the first __any_sync; the forward scan for the
//                    next seed is a ballot over 32 path voxels at a time.
// Every output is a function of the masks and the sequential rule, and the statistics are integer sums: nothing depends on the
// schedule.
#include <algorithm>
#include "fb_map.h"
#include "fb_corridor.h"

#define CORR_WARPS 8
#define CORR_BATCH 4

struct FbCorrCtr {
  unsigned long long boxes, tested, grown;   // boxes written (seeds inflated), layer tests, grown layers
};

__global__ void k_corr_mask(FbGeom g, const uint32_t *__restrict__ cobs, FbCorrMask M, double r, int unknown_blocks, uint32_t *mask) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < M.zwords; w += nwarps) {
    const long long row = w / M.wz;
    const int z = (int)(w - row * M.wz) * 32 + lane;
    bool ok = false;
    if (z < M.n[2]) {
      const int v[3] = {M.lo[0] + (int)(row / M.n[1]), M.lo[1] + (int)(row % M.n[1]), M.lo[2] + z};
      double d;
      ok = !fb_seg_blocks(g, cobs, v, r, unknown_blocks != 0, d);
    }
    const unsigned b = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) mask[w] = b;
  }
}

__global__ void k_corr_transpose(FbCorrMask M, uint32_t *mask) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5), ywords = (long long)M.n[2] * M.n[0] * M.wy;
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < ywords; w += nwarps) {
    const long long row = w / M.wy;                                       // row = z * n.x + x
    const int y = (int)(w - row * M.wy) * 32 + lane, z = (int)(row / M.n[0]), x = (int)(row % M.n[0]);
    bool ok = false;
    if (y < M.n[1]) ok = (mask[((long long)x * M.n[1] + y) * M.wz + (z >> 5)] >> (z & 31)) & 1u;
    const unsigned b = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) mask[M.zwords + w] = b;
  }
}

// The warp's accessor for fb_corridor.h: every lane calls every member with the same arguments.
struct CorrWarp {
  FbCorrMask M;
  const uint32_t *mask;
  const int32_t *P;           // the path's voxels (xyz), n of them
  int n, lane;
  int32_t *o_lo, *o_hi, *o_first;

  __device__ bool box_free(const int *lo, const int *hi) const {
    int a[3], b[3];
    for (int k = 0; k < 3; ++k) { a[k] = lo[k] - M.lo[k]; b[k] = hi[k] - M.lo[k]; }
    // rows (u, v) and words along the rows' bit axis [c0, c1]: y-rows for a layer one voxel thick in z, z-rows otherwise
    const bool zl = a[2] == b[2] && b[1] > a[1];
    const uint32_t *base = zl ? mask + M.zwords : mask;
    const int u0 = zl ? a[2] : a[0], nu = zl ? 1 : b[0] - a[0] + 1;
    const int v0 = zl ? a[0] : a[1], nv = zl ? b[0] - a[0] + 1 : b[1] - a[1] + 1, vs = zl ? M.n[0] : M.n[1];
    const int c0 = zl ? a[1] : a[2], c1 = zl ? b[1] : b[2], W = zl ? M.wy : M.wz;
    const int w0 = c0 >> 5, nw = (c1 >> 5) - w0 + 1;
    const unsigned fm = ~0u << (c0 & 31), lm = ~0u >> (31 - (c1 & 31));
    const long long total = (long long)nu * nv * nw;
    for (long long t0 = 0; t0 < total; t0 += 32 * CORR_BATCH) {
      uint32_t wd[CORR_BATCH], m[CORR_BATCH];
#pragma unroll
      for (int k = 0; k < CORR_BATCH; ++k) {
        const long long t = t0 + k * 32 + lane;
        wd[k] = 0u;
        m[k] = 0u;
        if (t < total) {
          const long long rr = t / nw;
          const int wi = (int)(t - rr * nw), v = (int)(rr % nv), u = (int)(rr / nv);
          m[k] = (wi == 0 ? fm : ~0u) & (wi == nw - 1 ? lm : ~0u);
          wd[k] = __ldg(&base[((long long)(u0 + u) * vs + (v0 + v)) * W + w0 + wi]);
        }
      }
      bool bad = false;
#pragma unroll
      for (int k = 0; k < CORR_BATCH; ++k) bad |= (wd[k] & m[k]) != m[k];
      if (__any_sync(0xffffffffu, bad)) return false;
    }
    return true;
  }
  __device__ void vox(int i, int *v) const { v[0] = P[3 * i]; v[1] = P[3 * i + 1]; v[2] = P[3 * i + 2]; }
  __device__ bool outside(int i, const int *lo, const int *hi) const {
    int v[3];
    vox(i, v);
    return !fb_corr_inside(v, lo, hi);
  }
  __device__ bool any_outside(const int *lo, const int *hi) const {
    for (int b = 0; b < n; b += 32)
      if (__any_sync(0xffffffffu, b + lane < n && outside(b + lane, lo, hi))) return true;
    return false;
  }
  __device__ int next_outside(int j, const int *lo, const int *hi) const {
    for (int b = j + 1; b < n; b += 32) {
      const unsigned bits = __ballot_sync(0xffffffffu, b + lane < n && outside(b + lane, lo, hi));
      if (bits) return b + __ffs(bits) - 1;
    }
    return n;
  }
  __device__ void emit(int k, const int *lo, const int *hi, int j) const {
    if (lane != 0) return;
    for (int a = 0; a < 3; ++a) { o_lo[3 * k + a] = lo[a]; o_hi[3 * k + a] = hi[a]; }
    o_first[k] = j;
  }
};

__device__ __forceinline__ void corr_count(FbCorrCtr *ctr, int lane, unsigned long long boxes, const FbCorrCount &c) {
  if (lane != 0) return;
  if (boxes) atomicAdd(&ctr->boxes, boxes);
  if (c.tested) atomicAdd(&ctr->tested, (unsigned long long)c.tested);
  if (c.grown) atomicAdd(&ctr->grown, (unsigned long long)c.grown);
}

__global__ void __launch_bounds__(32 * CORR_WARPS) k_corr_inflate(FbCorrMask M, const uint32_t *__restrict__ mask, int3 max_steps,
                                                                  const int32_t *__restrict__ seeds, long long n, int32_t *status,
                                                                  int32_t *out_lo, int32_t *out_hi, FbCorrCtr *ctr) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n) return;                                                    // whole warps
  CorrWarp acc{M, mask, nullptr, 0, (int)(threadIdx.x & 31), nullptr, nullptr, nullptr};
  int L_lo[3], L_hi[3], lo[3], hi[3];
  const int ms[3] = {max_steps.x, max_steps.y, max_steps.z};
  for (int k = 0; k < 3; ++k) {
    L_lo[k] = M.lo[k];
    L_hi[k] = M.lo[k] + M.n[k] - 1;
    lo[k] = seeds[3 * i + k];
    hi[k] = seeds[3 * (n + i) + k];
  }
  FbCorrCount c{0, 0};
  const int st = fb_corr_seed(acc, L_lo, L_hi, ms, lo, hi, c);
  if (acc.lane == 0) {
    status[i] = st;
    for (int k = 0; k < 3; ++k) {
      out_lo[3 * i + k] = st == FB_CORR_OK ? lo[k] : -1;
      out_hi[3 * i + k] = st == FB_CORR_OK ? hi[k] : -1;
    }
  }
  corr_count(ctr, acc.lane, st == FB_CORR_OK, c);
}

__global__ void __launch_bounds__(32 * CORR_WARPS) k_corr_chain(FbCorrMask M, const uint32_t *__restrict__ mask, int3 max_steps,
                                                                const int32_t *__restrict__ P, const int64_t *__restrict__ off,
                                                                long long n_paths, int32_t *status, int32_t *n_boxes, int32_t *blocked_at,
                                                                int32_t *box_lo, int32_t *box_hi, int32_t *first, FbCorrCtr *ctr) {
  const long long p = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (p >= n_paths) return;
  const long long o = off[p];
  CorrWarp acc{M, mask, P + 3 * o, (int)(off[p + 1] - o), (int)(threadIdx.x & 31), box_lo + 3 * o, box_hi + 3 * o, first + o};
  int L_lo[3], L_hi[3];
  const int ms[3] = {max_steps.x, max_steps.y, max_steps.z};
  for (int k = 0; k < 3; ++k) { L_lo[k] = M.lo[k]; L_hi[k] = M.lo[k] + M.n[k] - 1; }
  FbCorrCount c{0, 0};
  int nb, bl;
  const int st = fb_corr_chain(acc, acc.n, L_lo, L_hi, ms, &nb, &bl, c);
  if (acc.lane == 0) { status[p] = st; n_boxes[p] = nb; blocked_at[p] = bl; }
  corr_count(ctr, acc.lane, (unsigned long long)nb, c);
}

// ---------------------------------------------------------------- entry points (include/fiesta_b200.h)
static bool corridor_args_ok(const char *fn, const fiesta_map *m, const int *box_lo, const int *box_hi, const int32_t *max_steps,
                             int64_t n, double clearance, int flags, bool buffers) {
  if (!m || !box_lo || !box_hi || !max_steps) { fb_set_error("%s: null argument", fn); return false; }
  if (!count_buffers_ok(fn, n, buffers) || !clearance_flags_ok(fn, clearance, flags)) return false;
  for (int k = 0; k < 3; ++k) {                                           // per axis: the box, then its max_steps
    if (!box_axis_ok(fn, m->g, box_lo, box_hi, k)) return false;
    if (max_steps[k] < 0) { fb_set_error("%s: max_steps must be >= 0", fn); return false; }
  }
  return true;
}
// Grow the buffers, then record the start event and build the limit box's masks (2 launches).
static int corridor_begin(fiesta_map *m, const char *fn, const int *box_lo, const int *box_hi, double clearance, int flags,
                          size_t in_words, size_t off_words, size_t out_words) {
  FbCorrBufs &B = m->corr;
  const FbCorrMask M = fb_corr_mask_geom(box_lo, box_hi);
  const cudaStream_t s = m->stream;
  CK(cudaSetDevice(m->device));
  cudaError_t e = B.mask.grow((size_t)fb_corr_mask_words(M), s);
  if (e == cudaSuccess) e = B.in.grow(in_words, s);
  if (e == cudaSuccess && off_words) e = B.off.grow(off_words, s);
  if (e == cudaSuccess) e = B.out.grow(out_words, s);
  if (e == cudaSuccess) e = B.ctr.grow(1, s);
  if (e == cudaSuccess && !B.h_ctr) e = B.h_ctr.alloc(1);
  if (e != cudaSuccess) return alloc_failed(e, "%s: cannot allocate the buffers", fn);
  CK(cudaEventRecord(m->ev[0], s));
  CK(cudaMemsetAsync(B.ctr, 0, sizeof(FbCorrCtr), s));
  const long long ywords = fb_corr_mask_words(M) - M.zwords;
  const long long cap = (long long)FB_SMS * 64;                          // blocks of 8 warps, grid-stride beyond
  k_corr_mask<<<(unsigned)std::min((M.zwords + 7) / 8, cap), 256, 0, s>>>(m->g, m->cobs, M, clearance, flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS,
                                                                           B.mask);
  CK(cudaGetLastError());
  k_corr_transpose<<<(unsigned)std::min((ywords + 7) / 8, cap), 256, 0, s>>>(M, B.mask);
  CK(cudaGetLastError());
  m->st.kernel_launches += 2;
  return FIESTA_OK;
}
// After the copies out have been enqueued: synchronise and fill the statistics.
static int corridor_end(fiesta_map *m, const int *box_lo, const int *box_hi, fiesta_corridor_stats *stats) {
  FbCorrBufs &B = m->corr;
  CK(cudaEventRecord(m->ev[1], m->stream));
  CK(cudaMemcpyAsync(B.h_ctr, B.ctr, sizeof(FbCorrCtr), cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  if (stats) {
    *stats = fiesta_corridor_stats{};
    stats->boxes = (int64_t)B.h_ctr->boxes;
    stats->layers_tested = (int64_t)B.h_ctr->tested;
    stats->layers_grown = (int64_t)B.h_ctr->grown;
    stats->mask_voxels = 1;
    for (int k = 0; k < 3; ++k) stats->mask_voxels *= (int64_t)(box_hi[k] - box_lo[k] + 1);
    CK(cudaEventElapsedTime(&stats->ms_compute, m->ev[0], m->ev[1]));
  }
  return FIESTA_OK;
}
int fiesta_inflate_boxes(fiesta_map *m, const int box_lo[3], const int box_hi[3], const int32_t *seed_lo_xyz, const int32_t *seed_hi_xyz,
                         int64_t n, const int32_t max_steps[3], double clearance, int flags, int32_t *status, int32_t *out_lo_xyz,
                         int32_t *out_hi_xyz, fiesta_corridor_stats *stats) {
  const char *fn = "fiesta_inflate_boxes";
  if (!corridor_args_ok(fn, m, box_lo, box_hi, max_steps, n, clearance, flags, seed_lo_xyz && seed_hi_xyz && status && out_lo_xyz && out_hi_xyz))
    return FIESTA_ERR_INVALID;
  if (n >= 0x7fffffffll) { fb_set_error("%s: at most 2^31 - 2 seeds per call", fn); return FIESTA_ERR_LIMIT; }
  if (stats) *stats = fiesta_corridor_stats{};
  if (n == 0) return FIESTA_OK;
  int r;
  if ((r = corridor_begin(m, fn, box_lo, box_hi, clearance, flags, (size_t)n * 6, 0, (size_t)n * 7))) return r;
  FbCorrBufs &B = m->corr;
  const cudaStream_t s = m->stream;
  int32_t *d_st = B.out, *d_lo = d_st + n, *d_hi = d_lo + 3 * n;
  CK(cudaMemcpyAsync(B.in, seed_lo_xyz, (size_t)n * 12, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(B.in + 3 * n, seed_hi_xyz, (size_t)n * 12, cudaMemcpyHostToDevice, s));
  k_corr_inflate<<<(unsigned)((n + CORR_WARPS - 1) / CORR_WARPS), 32 * CORR_WARPS, 0, s>>>(
      fb_corr_mask_geom(box_lo, box_hi), B.mask, make_int3(max_steps[0], max_steps[1], max_steps[2]), B.in, n, d_st, d_lo, d_hi, B.ctr);
  CK(cudaGetLastError());
  m->st.kernel_launches++;
  CK(cudaMemcpyAsync(status, d_st, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out_lo_xyz, d_lo, (size_t)n * 12, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out_hi_xyz, d_hi, (size_t)n * 12, cudaMemcpyDeviceToHost, s));
  return corridor_end(m, box_lo, box_hi, stats);
}
int fiesta_corridors(fiesta_map *m, const int box_lo[3], const int box_hi[3], const int32_t *path_vox_xyz, const int64_t *path_off,
                     int64_t n_paths, const int32_t max_steps[3], double clearance, int flags, int32_t *status, int32_t *n_boxes,
                     int32_t *blocked_at, int32_t *box_lo_xyz, int32_t *box_hi_xyz, int32_t *first, fiesta_corridor_stats *stats) {
  const char *fn = "fiesta_corridors";
  if (!corridor_args_ok(fn, m, box_lo, box_hi, max_steps, n_paths, clearance, flags, path_off && status && n_boxes && blocked_at))
    return FIESTA_ERR_INVALID;
  if (n_paths > 0 && path_off[0] != 0) { fb_set_error("%s: path_off[0] must be 0", fn); return FIESTA_ERR_INVALID; }
  for (int64_t p = 0; p < n_paths; ++p)
    if (path_off[p + 1] < path_off[p]) { fb_set_error("%s: path_off decreases at %lld", fn, (long long)p); return FIESTA_ERR_INVALID; }
  const int64_t total = n_paths > 0 ? path_off[n_paths] : 0;
  if (total > 0 && !(path_vox_xyz && box_lo_xyz && box_hi_xyz && first)) { fb_set_error("%s: null buffer", fn); return FIESTA_ERR_INVALID; }
  if (total >= 0x7fffffffll) { fb_set_error("%s: at most 2^31 - 2 path voxels per call", fn); return FIESTA_ERR_LIMIT; }
  if (stats) *stats = fiesta_corridor_stats{};
  if (total == 0) {                                                       // only empty paths: status 0, no boxes
    for (int64_t p = 0; p < n_paths; ++p) { status[p] = FB_CORR_OK; n_boxes[p] = 0; blocked_at[p] = -1; }
    return FIESTA_OK;
  }
  const size_t T = (size_t)total, np = (size_t)n_paths;
  int r;
  if ((r = corridor_begin(m, fn, box_lo, box_hi, clearance, flags, T * 3, np + 1, np * 3 + T * 7))) return r;
  FbCorrBufs &B = m->corr;
  const cudaStream_t s = m->stream;
  int32_t *d_st = B.out, *d_nb = d_st + np, *d_bl = d_nb + np, *d_lo = d_bl + np, *d_hi = d_lo + 3 * T, *d_first = d_hi + 3 * T;
  CK(cudaMemcpyAsync(B.in, path_vox_xyz, T * 12, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(B.off, path_off, (np + 1) * 8, cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(d_lo, 0xff, T * 28, s));                            // -1 in every slot no box is written to
  k_corr_chain<<<(unsigned)((n_paths + CORR_WARPS - 1) / CORR_WARPS), 32 * CORR_WARPS, 0, s>>>(
      fb_corr_mask_geom(box_lo, box_hi), B.mask, make_int3(max_steps[0], max_steps[1], max_steps[2]), B.in, B.off, n_paths, d_st, d_nb, d_bl,
      d_lo, d_hi, d_first, B.ctr);
  CK(cudaGetLastError());
  m->st.kernel_launches++;
  CK(cudaMemcpyAsync(status, d_st, np * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(n_boxes, d_nb, np * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(blocked_at, d_bl, np * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(box_lo_xyz, d_lo, T * 12, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(box_hi_xyz, d_hi, T * 12, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(first, d_first, T * 4, cudaMemcpyDeviceToHost, s));
  return corridor_end(m, box_lo, box_hi, stats);
}
