// fiesta_b200 -- device side of map snapshots (fb_snapshot.h, DESIGN.md §3.12): the classification of the 8^3 tiles that hold
// anything but the default state, and the pack / unpack of their payload through bounded staging, with per-tile checksums and,
// on load, the validation of every word before any other kernel can read it.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <string.h>
#include "fb_common.cuh"
#include "fb_snapshot.h"

static_assert(FB_SNAP_MAX_GX == FB_MAX_GX && FB_SNAP_MAX_GY == FB_MAX_GY && FB_SNAP_MAX_GZ == FB_MAX_GZ, "grid limits");
static_assert(FB_SNAP_MAX_PTOTAL == (long long)FB_LIST_IDX_MASK, "voxel limit");

#define SNAP_THREADS 256

// global index of the k-th in-grid voxel (z fastest) of the tile at tile coordinates tc with extents n
__device__ __forceinline__ long long snap_voxel(const FbGeom &g, const int *tc, const int *n, int k) {
  const int nyz = n[1] * n[2];
  const int lx = k / nyz, r = k - lx * nyz, ly = r / n[2], lz = r - ly * n[2];
  return fb_ii(g, tc[0] * 8 + lx, tc[1] * 8 + ly, tc[2] * 8 + lz);
}

// One warp per tile: flag[t] = some in-grid voxel of tile t differs from cobs 0 / occ +0.0 / cnt 0 / LS 0.
__global__ void k_snap_classify(FbGeom g, const uint32_t *cobs, const double *occ, const unsigned long long *cnt, const unsigned long long *LS,
                                uint8_t *flag) {
  const unsigned t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (t >= (unsigned)g.ntiles) return;
  int tc[3], n[3];
  fb_snap_tile_dims(g.gx, g.gy, g.gz, t, tc, n);
  const int nv = n[0] * n[1] * n[2];
  bool nd = false;
  for (int k = lane; k < nv && !nd; k += 32) {
    const long long v = snap_voxel(g, tc, n, k);
    nd = __ldcs(&cobs[v]) != 0u || __double_as_longlong(__ldcs(&occ[v])) != 0ll || __ldcs(&cnt[v]) != 0ull || (LS && __ldcs(&LS[v]) != 0ull);
  }
  nd = __any_sync(0xffffffffu, nd);
  if (lane == 0) flag[t] = nd ? 1 : 0;
}

__device__ __forceinline__ unsigned long long snap_block_sum(unsigned long long v, unsigned long long *sm) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long s = 0;
  if (threadIdx.x == 0) for (int w = 0; w < SNAP_THREADS / 32; ++w) s += sm[w];
  return s;                                                  // thread 0 only
}

// One CTA per listed tile of the chunk [first, first + gridDim.x): its payload words (fb_snapshot.h) and checksum, at its offset
// from the chunk's first tile.
__global__ void __launch_bounds__(SNAP_THREADS) k_snap_pack(FbGeom g, const uint32_t *cobs, const double *occ, const unsigned long long *cnt,
                                                             const unsigned long long *LS, const uint32_t *list, const unsigned long long *off,
                                                             unsigned first, unsigned long long *out) {
  __shared__ unsigned long long sm[SNAP_THREADS / 32];
  const unsigned t = first + blockIdx.x;
  int tc[3], n[3];
  fb_snap_tile_dims(g.gx, g.gy, g.gz, list[t], tc, n);
  const int nv = n[0] * n[1] * n[2], nf = LS ? 3 : 2;
  const uint32_t W = fb_snap_tile_words(nv, LS != nullptr);
  unsigned long long *o = out + (off[t] - off[first]) / 8;
  unsigned long long acc = 0;
  for (uint32_t j = threadIdx.x; j < W; j += SNAP_THREADS) {
    unsigned long long w;
    if (j < (uint32_t)(nf * nv)) {
      const int f = (int)(j / (uint32_t)nv), k = (int)(j - (uint32_t)f * nv);
      const long long v = snap_voxel(g, tc, n, k);
      w = f == 0 ? (unsigned long long)__double_as_longlong(__ldcs(&occ[v])) : f == 1 ? __ldcs(&cnt[v]) : __ldcs(&LS[v]);
    } else {
      const int k = 2 * (int)(j - (uint32_t)(nf * nv));
      w = __ldcs(&cobs[snap_voxel(g, tc, n, k)]);
      if (k + 1 < nv) w |= (unsigned long long)__ldcs(&cobs[snap_voxel(g, tc, n, k + 1)]) << 32;
    }
    o[j] = w;
    acc += fb_snap_term(w, j);
  }
  const unsigned long long s = snap_block_sum(acc, sm);
  if (threadIdx.x == 0) o[W] = fb_snap_final(s, W);
}

// The reverse of k_snap_pack into a freshly created map, with every word validated: err[0] = lowest bad tile position, err[1] |=
// the FB_SNAP_BAD_* reasons.
__device__ __forceinline__ unsigned snap_check_record(const FbGeom &g, uint32_t c, bool exact) {
  unsigned bad = 0;
  if (c & FB_DINF) { if (!exact || (c & FB_CODE_MASK) < 2u) bad |= FB_SNAP_BAD_BIT31; }
  c &= FB_CODE_MASK;
  if (c >= 2u) {
    int x, y, z;
    fb_unpack(c, x, y, z);
    if (!fb_in_grid(g, x, y, z)) bad |= FB_SNAP_BAD_COBS;
  }
  return bad;
}
__global__ void __launch_bounds__(SNAP_THREADS) k_snap_unpack(FbGeom g, uint32_t *cobs, double *occ, unsigned long long *cnt, unsigned long long *LS,
                                                               const uint32_t *list, const unsigned long long *off, unsigned first,
                                                               const unsigned long long *in, unsigned long long tclock, unsigned *err) {
  __shared__ unsigned long long sm[SNAP_THREADS / 32];
  const unsigned t = first + blockIdx.x;
  int tc[3], n[3];
  fb_snap_tile_dims(g.gx, g.gy, g.gz, list[t], tc, n);
  const int nv = n[0] * n[1] * n[2], nf = LS ? 3 : 2;
  const uint32_t W = fb_snap_tile_words(nv, LS != nullptr);
  const unsigned long long *p = in + (off[t] - off[first]) / 8;
  unsigned long long acc = 0;
  unsigned bad = 0;
  for (uint32_t j = threadIdx.x; j < W; j += SNAP_THREADS) {
    const unsigned long long w = p[j];
    acc += fb_snap_term(w, j);
    if (j < (uint32_t)(nf * nv)) {
      const int f = (int)(j / (uint32_t)nv), k = (int)(j - (uint32_t)f * nv);
      const long long v = snap_voxel(g, tc, n, k);
      if (f == 0) {
        const double d = __longlong_as_double((long long)w);
        if (!isfinite(d)) bad |= FB_SNAP_BAD_OCC;
        occ[v] = d;
      } else if (f == 1) {
        if ((w >> 32) > (w & 0xffffffffull)) bad |= FB_SNAP_BAD_CNT;
        cnt[v] = w;
      } else {
        if (w >= tclock) bad |= FB_SNAP_BAD_LS;
        LS[v] = w;
      }
    } else {
      const int k = 2 * (int)(j - (uint32_t)(nf * nv));
      const uint32_t lo = (uint32_t)w, hi = (uint32_t)(w >> 32);
      bad |= snap_check_record(g, lo, LS != nullptr);
      cobs[snap_voxel(g, tc, n, k)] = lo;
      if (k + 1 < nv) { bad |= snap_check_record(g, hi, LS != nullptr); cobs[snap_voxel(g, tc, n, k + 1)] = hi; }
      else if (hi) bad |= FB_SNAP_BAD_COBS;
    }
  }
  bad = __reduce_or_sync(0xffffffffu, bad);
  if (bad && (threadIdx.x & 31) == 0) { atomicMin(&err[0], t); atomicOr(&err[1], bad); }
  const unsigned long long s = snap_block_sum(acc, sm);
  if (threadIdx.x == 0 && fb_snap_final(s, W) != p[W]) { atomicMin(&err[0], t); atomicOr(&err[1], FB_SNAP_BAD_SUM); }
}

// ====================================================================== host side
int fb_snap_list_tiles(const FbSnapArrays &A, FbSnapBufs &B, unsigned *n_out, cudaStream_t s) {
  const FbGeom &g = A.g;
  const unsigned T = (unsigned)g.ntiles;
  CK(B.flag.alloc(T)); CK(B.list.alloc(T)); CK(B.d_n.alloc(1)); CK(B.h_n.alloc(1));
  k_snap_classify<<<(unsigned)(((size_t)T * 32 + 255) / 256), 256, 0, s>>>(g, A.cobs, A.occ, A.cnt, A.LS, B.flag);
  CK(cudaGetLastError());
  size_t bytes = 0;
  thrust::counting_iterator<uint32_t> it(0);
  CK(cub::DeviceSelect::Flagged(nullptr, bytes, it, B.flag.p, B.list.p, B.d_n.p, (int)T, s));
  CK(B.tmp.grow(bytes, s));
  CK(cub::DeviceSelect::Flagged(B.tmp.p, bytes, it, B.flag.p, B.list.p, B.d_n.p, (int)T, s));
  CK(cudaMemcpyAsync(B.h_n.p, B.d_n.p, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  *n_out = *B.h_n.p;
  return FIESTA_OK;
}

// Staging of one save or load: two device and two pinned chunk buffers, a copy stream and its events.
namespace {
struct SnapIo {
  FbDevBuf<unsigned long long> dst[2];
  FbHostBuf<unsigned long long> hst[2];
  cudaStream_t cs = nullptr;
  cudaEvent_t done_dev[2] = {}, done_copy[2] = {};
  ~SnapIo() {
    if (cs) cudaStreamSynchronize(cs);
    for (int b = 0; b < 2; ++b) { if (done_dev[b]) cudaEventDestroy(done_dev[b]); if (done_copy[b]) cudaEventDestroy(done_copy[b]); }
    if (cs) cudaStreamDestroy(cs);
  }
  int init() {
    for (int b = 0; b < 2; ++b) {
      CK(dst[b].alloc(FB_SNAP_STAGE / 8)); CK(hst[b].alloc(FB_SNAP_STAGE / 8));
      CK(cudaEventCreateWithFlags(&done_dev[b], cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&done_copy[b], cudaEventDisableTiming));
    }
    CK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    return FIESTA_OK;
  }
};
// chunk boundaries: consecutive tiles whose payload fits one staging buffer (a tile is at most 14.4 KB)
void snap_chunks(const std::vector<unsigned long long> &off, std::vector<unsigned> &first) {
  const unsigned n = (unsigned)off.size() - 1;
  first.clear();
  for (unsigned t = 0; t < n;) {
    first.push_back(t);
    unsigned e = t + 1;
    while (e < n && off[e + 1] - off[t] <= FB_SNAP_STAGE) ++e;
    t = e;
  }
  first.push_back(n);
}
}  // namespace

int fb_snap_pack(const FbSnapArrays &A, FbSnapBufs &B, const std::vector<unsigned long long> &off, uint8_t *dst, cudaStream_t s, int *launches) {
  const unsigned n = (unsigned)off.size() - 1;
  if (n == 0) return FIESTA_OK;
  CK(B.off.alloc(n + 1));
  CK(cudaMemcpyAsync(B.off.p, off.data(), (n + 1) * 8, cudaMemcpyHostToDevice, s));
  SnapIo io;
  int r;
  if ((r = io.init())) return r;
  std::vector<unsigned> first;
  snap_chunks(off, first);
  const size_t nc = first.size() - 1;
  // chunk c: pack on the map's stream into device buffer c % 2, copy to pinned buffer c % 2 on the copy stream; the host copies
  // chunk c - 1 out of its pinned buffer while the device packs chunk c and copies it
  for (size_t c = 0; c <= nc; ++c) {
    const int b = (int)(c & 1);
    if (c < nc) {
      if (c >= 2) CK(cudaStreamWaitEvent(s, io.done_copy[b], 0));       // device buffer b has been copied out (chunk c - 2)
      k_snap_pack<<<first[c + 1] - first[c], SNAP_THREADS, 0, s>>>(A.g, A.cobs, A.occ, A.cnt, A.LS, B.list, B.off, first[c], io.dst[b]);
      CK(cudaGetLastError());
      ++*launches;
      CK(cudaEventRecord(io.done_dev[b], s));
      CK(cudaStreamWaitEvent(io.cs, io.done_dev[b], 0));
      CK(cudaMemcpyAsync(io.hst[b].p, io.dst[b].p, off[first[c + 1]] - off[first[c]], cudaMemcpyDeviceToHost, io.cs));
      CK(cudaEventRecord(io.done_copy[b], io.cs));
    }
    if (c >= 1) {
      const int pb = b ^ 1;
      CK(cudaEventSynchronize(io.done_copy[pb]));
      memcpy(dst + off[first[c - 1]], io.hst[pb].p, off[first[c]] - off[first[c - 1]]);
    }
  }
  return FIESTA_OK;
}

int fb_snap_unpack(const FbSnapArrays &A, FbSnapBufs &B, const uint32_t *h_list, const std::vector<unsigned long long> &off, const uint8_t *src,
                   unsigned long long tclock, unsigned *bad_tile, unsigned *reasons, cudaStream_t s, int *launches) {
  const unsigned n = (unsigned)off.size() - 1;
  *bad_tile = 0xffffffffu; *reasons = 0;
  if (n == 0) return FIESTA_OK;
  CK(B.list.alloc(n)); CK(B.off.alloc(n + 1)); CK(B.d_n.alloc(2)); CK(B.h_n.alloc(2));
  CK(cudaMemcpyAsync(B.list.p, h_list, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(B.off.p, off.data(), (n + 1) * 8, cudaMemcpyHostToDevice, s));
  const unsigned init[2] = {0xffffffffu, 0u};
  CK(cudaMemcpyAsync(B.d_n.p, init, 8, cudaMemcpyHostToDevice, s));
  CK(cudaStreamSynchronize(s));                               // the pageable sources above are copied
  SnapIo io;
  int r;
  if ((r = io.init())) return r;
  std::vector<unsigned> first;
  snap_chunks(off, first);
  const size_t nc = first.size() - 1;
  // chunk c: the host fills pinned buffer c % 2 (free once its copy of chunk c - 2 is done), the copy stream moves it to device
  // buffer c % 2 (free once the unpack of chunk c - 2 is done), the map's stream unpacks it
  for (size_t c = 0; c < nc; ++c) {
    const int b = (int)(c & 1);
    const size_t bytes = off[first[c + 1]] - off[first[c]];
    if (c >= 2) CK(cudaEventSynchronize(io.done_copy[b]));
    memcpy(io.hst[b].p, src + off[first[c]], bytes);
    if (c >= 2) CK(cudaStreamWaitEvent(io.cs, io.done_dev[b], 0));
    CK(cudaMemcpyAsync(io.dst[b].p, io.hst[b].p, bytes, cudaMemcpyHostToDevice, io.cs));
    CK(cudaEventRecord(io.done_copy[b], io.cs));
    CK(cudaStreamWaitEvent(s, io.done_copy[b], 0));
    k_snap_unpack<<<first[c + 1] - first[c], SNAP_THREADS, 0, s>>>(A.g, A.cobs, A.occ, A.cnt, A.LS, B.list, B.off, first[c], io.dst[b], tclock, B.d_n);
    CK(cudaGetLastError());
    ++*launches;
    CK(cudaEventRecord(io.done_dev[b], s));
  }
  CK(cudaMemcpyAsync(B.h_n.p, B.d_n.p, 8, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  *bad_tile = B.h_n.p[0]; *reasons = B.h_n.p[1];
  return FIESTA_OK;
}
