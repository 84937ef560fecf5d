// fiesta_b200 -- map snapshots (format: fb_snapshot.h, DESIGN.md §3.12): the classification of the 8^3 tiles that hold anything
// but the default state, the pack / unpack of their payload through bounded staging, with per-tile checksums and, on load, the
// validation of every word before any other kernel can read it; and fiesta_snapshot_save / fiesta_snapshot_load around them.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <string.h>
#include <vector>
#include "fb_map.h"
#include "fb_snapshot.h"

static_assert(FB_SNAP_MAX_GX == FB_MAX_GX && FB_SNAP_MAX_GY == FB_MAX_GY && FB_SNAP_MAX_GZ == FB_MAX_GZ, "grid limits");
static_assert(FB_SNAP_MAX_PTOTAL == (long long)FB_LIST_IDX_MASK, "voxel limit");

#define SNAP_THREADS 256
#define FB_SNAP_STAGE (16u << 20)  // bytes of each of the two device and two pinned staging buffers of a save or load
struct FbSnapArrays {              // the per-voxel state a snapshot carries; LS is null in FAST mode
  FbGeom g;
  uint32_t *cobs;
  double *occ;
  unsigned long long *cnt, *LS;
};
struct FbSnapBufs {                // per-tile scratch of one save or load
  FbDevBuf<uint8_t> flag;          // per grid tile: holds non-default state
  FbDevBuf<uint32_t> list, d_n;    // stored tiles ascending; selection count, or {first bad tile, reasons} on load
  FbDevBuf<unsigned long long> off;  // per stored tile: payload offset, and the end
  FbHostBuf<uint32_t> h_n;
  FbDevBuf<char> tmp;              // CUB temporary storage
};

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
// Lists the tiles with non-default state into B.list (ascending) and their count into *n_out.
static int snap_list_tiles(const FbSnapArrays &A, FbSnapBufs &B, unsigned *n_out, cudaStream_t s, int *launches) {
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
  *launches += 2;
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

// Payload of the B.list tiles, whose offsets (and the end) are `off`, written to host memory dst + off[t].
static int snap_pack(const FbSnapArrays &A, FbSnapBufs &B, const std::vector<unsigned long long> &off, uint8_t *dst, cudaStream_t s,
                     int *launches) {
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

// Scatters the payload at src + off[t] of the h_list tiles into A; *bad_tile = the first tile position that failed validation
// (0xffffffff: none), *reasons = the FB_SNAP_BAD_* bits.
static int snap_unpack(const FbSnapArrays &A, FbSnapBufs &B, const uint32_t *h_list, const std::vector<unsigned long long> &off,
                       const uint8_t *src, unsigned long long tclock, unsigned *bad_tile, unsigned *reasons, cudaStream_t s, int *launches) {
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

// ====================================================================== entry points (include/fiesta_b200.h)
static FbSnapArrays snap_arrays(fiesta_map *m) {
  return FbSnapArrays{m->g, m->cobs, m->occ, m->cnt, m->mode == FIESTA_MODE_EXACT ? m->X.LS.p : nullptr};
}
// the fiesta_stats counters in snapshot order: every one but kernel_launches (raycast_rounds' slot is not used)
static int64_t *snap_stat(fiesta_stats &st, int i) {
  int64_t *f[FB_SNAP_NSTATS] = {&st.occupancy_updates, &st.inserts, &st.deletes, &st.voxels_changed, &st.expansions, &st.voxels_reset,
                                &st.tile_visits, &st.generations, &st.rays_cast, &st.rays_dropped, &st.ray_voxels, &st.raycast_rounds,
                                &st.touched_voxels};
  return f[i];
}
static std::vector<unsigned long long> snap_offsets(const FbGeom &g, int exact, const uint32_t *list, size_t n) {
  std::vector<unsigned long long> off(n + 1);
  off[0] = 0;
  for (size_t t = 0; t < n; ++t) off[t + 1] = off[t] + fb_snap_tile_bytes(g.gx, g.gy, g.gz, exact, list[t]);
  return off;
}
int fiesta_snapshot_save(fiesta_map *m, void *buf, int64_t cap, int64_t *size) {
  const char *fn = "fiesta_snapshot_save";
  if (!m || !size || cap < 0 || (cap > 0 && !buf)) { fb_set_error("%s: bad argument", fn); return FIESTA_ERR_INVALID; }
  *size = 0;
  if (m->n_ev > 0) { fb_set_error("%s: SetOccupancy events are staged (UpdateOccupancy has not run)", fn); return FIESTA_ERR_INVALID; }
  if (m->n_touch_tiles > 0) { fb_set_error("%s: the occupancy queue is not empty (UpdateOccupancy has not run)", fn); return FIESTA_ERR_INVALID; }
  if (m->n_ins > 0 || m->n_del > 0) { fb_set_error("%s: inserts or deletes are pending (UpdateESDF has not run)", fn); return FIESTA_ERR_INVALID; }
  if (m->shard_world > 1) { fb_set_error("%s: an x-slab shard cannot be saved", fn); return FIESTA_ERR_INVALID; }
  CK(cudaSetDevice(m->device));
  const FbSnapArrays A = snap_arrays(m);
  const int exact = m->mode == FIESTA_MODE_EXACT;
  FbSnapBufs B;
  unsigned n = 0;
  int r, launches = 0;
  if ((r = snap_list_tiles(A, B, &n, m->stream, &launches))) return r;
  m->st.kernel_launches += launches;
  std::vector<uint32_t> list(n);
  if (n) {
    CK(cudaMemcpyAsync(list.data(), B.list, (size_t)n * 4, cudaMemcpyDeviceToHost, m->stream));
    CK(cudaStreamSynchronize(m->stream));
  }
  const std::vector<unsigned long long> off = snap_offsets(m->g, exact, list.data(), n);
  const int64_t depth_pixels = m->image_cnt ? (int64_t)m->d_img[0].cap : 0;
  FbSnapLayout L;
  fb_snap_layout(n, off[n], depth_pixels, &L);
  *size = (int64_t)L.total;
  if (!buf) return FIESTA_OK;                                             // size query
  if (cap < *size) { fb_set_error("%s: the buffer holds %lld bytes, the snapshot needs %lld", fn, (long long)cap, (long long)*size); return FIESTA_ERR_LIMIT; }
  uint8_t *p = static_cast<uint8_t *>(buf);
  launches = 0;
  if ((r = snap_pack(A, B, off, p + L.payload_off, m->stream, &launches))) return r;
  m->st.kernel_launches += launches;
  memset(p + L.list_off, 0, L.payload_off - L.list_off);
  for (unsigned t = 0; t < n; ++t) fb_snap_st32(p + L.list_off + 4 * t, list[t]);
  memset(p + L.depth_off, 0, L.depth_bytes);
  if (depth_pixels) {
    CK(cudaMemcpyAsync(p + L.depth_off, m->d_img[m->image_cnt & 1], (size_t)depth_pixels * 2, cudaMemcpyDeviceToHost, m->stream));
    CK(cudaStreamSynchronize(m->stream));
  }
  FbSnapHeader h{};
  h.version = FB_SNAP_VERSION; h.mode = (uint32_t)m->mode;
  for (int i = 0; i < 3; ++i) {
    h.origin[i] = m->cfg.origin[i]; h.map_size[i] = m->cfg.map_size[i];
    h.min_vec[i] = m->g.min_vec[i]; h.max_vec[i] = m->g.max_vec[i]; h.last_min_vec[i] = m->g.last_min_vec[i]; h.last_max_vec[i] = m->g.last_max_vec[i];
  }
  h.resolution = m->cfg.resolution;
  h.grid[0] = m->g.gx; h.grid[1] = m->g.gy; h.grid[2] = m->g.gz;
  h.params_set = m->params_set ? 1 : 0;
  h.l_hit = m->l_hit; h.l_miss = m->l_miss; h.l_min = m->l_min; h.l_max = m->l_max; h.l_occ = m->l_occ;
  h.flags = m->local_box_seen ? FB_SNAP_LOCAL_BOX_SEEN : 0u;
  h.image_cnt = m->image_cnt;
  h.tclock = exact ? m->X.tclock : 0; h.key_base = exact ? m->X.key_base : 0;
  for (int i = 0; i < FB_SNAP_NSTATS; ++i) h.stats[i] = i == FB_SNAP_STAT_ROUNDS ? 0 : *snap_stat(m->st, i);
  h.depth_pixels = depth_pixels;
  h.n_tiles = n;
  h.list_sum = fb_snap_checksum(p + L.list_off, (L.payload_off - L.list_off) / 8);
  h.depth_sum = fb_snap_checksum(p + L.depth_off, L.depth_bytes / 8);
  fb_snap_encode(h, p);
  return FIESTA_OK;
}
int fiesta_snapshot_load(const void *buf, int64_t size, int32_t device, fiesta_map **out) {
  const char *fn = "fiesta_snapshot_load";
  if (!out) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  *out = nullptr;
  if (!buf || size < 0) { fb_set_error("%s: bad argument", fn); return FIESTA_ERR_INVALID; }
  const uint8_t *p = static_cast<const uint8_t *>(buf);
  FbSnapHeader h;
  FbSnapLayout L;
  char err[256];
  if (fb_snap_parse(p, size, &h, &L, err, (int)sizeof(err))) { fb_set_error("%s: %s", fn, err); return FIESTA_ERR_INVALID; }
  fiesta_config cfg{};
  for (int i = 0; i < 3; ++i) { cfg.origin[i] = h.origin[i]; cfg.map_size[i] = h.map_size[i]; }
  cfg.resolution = h.resolution; cfg.device = device; cfg.mode = (int32_t)h.mode;
  fiesta_map *raw = nullptr;
  int r;
  if ((r = create_map(&cfg, &raw, false))) return r;                     // the mode is the snapshot's, whatever FIESTA_B200_MODE says
  std::unique_ptr<fiesta_map, void (*)(fiesta_map *)> m(raw, fiesta_destroy);   // destroyed on any failure below
  FbGeom &g = m->g;
  if (g.gx != h.grid[0] || g.gy != h.grid[1] || g.gz != h.grid[2]) { fb_set_error("%s: the rebuilt grid differs from the stored one", fn); return FIESTA_ERR_INVALID; }
  m->params_set = h.params_set != 0;
  m->l_hit = h.l_hit; m->l_miss = h.l_miss; m->l_min = h.l_min; m->l_max = h.l_max; m->l_occ = h.l_occ;
  for (int i = 0; i < 3; ++i) {
    g.min_vec[i] = h.min_vec[i]; g.max_vec[i] = h.max_vec[i]; g.last_min_vec[i] = h.last_min_vec[i]; g.last_max_vec[i] = h.last_max_vec[i];
  }
  set_box_flag(g);
  m->local_box_seen = (h.flags & FB_SNAP_LOCAL_BOX_SEEN) != 0;
  if (m->mode == FIESTA_MODE_EXACT) { m->X.tclock = h.tclock; m->X.key_base = h.key_base; }
  for (int i = 0; i < FB_SNAP_NSTATS; ++i) if (i != FB_SNAP_STAT_ROUNDS) *snap_stat(m->st, i) = h.stats[i];
  std::vector<uint32_t> list((size_t)h.n_tiles);
  for (size_t t = 0; t < list.size(); ++t) list[t] = fb_snap_ld32(p + L.list_off + 4 * t);
  const std::vector<unsigned long long> off = snap_offsets(g, m->mode == FIESTA_MODE_EXACT, list.data(), list.size());
  FbSnapBufs B;
  unsigned bad = 0, why = 0;
  int launches = 0;
  if ((r = snap_unpack(snap_arrays(m.get()), B, list.data(), off, p + L.payload_off, h.tclock, &bad, &why, m->stream, &launches))) return r;
  m->st.kernel_launches += launches;
  if (why) {
    fb_set_error("%s: stored tile %u (grid tile %u) is malformed:%s%s%s%s%s%s", fn, bad, list[bad], (why & FB_SNAP_BAD_SUM) ? " checksum mismatch;" : "",
                 (why & FB_SNAP_BAD_COBS) ? " closest-obstacle record outside the grid;" : "", (why & FB_SNAP_BAD_BIT31) ? " bad bit 31 of a record;" : "",
                 (why & FB_SNAP_BAD_OCC) ? " log-odds not finite;" : "", (why & FB_SNAP_BAD_LS) ? " relink time not below the relink clock;" : "",
                 (why & FB_SNAP_BAD_CNT) ? " more hits than observations;" : "");
    return FIESTA_ERR_INVALID;
  }
  // rebuilt, not stored: the Exist() bitmap, and FAST mode's staging copy of the records
  if ((r = rebuild_occbits(m.get()))) return r;
  if (m->mode == FIESTA_MODE_FAST) CK(cudaMemcpyAsync(m->cobs_b, m->cobs, (size_t)g.ptotal * 4, cudaMemcpyDeviceToDevice, m->stream));
  if (h.depth_pixels > 0) {
    if ((r = alloc_depth(m.get(), (size_t)h.depth_pixels))) return r;
    CK(cudaMemcpyAsync(m->d_img[h.image_cnt & 1], p + L.depth_off, (size_t)h.depth_pixels * 2, cudaMemcpyHostToDevice, m->stream));
  }
  m->image_cnt = h.image_cnt;
  CK(cudaStreamSynchronize(m->stream));
  *out = m.release();
  return FIESTA_OK;
}
