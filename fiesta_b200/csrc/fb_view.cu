// fiesta_b200 -- viewpoint coverage kernels (definition: fb_view.h, DESIGN.md §3.7).
//
// k_view_setup : one thread per candidate: its status, and its work, fb_view_chunks(size of its cluster) chunks of 32 members
//                (0 when it is not scored); work[n] = 0.
// (CUB)        : exclusive scans (int64) of the kept clusters' sizes -> each cluster's first member in the member list, and in
//                place of the candidates' work -> each candidate's first chunk; work[n] becomes the total.
// k_view_score : persistent, one warp per (candidate, 32-member chunk) work item, fetched grid-stride from the flat chunk list
//                (the total is read on the device: no host read-back before the launch).  Lane l takes member 32k + l, tests
//                range and field of view, and walks the line of sight only when some orientation sees the member.  Per
//                orientation a ballot counts the visible members; lane j adds orientation j's count to score[i][j].
//
// Cluster sizes run from the minimum size to ~10^5 members, so a CTA per candidate would leave the tail to the few candidates of
// the largest clusters; the flat chunk list spreads every cluster over the whole GPU instead.  Members of one chunk are
// neighbours in the cluster's index order, so the lanes' walks have similar length and read the same cache lines.  Every output
// is an integer sum of per-pair integer decisions (integer atomics), so it does not depend on the schedule.
#include <cub/cub.cuh>
#include <cmath>
#include "fb_frontier.cuh"
#include "fb_view.h"

#define VIEW_WARPS 8

__global__ void k_view_setup(FbGeom g, const uint32_t *__restrict__ cobs, const double *__restrict__ pos, const int32_t *__restrict__ cluster,
                             long long n, double clearance, const int64_t *__restrict__ size, int32_t *status, long long *work, FbViewCtr *ctr) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool scored = false;
  if (i < n) {
    const double p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
    const int st = fb_view_status(g, cobs, p, clearance);
    status[i] = st;
    scored = st == 0;
    work[i] = scored ? fb_view_chunks(size[cluster[i]]) : 0;
  } else if (i == n) {
    work[n] = 0;
  }
  const unsigned c = __popc(__ballot_sync(0xffffffffu, scored));
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&ctr->scored, (unsigned long long)c);
}

__global__ void __launch_bounds__(32 * VIEW_WARPS) k_view_score(FbGeom g, const uint32_t *__restrict__ cobs, const double *__restrict__ pos,
                                                                const int32_t *__restrict__ cluster, long long n, const long long *__restrict__ first,
                                                                const long long *__restrict__ moff, const int64_t *__restrict__ size,
                                                                const int32_t *__restrict__ m_xyz, const double *__restrict__ orient, int n_orient,
                                                                double range2, double tan_h, double tan_v, int unknown_blocks, int32_t *score,
                                                                FbViewCtr *ctr) {
  __shared__ double R[9 * FB_VIEW_MAX_ORIENT];
  for (int t = threadIdx.x; t < 9 * n_orient; t += blockDim.x) R[t] = orient[t];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long total = first[n];
  const long long nwarps = (long long)gridDim.x * VIEW_WARPS;
  unsigned long long walked = 0, visible = 0;
  for (long long w = (long long)blockIdx.x * VIEW_WARPS + (threadIdx.x >> 5); w < total; w += nwarps) {
    const long long i = fb_view_find(first, n, w);
    const int cl = cluster[i];
    const long long j = (w - first[i]) * FB_VIEW_CHUNK + lane;         // this lane's member, within its cluster
    unsigned mask = 0u;
    bool vis = false;
    if (j < size[cl]) {
      const double p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
      const long long m = moff[cl] + j;
      const int v[3] = {m_xyz[3 * m], m_xyz[3 * m + 1], m_xyz[3 * m + 2]};
      double c[3], d[3];
      fb_view_offset(g, v, p, c, d);
      if (fb_view_in_range(d, range2)) mask = fb_view_mask(R, n_orient, d, tan_h, tan_v);
      if (mask) vis = fb_view_visible(g, cobs, p, c, unknown_blocks != 0);
    }
    walked += __popc(__ballot_sync(0xffffffffu, mask != 0u));
    const unsigned vb = __ballot_sync(0xffffffffu, vis);
    if (!vb) continue;
    visible += __popc(vb);
    int mine = 0;
    for (int o = 0; o < n_orient; ++o) {
      const int cnt = __popc(__ballot_sync(0xffffffffu, vis && ((mask >> o) & 1u)));
      if (lane == o) mine = cnt;
    }
    if (mine) atomicAdd(&score[i * n_orient + lane], mine);
  }
  if (lane == 0) {
    if (walked) atomicAdd(&ctr->walked, walked);
    if (visible) atomicAdd(&ctr->visible, visible);
  }
}

// ---------------------------------------------------------------- host side
// One CUB call with temporary storage from tmp (grown as needed).
template <class Call>
static int view_cub(FbDevBuf<char> &tmp, cudaStream_t s, Call call) {
  size_t bytes = 0;
  CK(call((void *)nullptr, bytes));
  const cudaError_t e = tmp.grow(bytes ? bytes : 16, s);
  if (e != cudaSuccess) return alloc_failed(e, "fiesta_frontiers_score_viewpoints: cannot allocate %zu bytes of scan storage", bytes);
  bytes = tmp.cap;
  CK(call((void *)tmp.p, bytes));
  return FIESTA_OK;
}

// Expects V.pos / cl / orient filled for n >= 1 candidates and V.score / ctr zeroed; size / m_xyz are the frontier result's.
static int view_score(const FbGeom &g, const uint32_t *cobs, const int64_t *size, const int32_t *m_xyz, unsigned K, FbViewBufs &V,
                      FbDevBuf<char> &tmp, long long n, int n_orient, const fiesta_sensor_model &sm, double clearance, int unknown_blocks,
                      cudaStream_t s, int *launches) {
  int rc;
  const unsigned setup_blocks = (unsigned)((n + 1 + 255) / 256);
  k_view_setup<<<setup_blocks, 256, 0, s>>>(g, cobs, V.pos, V.cl, n, clearance, size, V.status, V.work, V.ctr);
  CK(cudaGetLastError());
  if ((rc = view_cub(tmp, s, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, size, V.moff.p, (int)K, s); }))) return rc;
  if ((rc = view_cub(tmp, s, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, V.work.p, V.work.p, (int)(n + 1), s); })))
    return rc;
  int per_sm = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_view_score, 32 * VIEW_WARPS, 0));
  int dev = 0, sms = FB_SMS;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const unsigned blocks = (unsigned)((per_sm > 0 ? per_sm : 1) * sms);
  k_view_score<<<blocks, 32 * VIEW_WARPS, 0, s>>>(g, cobs, V.pos, V.cl, n, V.work, V.moff, size, m_xyz, V.orient, n_orient,
                                                  sm.max_range * sm.max_range, sm.tan_half_fov[0], sm.tan_half_fov[1], unknown_blocks,
                                                  V.score, V.ctr);
  CK(cudaGetLastError());
  *launches += 4;
  return FIESTA_OK;
}

// ---------------------------------------------------------------- entry point (include/fiesta_b200.h)
int fiesta_frontiers_score_viewpoints(fiesta_frontiers *f, const int32_t *cluster, const double *pos_xyz, int64_t n, const double *orient,
                                      int32_t n_orient, const fiesta_sensor_model *sensor, double clearance, int flags, int32_t *status,
                                      int32_t *score, fiesta_viewpoint_stats *stats) {
  const char *fn = "fiesta_frontiers_score_viewpoints";
  if (!f || !sensor || !orient) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  if (!count_buffers_ok(fn, n, cluster && pos_xyz && status && score) || !clearance_flags_ok(fn, clearance, flags)) return FIESTA_ERR_INVALID;
  if (!f->valid) { fb_set_error("%s: no frontiers have been computed", fn); return FIESTA_ERR_INVALID; }
  if (n_orient < 1) { fb_set_error("%s: n_orient must be >= 1", fn); return FIESTA_ERR_INVALID; }
  const fiesta_sensor_model sm = *sensor;
  const double sv[3] = {sm.max_range, sm.tan_half_fov[0], sm.tan_half_fov[1]};
  for (double x : sv)
    if (!(std::isfinite(x) && x > 0)) { fb_set_error("%s: max_range and tan_half_fov must be finite and > 0", fn); return FIESTA_ERR_INVALID; }
  if (n_orient > FIESTA_VIEWPOINT_MAX_ORIENT) {
    fb_set_error("%s: at most %d orientations per call", fn, FIESTA_VIEWPOINT_MAX_ORIENT);
    return FIESTA_ERR_LIMIT;
  }
  for (int k = 0; k < 9 * n_orient; ++k)
    if (!std::isfinite(orient[k])) { fb_set_error("%s: orientation entry %d is not finite", fn, k); return FIESTA_ERR_INVALID; }
  const int64_t K = f->st.kept_clusters;
  for (int64_t i = 0; i < n; ++i)
    if (!(cluster[i] >= 0 && cluster[i] < K)) {
      fb_set_error("%s: cluster[%lld] = %d is not a kept cluster id (there are %lld)", fn, (long long)i, (int)cluster[i], (long long)K);
      return FIESTA_ERR_INVALID;
    }
  if (n >= 0x7fffffffll) { fb_set_error("%s: at most 2^31 - 2 candidates per call", fn); return FIESTA_ERR_LIMIT; }
  if (stats) *stats = fiesta_viewpoint_stats{};
  if (n == 0) return FIESTA_OK;
  fiesta_map *m = f->m;
  const cudaStream_t s = m->stream;
  FbViewBufs &V = f->V;
  CK(cudaSetDevice(m->device));
  cudaError_t e = V.pos.grow((size_t)n * 3, s);
  if (e == cudaSuccess) e = V.cl.grow((size_t)n, s);
  if (e == cudaSuccess) e = V.status.grow((size_t)n, s);
  if (e == cudaSuccess) e = V.work.grow((size_t)n + 1, s);
  if (e == cudaSuccess) e = V.score.grow((size_t)n * n_orient, s);
  if (e == cudaSuccess) e = V.moff.grow((size_t)K, s);
  if (e == cudaSuccess) e = V.orient.grow(9 * FIESTA_VIEWPOINT_MAX_ORIENT, s);
  if (e == cudaSuccess) e = V.ctr.grow(1, s);
  if (e == cudaSuccess && !V.h_ctr) e = V.h_ctr.alloc(1);
  if (e != cudaSuccess) return alloc_failed(e, "%s: cannot allocate the buffers of %lld candidates", fn, (long long)n);
  CK(cudaMemcpyAsync(V.pos, pos_xyz, (size_t)n * 24, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(V.cl, cluster, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(V.orient, orient, (size_t)n_orient * 72, cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(V.score, 0, (size_t)n * n_orient * 4, s));
  CK(cudaMemsetAsync(V.ctr, 0, sizeof(FbViewCtr), s));
  int launches = 0;
  CK(cudaEventRecord(f->ev[0], s));
  const int r = view_score(m->g, m->cobs, f->B.o_size, f->B.m_xyz, (unsigned)K, V, f->B.tmp, (long long)n, (int)n_orient, sm, clearance,
                           flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS, s, &launches);
  m->st.kernel_launches += launches;
  if (r != FIESTA_OK) return r;
  CK(cudaEventRecord(f->ev[1], s));
  CK(cudaMemcpyAsync(V.h_ctr, V.ctr, sizeof(FbViewCtr), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(status, V.status, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(score, V.score, (size_t)n * n_orient * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (stats) {
    stats->candidates_scored = (int64_t)V.h_ctr->scored;
    stats->pairs_walked = (int64_t)V.h_ctr->walked;
    stats->pairs_visible = (int64_t)V.h_ctr->visible;
    CK(cudaEventElapsedTime(&stats->ms_compute, f->ev[0], f->ev[1]));
  }
  return FIESTA_OK;
}
