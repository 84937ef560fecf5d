// fiesta_b200 -- segment clearance kernel (definition and arithmetic: fb_segment.h, DESIGN.md §3.4).
//
// One warp per segment.  Segment lengths in one batch range from a voxel to thousands of crossings, so a thread per segment
// would leave a warp waiting for its longest segment.  Instead lane l of sweep k walks slab 32k + l (slabs partition the walked
// voxels in t order, each from its exactly computed entry voxel); the earliest lane whose slab blocks comes from a ballot, the
// minimum distance up to and including its blocking voxel from a warp reduction over the lanes up to it, and the warp stops
// after the first sweep that blocks.  The result equals fb_seg_check's sequential walk bit for bit.
#include "fb_map.h"
#include "fb_segment.h"

#define FB_SEG_WARPS 8

__global__ void __launch_bounds__(32 * FB_SEG_WARPS) k_segment_clearance(FbGeom g, const uint32_t *__restrict__ cobs, const double *__restrict__ ab,
                                                                        long long n, double r, int unknown_blocks, int32_t *status,
                                                                        int64_t *hit_idx, double *hit_t, double *min_dist) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * FB_SEG_WARPS;
  for (long long i = (long long)blockIdx.x * FB_SEG_WARPS + (threadIdx.x >> 5); i < n; i += nwarps) {
    double e[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) e[k] = __ldg(&ab[6 * i + k]);
    FbSeg s;
    if (!fb_seg_setup(g, e, s)) {
      if (lane == 0) fb_seg_outside(&status[i], &hit_idx[i], &hit_t[i], &min_dist[i]);
      continue;
    }
    double run = (double)FIESTA_INFINITY;
    bool blocked = false;
    for (int base = 0; base < s.nslabs && !blocked; base += 32) {
      const int j = base + lane;
      FbSegScan sc = fb_seg_scan(g, cobs, r, unknown_blocks != 0);
      if (j < s.nslabs) fb_seg_walk(s, j, j + 1, sc);
      const unsigned hits = __ballot_sync(0xffffffffu, sc.hit);
      const int first = hits ? __ffs(hits) - 1 : 32;
      double m = lane <= first ? sc.min_d : (double)FIESTA_INFINITY;
#pragma unroll
      for (int o = 16; o; o >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
      run = fmin(run, m);
      blocked = hits != 0u;
      if (blocked && lane == first) fb_seg_store(g, sc, run, &status[i], &hit_idx[i], &hit_t[i], &min_dist[i]);
    }
    if (!blocked && lane == 0) {
      const FbSegScan clear = fb_seg_scan(g, cobs, r, false);
      fb_seg_store(g, clear, run, &status[i], &hit_idx[i], &hit_t[i], &min_dist[i]);
    }
  }
}

// ---------------------------------------------------------------- entry points (include/fiesta_b200.h)
// Both forms, validated, on device buffers: the launch on stream s.
static int segments_launch(fiesta_map *m, const double *ab, int64_t n, double clearance, int flags, int32_t *status, int64_t *hit_idx,
                           double *hit_t, double *min_dist, cudaStream_t s) {
  if (n <= 0) return FIESTA_OK;
  const long long want = (n + FB_SEG_WARPS - 1) / FB_SEG_WARPS;
  const unsigned blocks = (unsigned)(want < FB_SMS * 64ll ? want : FB_SMS * 64ll);
  k_segment_clearance<<<blocks, 32 * FB_SEG_WARPS, 0, s>>>(m->g, m->cobs, ab, n, clearance, flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS, status,
                                                           hit_idx, hit_t, min_dist);
  CK(cudaGetLastError());
  m->st.kernel_launches++;
  return FIESTA_OK;
}

int fiesta_check_segments(fiesta_map *m, const double *ab, int64_t n, double clearance, int flags, int32_t *status, int64_t *hit_idx,
                          double *hit_t, double *min_dist) {
  const char *fn = "fiesta_check_segments";
  if (!m || !count_buffers_ok(fn, n, ab && status && hit_idx && hit_t && min_dist) || !clearance_flags_ok(fn, clearance, flags))
    return FIESTA_ERR_INVALID;
  if (n == 0) return FIESTA_OK;
  CK(cudaSetDevice(m->device));
  CK(m->d_seg.grow((size_t)n * 76, m->stream));
  double *d_ab = reinterpret_cast<double *>(m->d_seg.p), *d_t = d_ab + 6 * n, *d_min = d_t + n;
  int64_t *d_idx = reinterpret_cast<int64_t *>(d_min + n);
  int32_t *d_st = reinterpret_cast<int32_t *>(d_idx + n);
  CK(cudaMemcpyAsync(d_ab, ab, (size_t)n * 48, cudaMemcpyHostToDevice, m->stream));
  int r;
  if ((r = segments_launch(m, d_ab, n, clearance, flags, d_st, d_idx, d_t, d_min, m->stream))) return r;
  CK(cudaMemcpyAsync(status, d_st, (size_t)n * 4, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(hit_idx, d_idx, (size_t)n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(hit_t, d_t, (size_t)n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(min_dist, d_min, (size_t)n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}

int fiesta_check_segments_device(fiesta_map *m, const double *d_ab, int64_t n, double clearance, int flags, int32_t *d_status,
                                 int64_t *d_hit_idx, double *d_hit_t, double *d_min_dist, void *stream) {
  const char *fn = "fiesta_check_segments_device";
  if (!m || !count_buffers_ok(fn, n, d_ab && d_status && d_hit_idx && d_hit_t && d_min_dist) || !clearance_flags_ok(fn, clearance, flags))
    return FIESTA_ERR_INVALID;
  const cudaStream_t s = (cudaStream_t)stream;
  int r;
  if ((r = device_query_begin(m, fn, s)) || (r = segments_launch(m, d_ab, n, clearance, flags, d_status, d_hit_idx, d_hit_t, d_min_dist, s)))
    return r;
  return device_query_end(m, s);
}
