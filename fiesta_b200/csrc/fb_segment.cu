// fiesta_b200 -- segment clearance kernel (definition and arithmetic: fb_segment.h, DESIGN.md §3.4).
//
// One warp per segment.  Segment lengths in one batch range from a voxel to thousands of crossings, so a thread per segment
// would leave a warp waiting for its longest segment.  Instead lane l of sweep k walks slab 32k + l (slabs partition the walked
// voxels in t order, each from its exactly computed entry voxel); the earliest lane whose slab blocks comes from a ballot, the
// minimum distance up to and including its blocking voxel from a warp reduction over the lanes up to it, and the warp stops
// after the first sweep that blocks.  The result equals fb_seg_check's sequential walk bit for bit.
#include "fb_common.cuh"
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

cudaError_t fb_segment_clearance(const FbGeom &g, const uint32_t *cobs, const double *ab, long long n, double r, int unknown_blocks,
                                 int32_t *status, int64_t *hit_idx, double *hit_t, double *min_dist, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  const long long want = (n + FB_SEG_WARPS - 1) / FB_SEG_WARPS;
  const unsigned blocks = (unsigned)(want < FB_SMS * 64ll ? want : FB_SMS * 64ll);
  k_segment_clearance<<<blocks, 32 * FB_SEG_WARPS, 0, s>>>(g, cobs, ab, n, r, unknown_blocks, status, hit_idx, hit_t, min_dist);
  return cudaGetLastError();
}
