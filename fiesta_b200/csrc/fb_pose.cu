// fiesta_b200 -- robot-shaped collision check kernels (definition: fb_pose.h, DESIGN.md §3.10).
//
// k_pose_setup : one thread per pose: status 2 or 0, n_blocked = 0, hit_idx = INT64_MAX, and its work, fb_pose_chunks() work
//                items of whole candidate z-rows (0 for an invalid pose); work[n] = 0.
// (CUB)        : exclusive scan (int64) of the work in place -> each pose's first work item; work[n] becomes the total.
// k_pose_check : persistent; warp W takes a contiguous run of the flat work-item list (the total is read on the device), so it
//                finds its first pose once and then steps forward.  On each new pose lanes 0..14 write one separating axis and its
//                threshold to the warp's shared memory.  Lanes take consecutive candidate voxels of the item (consecutive z:
//                consecutive records); an in-grid voxel is tested against the record first, and only blocking voxels and
//                voxels outside the grid run the 15-axis test.  Per pose a warp adds its touched blocking voxels to n_blocked
//                (atomicAdd), lowers hit_idx (atomicMin) and sets an outside bit in status (atomicOr).
// k_pose_finish: one thread per pose: the final status, hit_idx -1 unless blocked.
//
// A drone-sized body has a few hundred candidate voxels, a car at 5 cm a few hundred thousand: a thread per pose would leave a
// warp waiting for its largest pose, and a warp per pose would idle most lanes on small ones; items of about FB_POSE_CHUNK
// voxels balance both.  All outputs are integer sums, minima and flags of per-voxel decisions: they do not depend on the schedule.
#include <cub/cub.cuh>
#include "fb_map.h"
#include "fb_pose.h"
#include "fb_view.h"      // fb_view_find: the owner of a position in a flat work list

#define POSE_WARPS 8
#define POSE_OUTSIDE 4    // status bit set while the kernel runs: the box touches a voxel outside the grid

struct FbPoseBody { double h[3]; };

__global__ void k_pose_setup(FbGeom g, const double *__restrict__ poses, long long n, FbPoseBody b, int32_t *status, int32_t *n_blocked,
                             int64_t *hit_idx, long long *work) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    double pose[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) pose[k] = poses[12 * i + k];
    const bool ok = fb_pose_valid(g, pose);
    long long w = 0;
    if (ok) {
      int lo[3], nn[3];
      for (int k = 0; k < 3; ++k) fb_pose_range(g, pose, b.h, k, lo[k], nn[k]);
      w = fb_pose_chunks(nn);
    }
    status[i] = ok ? 0 : 2;
    n_blocked[i] = 0;
    hit_idx[i] = INT64_MAX;
    work[i] = w;
  } else if (i == n) {
    work[n] = 0;
  }
}

// A warp's results for pose i: touched blocking voxels, the least index among them, and whether a lane saw an outside voxel.
__device__ __forceinline__ void pose_flush(int lane, long long i, int cnt, long long best, bool out, int32_t *status, int32_t *n_blocked,
                                           int64_t *hit_idx) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    const long long x = __shfl_xor_sync(0xffffffffu, best, o);
    best = x < best ? x : best;
  }
  const bool anyout = __any_sync(0xffffffffu, out);
  if (lane == 0) {
    if (cnt) { atomicAdd(&n_blocked[i], cnt); atomicMin((long long *)&hit_idx[i], best); }
    if (anyout) atomicOr(&status[i], POSE_OUTSIDE);
  }
}

__global__ void __launch_bounds__(32 * POSE_WARPS) k_pose_check(FbGeom g, const uint32_t *__restrict__ cobs, const double *__restrict__ poses,
                                                                long long n, FbPoseBody b, double clearance, int unknown_blocks,
                                                                const long long *__restrict__ first, int32_t *status, int32_t *n_blocked,
                                                                int64_t *hit_idx) {
  __shared__ double sL[POSE_WARPS][FB_POSE_AXES][3];
  __shared__ double sT[POSE_WARPS][FB_POSE_AXES];
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
  const long long total = first[n];
  const long long nwarps = (long long)gridDim.x * POSE_WARPS, W = (long long)blockIdx.x * POSE_WARPS + wi;
  const long long per = (total + nwarps - 1) / nwarps;
  long long w = W * per;
  const long long w_end = w + per < total ? w + per : total;
  if (w >= w_end) return;
  long long i = fb_view_find(first, n, w);
  double p[3];
  int lo[3], nn[3], rpc = 1;
  int cnt = 0;
  long long best = INT64_MAX;
  bool out = false;
  for (long long cur = -1; w < w_end; ++w) {
    while (first[i + 1] <= w) ++i;                                        // poses without work share their first[] with the next
    if (i != cur) {
      if (cur >= 0) {
        pose_flush(lane, cur, cnt, best, out, status, n_blocked, hit_idx);
        cnt = 0; best = INT64_MAX; out = false;
      }
      cur = i;
      const double *pose = poses + 12 * i;                                  // read in place: a copy indexed by lane would go to local memory
      __syncwarp();                                                       // the previous pose's axes are no longer read
      if (lane < FB_POSE_AXES) {
        fb_pose_axis(pose + 3, lane, sL[wi][lane]);
        sT[wi][lane] = fb_pose_threshold(pose + 3, b.h, 0.5 * g.res, sL[wi][lane]);
      }
      for (int k = 0; k < 3; ++k) { p[k] = pose[k]; fb_pose_range(g, pose, b.h, k, lo[k], nn[k]); }
      rpc = fb_pose_rows_per_chunk(nn[2]);
      __syncwarp();
    }
    const long long rows = (long long)nn[0] * nn[1];
    const long long r0 = (w - first[i]) * rpc;
    const int nr = (int)(rows - r0 < rpc ? rows - r0 : rpc);
    const int nvox = nr * nn[2];
    for (int t = lane; t < nvox; t += 32) {
      const int row = (int)r0 + t / nn[2];                               // r0 + nr <= 518^2
      const int v[3] = {lo[0] + row / nn[1], lo[1] + row % nn[1], lo[2] + t % nn[2]};
      double d[3];
      if (!fb_in_grid(g, v[0], v[1], v[2])) {
        if (!out) {
          fb_pose_offset(g, p, v, d);
          out = fb_pose_touches_at(sL[wi], sT[wi], d);
        }
      } else {
        double dist;
        if (fb_seg_blocks(g, cobs, v, clearance, unknown_blocks != 0, dist)) {
          fb_pose_offset(g, p, v, d);
          if (fb_pose_touches_at(sL[wi], sT[wi], d)) {
            ++cnt;
            const long long idx = (long long)v[0] * g.gyz + (long long)v[1] * g.gz + v[2];
            best = idx < best ? idx : best;
          }
        }
      }
    }
  }
  pose_flush(lane, i, cnt, best, out, status, n_blocked, hit_idx);
}

__global__ void k_pose_finish(long long n, int32_t *status, const int32_t *__restrict__ n_blocked, int64_t *hit_idx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int st = status[i];
  if (st == 2) { hit_idx[i] = -1; return; }
  if (n_blocked[i]) { status[i] = 1; return; }
  status[i] = (st & POSE_OUTSIDE) ? 3 : 0;
  hit_idx[i] = -1;
}

// ---------------------------------------------------------------- entry points (include/fiesta_b200.h)
// Both forms, validated (fb_pose.h limits), on device buffers: the four launches on stream s.
static int poses_launch(fiesta_map *m, const double *poses, long long n, const double *h, double clearance, int flags, int32_t *status,
                        int32_t *n_blocked, int64_t *hit_idx, cudaStream_t s) {
  if (n <= 0) return FIESTA_OK;
  FbPoseBufs &B = m->pose;
  const FbPoseBody body = {{h[0], h[1], h[2]}};
  size_t bytes = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, bytes, B.work.p, B.work.p, (int)(n + 1), s));
  cudaError_t e = B.work.grow((size_t)n + 1, s);
  if (e == cudaSuccess) e = B.tmp.grow(bytes ? bytes : 16, s);
  if (e != cudaSuccess) return alloc_failed(e, "fiesta_check_poses: cannot allocate %zu bytes of work-list storage", (size_t)(n + 1) * 8 + bytes);
  const unsigned setup_blocks = (unsigned)((n + 1 + 255) / 256);
  k_pose_setup<<<setup_blocks, 256, 0, s>>>(m->g, poses, n, body, status, n_blocked, hit_idx, B.work);
  CK(cudaGetLastError());
  bytes = B.tmp.cap;
  CK(cub::DeviceScan::ExclusiveSum(B.tmp.p, bytes, B.work.p, B.work.p, (int)(n + 1), s));
  int per_sm = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pose_check, 32 * POSE_WARPS, 0));
  int dev = 0, sms = FB_SMS;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const unsigned blocks = (unsigned)((per_sm > 0 ? per_sm : 1) * sms);
  k_pose_check<<<blocks, 32 * POSE_WARPS, 0, s>>>(m->g, m->cobs, poses, n, body, clearance, flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS, B.work,
                                                  status, n_blocked, hit_idx);
  CK(cudaGetLastError());
  k_pose_finish<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(n, status, n_blocked, hit_idx);
  CK(cudaGetLastError());
  m->st.kernel_launches += 4;
  return FIESTA_OK;
}

int fiesta_check_poses(fiesta_map *m, const double *poses, int64_t n, const double half_extents[3], double clearance, int flags,
                       int32_t *status, int32_t *n_blocked, int64_t *hit_idx) {
  const char *fn = "fiesta_check_poses";
  if (!m) return FIESTA_ERR_INVALID;
  int r;
  if ((r = pose_args(m, fn, n, half_extents, clearance, flags, poses && status && n_blocked && hit_idx))) return r;
  if (n == 0) return FIESTA_OK;
  CK(cudaSetDevice(m->device));
  CK(m->pose.io.grow((size_t)n * 112, m->stream));
  double *d_poses = reinterpret_cast<double *>(m->pose.io.p);
  int64_t *d_idx = reinterpret_cast<int64_t *>(d_poses + 12 * n);
  int32_t *d_st = reinterpret_cast<int32_t *>(d_idx + n), *d_nb = d_st + n;
  CK(cudaMemcpyAsync(d_poses, poses, (size_t)n * 96, cudaMemcpyHostToDevice, m->stream));
  if ((r = poses_launch(m, d_poses, n, half_extents, clearance, flags, d_st, d_nb, d_idx, m->stream))) return r;
  CK(cudaMemcpyAsync(status, d_st, (size_t)n * 4, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(n_blocked, d_nb, (size_t)n * 4, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaMemcpyAsync(hit_idx, d_idx, (size_t)n * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}

int fiesta_check_poses_device(fiesta_map *m, const double *d_poses, int64_t n, const double half_extents[3], double clearance, int flags,
                              int32_t *d_status, int32_t *d_n_blocked, int64_t *d_hit_idx, void *stream) {
  const char *fn = "fiesta_check_poses_device";
  if (!m) return FIESTA_ERR_INVALID;
  int r;
  if ((r = pose_args(m, fn, n, half_extents, clearance, flags, d_poses && d_status && d_n_blocked && d_hit_idx))) return r;
  const cudaStream_t s = (cudaStream_t)stream;
  if ((r = device_query_begin(m, fn, s)) ||
      (r = poses_launch(m, d_poses, n, half_extents, clearance, flags, d_status, d_n_blocked, d_hit_idx, s)))
    return r;
  return device_query_end(m, s);
}
