// fiesta_b200 -- the packed distance record, the grid geometry and the per-voxel distance read, shared by the kernels, the host
// code of the C ABI (pinned host mirror) and CPU tests.  Plain C++: no CUDA header is needed; under nvcc the functions are
// __host__ __device__ (FB_HD).  Record format: see fb_common.cuh.
#ifndef FB_RECORD_H_
#define FB_RECORD_H_
#include <math.h>
#include <stdint.h>
#include "../../include/fiesta_b200.h"

#ifdef __CUDACC__
#define FB_HD __host__ __device__ __forceinline__
#else
#define FB_HD inline
#endif

#define FB_UNKNOWN 0u
#define FB_INF 1u
// EXACT mode (which never uses FRESH) keeps in the same bit, between calls, "distance_ forced to +infinity_ while the closest
// obstacle and its dependant-list link are kept" -- the state UpdateOccupancy(false) leaves behind for a voxel outside the
// previous update box (ESDFMap.cpp:256-259).  Cleared by the next write of the record.
#define FB_DINF 0x80000000u
#define FB_CODE_MASK 0x7fffffffu

struct FbGeom {
  int gx, gy, gz, pz;          // grid_size_ and padded z pitch
  int gyz;                     // grid_size_yz_ (reference linear index)
  int total;                   // grid_total_size_
  long long ptotal;            // gx*gy*pz, size of the device arrays
  int tx, ty, tz, ntiles;      // 8^3 tile grid
  double origin[3], res, res_inv;
  double min_range[3], max_range[3];
  int min_vec[3], max_vec[3], last_min_vec[3], last_max_vec[3];
  int box_is_full;             // update box == whole grid (SetOriginalRange)
};

FB_HD uint32_t fb_pack(int x, int y, int z) {
  return ((uint32_t)(x + 1) << 20) | ((uint32_t)y << 10) | (uint32_t)z;
}
FB_HD void fb_unpack(uint32_t c, int &x, int &y, int &z) {
  x = (int)((c & FB_CODE_MASK) >> 20) - 1; y = (int)((c >> 10) & 1023u); z = (int)(c & 1023u);
}
FB_HD long long fb_ii(const FbGeom &g, int x, int y, int z) {
  return ((long long)x * g.gy + y) * g.pz + z;
}
FB_HD bool fb_in_grid(const FbGeom &g, int x, int y, int z) {
  return x >= 0 && x < g.gx && y >= 0 && y < g.gy && z >= 0 && z < g.gz;
}

// distance_buffer_ value of a record (ESDFMap.cpp:122-123, 198, 247): exact because the stored obstacle coordinate is exact.
// Host + device: the pinned host mirror (fiesta_host_mirror_*) evaluates the same expression on the same records.
FB_HD double fb_record_distance(uint32_t c, int x, int y, int z, double res) {
  const bool dinf = (c & FB_DINF) != 0u;                                    // between calls bit 31 is only ever set by EXACT mode's local-map reset
  c &= FB_CODE_MASK;
  if (c == FB_UNKNOWN) return (double)FIESTA_UNDEFINED;
  if (c == FB_INF || dinf) return (double)FIESTA_INFINITY;
  int ox, oy, oz;
  fb_unpack(c, ox, oy, oz);
  const double dx = (double)(ox - x), dy = (double)(oy - y), dz = (double)(oz - z);
  return sqrt((dx * dx + dy * dy) + dz * dz) * res;
}

FB_HD uint32_t fb_ld_record(const uint32_t *p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
// GetDistance(Vector3i) (ESDFMap.cpp:477-479): unknown reads +infinity_.  Out-of-grid coordinates (undefined behaviour
// in the reference) also read +infinity_.
FB_HD double fb_get_distance_vox(const FbGeom &g, const uint32_t *cobs, int x, int y, int z) {
  if (!fb_in_grid(g, x, y, z)) return (double)FIESTA_INFINITY;
  const double d = fb_record_distance(fb_ld_record(&cobs[fb_ii(g, x, y, z)]), x, y, z, g.res);
  return d < 0 ? (double)FIESTA_INFINITY : d;
}
// ESDFMap::PosInMap (ESDFMap.cpp:46-61): inclusive on both faces
FB_HD bool fb_pos_in_map(const FbGeom &g, const double *p) {
  if (p[0] < g.min_range[0] || p[1] < g.min_range[1] || p[2] < g.min_range[2]) return false;
  if (p[0] > g.max_range[0] || p[1] > g.max_range[1] || p[2] > g.max_range[2]) return false;
  return true;
}
// ESDFMap::Pos2Vox (ESDFMap.cpp:74-77)
FB_HD void fb_pos2vox(const FbGeom &g, const double *p, int *v) {
  for (int k = 0; k < 3; ++k) v[k] = (int)floor((p[k] - g.origin[k]) / g.res);
}
#endif
