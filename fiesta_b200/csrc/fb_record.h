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

// The point queries, generic in the voxel read: `rd(x, y, z)` is GetDistance(Vector3i) of the field being queried.  The map's
// own queries (device kernel, query plan, host mirror) read the records with FbRecordRead; the signed field (fb_signed.h) reads
// its signed values inside its box and the records elsewhere.  Every other operation is shared.
struct FbRecordRead {
  const FbGeom &g;
  const uint32_t *cobs;
  FB_HD double operator()(int x, int y, int z) const { return fb_get_distance_vox(g, cobs, x, y, z); }
};
// GetDistance(Vector3d) (ESDFMap.cpp:467-475)
template <class Read> FB_HD double fb_query_distance(const FbGeom &g, const Read &rd, const double *p) {
  if (!fb_pos_in_map(g, p)) return (double)FIESTA_UNDEFINED;
  int v[3];
  fb_pos2vox(g, p, v);
  return rd(v[0], v[1], v[2]);
}
// GetDistWithGradTrilinear (ESDFMap.cpp:481-540), operation for operation (fp64, no contraction: -fmad=false on the device,
// no FMA target on the host).
template <class Read> FB_HD double fb_query_trilinear(const FbGeom &g, const Read &rd, const double *p, double *grad) {
  if (!fb_pos_in_map(g, p)) { grad[0] = grad[1] = grad[2] = 0.0; return -1.0; }
  int b[3];
  double bp[3], f[3];
#ifdef __CUDACC__
#pragma unroll
#endif
  for (int k = 0; k < 3; ++k) {
    const double pm = p[k] - 0.5 * g.res * 1.0;                           // pos - 0.5*resolution_*Ones()
    b[k] = (int)floor((pm - g.origin[k]) / g.res);
    bp[k] = (b[k] + 0.5) * g.res + g.origin[k];                           // Vox2Pos
    f[k] = (p[k] - bp[k]) * g.res_inv;
  }
  double c[2][2][2];
#ifdef __CUDACC__
#pragma unroll
#endif
  for (int x = 0; x < 2; ++x)
#ifdef __CUDACC__
#pragma unroll
#endif
    for (int y = 0; y < 2; ++y)
#ifdef __CUDACC__
#pragma unroll
#endif
      for (int z = 0; z < 2; ++z) c[x][y][z] = rd(b[0] + x, b[1] + y, b[2] + z);
  const double v00 = (1 - f[0]) * c[0][0][0] + f[0] * c[1][0][0];
  const double v01 = (1 - f[0]) * c[0][0][1] + f[0] * c[1][0][1];
  const double v10 = (1 - f[0]) * c[0][1][0] + f[0] * c[1][1][0];
  const double v11 = (1 - f[0]) * c[0][1][1] + f[0] * c[1][1][1];
  const double v0 = (1 - f[1]) * v00 + f[1] * v10;
  const double v1 = (1 - f[1]) * v01 + f[1] * v11;
  grad[2] = (v1 - v0) * g.res_inv;
  grad[1] = ((1 - f[2]) * (v10 - v00) + f[2] * (v11 - v01)) * g.res_inv;
  double g0 = (1 - f[2]) * (1 - f[1]) * (c[1][0][0] - c[0][0][0]);
  g0 += (1 - f[2]) * f[1] * (c[1][1][0] - c[0][1][0]);
  g0 += f[2] * (1 - f[1]) * (c[1][0][1] - c[0][0][1]);
  g0 += f[2] * f[1] * (c[1][1][1] - c[0][1][1]);
  g0 *= g.res_inv;
  grad[0] = g0;
  return (1 - f[2]) * v0 + f[2] * v1;
}
#endif
