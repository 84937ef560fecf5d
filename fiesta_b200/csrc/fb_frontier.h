// fiesta_b200 -- frontier extraction for exploration planners: the per-voxel frontier predicate and the cluster centroid.  Plain
// C++ shared by the kernels (fb_frontier.cu) and CPU tests (tests/cpp/frontier_test.cpp, g++).
//
// Definition (DESIGN.md §3.6).  A grid voxel is unknown when its record decodes to FB_UNKNOWN (export_distance() reads -10000
// there); FB_DINF and unreached records are observed.  A voxel v of the inclusive box [lo, hi] is a frontier voxel when
//   1. it is observed,
//   2. it is not occupied: occ <= l_occ (GetOccupancy(Vector3i), as k_query evaluates it),
//   3. it does not block at clearance r in the sense of fb_seg_blocks with the unknown flag off, so it is a traversable voxel of a
//      cost-to-go field computed at the same clearance, and
//   4. at least one of its 6 face neighbours inside the grid is unknown (outside the box counts; outside the grid does not).
// Clusters are the 26-connected components of the frontier voxels of the box, numbered by their smallest box index
// (fb_nav_idx), which is also the reference's x, y, z loop order.  Clusters smaller than a minimum size are dropped.
#ifndef FB_FRONTIER_H_
#define FB_FRONTIER_H_
#include "fb_nav.h"       // FbNavBox, fb_nav_idx: the frontier labels use the cost-to-go field's box layout
#include "fb_segment.h"   // fb_seg_blocks

FB_HD bool fb_fr_unknown(const FbGeom &g, const uint32_t *rec, int x, int y, int z) {
  return (fb_ld_record(&rec[fb_ii(g, x, y, z)]) & FB_CODE_MASK) == FB_UNKNOWN;
}

// Is grid voxel v a frontier voxel at clearance r?  rec / occ are the map's records and log-odds in the device layout (fb_ii).
FB_HD bool fb_fr_is_frontier(const FbGeom &g, const uint32_t *rec, const double *occ, double l_occ, const int *v, double r) {
  const int x = v[0], y = v[1], z = v[2];
  if (fb_fr_unknown(g, rec, x, y, z)) return false;
  if (occ[fb_ii(g, x, y, z)] > l_occ) return false;
  double d;
  if (fb_seg_blocks(g, rec, v, r, false, d)) return false;
  return (x > 0 && fb_fr_unknown(g, rec, x - 1, y, z)) || (x + 1 < g.gx && fb_fr_unknown(g, rec, x + 1, y, z)) ||
         (y > 0 && fb_fr_unknown(g, rec, x, y - 1, z)) || (y + 1 < g.gy && fb_fr_unknown(g, rec, x, y + 1, z)) ||
         (z > 0 && fb_fr_unknown(g, rec, x, y, z - 1)) || (z + 1 < g.gz && fb_fr_unknown(g, rec, x, y, z + 1));
}

// Centroid coordinate of a cluster of n voxels whose grid coordinates sum to s on this axis: Vox2Pos's operation order applied to
// the mean, ((double)s / (double)n + 0.5) * res + origin, each operation rounded on its own (no contraction).
FB_HD double fb_fr_centroid(long long s, long long n, double res, double origin) {
  return ((double)s / (double)n + 0.5) * res + origin;
}
#endif
