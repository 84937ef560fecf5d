// fiesta_b200 -- cost-to-go field for planners: geodesic distance to a goal set through free space at a clearance, and the path
// rule that walks it back to a goal.  Plain C++ shared by the kernels (fb_nav.cu) and CPU tests (tests/cpp/nav_test.cpp, g++).
//
// Definition (DESIGN.md §3.5).  The field covers an inclusive voxel box [lo, hi] of the grid, indexed
// ((x - lo.x) * By + (y - lo.y)) * Bz + (z - lo.z).  A voxel is traversable when fb_seg_blocks says it does not block; voxels
// outside the box count as blocked.  A move u -> u + d, d in {-1,0,1}^3 \ {0}, is allowed iff every voxel of the axis-aligned
// box spanned by u and u + d (2, 4 or 8 voxels) is traversable, so no move cuts a corner between obstacles; its weight is
// w(d) = res * sqrt(k), k = the number of non-zero components of d.  D(goal) = 0 and elsewhere D is the least fixpoint of
// D(v) = min over allowed moves u -> v of fl(D(u) + w), +inf where no goal is reachable, and -1 on blocked voxels.  So the field
// itself carries the traversability: a voxel is traversable iff it lies in the box and D >= 0.
#ifndef FB_NAV_H_
#define FB_NAV_H_
#include "fb_record.h"

#define FB_NAV_BLOCKED (-1.0)

struct FbNavBox {
  int lo[3], n[3];   // lower corner (grid voxel) and extents
};

FB_HD long long fb_nav_idx(const FbNavBox &b, int x, int y, int z) {   // box-local coordinates
  return ((long long)x * b.n[1] + y) * b.n[2] + z;
}
FB_HD bool fb_nav_in_box(const FbNavBox &b, int x, int y, int z) {
  return x >= 0 && x < b.n[0] && y >= 0 && y < b.n[1] && z >= 0 && z < b.n[2];
}

// Direction k in 0..26 (13 = no move), in path order: (dx, dy, dz) lexicographic with dx slowest and -1 first.
FB_HD void fb_nav_dir(int k, int *d) { d[0] = k / 9 - 1; d[1] = k / 3 % 3 - 1; d[2] = k % 3 - 1; }

// Pos2Vox of p into box-local coordinates; false when p has a NaN coordinate or its voxel is outside the box.  floor() is taken in
// fp64 and compared before the conversion, so positions far outside the grid never reach an out-of-range int conversion.
FB_HD bool fb_nav_locate(const FbGeom &g, const FbNavBox &b, const double *p, int *v) {
  for (int k = 0; k < 3; ++k) {
    const double f = floor((p[k] - g.origin[k]) / g.res);
    if (!(f >= (double)b.lo[k] && f < (double)(b.lo[k] + b.n[k]))) return false;
    v[k] = (int)f - b.lo[k];
  }
  return true;
}

FB_HD bool fb_nav_traversable(const FbNavBox &b, const double *D, int x, int y, int z) {
  return fb_nav_in_box(b, x, y, z) && D[fb_nav_idx(b, x, y, z)] >= 0.0;
}
// Is the move from v in direction d allowed?  (Moves are symmetric: the spanned box is the same from either end.)
FB_HD bool fb_nav_move_ok(const FbNavBox &b, const double *D, const int *v, const int *d) {
  for (int ex = d[0] < 0 ? -1 : 0; ex <= (d[0] > 0 ? 1 : 0); ++ex)
    for (int ey = d[1] < 0 ? -1 : 0; ey <= (d[1] > 0 ? 1 : 0); ++ey)
      for (int ez = d[2] < 0 ? -1 : 0; ez <= (d[2] > 0 ? 1 : 0); ++ez)
        if (!fb_nav_traversable(b, D, v[0] + ex, v[1] + ey, v[2] + ez)) return false;
  return true;
}

// Move mask of a voxel (cost matrices, fb_navmatrix.cu) from the traversability of its 3x3x3 neighbourhood, nb bit e = voxel +
// fb_nav_dir(e) traversable (bit 13: the voxel itself).  Bit 13 of the result: the voxel is traversable; bit k != 13: the move from
// neighbour k into the voxel is allowed, i.e. the box the two span is traversable.  0 for a blocked voxel.
FB_HD unsigned fb_nav_move_bits(unsigned nb) {
  if (!(nb & (1u << 13))) return 0;
  unsigned out = 1u << 13;
  for (int k = 0; k < 27; ++k) {
    if (k == 13) continue;
    int d[3];
    fb_nav_dir(k, d);
    unsigned need = 0;
    for (int ex = d[0] < 0 ? -1 : 0; ex <= (d[0] > 0 ? 1 : 0); ++ex)
      for (int ey = d[1] < 0 ? -1 : 0; ey <= (d[1] > 0 ? 1 : 0); ++ey)
        for (int ez = d[2] < 0 ? -1 : 0; ez <= (d[2] > 0 ? 1 : 0); ++ez) need |= 1u << ((ex + 1) * 9 + (ey + 1) * 3 + ez + 1);
    if ((nb & need) == need) out |= 1u << k;
  }
  return out;
}

// Field update (fiesta_nav_update, DESIGN.md §3.11).  u = v + fb_nav_dir(k) is a tight support of v when the move u -> v was allowed
// under the old traversability (fb_nav_move_bits of the old signs), D_old(u) is finite and fl(D_old(u) + w) == D_old(v).  Weights are positive, so a support always has the smaller cost and the relation is acyclic.
FB_HD bool fb_nav_is_support(bool old_allowed, double du, double w, double dv) {
  return old_allowed && du < (double)INFINITY && du + w == dv;
}
FB_HD double fb_nav_weight(int k, const double *w) {   // weight of a move in direction k != 13
  int d[3];
  fb_nav_dir(k, d);
  const int nz = (d[0] != 0) + (d[1] != 0) + (d[2] != 0);
  return nz == 1 ? w[0] : nz == 2 ? w[1] : w[2];
}
// All tight supports of a voxel from its 3x3x3 neighbourhood of old costs d27 (d27[13]: the voxel; -1 outside the box): bit k set
// when neighbour k is one.  0 for a blocked voxel.
FB_HD unsigned fb_nav_support_bits(const double *d27, const double *w) {
  unsigned nb = 0;
  for (int e = 0; e < 27; ++e) nb |= (d27[e] >= 0.0 ? 1u : 0u) << e;
  const unsigned old_bits = fb_nav_move_bits(nb);
  unsigned out = 0;
  for (int k = 0; k < 27; ++k)
    if (k != 13 && fb_nav_is_support((old_bits >> k) & 1u, d27[k], fb_nav_weight(k, w), d27[13])) out |= 1u << k;
  return out;
}
// Per box voxel scratch byte of an update
#define FB_NAVU_NEWT 1u      // traversable on the current records
#define FB_NAVU_CHG 2u       // traversability changed since the field was last brought up to date
#define FB_NAVU_WD 4u        // withdrawn: still traversable, finite old cost, no kept support

// One step of the path rule: the first allowed neighbour u of v, in direction order, with fl(D(u) + w) == D(v).  False when there
// is none (never at the fixpoint, for a reached voxel other than a goal).
FB_HD bool fb_nav_step(const FbNavBox &b, const double *D, const double *w, int *v) {
  const double dv = D[fb_nav_idx(b, v[0], v[1], v[2])];
  for (int k = 0; k < 27; ++k) {
    if (k == 13) continue;
    int d[3];
    fb_nav_dir(k, d);
    const int u[3] = {v[0] + d[0], v[1] + d[1], v[2] + d[2]};
    if (!fb_nav_move_ok(b, D, v, d)) continue;
    const int nz = (d[0] != 0) + (d[1] != 0) + (d[2] != 0);
    const double c = D[fb_nav_idx(b, u[0], u[1], u[2])] + (nz == 1 ? w[0] : nz == 2 ? w[1] : w[2]);
    if (c == dv) { v[0] = u[0]; v[1] = u[1]; v[2] = u[2]; return true; }
  }
  return false;
}

// Path status (fiesta_nav_paths)
#define FB_NAV_REACHED 0
#define FB_NAV_UNREACHABLE 1
#define FB_NAV_INVALID_START 2
#define FB_NAV_TRUNCATED 3

// The path from box-local voxel v down the field to a goal: at most max_len >= 1 grid voxels (xyz) into vox, *len of them; *cost
// = D(start) (+inf when unreachable, NaN for a blocked start).  Stops with TRUNCATED after max_len voxels, which also bounds the
// walk where fl(D(u) + w) == D(u) would let it stand still.
FB_HD int fb_nav_path(const FbNavBox &b, const double *D, const double *w, int *v, int max_len, int32_t *vox, int32_t *len, double *cost) {
  const double d0 = D[fb_nav_idx(b, v[0], v[1], v[2])];
  *len = 0;
  *cost = d0 < 0.0 ? nan("") : d0;
  if (d0 < 0.0) return FB_NAV_INVALID_START;
  if (!(d0 < (double)INFINITY)) return FB_NAV_UNREACHABLE;
  for (int n = 0;; ++n) {
    if (n == max_len) { *len = n; return FB_NAV_TRUNCATED; }
    for (int k = 0; k < 3; ++k) vox[3 * n + k] = b.lo[k] + v[k];
    *len = n + 1;
    if (D[fb_nav_idx(b, v[0], v[1], v[2])] == 0.0) return FB_NAV_REACHED;
    if (!fb_nav_step(b, D, w, v)) return FB_NAV_TRUNCATED;   // no predecessor: only on a field that is not the fixpoint
  }
}

// Cost matrix (fiesta_nav_matrix, DESIGN.md §3.9): cost[i][j] = D_i(voxel of target j), D_i the field above with goals = {source i},
// when both points have status 0; NaN otherwise.  The status of a source or a target:
#define FB_NAVM_PLACED 0     // its voxel is a traversable box voxel
#define FB_NAVM_BLOCKED 1    // its voxel is in the box but blocked
#define FB_NAVM_OUTSIDE 2    // a NaN coordinate, fails PosInMap, or its voxel is outside the box
#endif
