// fiesta_b200 -- robot-shaped collision checks: does an oriented box at a pose touch a voxel that blocks?  Pose validation, the
// per-pose constants (15 separating axes, their thresholds, the candidate voxel range), the exact touch test and the sequential
// check of one pose, shared by the kernel (fb_pose.cu), the pinned host mirror and CPU tests (tests/cpp/pose_test.cpp, g++).
//
// Definition (DESIGN.md §3.10).  A pose is 12 doubles {px, py, pz, R00 .. R22}: the box centre p in metres and a row-major 3x3
// world-to-body matrix whose rows u_0, u_1, u_2 are the box axes in world coordinates, used as given.  The half extents h (metres,
// finite, >= 0) are shared by all poses of a call.  Voxel v (any integer triple) has centre c_k = ((double)v_k + 0.5) * res +
// origin_k (Vox2Pos), offset d_k = c_k - p_k and half-edge r = 0.5 * res.  The box touches v iff no axis L of the separating-axis
// test over the world axes e_k, the box axes u_j and the nine products e_k x u_j separates the closed cube from the closed box:
// !(fabs(proj_L) > T_L) for all 15, each fp64 operation rounded on its own, with
//   proj_L = (L0*d0 + L1*d1) + L2*d2
//   T_L    = r * ((fabs(L0) + fabs(L1)) + fabs(L2)) + ((h0 * fabs(u_0.L) + h1 * fabs(u_1.L)) + h2 * fabs(u_2.L)),
//   u_j.L  = (u_j0*L0 + u_j1*L1) + u_j2*L2.
// A touched in-grid voxel blocks by fb_seg_blocks.  Status 0 clear, 1 some touched in-grid voxel blocks (n_blocked of them, hit_idx
// = the least reference index x*Gy*Gz + y*Gz + z among them), 2 invalid pose, 3 not blocked but the box touches a voxel outside
// the grid.
//
// Candidates: e_k = (h0*|u_0k| + h1*|u_1k|) + h2*|u_2k| bounds the box along world axis k, and every touched voxel lies in
// lo_k = floor((p_k - e_k - origin_k) / res) - 1 .. hi_k = floor((p_k + e_k - origin_k) / res) + 1 (DESIGN.md §3.10 argues it).
// With h0 + h1 + h2 <= 256 * res a range holds at most 518 voxels per axis.
#ifndef FB_POSE_H_
#define FB_POSE_H_
#include "fb_segment.h"   // fb_seg_blocks: the blocking rule of segment clearance

#define FB_POSE_AXES 15
#define FB_POSE_MAX_SPAN 256          // h0 + h1 + h2 <= 256 * res (FIESTA_ERR_LIMIT beyond)
#define FB_POSE_R_MAX (1.0 + 1.0 / 1048576.0)   // |R_jk| <= 1 + 2^-20, else status 2
#define FB_POSE_CHUNK 256             // candidate voxels per work item of the kernel (whole z-rows, at least one)

struct FbPose {
  double p[3];
  double L[FB_POSE_AXES][3];
  double T[FB_POSE_AXES];
  int lo[3], n[3];                    // candidate range: lo_k .. lo_k + n_k - 1
};

// Status 2 rule: p has a NaN or fails PosInMap, an R entry is non-finite or some |R_jk| > 1 + 2^-20.
FB_HD bool fb_pose_valid(const FbGeom &g, const double *pose) {
  if (pose[0] != pose[0] || pose[1] != pose[1] || pose[2] != pose[2] || !fb_pos_in_map(g, pose)) return false;
  for (int k = 3; k < 12; ++k)
    if (!(fabs(pose[k]) <= FB_POSE_R_MAX)) return false;                // NaN and +-inf fail too
  return true;
}

// Axis a of the separating-axis test: e_a (a < 3), u_{a-3} (a < 6), else e_k x u_j with k = (a - 6) / 3, j = (a - 6) % 3 (exact:
// every component is 0 or +- an entry of u_j).
FB_HD void fb_pose_axis(const double *R, int a, double *L) {
  if (a < 3) { L[0] = a == 0 ? 1.0 : 0.0; L[1] = a == 1 ? 1.0 : 0.0; L[2] = a == 2 ? 1.0 : 0.0; return; }
  if (a < 6) { for (int i = 0; i < 3; ++i) L[i] = R[3 * (a - 3) + i]; return; }
  const int k = (a - 6) / 3;
  const double *u = R + 3 * ((a - 6) % 3);
  if (k == 0) { L[0] = 0.0; L[1] = -u[2]; L[2] = u[1]; }
  else if (k == 1) { L[0] = u[2]; L[1] = 0.0; L[2] = -u[0]; }
  else { L[0] = -u[1]; L[1] = u[0]; L[2] = 0.0; }
}

FB_HD double fb_pose_dot(const double *a, const double *b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// T_L: the cube's and the box's projected radii on L.
FB_HD double fb_pose_threshold(const double *R, const double *h, double r, const double *L) {
  return r * ((fabs(L[0]) + fabs(L[1])) + fabs(L[2])) +
         ((h[0] * fabs(fb_pose_dot(R, L)) + h[1] * fabs(fb_pose_dot(R + 3, L))) + h[2] * fabs(fb_pose_dot(R + 6, L)));
}

// Candidate range on world axis k.
FB_HD void fb_pose_range(const FbGeom &g, const double *pose, const double *h, int k, int &lo, int &n) {
  const double *R = pose + 3;
  const double e = (h[0] * fabs(R[k]) + h[1] * fabs(R[3 + k])) + h[2] * fabs(R[6 + k]);
  lo = (int)floor((pose[k] - e - g.origin[k]) / g.res) - 1;
  n = (int)floor((pose[k] + e - g.origin[k]) / g.res) + 1 - lo + 1;
}

// Per-pose constants of a valid pose.
FB_HD void fb_pose_setup(const FbGeom &g, const double *pose, const double *h, FbPose &P) {
  const double r = 0.5 * g.res;
  for (int k = 0; k < 3; ++k) P.p[k] = pose[k];
  for (int a = 0; a < FB_POSE_AXES; ++a) {
    fb_pose_axis(pose + 3, a, P.L[a]);
    P.T[a] = fb_pose_threshold(pose + 3, h, r, P.L[a]);
  }
  for (int k = 0; k < 3; ++k) fb_pose_range(g, pose, h, k, P.lo[k], P.n[k]);
}

// Separating-axis test on voxel v given its offset from the pose centre; L / T are the pose's axes and thresholds.
FB_HD bool fb_pose_touches_at(const double (*L)[3], const double *T, const double *d) {
  for (int a = 0; a < FB_POSE_AXES; ++a)
    if (fabs(fb_pose_dot(L[a], d)) > T[a]) return false;
  return true;
}
FB_HD void fb_pose_offset(const FbGeom &g, const double *p, const int *v, double *d) {
  for (int k = 0; k < 3; ++k) d[k] = (((double)v[k] + 0.5) * g.res + g.origin[k]) - p[k];
}
FB_HD bool fb_pose_touches(const FbGeom &g, const FbPose &P, const int *v) {
  double d[3];
  fb_pose_offset(g, P.p, v, d);
  return fb_pose_touches_at(P.L, P.T, d);
}

// Work items of a valid pose in the kernel: chunks of whole candidate z-rows (x slowest), FB_POSE_CHUNK voxels or one row each.
FB_HD int fb_pose_rows_per_chunk(int nz) { return nz >= FB_POSE_CHUNK ? 1 : FB_POSE_CHUNK / nz; }
FB_HD long long fb_pose_chunks(const int *n) {
  const long long rows = (long long)n[0] * n[1], rpc = fb_pose_rows_per_chunk(n[2]);
  return (rows + rpc - 1) / rpc;
}

// One pose, sequentially (host side of the pinned mirror; the reference for the kernel).
FB_HD void fb_pose_check(const FbGeom &g, const uint32_t *rec, const double *pose, const double *h, double clearance, bool unknown_blocks,
                         int32_t *status, int32_t *n_blocked, int64_t *hit_idx) {
  *n_blocked = 0;
  *hit_idx = -1;
  if (!fb_pose_valid(g, pose)) { *status = 2; return; }
  FbPose P;
  fb_pose_setup(g, pose, h, P);
  bool outside = false;
  int32_t cnt = 0;
  int64_t best = -1;
  int v[3];
  for (v[0] = P.lo[0]; v[0] < P.lo[0] + P.n[0]; ++v[0])
    for (v[1] = P.lo[1]; v[1] < P.lo[1] + P.n[1]; ++v[1])
      for (v[2] = P.lo[2]; v[2] < P.lo[2] + P.n[2]; ++v[2]) {
        double dist;
        if (!fb_in_grid(g, v[0], v[1], v[2])) {
          if (!outside && fb_pose_touches(g, P, v)) outside = true;
        } else if (fb_seg_blocks(g, rec, v, clearance, unknown_blocks, dist) && fb_pose_touches(g, P, v)) {
          const int64_t idx = (int64_t)v[0] * g.gyz + (int64_t)v[1] * g.gz + v[2];
          if (cnt == 0) best = idx;                                       // loop order is index order: the first is the least
          ++cnt;
        }
      }
  *status = cnt ? 1 : (outside ? 3 : 0);
  *n_blocked = cnt;
  *hit_idx = best;
}
#endif
