// fiesta_b200 -- viewpoint coverage for exploration planners: how many members of a frontier cluster would a sensor at a candidate
// pose see?  The candidate status, the range and field-of-view tests of one (candidate, member) pair and the line-of-sight visitor,
// shared by the kernels (fb_view.cu) and CPU tests (tests/cpp/viewpoint_test.cpp, g++).
//
// Definition (DESIGN.md §3.7).  A candidate p (metres) has status 2 when it fails PosInMap or has a NaN coordinate (the segment
// query's rule), 1 when its voxel Pos2Vox(p) is outside the grid, never observed or has GetDistance(Vector3i) <= clearance (unknown
// space always counts, whatever the flags), else 0.  For a status-0 candidate and a member voxel v of its cluster, each fp64
// operation rounded on its own:
//   c_k = ((double)v_k + 0.5) * res + origin_k          (Vox2Pos)        d_k = c_k - p_k
//   in range   (d0*d0 + d1*d1) + d2*d2 <= max_range * max_range
//   in view j  s_k = (R[k][0]*d0 + R[k][1]*d1) + R[k][2]*d2,  s0 > 0 && fabs(s1) <= tan_h * s0 && fabs(s2) <= tan_v * s0
//   visible    fiesta_check_segments on {p, c} at clearance 0 with the caller's flags returns status 0: no voxel of the exact walk
//              of fb_segment.h is an obstacle (GetDistance(Vector3i) == 0) nor, with FIESTA_SEGMENT_UNKNOWN_BLOCKS, never observed.
// score[i][j] counts the members that are in range, in view for orientation j and visible.
//
// Work decomposition: candidate i with status 0 owns fb_view_chunks(size of its cluster) chunks of 32 consecutive members; the
// chunks of all candidates form one flat list in candidate order, and fb_view_find maps a position in it back to its candidate.
#ifndef FB_VIEW_H_
#define FB_VIEW_H_
#include "fb_segment.h"   // fb_seg_setup / fb_seg_walk / fb_seg_blocks: the line of sight is the segment query's walk at r = 0

#define FB_VIEW_MAX_ORIENT 32   // one bit per orientation in a 32-bit mask
#define FB_VIEW_CHUNK 32        // members per work item: one per lane of a warp

FB_HD int fb_view_status(const FbGeom &g, const uint32_t *rec, const double *p, double clearance) {
  if (p[0] != p[0] || p[1] != p[1] || p[2] != p[2] || !fb_pos_in_map(g, p)) return 2;
  int v[3];
  fb_pos2vox(g, p, v);
  double d;
  if (!fb_in_grid(g, v[0], v[1], v[2]) || fb_seg_blocks(g, rec, v, clearance, true, d)) return 1;
  return 0;
}

FB_HD long long fb_view_chunks(long long size) { return (size + FB_VIEW_CHUNK - 1) / FB_VIEW_CHUNK; }

// The last candidate i in [0, n) with first[i] <= w, for first = the exclusive prefix sum of the candidates' chunk counts and
// 0 <= w < first[n]: the candidate that owns chunk w (candidates without work share their first[] with the next one and lose).
FB_HD long long fb_view_find(const long long *first, long long n, long long w) {
  long long lo = 0, hi = n;   // first[lo] <= w < first[hi]
  while (hi - lo > 1) {
    const long long mid = lo + (hi - lo) / 2;
    if (first[mid] <= w) lo = mid; else hi = mid;
  }
  return lo;
}

// Member voxel v seen from p: its centre c and the offset d = c - p.
FB_HD void fb_view_offset(const FbGeom &g, const int *v, const double *p, double *c, double *d) {
  for (int k = 0; k < 3; ++k) {
    c[k] = ((double)v[k] + 0.5) * g.res + g.origin[k];
    d[k] = c[k] - p[k];
  }
}

FB_HD bool fb_view_in_range(const double *d, double range2) { return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] <= range2; }

// Bit j set when d is inside the field of view of orientation j: R holds n_orient row-major 3x3 world-to-sensor matrices.
FB_HD unsigned fb_view_mask(const double *R, int n_orient, const double *d, double tan_h, double tan_v) {
  unsigned mask = 0u;
  for (int j = 0; j < n_orient; ++j) {
    const double *r = R + 9 * j;
    const double s0 = (r[0] * d[0] + r[1] * d[1]) + r[2] * d[2];
    const double s1 = (r[3] * d[0] + r[4] * d[1]) + r[5] * d[2];
    const double s2 = (r[6] * d[0] + r[7] * d[1]) + r[8] * d[2];
    if (s0 > 0 && fabs(s1) <= tan_h * s0 && fabs(s2) <= tan_v * s0) mask |= 1u << j;
  }
  return mask;
}

// Visitor for fb_seg_walk: stops at the first voxel that blocks at r = 0.
struct FbViewLos {
  const FbGeom *g;
  const uint32_t *rec;
  bool unknown_blocks;
  bool blocked;
  FB_HD bool operator()(const int *v, long long, long long) {
    double d;
    blocked = fb_seg_blocks(*g, rec, v, 0.0, unknown_blocks, d);
    return blocked;
  }
};

// Is the segment p-c clear at clearance 0 (status 0 of fiesta_check_segments)?
FB_HD bool fb_view_visible(const FbGeom &g, const uint32_t *rec, const double *p, const double *c, bool unknown_blocks) {
  const double ab[6] = {p[0], p[1], p[2], c[0], c[1], c[2]};
  FbSeg s;
  if (!fb_seg_setup(g, ab, s)) return false;
  FbViewLos los{&g, rec, unknown_blocks, false};
  fb_seg_walk(s, 0, s.nslabs, los);
  return !los.blocked;
}
#endif
