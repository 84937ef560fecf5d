// fiesta_b200 -- topological roadmaps for planners: the voxel skeleton of a box's free space on the discrete generalized Voronoi
// diagram of the map's obstacles, and its graph of junctions and edges.  Plain C++ shared by the kernels (fb_skel.cu) and CPU tests
// (tests/cpp/skeleton_test.cpp, g++).
//
// Definition (DESIGN.md §3.14).  Inputs: an inclusive box B = [lo, hi], a clearance r, flags (FIESTA_SEGMENT_*), max_cos in [-1, 1)
// and min_branch >= 0.  Box indices are fb_nav_idx's, as in fiesta_nav_export.
//   1. Object.  X0 = the traversable voxels of B: fb_seg_blocks says they do not block (as a cost-to-go field at the same clearance
//      and flags).  Voxels outside B are background.
//   2. Closest obstacle.  o(v) = the obstacle coordinate of v's record, defined when the code is neither FB_UNKNOWN nor FB_INF and
//      the FB_DINF bit is clear (fb_sk_obstacle).
//   3. GVD anchor.  v in X0 with o(v) defined is an anchor when a face neighbour u in X0 (inside B) has o(u) defined, o(u) != o(v),
//      and with a = o(v) - v, b = o(u) - u (exact int64 dot products), each fp64 operation rounded on its own:
//        (double)(a.b) <= max_cos * sqrt((double)(a.a) * (double)(b.b))                                     (fb_sk_anchor_pair)
//   4. Simple point (26/6 topology).  T26(v) = the number of 26-components of X n N26*(v); T6(v) = the number of 6-components of
//      the complement of X in N18*(v) that contain one of v's 6 face neighbours; v is simple iff T26 = 1 and T6 = 1 (fb_sk_simple).
//   5. Thinning.  The subfield of v is s = 4((x-lo.x)&1) + 2((y-lo.y)&1) + ((z-lo.z)&1).  An iteration is 8 passes s = 0..7; pass s
//      deletes every voxel of subfield s that satisfies the phase's rule on X as it stands at the start of the pass.  No two voxels
//      of one subfield are 26-neighbours, so a pass equals deleting them one at a time in any order.  Phase 1 deletes simple voxels
//      that are not anchors, phase 2 simple voxels with at least two 26-neighbours in X (endpoints stay); each phase runs until an
//      iteration deletes nothing (that iteration is counted).
//   6. Graph of a set S.  deg(v) = v's 26-neighbours in S.  Vertex voxels: deg != 2, plus the smallest-index voxel of every
//      26-component of S whose voxels all have deg 2 (a pure cycle).  Vertices are the 26-components of the vertex voxels, chains
//      the 26-components of the others; both are numbered by smallest box index.  A chain is a simple path whose end voxels each
//      attach to exactly one vertex voxel (a 1-voxel chain to two).  Its edge is the voxel path attach_p, chain..., attach_q,
//      oriented so that (vertex id, attach box index, adjacent chain voxel box index) is lexicographically smaller at its start.
//      Per edge: u, v, the path's voxel count, length = the left fold of fb_nav_weight over its steps from the start, and min_dist =
//      the least GetDistance(Vector3i) over the path.  Per vertex: size, rep (its first voxel), the frontier's centroid formula and
//      degree (edge ends attached; a self-loop counts twice).
//   7. Spur pruning, in rounds on the graph of the current set until a round removes nothing (that round is counted); a round
//      removes at once (a) every edge of fewer than min_branch path voxels (the leaf voxel counted, the other attachment not) from
//      a leaf -- a vertex made of one deg-1 voxel -- to a different vertex that is not a leaf: its chain and its leaf voxel, and
//      (b) if min_branch >= 2, every deg-1 voxel whose only neighbour has deg >= 3.  No component is ever removed and the topology
//      is kept.  The skeleton is the graph of the pruned set; min_branch <= 1 disables pruning (0 rounds).
#ifndef FB_SKEL_H_
#define FB_SKEL_H_
#include "fb_nav.h"       // FbNavBox, fb_nav_idx, fb_nav_dir, fb_nav_weight
#include "fb_segment.h"   // fb_seg_blocks

// Per box voxel state byte
#define FB_SK_TRAV 1u     // in X0
#define FB_SK_ANCHOR 2u   // GVD anchor
#define FB_SK_IN 4u       // in the current set X (after the compute: the final skeleton)

// 3x3x3 neighbourhood codes: bit e = (dx+1)*9 + (dy+1)*3 + (dz+1) (fb_nav_dir's order), bit 13 the voxel itself.
#define FB_SK_FULL 0x7ffffffu
#define FB_SK_CENTER (1u << 13)
#define FB_SK_ZLO 0x1249249u      // dz = -1
#define FB_SK_ZHI 0x4924924u      // dz = +1
#define FB_SK_YLO 0x01c0e07u      // dy = -1
#define FB_SK_YHI 0x70381c0u      // dy = +1
#define FB_SK_XLO 0x00001ffu      // dx = -1
#define FB_SK_XHI 0x7fc0000u      // dx = +1
#define FB_SK_N6 ((1u << 4) | (1u << 10) | (1u << 12) | (1u << 14) | (1u << 16) | (1u << 22))
#define FB_SK_CORNERS ((1u << 0) | (1u << 2) | (1u << 6) | (1u << 8) | (1u << 18) | (1u << 20) | (1u << 24) | (1u << 26))
#define FB_SK_N18 (FB_SK_FULL & ~FB_SK_CORNERS)

FB_HD unsigned fb_sk_popc(unsigned a) {
#ifdef __CUDA_ARCH__
  return (unsigned)__popc(a);
#else
  return (unsigned)__builtin_popcount(a);
#endif
}
// One step of 6- or 26-dilation inside the 3x3x3 cube (the masks stop shifts from wrapping to the next row).
FB_HD unsigned fb_sk_dil6(unsigned a) {
  return a | ((a & ~FB_SK_ZHI) << 1) | ((a & ~FB_SK_ZLO) >> 1) | ((a & ~FB_SK_YHI) << 3) | ((a & ~FB_SK_YLO) >> 3) |
         ((a & ~FB_SK_XHI) << 9) | ((a & ~FB_SK_XLO) >> 9);
}
FB_HD unsigned fb_sk_dil26(unsigned a) {
  a |= ((a & ~FB_SK_ZHI) << 1) | ((a & ~FB_SK_ZLO) >> 1);
  a |= ((a & ~FB_SK_YHI) << 3) | ((a & ~FB_SK_YLO) >> 3);
  return a | ((a & ~FB_SK_XHI) << 9) | ((a & ~FB_SK_XLO) >> 9);
}
// The part of `set` connected to `seed` (a subset of it), by repeated dilation: a bit-parallel flood fill in registers.
FB_HD unsigned fb_sk_flood(unsigned seed, unsigned set, bool six) {
  for (;;) {
    const unsigned n = (six ? fb_sk_dil6(seed) : fb_sk_dil26(seed)) & set;
    if (n == seed) return seed;
    seed = n;
  }
}
// Is the centre simple for the set whose neighbourhood code is `code` (the centre bit is ignored)?
FB_HD bool fb_sk_simple(unsigned code) {
  const unsigned fg = code & FB_SK_FULL & ~FB_SK_CENTER;
  if (!fg) return false;                                                       // T26 = 0
  if (fb_sk_flood(fg & (0u - fg), fg, false) != fg) return false;            // T26 >= 2
  const unsigned bg = ~code & FB_SK_N18 & ~FB_SK_CENTER, faces = bg & FB_SK_N6;
  if (!faces) return false;                                                    // T6 = 0
  return (faces & ~fb_sk_flood(faces & (0u - faces), bg, true)) == 0;        // T6 = 1
}
// The thinning rule of a phase (1 or 2) for a voxel of X with neighbourhood code `code`.
FB_HD bool fb_sk_deletable(unsigned code, bool anchor, int phase) {
  if (phase == 1 && anchor) return false;
  if (phase == 2 && fb_sk_popc(code & FB_SK_FULL & ~FB_SK_CENTER) < 2) return false;
  return fb_sk_simple(code);
}
FB_HD int fb_sk_subfield(const FbNavBox &, int x, int y, int z) {   // box-local coordinates: their parity is relative to lo
  return 4 * (x & 1) + 2 * (y & 1) + (z & 1);
}

// o(v) from a packed record: false when undefined.
FB_HD bool fb_sk_obstacle(uint32_t c, int *o) {
  if (c & FB_DINF) return false;
  c &= FB_CODE_MASK;
  if (c == FB_UNKNOWN || c == FB_INF) return false;
  fb_unpack(c, o[0], o[1], o[2]);
  return true;
}
// The anchor test between a voxel v with obstacle ov and a face neighbour u with obstacle ou (both defined).
FB_HD bool fb_sk_anchor_pair(const int *v, const int *ov, const int *u, const int *ou, double max_cos) {
  if (ov[0] == ou[0] && ov[1] == ou[1] && ov[2] == ou[2]) return false;
  long long a[3], b[3];
  for (int k = 0; k < 3; ++k) { a[k] = (long long)ov[k] - v[k]; b[k] = (long long)ou[k] - u[k]; }
  const long long ab = a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
  const long long aa = a[0] * a[0] + a[1] * a[1] + a[2] * a[2];
  const long long bb = b[0] * b[0] + b[1] * b[1] + b[2] * b[2];
  const double p = (double)aa * (double)bb;
  const double s = sqrt(p);
  const double rhs = max_cos * s;
  return (double)ab <= rhs;
}
#endif
