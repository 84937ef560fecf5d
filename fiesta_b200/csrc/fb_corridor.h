// fiesta_b200 -- safe flight corridors for planners: free axis-aligned voxel boxes inflated face by face, and chains of them along
// a path in which consecutive boxes share a voxel.  Plain C++ shared by the kernels (fb_corridor.cu, one warp per seed or path) and
// the CPU test (tests/cpp/corridor_test.cpp, g++).
//
// Definition (DESIGN.md §3.8).  All boxes are inclusive voxel boxes [lo, hi].  A voxel is traversable when it lies in the limit box
// L and fb_seg_blocks says it does not block at the clearance with the caller's flags -- the predicate of the cost-to-go field.
//   inflate  B = S (a seed box whose voxels are all traversable), all six faces active.  Rounds visit the faces in the order
//            -x, +x, -y, +y, -z, +z; an active face that has reached L or max_steps[axis] layers beyond the seed's face is
//            deactivated; otherwise the one-voxel-thick layer just outside it, spanning B's current extent on the other two axes,
//            is tested: all traversable -> B grows by it, else the face is deactivated for good (the other faces only grow, so a
//            later layer on this face would still hold the blocking voxel).  Stops when no face is active.
//   chain    a path P[0..n-1] of grid voxels: status 2 (no boxes) when some P[i] is outside L.  The first seed is {P[0]}; after a
//            box whose seed index is j, let i be the first index > j with P[i] outside the box: none -> status 0; otherwise the next
//            seed is AABB(P[i-1], P[i]) with seed index i.  A seed holding a non-traversable voxel stops the chain with status 1 and
//            blocked_at = its seed index; the boxes before it are kept.
// The access to the voxels is the accessor's: the CPU test evaluates the predicate voxel by voxel, the kernel reads bit masks with
// a whole warp.  The rule itself is only here.
#ifndef FB_CORRIDOR_H_
#define FB_CORRIDOR_H_
#include "fb_segment.h"

#define FB_CORR_OK 0
#define FB_CORR_BLOCKED 1
#define FB_CORR_OUTSIDE 2

struct FbCorrCount {
  long long tested, grown;   // layer tests of the rule (grown + refused), and grown layers
};

// Inflate [lo, hi] in place.  Acc: bool box_free(const int *lo, const int *hi) -- every voxel of the box is traversable.
template <class Acc>
FB_HD void fb_corr_inflate(Acc &acc, const int *L_lo, const int *L_hi, const int *max_steps, int *lo, int *hi, FbCorrCount &c) {
  long long stop_lo[3], stop_hi[3];                                      // 64-bit: max_steps may be as large as INT_MAX
  for (int k = 0; k < 3; ++k) {
    const long long a = (long long)lo[k] - max_steps[k], b = (long long)hi[k] + max_steps[k];
    stop_lo[k] = a > L_lo[k] ? a : L_lo[k];
    stop_hi[k] = b < L_hi[k] ? b : L_hi[k];
  }
  unsigned active = 0x3fu;
  while (active) {
    for (int f = 0; f < 6; ++f) {
      if (!((active >> f) & 1u)) continue;
      const int a = f >> 1;
      const bool up = (f & 1) != 0;
      if (up ? hi[a] >= stop_hi[a] : lo[a] <= stop_lo[a]) { active &= ~(1u << f); continue; }
      int llo[3] = {lo[0], lo[1], lo[2]}, lhi[3] = {hi[0], hi[1], hi[2]};
      llo[a] = lhi[a] = up ? hi[a] + 1 : lo[a] - 1;
      ++c.tested;
      if (acc.box_free(llo, lhi)) {
        if (up) ++hi[a]; else --lo[a];
        ++c.grown;
      } else {
        active &= ~(1u << f);
      }
    }
  }
}

FB_HD bool fb_corr_inside(const int *v, const int *lo, const int *hi) {
  return v[0] >= lo[0] && v[0] <= hi[0] && v[1] >= lo[1] && v[1] <= hi[1] && v[2] >= lo[2] && v[2] <= hi[2];
}

// The chain of one path of n voxels.  Acc: box_free as above; void vox(int i, int *v) -- P[i]; bool any_outside(lo, hi) -- some
// P[i] lies outside the box; int next_outside(int j, lo, hi) -- the first i > j with P[i] outside the box, n if none;
// void emit(int k, lo, hi, int j) -- box k with seed index j.  Returns the status; *n_boxes and *blocked_at (-1 unless status 1).
template <class Acc>
FB_HD int fb_corr_chain(Acc &acc, int n, const int *L_lo, const int *L_hi, const int *max_steps, int *n_boxes, int *blocked_at,
                        FbCorrCount &c) {
  *n_boxes = 0;
  *blocked_at = -1;
  if (n == 0) return FB_CORR_OK;
  if (acc.any_outside(L_lo, L_hi)) return FB_CORR_OUTSIDE;
  int lo[3], hi[3], j = 0;
  acc.vox(0, lo);
  acc.vox(0, hi);
  for (;;) {
    if (!acc.box_free(lo, hi)) { *blocked_at = j; return FB_CORR_BLOCKED; }
    fb_corr_inflate(acc, L_lo, L_hi, max_steps, lo, hi, c);
    acc.emit(*n_boxes, lo, hi, j);
    ++*n_boxes;
    const int i = acc.next_outside(j, lo, hi);
    if (i >= n) return FB_CORR_OK;
    int a[3], b[3];
    acc.vox(i - 1, a);
    acc.vox(i, b);
    for (int k = 0; k < 3; ++k) { lo[k] = a[k] < b[k] ? a[k] : b[k]; hi[k] = a[k] < b[k] ? b[k] : a[k]; }
    j = i;
  }
}

// One independent seed: FB_CORR_OUTSIDE when it is inverted or not inside L, FB_CORR_BLOCKED when it holds a non-traversable
// voxel, else it is inflated in place.
template <class Acc>
FB_HD int fb_corr_seed(Acc &acc, const int *L_lo, const int *L_hi, const int *max_steps, int *lo, int *hi, FbCorrCount &c) {
  for (int k = 0; k < 3; ++k)
    if (!(lo[k] <= hi[k] && lo[k] >= L_lo[k] && hi[k] <= L_hi[k])) return FB_CORR_OUTSIDE;
  if (!acc.box_free(lo, hi)) return FB_CORR_BLOCKED;
  fb_corr_inflate(acc, L_lo, L_hi, max_steps, lo, hi, c);
  return FB_CORR_OK;
}

// Bit masks of the traversable voxels of L (box-local coordinates, L's extents n[3]): bit 1 = traversable.
//   z-rows  per (x, y): wz = ceil(n.z / 32) words, word ((x * n.y + y) * wz + z / 32), bit z % 32   (layers of the +-x, +-y faces)
//   y-rows  per (z, x): wy = ceil(n.y / 32) words, word ((z * n.x + x) * wy + y / 32), bit y % 32   (layers of the +-z faces)
struct FbCorrMask {
  int lo[3], n[3];
  int wz, wy;
  long long zwords;          // n.x * n.y * wz: the y-rows follow the z-rows
};
FB_HD FbCorrMask fb_corr_mask_geom(const int *L_lo, const int *L_hi) {
  FbCorrMask M;
  for (int k = 0; k < 3; ++k) { M.lo[k] = L_lo[k]; M.n[k] = L_hi[k] - L_lo[k] + 1; }
  M.wz = (M.n[2] + 31) >> 5;
  M.wy = (M.n[1] + 31) >> 5;
  M.zwords = (long long)M.n[0] * M.n[1] * M.wz;
  return M;
}
FB_HD long long fb_corr_mask_words(const FbCorrMask &M) { return M.zwords + (long long)M.n[2] * M.n[0] * M.wy; }
#endif
