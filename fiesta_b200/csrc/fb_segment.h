// fiesta_b200 -- segment clearance: is the straight segment a-b at least r away from every obstacle, and if not, where does it
// first come too close?  The exact voxel walk and the per-voxel test, shared by the kernel (fb_segment.cu, one warp per segment)
// and the pinned host mirror (sequential).  Plain C++: tests/cpp/segment_test.cpp checks it on the CPU with g++.
//
// Definition (DESIGN.md §3.4).  An endpoint p maps to voxel units with Pos2Vox's own expression, u = (p - origin) / res in fp64,
// and is truncated to a fixed-point lattice, q = floor(u * 2^20) (exact; floor(q / 2^20) == Pos2Vox(p)).  The voxels walked are
// V = { floor(p(t)) : t in [0,1] }, p(t) = qa + t (qb - qa), in t order: at a crossing, axes moving up step AT the crossing
// parameter t*, axes moving down step just after it, so an edge or corner crossing yields the one or two voxels the floor gives
// there and no others.  A voxel blocks when GetDistance(Vector3i) <= r, or, with FIESTA_SEGMENT_UNKNOWN_BLOCKS, when it was never
// observed.  Upper-face coordinates == G read +10000 and never block.
//
// Arithmetic: grids have <= 2046 voxels per axis, so 0 <= q < 2^31.  A crossing parameter is n / den with n <= den = |qb - qa|
// < 2^31 (one axis' displacement); comparisons cross-multiply (< 2^62), and a voxel at a given crossing is one floor division of
// c * den < 2^62.  Everything is exact 64-bit integer arithmetic: host and device decide ties and near-ties identically.
//
// Slabs: the crossings of the axis with the largest displacement (the slab axis) cut V into nslabs = 1 + (number of those
// crossings) consecutive runs.  Slab j >= 1 starts at the slab axis' j-th crossing -- at t* for an axis moving up, just after t*
// for one moving down -- and ends where slab j + 1 starts; slab 0 starts at t = 0.  The slabs partition V in order, with no gap and
// no duplicate, and each can be walked on its own from its exactly computed entry voxel.
#ifndef FB_SEGMENT_H_
#define FB_SEGMENT_H_
#include "fb_record.h"

#define FB_SEG_QBITS 20
#define FB_SEG_Q (1ll << FB_SEG_QBITS)

struct FbSeg {
  long long qa[3], qb[3];   // endpoints on the 2^-20 voxel lattice
  long long den[3];         // |qb - qa|
  int dir[3];               // sign of qb - qa
  int v0[3];                // start voxel, floor(qa / 2^20)
  int dom;                  // slab axis: the largest |qb - qa|, lowest axis on a tie
  int nslabs;
};

// Endpoint setup.  False when an endpoint fails PosInMap (ESDFMap.cpp:46-61) or has a NaN coordinate (which PosInMap's
// comparisons let through); the box is convex, so two endpoints in the map put the whole segment in it.
FB_HD bool fb_seg_setup(const FbGeom &g, const double *ab, FbSeg &s) {
  for (int k = 0; k < 6; ++k)
    if (ab[k] != ab[k]) return false;
  if (!fb_pos_in_map(g, ab) || !fb_pos_in_map(g, ab + 3)) return false;
  s.dom = 0;
  for (int k = 0; k < 3; ++k) {
    const double ua = (ab[k] - g.origin[k]) / g.res, ub = (ab[k + 3] - g.origin[k]) / g.res;
    s.qa[k] = (long long)floor(ua * (double)FB_SEG_Q);
    s.qb[k] = (long long)floor(ub * (double)FB_SEG_Q);
    const long long d = s.qb[k] - s.qa[k];
    s.dir[k] = d > 0 ? 1 : (d < 0 ? -1 : 0);
    s.den[k] = d < 0 ? -d : d;
    s.v0[k] = (int)(s.qa[k] >> FB_SEG_QBITS);
    if (s.den[k] > s.den[s.dom]) s.dom = k;
  }
  const int a = s.dom, va1 = (int)(s.qb[a] >> FB_SEG_QBITS);
  s.nslabs = 1 + (va1 > s.v0[a] ? va1 - s.v0[a] : s.v0[a] - va1);
  return true;
}

// Entry of slab j: its first voxel v and the parameter tn / td at which V enters it.
FB_HD void fb_seg_entry(const FbSeg &s, int j, int *v, long long &tn, long long &td) {
  if (j == 0) {
    for (int k = 0; k < 3; ++k) v[k] = s.v0[k];
    tn = 0; td = 1;
    return;
  }
  const int a = s.dom;
  const bool up = s.dir[a] > 0;
  const long long plane = (long long)(up ? s.v0[a] + j : s.v0[a] - j + 1) * FB_SEG_Q;
  tn = up ? plane - s.qa[a] : s.qa[a] - plane;
  td = s.den[a];
  const long long D = FB_SEG_Q * td;
  for (int k = 0; k < 3; ++k) {
    const long long X = s.qa[k] * td + s.dir[k] * (tn * s.den[k]);     // coordinate at t* times td: 0 <= X <= td * max(qa, qb) < 2^62
    // floor at t* itself; an axis moving down whose coordinate sits on a plane has already stepped when the slab axis steps just after t*
    v[k] = (int)((!up && s.dir[k] < 0) ? (X + D - 1) / D - 1 : X / D);
  }
}

// Walk slabs [j0, j1) in t order; visit(v, tn, td) is called for every voxel of V with the parameter at which it is entered and
// returns true to stop.
template <class Visit>
FB_HD void fb_seg_walk(const FbSeg &s, int j0, int j1, Visit &visit) {
  int v[3];
  long long tn, td;
  fb_seg_entry(s, j0, v, tn, td);
  if (visit(v, tn, td)) return;
  const int a = s.dom;
  for (;;) {
    long long n[3], bn = 0, bd = 1;
    bool ok[3], any = false;
    for (int k = 0; k < 3; ++k) {                                       // next crossing of each axis, as n[k] / den[k]
      ok[k] = false;
      n[k] = 0;
      if (s.dir[k] > 0) { const long long p = (long long)(v[k] + 1) * FB_SEG_Q; ok[k] = p <= s.qb[k]; n[k] = p - s.qa[k]; }
      else if (s.dir[k] < 0) { const long long p = (long long)v[k] * FB_SEG_Q; ok[k] = p > s.qb[k]; n[k] = s.qa[k] - p; }
      if (ok[k] && (!any || n[k] * bd < bn * s.den[k])) { bn = n[k]; bd = s.den[k]; any = true; }
    }
    if (!any) return;
    bool at[3];
    for (int k = 0; k < 3; ++k) at[k] = ok[k] && n[k] * bd == bn * s.den[k];
    const int done = s.dir[a] > 0 ? v[a] - s.v0[a] : s.v0[a] - v[a];
    const bool end = at[a] && done + 1 == j1;                           // the slab axis' next step starts slab j1
    if (end && s.dir[a] > 0) return;
    bool step = false;
    for (int k = 0; k < 3; ++k)
      if (at[k] && s.dir[k] > 0) { ++v[k]; step = true; }
    if (step && visit(v, bn, bd)) return;
    if (end) return;
    step = false;
    for (int k = 0; k < 3; ++k)
      if (at[k] && s.dir[k] < 0) { --v[k]; step = true; }
    if (step && visit(v, bn, bd)) return;
  }
}

// Block test on a packed record: d = GetDistance(Vector3i) of voxel v (+10000 when unknown, unreached, FB_DINF or outside the
// grid, as fb_get_distance_vox reads it).  Callers keep r < +10000, so +10000 never blocks.
FB_HD bool fb_seg_blocks(const FbGeom &g, const uint32_t *rec, const int *v, double r, bool unknown_blocks, double &d) {
  if (!fb_in_grid(g, v[0], v[1], v[2])) { d = (double)FIESTA_INFINITY; return false; }
  d = fb_record_distance(fb_ld_record(&rec[fb_ii(g, v[0], v[1], v[2])]), v[0], v[1], v[2], g.res);
  if (d < 0) { d = (double)FIESTA_INFINITY; return unknown_blocks; }
  return d <= r;
}

// Visitor: the minimum distance over the voxels walked and the first blocking voxel; stops there.
struct FbSegScan {
  const FbGeom *g;
  const uint32_t *rec;
  double r;
  bool unknown_blocks;
  double min_d;
  bool hit;
  int hv[3];
  long long tn, td;
  FB_HD bool operator()(const int *v, long long n, long long d) {
    double dist;
    const bool b = fb_seg_blocks(*g, rec, v, r, unknown_blocks, dist);
    if (dist < min_d) min_d = dist;
    if (!b) return false;
    hit = true;
    hv[0] = v[0]; hv[1] = v[1]; hv[2] = v[2];
    tn = n; td = d;
    return true;
  }
};
FB_HD FbSegScan fb_seg_scan(const FbGeom &g, const uint32_t *rec, double r, bool unknown_blocks) {
  FbSegScan sc;
  sc.g = &g; sc.rec = rec; sc.r = r; sc.unknown_blocks = unknown_blocks;
  sc.min_d = (double)FIESTA_INFINITY; sc.hit = false;
  sc.hv[0] = sc.hv[1] = sc.hv[2] = 0; sc.tn = 0; sc.td = 1;
  return sc;
}

// The four outputs: status 0 clear / 1 blocked / 2 outside the map; hit_idx = x*Gy*Gz + y*Gz + z of the first blocking voxel or -1;
// hit_t = the parameter at which it is entered (one correctly rounded division of two exact integers) or NaN; min_dist.
FB_HD void fb_seg_outside(int32_t *status, int64_t *hit_idx, double *hit_t, double *min_dist) {
  *status = 2; *hit_idx = -1; *hit_t = nan(""); *min_dist = (double)FIESTA_UNDEFINED;
}
FB_HD void fb_seg_store(const FbGeom &g, const FbSegScan &sc, double min_d, int32_t *status, int64_t *hit_idx, double *hit_t,
                        double *min_dist) {
  *status = sc.hit ? 1 : 0;
  *hit_idx = sc.hit ? (int64_t)sc.hv[0] * g.gyz + (int64_t)sc.hv[1] * g.gz + sc.hv[2] : -1;
  *hit_t = sc.hit ? (double)sc.tn / (double)sc.td : nan("");
  *min_dist = min_d;
}

// One segment, sequentially (host side of the pinned mirror; the reference for the kernel).
FB_HD void fb_seg_check(const FbGeom &g, const uint32_t *rec, const double *ab, double r, bool unknown_blocks, int32_t *status,
                        int64_t *hit_idx, double *hit_t, double *min_dist) {
  FbSeg s;
  if (!fb_seg_setup(g, ab, s)) { fb_seg_outside(status, hit_idx, hit_t, min_dist); return; }
  FbSegScan sc = fb_seg_scan(g, rec, r, unknown_blocks);
  fb_seg_walk(s, 0, s.nslabs, sc);
  fb_seg_store(g, sc, sc.min_d, status, hit_idx, hit_t, min_dist);
}
#endif
