// fiesta_b200 -- the frontier handle and the buffer types shared by fb_frontier.cu (extraction) and fb_view.cu (viewpoint coverage
// of its clusters).  The definitions are in fb_frontier.h and fb_view.h.
#pragma once
#include "fb_map.h"
#include "fb_nav.h"       // FbNavBox: the frontier box uses the cost-to-go field's box layout

// Union-find by index in global memory, shared by the frontier's clusters (over the box) and the skeleton's graph (over its
// compacted voxels, fb_skel.cu).  Parent words only ever decrease and point at a smaller index of the same component, so after
// the unions every component is one tree rooted at its smallest index, whatever order they ran in.
//
// Root of x, halving the path on the way.  The shortcut is an atomicMin, so it can only lower a parent word to another ancestor
// and never undo a concurrent hook.
static __device__ unsigned fr_find(uint32_t *P, unsigned x) {
  unsigned p = __ldcg(&P[x]);
  while (p != x) {
    const unsigned gp = __ldcg(&P[p]);
    if (gp < p) atomicMin(&P[x], gp);
    x = p; p = gp;
  }
  return x;
}
static __device__ void fr_union(uint32_t *P, unsigned a, unsigned b) {
  for (;;) {
    a = fr_find(P, a); b = fr_find(P, b);
    if (a == b) return;
    if (a > b) { const unsigned t = a; a = b; b = t; }
    const unsigned old = atomicMin(&P[b], a);
    if (old == b) return;
    b = old;
  }
}

struct FbFrCtr {
  unsigned long long frontier;     // frontier voxels of the box
  unsigned long long roots;        // clusters before the size filter
  unsigned long long kept_voxels;  // members of the kept clusters
  unsigned sel[3];                 // CUB selection counts: roots, kept clusters, kept members
  unsigned pad;
};
struct FbFrBufs {                  // device buffers of one fiesta_frontiers object, grown by fiesta_frontiers_compute
  FbDevBuf<uint32_t> P;            // box: union-find parent words (FR_NONE off the frontier)
  FbDevBuf<int32_t> L;             // box: cluster label, -1 elsewhere (fiesta_frontiers_export)
  // per cluster before the size filter (C of them): root box index, size, kept ids in order, pre-filter id -> kept id or -1,
  // grid-coordinate sums [3C], bounding boxes [lo 3C][hi 3C]
  FbDevBuf<uint32_t> roots, size, kept;
  FbDevBuf<int32_t> newid, box;
  FbDevBuf<unsigned long long> sum;
  // outputs per kept cluster, at pre-filter capacity C: size, [rep 3C][bbox lo 3C][bbox hi 3C], centroid [3C]
  FbDevBuf<int64_t> o_size;
  FbDevBuf<int32_t> o_i32;
  FbDevBuf<double> o_cen;
  // per member: sort keys and box indices (double-buffered), then the grid xyz of the sorted members
  FbDevBuf<uint32_t> mkey[2], mval[2];
  FbDevBuf<int32_t> m_xyz;
  FbDevBuf<char> tmp;              // CUB temporary storage
  FbDevBuf<FbFrCtr> ctr;
  FbHostBuf<FbFrCtr> h_ctr;
  unsigned C = 0;                  // pre-filter clusters of the last compute: the stride of o_i32
};
// viewpoint coverage of frontier clusters (fb_view.cu)
struct FbViewCtr {
  unsigned long long scored, walked, visible;   // status-0 candidates, pairs in range and view, walked pairs with a clear line of sight
};
struct FbViewBufs {                // device buffers of fiesta_frontiers_score_viewpoints, kept on the frontier object
  FbDevBuf<double> pos;            // per candidate: position [3n]
  FbDevBuf<int32_t> cl, status;    //                cluster id, status
  FbDevBuf<long long> work;        //                [n + 1] chunk counts, scanned in place to each one's first chunk (work[n]: total)
  FbDevBuf<int32_t> score;         //                [n * n_orient]
  FbDevBuf<long long> moff;        // per kept cluster: its first member in the member list
  FbDevBuf<double> orient;         // [9 * n_orient]
  FbDevBuf<FbViewCtr> ctr;
  FbHostBuf<FbViewCtr> h_ctr;
};

struct fiesta_frontiers {
  fiesta_map *m = nullptr;
  FbFrBufs B;
  FbViewBufs V;                     // fiesta_frontiers_score_viewpoints
  cudaEvent_t ev[2] = {};
  FbNavBox box{};
  fiesta_frontier_stats st{};
  bool valid = false;               // B holds the result of a compute over `box`
  ~fiesta_frontiers() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
  }
};
