// fiesta_b200 -- the skeleton handle (fiesta_skeleton_*) and its device buffers.  The definition is in fb_skel.h, the kernels in
// fb_skel.cu.
#pragma once
#include "fb_map.h"
#include "fb_nav.h"       // FbNavBox: the skeleton box uses the cost-to-go field's box layout

#define FB_SK_BATCH 8     // thinning iterations queued between two reads of their deletion counts

struct FbSkCtr {
  unsigned long long trav, anchors;          // X0 and its anchors
  unsigned long long del[FB_SK_BATCH];       // deletions per iteration of the current batch
  unsigned long long path_voxels;            // edge path voxels of the final graph
  unsigned n;                                // skeleton voxels selected from the box
  unsigned sel[3];                           // CUB selection counts: vertex roots, edge roots, voxels kept by a pruning round
  unsigned removed;                          // voxels a pruning round removes
  unsigned pad;
};
struct FbSkBufs {                  // device buffers of one fiesta_skeleton object, grown by fiesta_skeleton_compute
  FbDevBuf<uint8_t> st;            // box: state byte (FB_SK_TRAV | FB_SK_ANCHOR | FB_SK_IN), the export mask
  FbDevBuf<int32_t> M;             // box: compact id of a skeleton voxel, -1 elsewhere; after the compute the export labels
  // per skeleton voxel (capacity: the voxels thinning leaves; pruning only removes): box index in index order (double-buffered
  // across pruning rounds), 26-neighbourhood code, union-find parent word, class (1 vertex voxel, 0 chain voxel), scratch flags
  FbDevBuf<uint32_t> idx[2], code, par;
  FbDevBuf<uint8_t> cls, flag;
  // per vertex / per edge, at the same capacity: roots, sizes, coordinate sums, chain ends, orientation, pruning marks
  FbDevBuf<uint32_t> vroot, eroot, vsize, esize, end_lo, end_hi, e_att, e_first;
  FbDevBuf<unsigned long long> vsum;
  FbDevBuf<uint8_t> vrm, erm;
  FbDevBuf<long long> off;         // edge path offsets (exclusive scan of n_vox)
  // outputs: vertex size, rep [3V], centroid [3V], degree; edge uv [2E], n_vox, length, min_dist; path voxels [3 path_voxels]
  FbDevBuf<int64_t> o_vsize, o_nvox;
  FbDevBuf<int32_t> o_rep, o_vdeg, o_uv, o_vox;
  FbDevBuf<double> o_cen, o_len, o_mind;
  FbDevBuf<char> tmp;              // CUB temporary storage
  FbDevBuf<FbSkCtr> ctr;
  FbHostBuf<FbSkCtr> h_ctr;
};

struct fiesta_skeleton {
  fiesta_map *m = nullptr;
  FbSkBufs B;
  cudaEvent_t ev[4] = {};           // start, after init, after thinning, end
  FbNavBox box{};
  fiesta_skeleton_stats st{};
  bool valid = false;               // B holds the result of a compute over `box`
  ~fiesta_skeleton() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
  }
};
