// fiesta_b200 -- the cost-to-go field handle and the launch types shared by fb_nav.cu (fields, updates, paths) and
// fb_navmatrix.cu (cost matrices).  The field's definition and box layout are in fb_nav.h.
#pragma once
#include "fb_map.h"
#include "fb_nav.h"

struct FbNavCtr {
  unsigned n[3];               // tile work-list lengths, rotating by generation (k_nav_relax)
  unsigned next[3];            // dynamic tile fetch counters, rotating the same way
  unsigned generations, pad;
  unsigned long long goals_placed, blocked, reached, tile_visits;
};
struct FbNavArgs {
  double *D;                   // the field, box layout (fb_nav.h)
  FbNavBox b;
  int tn[3];                   // 8^3 tiles per box axis
  double w[3];                 // res * sqrt(1), res * sqrt(2), res * sqrt(3)
  uint32_t *stamp;             // per tile: stamp of the generation it is queued for (generation g has stamp g + 1)
  uint32_t *list[2];           // tile work lists by generation parity
  FbNavCtr *ctr;
};
// field update (DESIGN.md §3.11)
struct FbNavUCtr {
  FbNavCtr wave;               // the withdrawal wave's work lists, generations and tile visits
  unsigned long long became_blocked, became_free, withdrawn, goals_new;
  unsigned seed_tiles, pad;
};
// cost matrices: up to FB_NAVM_CH sources' fields relaxed together, one channel each
#define FB_NAVM_CH 32
struct FbNavMCtr {                 // per pass; zeroed before it
  unsigned n[3], next[3];          // work-list lengths and fetch counters, rotating by generation as in FbNavCtr
  unsigned long long mmin[FB_NAVM_CH][3];   // per channel: bits of the least value written in generation g, slot g % 3
  unsigned queued[FB_NAVM_CH][3];           // per channel: work items queued for generation g, slot g % 3
  unsigned retired[FB_NAVM_CH];             // the channel's targets are final: its work items are dropped
};
struct FbNavMTot {                 // summed over the passes of a call
  unsigned long long generations, tile_visits, retired_early;
};
struct FbNavMArgs {
  double *D;                       // [channel][box index] (fb_nav.h layout); +inf until reached
  const uint32_t *M;               // per box voxel: fb_nav_move_bits
  FbNavBox b;
  int tn[3];                       // 8^3 tiles per box axis
  unsigned nt;                     // tiles per channel; a work item is channel * nt + tile
  long long nv;                    // box voxels
  double w[3];
  uint32_t *stamp;                 // per work item: stamp of the generation it is queued for (generation g has stamp g + 1)
  uint32_t *list[2];               // work lists by generation parity
  FbNavMCtr *ctr;
  FbNavMTot *tot;
  const long long *tgt;            // box indices of the status-0 targets
  int n_tgt, nch;                  // status-0 targets, channels of this pass
};
int fb_navm_relax_blocks(int device);   // co-resident CTAs of k_navm_relax (fb_navmatrix.cu)

struct fiesta_nav_field {
  fiesta_map *m = nullptr;
  int blocks = 0;                   // co-resident CTAs of k_nav_relax (cooperative launch)
  int wblocks = 0;                  // co-resident CTAs of k_navu_withdraw
  FbDevBuf<double> D, d_goals;
  FbDevBuf<uint32_t> stamp, list[2];
  FbDevBuf<FbNavCtr> ctr;
  FbHostBuf<FbNavCtr> h_ctr;
  FbDevBuf<double> d_pd;            // fiesta_nav_paths: [starts 3n][cost n]
  FbDevBuf<int32_t> d_pi;           //                   [status n][len n][vox 3 n max_len]
  FbDevBuf<uint8_t> u_flags;        // fiesta_nav_update: one scratch byte per box voxel
  FbDevBuf<FbNavUCtr> u_ctr;
  FbHostBuf<FbNavUCtr> h_uctr;
  // fiesta_nav_matrix: its own buffers, so that a matrix leaves the last field, export and paths as they were
  int mblocks = 0;                  // co-resident CTAs of k_navm_relax
  FbDevBuf<uint32_t> M;             // per box voxel: move mask
  FbDevBuf<double> MD, m_pts, m_cost;   // [channel][box voxel] fields; points [sources 3 n_src][targets 3 n_tgt]; cost
  FbDevBuf<uint32_t> m_stamp, m_list[2];  // per (channel, tile)
  FbDevBuf<int32_t> m_st, m_rows;   // per point: status; rows: placed sources in index order, then the others
  FbDevBuf<long long> m_idx, m_src, m_tgt;  // per point: box index or -1; placed sources' box indices; placed targets' box indices
  FbDevBuf<FbNavMCtr> m_ctr;
  FbDevBuf<FbNavMTot> m_tot;
  FbHostBuf<FbNavMTot> h_mtot;
  cudaEvent_t ev[2] = {};
  FbNavBox box{};
  double w[3]{};
  bool valid = false;               // D holds a field computed for `box`
  long long n_goals = 0;            // goals (in d_goals), clearance and flags of the last compute: what fiesta_nav_update keeps
  double clearance = 0.0;
  int flags = 0;
  ~fiesta_nav_field() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
  }
};
