// fiesta_b200 -- host state of a map, and the map functions and argument checks the planner modules share (defined in fb_map.cu).
//
// Internal to the library: the C ABI is include/fiesta_b200.h.  A feature's entry points live beside its kernels and reach the
// map through this header.
#pragma once
#include <memory>
#include <new>
#include "../../include/fiesta_b200.h"
#include "fb_common.cuh"
#include "fb_exact.h"

struct FbNavBox;
// Defined in fb_corridor.cu, the only file that reads or writes it.  The map only holds the two buffers, and FbBuf<T> needs the
// complete type for nothing but alloc / grow (sizeof(T)), which only fb_corridor.cu calls.
struct FbCorrCtr;
struct FbCorrBufs {                // device buffers of fiesta_inflate_boxes / fiesta_corridors, kept on the map
  FbDevBuf<uint32_t> mask;         // the limit box's traversable bits, z-rows then y-rows (fb_corridor.h)
  FbDevBuf<int32_t> in;            // seeds [lo 3n][hi 3n], or path voxels [3 total]
  FbDevBuf<int64_t> off;           // path offsets [n_paths + 1]
  FbDevBuf<int32_t> out;           // seeds: [status n][lo 3n][hi 3n]; paths: [status][n_boxes][blocked_at] x n_paths, [lo 3T][hi 3T][first T]
  FbDevBuf<FbCorrCtr> ctr;
  FbHostBuf<FbCorrCtr> h_ctr;
};
struct FbPoseBufs {                // device buffers of fiesta_check_poses(_device), kept on the map
  FbDevBuf<char> io;               // host form: [poses 12n][hit_idx n] 8-byte words, [status n][n_blocked n] int32
  FbDevBuf<long long> work;        // [n + 1] chunk counts, scanned in place to each pose's first work item (work[n]: total)
  FbDevBuf<char> tmp;              // CUB temporary storage
};

struct fiesta_map {
  FbGeom g{};
  fiesta_config cfg{};              // as given at create, with the device and the mode in force (fiesta_get_config, snapshots)
  int device = 0;
  cudaStream_t stream = nullptr;
  bool params_set = false;
  double l_hit = 0, l_miss = 0, l_min = 0, l_max = 0, l_occ = 0;
  double l_cornor[3]{}, r_cornor[3]{};
  // per-voxel state
  FbDevBuf<uint32_t> cobs, cobs_b, stamp[2], occbits;
  FbDevBuf<double> occ;
  FbDevBuf<unsigned long long> cnt;
  // tiles
  FbDevBuf<uint32_t> tile_flag, nb_flag, list[2], changed[2], changed_bbox[2];
  CUtensorMap tmap{};
  int wf_blocks = 0, rr_blocks = 0;
  // queues
  FbDevBuf<uint32_t> touch_flag, touch_list;
  unsigned touch_epoch = 0;
  FbDevBuf<uint32_t> ins, del;
  unsigned n_touch_tiles = 0, n_ins = 0, n_del = 0;  // host view (valid after the last sync)
  FbDevBuf<FbCounters> d_ctr;
  FbHostBuf<FbCounters> h_ctr;
  // per-call SetOccupancy staging
  FbHostBuf<uint32_t> h_ev;
  FbDevBuf<uint32_t> d_ev;
  size_t n_ev = 0;
  // ray casting
  FbDevBuf<float> d_xyz;
  FbDevBuf<uint32_t> ray_list;
  FbDevBuf<int> ray_len, ray_reach;
  FbDevBuf<unsigned> ray_dirty;
  unsigned frame_tag = 0, owner_tag = 0;
  // queries
  FbDevBuf<double> d_qin, d_qout;
  FbDevBuf<char> d_seg;             // fiesta_check_segments: [ab 6n][hit_t n][min_dist n] doubles, [hit_idx n] int64, [status n] int32
  FbCorrBufs corr;                  // fiesta_inflate_boxes / fiesta_corridors
  FbPoseBufs pose;                  // fiesta_check_poses / fiesta_check_poses_device
  cudaEvent_t ev[4] = {};
  cudaEvent_t ev_q[2] = {};         // device queries: map stream -> caller's stream, and back
  FbDevBuf<unsigned long long> d_dbg;
  // depth front end (next #1)
  FbDevBuf<uint16_t> d_img[2];
  unsigned image_cnt = 0;
  FbDevBuf<float> d_dpts, d_dcloud;
  FbDevBuf<uint8_t> d_dflags;
  FbDevBuf<uint32_t> d_dsel;
  FbDevBuf<unsigned> d_dcount;
  FbDevBuf<char> d_dtmp;
  unsigned last_cloud_n = 0;
  int mode = FIESTA_MODE_EXACT;
  int shard_rank = 0, shard_world = 1, tile_x_lo = 0, tile_x_hi = 0;
  FbDevBuf<unsigned> d_halo_changed;
  // FAST mode: some relaxation (UpdateESDF / shard_relax) ran under an update box that is not the whole grid, so voxels
  // outside it may hold values their neighbours never offered them; from then on every queued voxel pulls (DESIGN 3.3)
  bool local_box_seen = false;
  FbExact X;
  fiesta_stats st{};
  // pinned host mirror (next #3): union of the update boxes that were current while records could change
  struct fiesta_host_mirror *mirror = nullptr;
  int dirty_lo[3]{}, dirty_hi[3]{};
  bool dirty_any = false, pending_obs = false;  // pending_obs: observations counted under the current box and not integrated yet
  // records epoch: incremented by every call that can change the records (UpdateOccupancy, UpdateESDF, shard ingest / relax);
  // a signed field (fb_signed.cu) computed under an older epoch refuses to be read
  unsigned long long records_epoch = 0;
};

// Map functions: FIESTA_OK or a FIESTA_ERR_* code with fiesta_last_error() set.
int flush_events(fiesta_map *m);                                          // applies the staged SetOccupancy events; synchronises
// fiesta_create; a snapshot load passes honour_env = false, so that the mode it restores is not overridden by FIESTA_B200_MODE
int create_map(const fiesta_config *cfg, fiesta_map **out, bool honour_env);
int alloc_depth(fiesta_map *m, size_t N);                                 // depth buffers for images of N pixels, none kept
void set_box_flag(FbGeom &g);
int rebuild_occbits(fiesta_map *m);                                       // the Exist() bitmap from occ under the current l_occ
// Queries on device buffers, ordered on the caller's stream s (fb_map.cu explains the two cross-stream waits).
int device_query_begin(fiesta_map *m, const char *fn, cudaStream_t s);
int device_query_end(fiesta_map *m, cudaStream_t s);

// Argument checks of the entry points: false (or the FIESTA_ERR_* code) with the message "<fn>: ..." set.
bool count_buffers_ok(const char *fn, int64_t n, bool buffers);           // n >= 0, and buffers when n > 0
bool clearance_flags_ok(const char *fn, double clearance, int flags);     // clearance in [0, +10000), flags in FIESTA_SEGMENT_*
int pose_args(const fiesta_map *m, const char *fn, int64_t n, const double *h, double clearance, int flags, bool buffers);
bool box_axis_ok(const char *fn, const FbGeom &g, const int *lo, const int *hi, int k);     // axis k: 0 <= lo <= hi < grid
bool box_arg(const char *fn, const FbGeom &g, const int *lo, const int *hi, FbNavBox *b);   // every axis; b (if any) := the box
// A buffer allocation that failed: clears the (not sticky) error, sets the message fmt with ": <CUDA error>" appended, FIESTA_ERR_CUDA.
int alloc_failed(cudaError_t e, const char *fmt, ...);

// Handles on a map (cost-to-go field, frontiers, query plan, host mirror): a type T with a member `fiesta_map *m` whose
// destructor releases what it holds beyond its buffers.  Destruction waits for the map's stream, so nothing queued still uses them.
template <class T> void handle_destroy(T *h) {
  if (!h) return;
  cudaSetDevice(h->m->device);
  cudaStreamSynchronize(h->m->stream);
  delete h;
}
struct FbHandleDelete {
  template <class T> void operator()(T *h) const { handle_destroy(h); }
};
template <class T> using FbHandle = std::unique_ptr<T, FbHandleDelete>;
// A new handle on m, made on m's device; h stays null (no message) when host memory runs out.
template <class T> int handle_new(fiesta_map *m, FbHandle<T> &h) {
  CK(cudaSetDevice(m->device));
  h.reset(new (std::nothrow) T());
  if (h) h->m = m;
  return FIESTA_OK;
}
