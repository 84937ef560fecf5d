/*
 * fiesta_b200 -- C ABI of the H100-native FIESTA hot path.
 *
 * This is the drop-in boundary: every entry point below replaces one method of the reference's
 * `fiesta::ESDFMap` (or the one `Fiesta` member that drives it) and keeps its argument meaning, return
 * sentinels and error behaviour.  Citations are into the reference tree (HKUST-Aerial-Robotics/FIESTA).
 * Plain pointers and sizes only; no C++/torch types.  All functions are synchronous with respect to the
 * caller unless stated otherwise (work is enqueued on the map's CUDA stream and waited for where a
 * value is returned).
 *
 * Voxel index convention (ESDFMap.cpp:84-93): idx = x*Gy*Gz + y*Gz + z, z fastest.
 * Sentinels (ESDFMap.cpp:181-185): -10000 = undefined / out of map, +10000 = infinity.
 */
#ifndef FIESTA_B200_H_
#define FIESTA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fiesta_map fiesta_map;

#define FIESTA_UNDEFINED (-10000)
#define FIESTA_INFINITY (10000)

enum {
  FIESTA_OK = 0,
  FIESTA_ERR_INVALID = 1,   /* bad argument */
  FIESTA_ERR_CUDA = 2,      /* CUDA runtime/driver error, see fiesta_last_error() */
  FIESTA_ERR_NO_DEVICE = 3, /* no usable sm_90 device: there is NO CPU fallback */
  FIESTA_ERR_LIMIT = 4      /* grid or frame exceeds a documented limit */
};

/* Ordering mode of UpdateOccupancy / UpdateESDF.
 *  EXACT (the default, = a zero-initialised fiesta_config): reproduces the reference's sequential FIFO order on the device
 *         (insert/delete queue order, LIFO dependant lists, dirs_ order, intra-queue visibility): closest_obstacle_ and
 *         distance_ equal the reference bit for bit in every scene, and the expansion count equals the reference's
 *         "Expanding N nodes".  This is the mode that reproduces the reference.
 *  FAST : order-free parallel wavefront, several times faster.  Occupancy, counters and queries are bit-exact; distance_ is
 *         bit-exact wherever the reference's result does not depend on its FIFO arrival order (fully observed scenes with
 *         sparse obstacles); on partially observed scenes (every ray-cast map) a fraction of a percent to a few percent of
 *         the distances differ from the reference by up to a few voxels, and exact distance ties keep the smallest obstacle
 *         coordinate instead of the first arrival.  Opt in explicitly.
 * The environment variable FIESTA_B200_MODE=exact|fast, when set, overrides fiesta_config.mode in fiesta_create (a knob for
 * callers that construct the map through the C++ facade without touching its arguments). */
enum { FIESTA_MODE_EXACT = 0, FIESTA_MODE_FAST = 1 };

/* ESDFMap::ESDFMap(origin, resolution, map_size) arguments (ESDFMap.h:116, ESDFMap.cpp:171-213) plus placement. */
typedef struct fiesta_config {
  double origin[3];     /* l_cornor_ : lower corner of the map, metres */
  double resolution;    /* voxel edge, metres */
  double map_size[3];   /* r_cornor_ - l_cornor_, metres; grid = ceil(map_size / resolution) */
  int32_t device;       /* CUDA device ordinal */
  int32_t mode;         /* FIESTA_MODE_EXACT (0, default) or FIESTA_MODE_FAST (1), see above */
  int32_t reserved[6];  /* must be zero */
} fiesta_config;

/* Fiesta::RaycastProcess parameters (parameters.h:148-149, Fiesta.h:209-245). */
typedef struct fiesta_raycast_params {
  double min_ray_length; /* parameters_.min_ray_length_ */
  double max_ray_length; /* parameters_.max_ray_length_ */
} fiesta_raycast_params;

/* What the reference prints inside its hot path (ESDFMap.cpp:237,277,394) plus device timings. */
typedef struct fiesta_stats {
  int64_t occupancy_updates;   /* occupancy_queue_ size drained by the last UpdateOccupancy          (:237) */
  int64_t inserts, deletes;    /* insert_queue_/delete_queue_ sizes seen by the last UpdateESDF        (:277) */
  int64_t voxels_changed;      /* voxels whose (distance, closest obstacle) record changed in the last UpdateESDF */
  int64_t expansions;          /* EXACT mode: non-stale queue pops = the reference's "Expanding N nodes" (ESDFMap.cpp:394); FAST: 0 */
  int64_t voxels_reset;        /* dependants of deleted obstacles cleared by the last UpdateESDF (E2) */
  int64_t tile_visits;         /* 8^3 tile relaxations run by the last UpdateESDF */
  int64_t generations;         /* wavefront generations of the last UpdateESDF */
  int64_t rays_cast;           /* rays traversed by the last raycast frame (after endpoint dedupe, Fiesta.h:221-231) */
  int64_t rays_dropped;        /* rays the reference Raycast() would never return from / would throw on */
  int64_t ray_voxels;          /* DDA voxels emitted by the last raycast frame */
  int64_t raycast_rounds;      /* stamp-resolution rounds of the last raycast frame */
  int64_t touched_voxels;      /* voxels currently waiting in the occupancy queue */
  int64_t kernel_launches;     /* kernels launched by this map since creation */
  float ms_raycast;            /* device time of the last raycast frame */
  float ms_update_occupancy;   /* device time of the last UpdateOccupancy */
  float ms_update_esdf;        /* device time of the last UpdateESDF (whole call) */
  float ms_esdf_delete_scan;   /* ... of which: dense dependant scan (E2) */
  float ms_esdf_wavefront;     /* ... of which: tile wavefront kernel (E3) */
  float reserved_f[1];
} fiesta_stats;

/* ---- lifetime: `new ESDFMap(...)` / `delete` (Fiesta.h:96,137) ---- */
int fiesta_create(const fiesta_config *cfg, fiesta_map **out);
void fiesta_destroy(fiesta_map *m);
/* Thread-local description of the last failure on this thread ("" if none). */
const char *fiesta_last_error(void);

/* ESDFMap::SetParameters (ESDFMap.h:124, ESDFMap.cpp:218-224). */
int fiesta_set_parameters(fiesta_map *m, double p_hit, double p_miss, double p_min, double p_max, double p_occ);
/* public field ESDFMap::grid_total_size_ (ESDFMap.h:115) and grid_size_ (ESDFMap.cpp:175-176). */
int fiesta_grid_total_size(const fiesta_map *m);
int fiesta_grid_size(const fiesta_map *m, int out[3]);

/* ---- occupancy input ---- */
/* int ESDFMap::SetOccupancy(Eigen::Vector3d pos, int occ) (ESDFMap.cpp:401-415): -10000 for occ not in {0,1} or pos
 * outside the map, else the linear voxel index (also when the voxel is outside the update box and is not counted). */
int fiesta_set_occupancy_pos(fiesta_map *m, const double pos[3], int occ);
/* int ESDFMap::SetOccupancy(Eigen::Vector3i vox, int occ) (ESDFMap.cpp:417-437). */
int fiesta_set_occupancy_vox(fiesta_map *m, const int vox[3], int occ);
/* The same call for n events in order; out_idx (nullable) receives each return value. Host pointers. */
int fiesta_set_occupancy_batch_pos(fiesta_map *m, const double *pos_xyz, const uint8_t *occ, int64_t n, int *out_idx);
int fiesta_set_occupancy_batch_vox(fiesta_map *m, const int *vox_xyz, const uint8_t *occ, int64_t n, int *out_idx);

/* SetOccupancy(Vector3i, occ) for n events whose arrays already live in DEVICE memory (vox: 3 ints each, occ: 0/1); events
 * outside the update box or the grid are ignored exactly like the host call ignores them.  FAST mode only (no serial order). */
int fiesta_set_occupancy_batch_vox_device(fiesta_map *m, const int *d_vox_xyz, const uint8_t *d_occ, int64_t n);

/* Fiesta::RaycastMultithread + RaycastProcess, serial semantics (Fiesta.h:194-303), fused with Raycast()
 * (raycast.cpp:56-158) and the counter part of SetOccupancy.  xyz: n points (pcl::PointXYZ, 3 floats each) in the
 * sensor frame; T: row-major 4x4 `transform_` (Fiesta.h:415-419); raycast_origin_ = T[:3,3]/T[3,3] (Fiesta.h:420).
 * `fiesta_raycast_frame` takes a HOST pointer; `_device` takes a DEVICE pointer valid on the map's device.  Both return after
 * the frame's counters are complete (the call reads back the frame statistics).
 * Limits (FIESTA_ERR_LIMIT, nothing is truncated): n <= 524286 points per call (split larger clouds into ordered sub-frames);
 * 1500 voxels per ray as in the reference (raycast.cpp:127-130); EXACT mode: at most 16383 frames between two
 * fiesta_update_occupancy calls (observation time stamps are 44 bits per integration epoch). */
int fiesta_raycast_frame(fiesta_map *m, const float *xyz, int64_t n, const double T[16], const fiesta_raycast_params *p);
int fiesta_raycast_frame_device(fiesta_map *m, const float *d_xyz, int64_t n, const double T[16],
                                const fiesta_raycast_params *p);

/* Fiesta::DepthConversion + RaycastMultithread in one call (Fiesta.h:319-382, then :281-303): `depth` is a HOST rows x cols
 * uint16 image in millimetres (sensor_msgs::Image TYPE_16UC1, Fiesta.h:326-332).  Back-projection, the temporal depth filter
 * against the previous image of this map and the pixel-order compaction run on the device; the cloud never leaves HBM.
 * m_rel = last_transform_.inverse() * transform_ (row-major; only read when use_depth_filter != 0 and this is not the first
 * image).  *n_points receives the size of the cloud that was ray cast (0 for the first filtered image, Fiesta.h:353). */
typedef struct fiesta_depth_params {
  double focal_x, focal_y, center_x, center_y;      /* parameters.h:139-140 */
  int32_t use_depth_filter, depth_filter_margin;    /* parameters.h:143,145 */
  double depth_filter_max_dist, depth_filter_min_dist, depth_filter_tolerance;
} fiesta_depth_params;
int fiesta_depth_frame(fiesta_map *m, const uint16_t *depth, int rows, int cols, const fiesta_depth_params *dp, const double T[16],
                       const double m_rel[16], const fiesta_raycast_params *rp, int64_t *n_points);
/* The cloud produced by the last fiesta_depth_frame (3 floats per point, pixel order), for inspection / parity tests. */
int fiesta_last_depth_cloud(fiesta_map *m, float *out_xyz, int64_t cap, int64_t *n_points);

/* ---- per-frame driver: Fiesta::UpdateEsdfEvent (Fiesta.h:507-514) ---- */
/* bool ESDFMap::CheckUpdate() (ESDFMap.cpp:227-233): 1 if the occupancy queue is non-empty. */
int fiesta_check_update(fiesta_map *m);
/* bool ESDFMap::UpdateOccupancy(bool global_map) (ESDFMap.cpp:235-271): 1 if inserts or deletes are pending, 0 if not,
 * negative error code on failure. */
int fiesta_update_occupancy(fiesta_map *m, int global_map);
/* void ESDFMap::UpdateESDF() (ESDFMap.cpp:273-398). */
int fiesta_update_esdf(fiesta_map *m);
/* ESDFMap::SetUpdateRange / SetOriginalRange (ESDFMap.cpp:792-824). */
int fiesta_set_update_range(fiesta_map *m, const double min_pos[3], const double max_pos[3], int new_vec);
int fiesta_set_original_range(fiesta_map *m);

/* ---- queries (ESDFMap.cpp:452-540) ---- */
double fiesta_get_distance_pos(fiesta_map *m, const double pos[3]);  /* -10000 outside the map; unknown reads +10000 */
double fiesta_get_distance_vox(fiesta_map *m, const int vox[3]);
int fiesta_get_occupancy_pos(fiesta_map *m, const double pos[3]);    /* -10000 outside the map, else 0/1 */
int fiesta_get_occupancy_vox(fiesta_map *m, const int vox[3]);
/* double ESDFMap::GetDistWithGradTrilinear(pos, grad) (ESDFMap.cpp:481-540): -1 outside the map. */
double fiesta_get_dist_grad_trilinear(fiesta_map *m, const double pos[3], double grad[3]);
/* Batched forms (host pointers): n positions -> n distances (+ n gradients). */
int fiesta_get_distance_batch_pos(fiesta_map *m, const double *pos_xyz, int64_t n, double *out_dist);
int fiesta_get_dist_grad_trilinear_batch(fiesta_map *m, const double *pos_xyz, int64_t n, double *out_dist,
                                         double *out_grad_xyz);

/* Planner query plan (SURVEY.md 8(f) #3): GetDistWithGradTrilinear (ESDFMap.cpp:481-540) for a FIXED number of positions per
 * call, as trajectory optimisers issue it every iteration.  The plan owns pinned host buffers and a CUDA graph of
 * {copy positions in, query kernel, copy distances + gradients out}; a run is one graph launch and one synchronisation.
 * Write the n positions to fiesta_query_plan_positions() (xyz triples), call fiesta_query_plan_run(), read n distances and n
 * gradient triples.  Results equal fiesta_get_dist_grad_trilinear_batch bit for bit.  Create it after SetParameters; destroy it
 * before the map. */
typedef struct fiesta_query_plan fiesta_query_plan;
int fiesta_query_plan_create(fiesta_map *m, int64_t n, fiesta_query_plan **out);
void fiesta_query_plan_destroy(fiesta_query_plan *p);
double *fiesta_query_plan_positions(fiesta_query_plan *p);
const double *fiesta_query_plan_distances(const fiesta_query_plan *p);
const double *fiesta_query_plan_gradients(const fiesta_query_plan *p);
int fiesta_query_plan_run(fiesta_query_plan *p);

/* Pinned host mirror of the distance field (SURVEY.md 8(f) #3): for consumers that call GetDistance / GetDistWithGradTrilinear
 * (ESDFMap.cpp:467-540) one position at a time from host code, where a device round trip per call would dominate.  The mirror
 * keeps the packed 4-byte distance records (obstacle coordinate per voxel) of the whole grid in page-locked host memory;
 * fiesta_host_mirror_refresh() -- call it after UpdateESDF -- compares the union of the update boxes used since the previous
 * refresh with a device-side shadow of what the host holds, copies only the changed (index, record) pairs and patches them in
 * (more changes than grid/32: one bulk copy).  The getters are pure host code (no CUDA call, no lock) and return the same bits
 * as fiesta_get_distance_pos / _vox / fiesta_get_dist_grad_trilinear would for the map as of the last refresh.  A record is one
 * aligned 32-bit word, so a reader running concurrently with a refresh sees a voxel's old or new value, never a mixture.
 * One mirror per map; costs 4 bytes per voxel of pinned host memory and 4 of device memory.  Destroy it before the map (a
 * mirror still attached is destroyed with its map). */
typedef struct fiesta_host_mirror fiesta_host_mirror;
int fiesta_host_mirror_create(fiesta_map *m, fiesta_host_mirror **out);
void fiesta_host_mirror_destroy(fiesta_host_mirror *p);
int fiesta_host_mirror_refresh(fiesta_host_mirror *p, int64_t *n_changed);   /* n_changed (may be NULL): records patched */
double fiesta_host_mirror_get_distance_pos(const fiesta_host_mirror *p, const double pos[3]);
double fiesta_host_mirror_get_distance_vox(const fiesta_host_mirror *p, const int vox[3]);
double fiesta_host_mirror_get_dist_grad_trilinear(const fiesta_host_mirror *p, const double pos[3], double grad[3]);
int fiesta_host_mirror_get_distance_batch_pos(const fiesta_host_mirror *p, const double *pos_xyz, int64_t n, double *out_dist);
int fiesta_host_mirror_get_dist_grad_trilinear_batch(const fiesta_host_mirror *p, const double *pos_xyz, int64_t n,
                                                     double *out_dist, double *out_grad_xyz);
/* the pinned records themselves (device layout: index = (x*Gy + y)*Pz + z, Pz = Gz rounded up as fiesta_create reports) and
 * {records patched by the last refresh, voxels it scanned, refreshes so far, bulk copies so far} */
const uint32_t *fiesta_host_mirror_records(const fiesta_host_mirror *p);
int fiesta_host_mirror_stats(const fiesta_host_mirror *p, int64_t out[4]);

/* ---- state dumps in the reference's own representation (parity harness; host pointers, grid_total_size entries) ---- */
int fiesta_export_distance(fiesta_map *m, double *out);             /* distance_buffer_: -10000 unknown, +10000 unreached */
int fiesta_export_closest_obstacle(fiesta_map *m, int *out_xyz);    /* closest_obstacle_: 3 ints, -10000 = none */
int fiesta_export_occupancy(fiesta_map *m, double *out);            /* occupancy_buffer_ log-odds */
int fiesta_export_counters(fiesta_map *m, int *num_hit, int *num_total); /* num_hit_, num_miss_ (all observations) */

/* ---- multi-GPU: x-slab sharding of UpdateESDF (one process per GPU; the caller moves the ghost layers, e.g. with NCCL) ----
 * Every rank holds the whole grid and integrates every frame identically (ray casting and UpdateOccupancy are replicated),
 * but relaxes only the tile columns of its own x-slab.  dirs_ reaches 2 voxels (parameters.h:66-68), so the ghost layer is 2
 * x-layers on each internal face; one x-layer is Gy*Pz contiguous records, so layers are sent as they lie in memory.
 * Protocol per UpdateESDF:  fiesta_update_esdf();  repeat { fiesta_shard_pack -> exchange with rank-1 / rank+1 ->
 * fiesta_shard_ingest -> fiesta_shard_relax; all-reduce the number of changed records } until it is 0 on every rank. */
typedef struct fiesta_shard_info {
  int32_t rank, world;
  int32_t x_begin, x_end;        /* voxel x range owned by this rank */
  int32_t has_lo, has_hi;        /* neighbours rank-1 / rank+1 exist */
  int64_t layer_words;           /* 32-bit words in one ghost exchange buffer = 2 * Gy * Pz */
} fiesta_shard_info;
int fiesta_set_shard(fiesta_map *m, int rank, int world, fiesta_shard_info *out);
/* Copy this rank's two lowest / two highest owned x-layers into the DEVICE buffers d_lo / d_hi (layer_words words each). */
int fiesta_shard_pack(fiesta_map *m, uint32_t *d_lo, uint32_t *d_hi);
/* Take the neighbours' boundary layers (DEVICE buffers; nullable where no neighbour exists): d_from_lo = rank-1's highest
 * two layers, d_from_hi = rank+1's lowest two.  *changed = number of ghost records that differed. */
int fiesta_shard_ingest(fiesta_map *m, const uint32_t *d_from_lo, const uint32_t *d_from_hi, int64_t *changed);
/* Relax the slab again from the queued tiles; *changed = records changed inside the slab. */
int fiesta_shard_relax(fiesta_map *m, int64_t *changed);

/* ---- visualisation extraction on the device (the step right after the path) ----
 * ESDFMap::GetPointCloud (ESDFMap.cpp:544-582): centres (3 floats each, geometry_msgs::Point32) of the occupied voxels inside the
 * update box with vis_lower <= z index <= vis_upper, in the reference's loop order.  *count = number found (may exceed cap). */
int fiesta_get_point_cloud(fiesta_map *m, int vis_lower_bound, int vis_upper_bound, float *out_xyz, int64_t cap, int64_t *count);
/* ESDFMap::GetSliceMarker (ESDFMap.cpp:639-699): points (3 doubles) and RainbowColorMap colours (4 floats rgba) of the voxels of
 * z-slice `slice` inside the update box whose distance is in [0, +10000). */
int fiesta_get_slice_marker(fiesta_map *m, int slice, double max_dist, double *out_xyz, float *out_rgba, int64_t cap, int64_t *count);

int fiesta_get_stats(fiesta_map *m, fiesta_stats *out);
/* Block until all work queued on the map's stream has finished. */
int fiesta_synchronize(fiesta_map *m);

#ifdef __cplusplus
}
#endif
#endif /* FIESTA_B200_H_ */
