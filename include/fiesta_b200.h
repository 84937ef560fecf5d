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
 * fiesta_update_occupancy calls (observation time stamps are 44 bits per integration epoch).
 * The environment variable FIESTA_RAY_LATTICE=0, read on every call, turns off the lattice fast path (per-voxel Pos2Vox
 * skipped when the map's voxels line up with the DDA's, DESIGN.md 3.1) so that tests can run any map through the general
 * per-voxel path; the results are the same either way. */
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

/* ---- segment clearance (planners: RRT/PRM edges, line of sight, trajectory checks between waypoints) ----
 * Is the straight segment a-b (metres) at least `clearance` away from every obstacle, and if not, where does it first come too
 * close?  Each endpoint is mapped to voxel units as Pos2Vox does ((p - origin) / resolution, fp64) and truncated to a 2^-20 voxel
 * lattice; every voxel the lattice segment touches is walked in order, with exact integer arithmetic.  A voxel blocks when
 * GetDistance(Vector3i) <= clearance or, with FIESTA_SEGMENT_UNKNOWN_BLOCKS, when it was never observed.  In other words: a segment
 * is clear iff GetDistance(p) > clearance at every point p of it (and, with the flag, no point of it lies in unknown space).
 * Outputs per segment:
 *   status   0 = clear, 1 = blocked, 2 = an endpoint is outside the map (PosInMap, ESDFMap.cpp:46-61) or NaN
 *   hit_idx  linear index x*Gy*Gz + y*Gz + z of the first blocking voxel, else -1
 *   hit_t    parameter in [0,1] at which the segment enters that voxel (0 for the start voxel), else NaN
 *   min_dist minimum GetDistance(Vector3i) over the voxels walked up to and including the first blocking one (all of them when
 *            clear); -10000 when outside
 * `ab` holds n segments as {ax, ay, az, bx, by, bz}.  FIESTA_ERR_INVALID for a NaN, negative or >= +10000 clearance, unknown flag
 * bits, or null buffers with n > 0.  All variants return identical arrays for the same records. */
#define FIESTA_SEGMENT_UNKNOWN_BLOCKS 1
/* host pointers; synchronous like the other batch queries */
int fiesta_check_segments(fiesta_map *m, const double *ab, int64_t n, double clearance, int flags, int32_t *status, int64_t *hit_idx,
                          double *hit_t, double *min_dist);
/* pure host code on the pinned records, as of the last refresh */
int fiesta_host_mirror_check_segments(const fiesta_host_mirror *p, const double *ab, int64_t n, double clearance, int flags,
                                      int32_t *status, int64_t *hit_idx, double *hit_t, double *min_dist);

/* ---- robot-shaped collision checks (planners: hybrid A* / lattice motion primitives, MPPI rollouts, any robot that is not a sphere) ----
 * Does an oriented box at a pose touch a voxel that blocks?  The half extents h[3] (metres, finite, >= 0; zeros give a plate, a
 * segment or a point) are shared by the n poses of a call.  A pose is 12 doubles {px, py, pz, R00 .. R22}: p is the box centre in
 * metres, R a row-major 3x3 world-to-body matrix whose rows u_0, u_1, u_2 are the box axes in world coordinates (the convention of
 * the viewpoint orientations).  The rows are used exactly as given: no orthonormality check, no trigonometry; the result describes
 * a box only when R is a rotation.
 *   touched   voxel v (any integer triple, in the grid or not) with centre c_k = ((double)v_k + 0.5) * resolution + origin_k and
 *             d_k = c_k - p_k is touched iff the closed cube of half-edge r = resolution / 2 and the closed box intersect, decided
 *             by the separating-axis test over the world axes e_k, the box axes u_j and the nine products e_k x u_j: no L has
 *             fabs(proj_L) > T_L, where, each fp64 operation rounded on its own,
 *               proj_L = (L0*d0 + L1*d1) + L2*d2,  u_j.L = (u_j0*L0 + u_j1*L1) + u_j2*L2,
 *               T_L = r * ((fabs(L0) + fabs(L1)) + fabs(L2)) + ((h0*fabs(u_0.L) + h1*fabs(u_1.L)) + h2*fabs(u_2.L)).
 *             Touching faces count: a body whose face touches an obstacle's face collides.
 *   blocking  a touched grid voxel blocks as in segment clearance: GetDistance(Vector3i) <= clearance (clearance 0: obstacle voxels
 *             only) or, with FIESTA_SEGMENT_UNKNOWN_BLOCKS, never observed.
 * Outputs per pose:
 *   status    0 = no touched grid voxel blocks and the box stays in the grid; 1 = some touched grid voxel blocks; 2 = invalid pose:
 *             p has a NaN or fails PosInMap, an R entry is non-finite or some |R_jk| > 1 + 2^-20; 3 = nothing blocks, but the box
 *             touches a voxel outside the grid (it leaves the map).  1 takes precedence over 3.  Voxels outside the grid are never
 *             read as records; a planner that wants the map's edge to block treats status 3 as blocked.
 *   n_blocked the number of touched blocking grid voxels (0 unless status 1)
 *   hit_idx   the least linear index x*Gy*Gz + y*Gz + z among them, else -1
 * Every output is an integer decided by fixed fp64 expressions and the records: the same bits on every run and as the sequential
 * definition (tests/poseref.py).  A union of boxes is the OR of the statuses of one call per box.  Errors, after which nothing is
 * written: FIESTA_ERR_INVALID for a NaN, infinite or negative half extent, a clearance or flags that fiesta_check_segments
 * rejects, n < 0, null half_extents, or null buffers with n > 0; FIESTA_ERR_LIMIT when h0 + h1 + h2 > 256 * resolution (at most
 * 518 candidate voxels per axis) or n >= 2^31 - 1.  Memory on the map, grown as needed: 8 bytes per pose (work list) plus scan
 * storage, and 112 bytes per pose for the host form's staging. */
/* host pointers; synchronous like the other batch queries */
int fiesta_check_poses(fiesta_map *m, const double *poses /* n * 12 */, int64_t n, const double half_extents[3], double clearance,
                       int flags, int32_t *status, int32_t *n_blocked, int64_t *hit_idx);
/* pure host code on the pinned records, as of the last refresh */
int fiesta_host_mirror_check_poses(const fiesta_host_mirror *p, const double *poses, int64_t n, const double half_extents[3],
                                   double clearance, int flags, int32_t *status, int32_t *n_blocked, int64_t *hit_idx);

/* ---- cost-to-go field (planners: A* / hybrid-A* heuristics, guide paths for trajectory optimisers, cost to frontier goals) ----
 * How far is the nearest goal through free space, keeping a clearance, and which way leads there?  The field covers an inclusive
 * voxel box [box_lo, box_hi] (0 <= lo <= hi < grid size on every axis) and is a snapshot of the records at the time of the call
 * (fiesta_nav_update brings it up to date).
 *   traversable  a voxel of the box that does not block in the sense of segment clearance: GetDistance(Vector3i) > clearance,
 *                and, with FIESTA_SEGMENT_UNKNOWN_BLOCKS, observed.  Voxels outside the box count as blocked.
 *   moves        u -> u+d for the 26 offsets d in {-1,0,1}^3 \ {0}, allowed iff every voxel of the axis-aligned box spanned by u
 *                and u+d (2, 4 or 8 voxels) is traversable: no corner cutting between diagonal obstacles.  Weight
 *                resolution * sqrt(k), k = the number of non-zero components of d.
 *   goals        positions (metres), mapped to voxels as Pos2Vox does; goals outside the box or on a blocked voxel are ignored
 *                (stats.goals_placed counts the others).  Duplicates are allowed.
 *   field        D = 0 on goals, else the least fixpoint of D(v) = min over allowed moves u -> v of fl(D(u) + w) in fp64 (the bits
 *                of a sequential Dijkstra, whatever order the device relaxes in); +inf where no goal is reachable; -1 on blocked
 *                voxels.  fiesta_nav_export writes it for the box, index ((x-lo.x)*By + (y-lo.y))*Bz + (z-lo.z), z fastest.
 *   paths        from each start position: the start voxel, then repeatedly the first allowed neighbour u, in (dx, dy, dz) order
 *                with dx slowest and -1 first, with fl(D(u) + w) == D(v), until D == 0.  vox_xyz receives max_len grid voxels
 *                (x, y, z) per start, -1 past len[i]; cost[i] = D(start).  Folding the weights from the goal back along the path
 *                reproduces D(start) bit for bit.  status 0 = reached, 1 = unreachable (cost +inf, len 0), 2 = start blocked,
 *                outside the box or the map (PosInMap) or NaN (cost NaN, len 0), 3 = truncated after max_len voxels.
 * The field object owns its device buffers, which grow to the largest box used: 8 bytes per box voxel plus 12 bytes per 8^3 tile,
 * with the library's 50 % growth headroom (about 1.6 GB for a 512^3 box; 6.5 GB for a 1024 x 1024 x 512 box, which next to an
 * EXACT map of that grid -- 68.1 GiB on a 79.2 GiB card -- is tight; a signed field of the same box takes as much, 8 bytes per
 * box voxel).  It runs on the map's stream; the calls are synchronous.
 * Destroy it before the map.  Errors:
 * FIESTA_ERR_INVALID for a box outside the grid or inverted, a clearance or flags that fiesta_check_segments rejects, null
 * buffers, max_len < 1, or export / paths before a compute; nothing changes then.  FIESTA_ERR_CUDA when the buffers cannot be
 * allocated; the map is untouched and the field must be computed again. */
typedef struct fiesta_nav_field fiesta_nav_field;
typedef struct fiesta_nav_stats {
  int64_t box_voxels, blocked, reached;   /* reached: voxels with a finite D, goals included */
  int64_t goals_placed;                   /* goals inside the box on a traversable voxel (duplicates counted) */
  int64_t generations, tile_visits;       /* grid-wide relaxation rounds and 8^3 tile relaxations of the device solver */
  float ms_compute;                       /* device time of the compute */
  float reserved_f[1];
} fiesta_nav_stats;
int fiesta_nav_create(fiesta_map *m, fiesta_nav_field **out);
void fiesta_nav_destroy(fiesta_nav_field *f);
int fiesta_nav_compute(fiesta_nav_field *f, const int box_lo[3], const int box_hi[3], const double *goals_xyz, int64_t n_goals,
                       double clearance, int flags, fiesta_nav_stats *stats /* nullable */);
int fiesta_nav_export(const fiesta_nav_field *f, double *out);   /* box_voxels doubles */
int fiesta_nav_paths(fiesta_nav_field *f, const double *starts_xyz, int64_t n, int32_t max_len, int32_t *status, int32_t *len,
                     double *cost, int32_t *vox_xyz /* n * max_len * 3 */);

/* ---- cost-to-go fields that follow the map (replanning at sensor rate: D* Lite / LPA*-style users of a live field) ----
 * fiesta_nav_update re-reads the map's records and repairs the field in place instead of recomputing it.  Afterwards the field,
 * fiesta_nav_export and fiesta_nav_paths are bit for bit what fiesta_nav_compute would give now with the box, goals, clearance and
 * flags of the last successful compute, in both map modes and after any sequence of frames, SetUpdateRange / local-map resets,
 * SetParameters and chained updates.  A goal ignored because its voxel was blocked counts again once the voxel is traversable,
 * and the reverse.  The old traversability is the field's own sign; voxels whose finite cost lost its support through a voxel
 * that became blocked are withdrawn, then the relaxation of fiesta_nav_compute runs from the repaired start state over the tiles
 * near the changes only (DESIGN.md §3.11), so a call with nothing changed does no relaxation (generations == tile_visits == 0).
 * fiesta_nav_matrix keeps its own buffers: a matrix between a compute and an update changes neither.  Memory: 1 scratch byte per
 * box voxel on the field object, grown like its other buffers (201 MB for a 512^3 box with the 50 % growth headroom).
 * Synchronous, on the map's stream.  Errors: FIESTA_ERR_INVALID for a null field or before any successful compute (nothing
 * changes); FIESTA_ERR_CUDA when the scratch cannot be allocated, in which case nothing has been written and the field is still
 * valid. */
typedef struct fiesta_nav_update_stats {
  int64_t box_voxels;
  int64_t became_blocked, became_free;   /* box voxels whose traversability changed since the field was last brought up to date */
  int64_t withdrawn;                     /* traversable voxels whose finite cost lost its support (DESIGN.md §3.11) */
  int64_t goals_placed, goals_new;       /* goals_placed as fiesta_nav_stats; goals_new: placed now, not placed before (duplicates
                                            counted), i.e. goals on a voxel that became free */
  int64_t seed_tiles;                    /* 8^3 tiles queued for the re-relaxation's generation 0 */
  int64_t withdraw_generations, generations, tile_visits;   /* withdrawal wave; re-relaxation (as fiesta_nav_stats) */
  int64_t blocked, reached;              /* of the repaired field, as fiesta_nav_stats */
  float ms_compute;                      /* device time of the whole update */
  float reserved_f[1];
} fiesta_nav_update_stats;
int fiesta_nav_update(fiesta_nav_field *f, fiesta_nav_update_stats *stats /* nullable */);

/* ---- cost matrices (tour planners, task allocation, roadmap edge costs): the geodesic cost from each of many sources to each of
 * many targets through free space at a clearance, in one call.
 *   box, clearance, flags   as fiesta_nav_compute (same rules, same errors).
 *   status       per source and per target (positions in metres): 0 = its voxel (Pos2Vox) is a traversable box voxel, 1 = the voxel
 *                is in the box but blocked, 2 = a NaN coordinate, outside the map (PosInMap) or the voxel is outside the box.
 *   cost         cost[i * n_tgt + j] = D_i(voxel of target j) when source i and target j both have status 0, where D_i is the field
 *                fiesta_nav_compute returns for the same box, clearance and flags with goals = {source i}: +inf when the target is
 *                unreachable in the box, 0 when it lies in the source's voxel; NaN otherwise.  Bit for bit, so it also equals the
 *                cost fiesta_nav_paths returns from target j on that field.  Duplicate points are allowed.  There is no symmetry:
 *                cost[i][j] is the left fold of the weights from source i, so with the roles swapped the same pair of points can
 *                differ in the last bits (fl-addition is not associative).
 * The sources' fields are relaxed together, up to 32 per pass (fewer when 8 bytes per box voxel per source would pass 2^32 bytes),
 * and a source stops as soon as all of its targets are provably final, so its time follows the distance to its farthest target
 * rather than the box size.  The call owns separate buffers on the field object, which grow to the largest use: 4 bytes per box
 * voxel (move masks), 8 bytes per box voxel and 12 bytes per 8^3 tile for each source of a pass (about 1.6 GB for 32 sources on a
 * 160^3 box, 6.4 GB for 4 on a 512^3 box, with the 50 % growth headroom), and 8 bytes per matrix entry.  It does not change the
 * field, export or paths of the last fiesta_nav_compute.  Synchronous, on the map's stream.  Errors, after which nothing has been
 * written: FIESTA_ERR_INVALID for what fiesta_nav_compute rejects, negative counts, or null buffers where there is work (statuses
 * for n > 0, cost when both counts are > 0); FIESTA_ERR_LIMIT when n_src * n_tgt >= 2^31; FIESTA_ERR_CUDA when the buffers
 * cannot be allocated.  n_src == 0 or n_tgt == 0 is valid: the statuses are still written. */
typedef struct fiesta_nav_matrix_stats {
  int64_t sources_placed, targets_placed;  /* status-0 points */
  int64_t passes;                          /* batches of sources resident together (0 when no source or no target is placed) */
  int64_t generations, tile_visits;        /* summed over passes */
  int64_t sources_retired_early;           /* sources stopped before their work list emptied */
  float ms_compute;                        /* device time of the whole call */
  float reserved_f[1];
} fiesta_nav_matrix_stats;
int fiesta_nav_matrix(fiesta_nav_field *f, const int box_lo[3], const int box_hi[3], const double *sources_xyz, int64_t n_src,
                      const double *targets_xyz, int64_t n_tgt, double clearance, int flags, int32_t *src_status, int32_t *tgt_status,
                      double *cost /* n_src * n_tgt, row i = source i */, fiesta_nav_matrix_stats *stats /* nullable */);

/* ---- signed distance (gradient-based trajectory optimisers: a way out for waypoints inside obstacles) ----
 * FIESTA's field is exactly 0 on every obstacle voxel, so a waypoint inside a wall sees distance 0 and gradient 0 there.  The
 * signed field of an inclusive voxel box B = [box_lo, box_hi] (0 <= lo <= hi < grid size on every axis) keeps FIESTA's distance
 * outside obstacles and goes negative inside them, by the depth to free space.  It is a snapshot of the records at the time of
 * fiesta_signed_compute.
 *   obstacle     a grid voxel whose distance reads exactly 0 in fiesta_export_distance (its closest obstacle is itself).  An
 *                EXACT-mode voxel under a local-map reset reads +10000 and is not one.  Every other voxel is a non-obstacle: free,
 *                unreached or never observed.
 *   depth        for an obstacle voxel v of B, q(v) = the least dx^2 + dy^2 + dz^2 (voxel units, exact integers) from v to a
 *                non-obstacle voxel OF B; voxels outside B are not candidates, so give the box a margin where true depths near its
 *                faces matter.
 *   S(v)         for a voxel of B, each fp64 operation rounded on its own: GetDistance(Vector3i v) for a non-obstacle (never
 *                observed reads +10000); (1.0 - sqrt((double)q(v))) * resolution for an obstacle, so surface voxels (q == 1) stay
 *                +0.0 and deeper ones go negative (the pos - neg + resolution convention of ESDF-based planners); -inf for an
 *                obstacle when B holds no non-obstacle voxel.  fiesta_signed_export writes S for the box, index as
 *                fiesta_nav_export.
 *   queries      fiesta_signed_get_distance_batch / _get_dist_grad_trilinear_batch run the expressions of
 *                fiesta_get_distance_batch_pos / fiesta_get_dist_grad_trilinear_batch operation for operation; only the voxel read
 *                differs: a voxel inside B reads S, one outside B (or outside the grid) reads what the map's queries read.  So a
 *                position none of whose 8 stencil voxels (its voxel, for the distance) is an obstacle with q > 1 gets the map
 *                query's bits exactly.  The _device forms follow the ordering rules of the stream-ordered queries below (and
 *                refuse a capturing stream) and return the host forms' bits.
 * Every output is a fixed integer or fp64 expression of the records: the same bits on every run and as an exact Euclidean
 * distance transform of the obstacle mask (tests/signedref.py: scipy.ndimage.distance_transform_edt).
 * Staleness: the map keeps a records epoch that fiesta_update_occupancy, fiesta_update_esdf, fiesta_shard_ingest and
 * fiesta_shard_relax increment.  Export and queries on a field computed under an older epoch return FIESTA_ERR_INVALID (compute
 * again), so the voxels inside and outside B always describe the same records.
 * Memory on the field object, grown as needed with the library's 50 % headroom: 4 bytes of q and 4 bytes of scratch per box voxel
 * (about 1.6 GB for a 512^3 box); export stages 8 bytes per box voxel for the duration of the call.  Host calls run on the map's
 * stream and are synchronous.  Destroy the field before the map.  Errors, after which nothing changes: FIESTA_ERR_INVALID for a
 * box outside the grid or inverted, null buffers where there is work or a negative n, export or queries before a compute or on
 * a stale field; FIESTA_ERR_CUDA when the buffers cannot be allocated, after which the field must be computed again. */
typedef struct fiesta_signed_field fiesta_signed_field;
typedef struct fiesta_signed_stats {
  int64_t box_voxels, obstacles;
  int64_t interior;                       /* obstacles with S < 0: q > 1, or every obstacle when B has no non-obstacle voxel */
  int64_t max_depth_sq;                   /* largest finite q, 0 if none; -1 when B has no non-obstacle voxel and obstacles > 0 */
  float ms_compute;                       /* device time of the three passes */
  float reserved_f[1];
} fiesta_signed_stats;
int fiesta_signed_create(fiesta_map *m, fiesta_signed_field **out);
void fiesta_signed_destroy(fiesta_signed_field *f);
int fiesta_signed_compute(fiesta_signed_field *f, const int box_lo[3], const int box_hi[3], fiesta_signed_stats *stats /* nullable */);
int fiesta_signed_export(const fiesta_signed_field *f, double *out);   /* box_voxels doubles */
int fiesta_signed_get_distance_batch(fiesta_signed_field *f, const double *pos_xyz, int64_t n, double *out_dist);
int fiesta_signed_get_dist_grad_trilinear_batch(fiesta_signed_field *f, const double *pos_xyz, int64_t n, double *out_dist,
                                                double *out_grad_xyz);
int fiesta_signed_get_distance_batch_device(fiesta_signed_field *f, const double *d_pos_xyz, int64_t n, double *d_dist, void *stream);
int fiesta_signed_get_dist_grad_trilinear_batch_device(fiesta_signed_field *f, const double *d_pos_xyz, int64_t n, double *d_dist,
                                                        double *d_grad_xyz, void *stream);

/* ---- frontier extraction (exploration planners: where does observed free space end?) ----
 * The free voxels of an inclusive voxel box [box_lo, box_hi] (0 <= lo <= hi < grid size on every axis) that border never-observed
 * space, grouped into clusters, as a snapshot of the integrated records and log-odds at the time of the call (observations that
 * UpdateOccupancy has not integrated yet are not part of it).
 *   unknown      a grid voxel whose distance reads -10000 in fiesta_export_distance (never observed).  Unreached voxels and
 *                voxels reset by a local-map update are observed.
 *   frontier     a box voxel that is observed, not occupied (GetOccupancy(Vector3i) == 0: log-odds <= l_occ), does not block at
 *                the clearance in the sense of fiesta_check_segments without FIESTA_SEGMENT_UNKNOWN_BLOCKS (so it is a
 *                traversable voxel of a cost-to-go field at the same clearance, usable as a nav goal or path start), and has
 *                an unknown face neighbour inside the grid; the neighbour may lie outside the box, the map's outer faces do not
 *                count.
 *   clusters     the 26-connected components of the box's frontier voxels (a cluster cut by a box face stays cut); clusters of
 *                fewer than min_cluster_size voxels are dropped; the kept ones are numbered 0..K-1 by their smallest member in
 *                x, y, z loop order (the box index below).
 *   per cluster  size; rep = its first member (grid voxel xyz); bbox lo / hi (grid voxels, inclusive); centroid (metres) =
 *                ((double)S / (double)size + 0.5) * resolution + origin per axis, S the exact sum of the members' grid
 *                coordinates, each operation rounded separately.
 *   voxels       the kept clusters' members as grid voxel xyz, cluster by cluster, in loop order within a cluster.
 *   labels       fiesta_frontiers_export: one int32 per box voxel, index ((x-lo.x)*By + (y-lo.y))*Bz + (z-lo.z) as in
 *                fiesta_nav_export: the cluster id, or -1 off the frontier or in a dropped cluster.
 * Every output is integer or one fixed fp64 expression: the same bits on every run and as a sequential definition
 * (tests/frontierref.py).  fiesta_frontiers_clusters / _voxels write the first min(cap, n) entries (n = stats.kept_clusters /
 * stats.kept_voxels of the last compute), as fiesta_get_point_cloud does.
 * The object owns its device buffers, which grow to the largest box and result used: 8 bytes per box voxel, plus 132 bytes per
 * cluster before the size filter and 28 bytes per kept member, with the library's 50 % growth headroom (about 1.6 GB for a
 * 512^3 box).  It runs on the map's stream; the calls are synchronous.  Destroy it before the map.  Errors:
 * FIESTA_ERR_INVALID for a box outside the grid or inverted, a clearance fiesta_check_segments rejects (NaN, < 0, >= 10000),
 * min_cluster_size < 1, null buffers, a negative cap, or reads before a compute; nothing changes then.  FIESTA_ERR_CUDA when the
 * buffers cannot be allocated; the map is untouched and a new compute is needed before the results can be read. */
typedef struct fiesta_frontiers fiesta_frontiers;
typedef struct fiesta_frontier_stats {
  int64_t box_voxels;
  int64_t frontier_voxels;                /* frontier voxels of the box, before the size filter */
  int64_t clusters, kept_clusters;        /* clusters before and after the size filter */
  int64_t kept_voxels;                    /* members of the kept clusters */
  float ms_compute;                       /* device time of the compute */
  float reserved_f[1];
} fiesta_frontier_stats;
int fiesta_frontiers_create(fiesta_map *m, fiesta_frontiers **out);
void fiesta_frontiers_destroy(fiesta_frontiers *f);
int fiesta_frontiers_compute(fiesta_frontiers *f, const int box_lo[3], const int box_hi[3], double clearance, int64_t min_cluster_size,
                             fiesta_frontier_stats *stats /* nullable */);
int fiesta_frontiers_clusters(const fiesta_frontiers *f, int64_t cap, int64_t *size, int32_t *rep_xyz /* cap * 3 */,
                              int32_t *bbox_lo_xyz /* cap * 3 */, int32_t *bbox_hi_xyz /* cap * 3 */, double *centroid_xyz /* cap * 3 */);
int fiesta_frontiers_voxels(const fiesta_frontiers *f, int64_t cap, int32_t *vox_xyz /* cap * 3 */);
int fiesta_frontiers_export(const fiesta_frontiers *f, int32_t *labels);   /* box_voxels int32 */

/* ---- viewpoint coverage (exploration planners: where should the sensor stand to look past a frontier?) ----
 * Scores candidate sensor poses by the members of a frontier cluster they would see.  Candidate i is a position pos[i] (metres)
 * tagged with a kept cluster id cluster[i] of the last fiesta_frontiers_compute; the n_orient (1..32) orientations are shared by
 * all candidates, each a row-major 3x3 world-to-sensor matrix R: row 0 is the optical axis, row 1 the axis the horizontal field of
 * view spans, row 2 the vertical one.  The rows are used exactly as given (no orthonormality check, no trigonometry).
 *   status     2 = pos fails PosInMap or has a NaN coordinate; 1 = its voxel Pos2Vox(pos) is outside the grid (upper faces),
 *              never observed or has GetDistance(Vector3i) <= clearance, whatever the flags (so every status-0 candidate is a
 *              traversable voxel of a cost-to-go field at the same clearance, with or without FIESTA_SEGMENT_UNKNOWN_BLOCKS);
 *              0 = scored.  A candidate with status 1 or 2 scores 0 for every orientation.
 *   pair       for a status-0 candidate p and a member voxel v of its cluster, each fp64 operation rounded on its own:
 *              c_k = ((double)v_k + 0.5) * resolution + origin_k (Vox2Pos), d_k = c_k - p_k;
 *              in range: (d0*d0 + d1*d1) + d2*d2 <= max_range * max_range;
 *              in view of orientation j: s_k = (R[k][0]*d0 + R[k][1]*d1) + R[k][2]*d2 with
 *              s0 > 0 && fabs(s1) <= tan_half_fov[0] * s0 && fabs(s2) <= tan_half_fov[1] * s0;
 *              visible: fiesta_check_segments on {p, c} at clearance 0 with `flags` returns status 0 (no obstacle voxel on the
 *              exact walk and, with FIESTA_SEGMENT_UNKNOWN_BLOCKS, no never-observed one).
 *   score      score[i * n_orient + j] = the members of cluster[i] in range, in view of orientation j and visible.
 * Line of sight reads the records at the time of the call; the members are those of the last compute.  Every output is an integer
 * decided by fixed fp64 expressions and the integer walk: the same bits on every run and as a sequential definition
 * (tests/viewref.py).  Memory on the frontier object, grown as needed: 40 + 4 * n_orient bytes per candidate and 8 per kept
 * cluster, plus scan storage.  Host pointers, the map's stream, synchronous.  Errors (nothing is written and the frontier result
 * stays valid): FIESTA_ERR_INVALID before any compute, for a cluster id outside [0, kept_clusters), n < 0, n_orient < 1, a
 * non-finite or <= 0 max_range or tangent, a non-finite orientation entry, a clearance or flags that fiesta_check_segments
 * rejects, or null buffers with n > 0 (sensor and orient are always needed); FIESTA_ERR_LIMIT for n_orient > 32 (call again
 * with the rest) or n >= 2^31 - 1; FIESTA_ERR_CUDA when the buffers cannot be allocated. */
typedef struct fiesta_sensor_model {
  double max_range;                       /* metres, Euclidean from the sensor position to the voxel centre */
  double tan_half_fov[2];                 /* horizontal (row 1), vertical (row 2) */
} fiesta_sensor_model;
typedef struct fiesta_viewpoint_stats {
  int64_t candidates_scored;              /* status-0 candidates */
  int64_t pairs_walked;                   /* (candidate, member) pairs in range and in view of at least one orientation */
  int64_t pairs_visible;                  /* walked pairs with a clear line of sight */
  float ms_compute;                       /* device time of the scoring */
  float reserved_f[1];
} fiesta_viewpoint_stats;
#define FIESTA_VIEWPOINT_MAX_ORIENT 32
int fiesta_frontiers_score_viewpoints(fiesta_frontiers *f, const int32_t *cluster, const double *pos_xyz, int64_t n,
                                      const double *orient /* n_orient * 9 */, int32_t n_orient, const fiesta_sensor_model *sensor,
                                      double clearance, int flags, int32_t *status, int32_t *score /* n * n_orient, row i = candidate i */,
                                      fiesta_viewpoint_stats *stats /* nullable */);

/* ---- topological roadmaps (global, topology-guided and exploration planners: a sparse graph of the free space) ----
 * The skeleton of the free space of an inclusive voxel box [box_lo, box_hi] (0 <= lo <= hi < grid size on every axis): voxels on the
 * discrete generalized Voronoi diagram of the map's obstacles (where the closest obstacle changes sharply between neighbours), thinned
 * to curves that keep the free space's topology, as a graph of junctions and edges.  A snapshot of the integrated records at the time
 * of the call; nothing in the map or in any other result changes.  Box indices are ((x-lo.x)*By + (y-lo.y))*Bz + (z-lo.z) as in
 * fiesta_nav_export.
 *   traversable  a box voxel that does not block at the clearance and flags in the sense of fiesta_check_segments (so a traversable
 *                voxel of a cost-to-go field at the same clearance and flags).  Voxels outside the box are not.
 *   o(v)         the voxel's closest obstacle (fiesta_export_closest_obstacle), defined on observed voxels that have one and are not
 *                under an EXACT local-map reset (their distance reads +10000).
 *   anchor       a traversable voxel v with o(v) defined and a traversable face neighbour u in the box with o(u) defined and
 *                different, where, with a = o(v) - v and b = o(u) - u (exact integer dot products, each fp64 operation rounded on its
 *                own), (double)(a.b) <= max_cos * sqrt((double)(a.a) * (double)(b.b)).
 *   thinning     from the traversable set, delete simple voxels (26/6 topology) in iterations of 8 passes over the parity subfields
 *                s = 4((x-lo.x)&1) + 2((y-lo.y)&1) + ((z-lo.z)&1): phase 1 deletes those that are not anchors, phase 2 those with at
 *                least two 26-neighbours left (endpoints stay), each until an iteration deletes nothing.  The result does not depend
 *                on any schedule.
 *   graph        deg(v) = v's 26-neighbours in the set.  Vertex voxels: deg != 2, and the smallest-index voxel of each component that
 *                is a pure cycle.  Vertices: the 26-components of vertex voxels; chains: the 26-components of the rest, each a simple
 *                path whose ends attach to one vertex voxel each.  Vertices and edges are numbered by their smallest box index
 *                (an edge by its chain's).  An edge is the voxel path attach, chain..., attach, oriented so that (vertex id, attach
 *                box index, adjacent chain voxel box index) is lexicographically smaller at its start.
 *   pruning      with min_branch >= 2, rounds until one removes nothing, each removing at once (a) every edge of fewer than min_branch
 *                path voxels (its leaf counted, the other attachment not) from a leaf (a vertex of one voxel with one neighbour) to a
 *                different vertex that is not a leaf, with its leaf, and (b) every voxel with one neighbour whose neighbour has >= 3.
 *                No component is removed.  min_branch 0 or 1: no pruning.
 *   per vertex   size; rep = its first voxel (grid xyz); centroid (metres) = ((double)S / (double)size + 0.5) * resolution + origin
 *                per axis, as the frontier clusters'; degree = edge ends attached to it (a self-loop counts twice).
 *   per edge     uv = (start vertex, end vertex); n_vox = the path's voxel count; length = the left fold, from the start, of the
 *                cost-to-go field's move weights (resolution * sqrt(non-zero components)); min_dist = the least
 *                GetDistance(Vector3i) over the path.  fiesta_skeleton_edge_voxels: the paths as grid xyz, concatenated in edge order.
 *   export       mask: one byte per box voxel, bit 1 traversable, bit 2 anchor, bit 4 final skeleton; label: one int32 per box voxel,
 *                the vertex id on vertex voxels, -2 - e on the chain voxels of edge e, -1 elsewhere.  Either pointer may be null.
 * Every output is integer or one fixed fp64 expression: the same bits on every run and as the sequential definition
 * (tests/skeletonref.py; fiesta_b200/csrc/fb_skel.h, DESIGN.md §3.14).  The _vertices / _edges / _edge_voxels reads write the first
 * min(cap, n) entries (n = stats.vertices / edges / edge_voxels).  The object owns its device buffers, which grow to the largest box
 * and result used: 5 bytes per box voxel, 164 per voxel left after thinning and 12 per edge path voxel, with the library's 50 %
 * growth headroom (about 1 GB for a 512^3 box).  It runs on the map's stream; the calls are synchronous.  Destroy it before the map.
 * Errors: FIESTA_ERR_INVALID for a box outside the grid or inverted, a clearance or flags fiesta_check_segments rejects, a max_cos
 * that is NaN or outside [-1, 1), min_branch < 0, null buffers, a negative cap, or reads before a compute; nothing is written then.
 * FIESTA_ERR_CUDA when the buffers cannot be allocated; a new compute is needed before the results can be read. */
typedef struct fiesta_skeleton fiesta_skeleton;
typedef struct fiesta_skeleton_stats {
  int64_t box_voxels;
  int64_t traversable, anchors;           /* voxels of X0, and the anchors among them */
  int64_t iterations[2];                  /* thinning iterations of phases 1 and 2, each counting the one that deleted nothing */
  int64_t prune_rounds;                   /* pruning rounds, counting the one that removed nothing (0 without pruning) */
  int64_t pruned_voxels;                  /* voxels pruning removed */
  int64_t skeleton_voxels, vertices, edges;
  int64_t edge_voxels;                    /* sum of the edges' n_vox: the length of fiesta_skeleton_edge_voxels */
  float ms_compute;                       /* device time of the compute, and of its three stages */
  float ms_init, ms_thin, ms_graph;
} fiesta_skeleton_stats;
int fiesta_skeleton_create(fiesta_map *m, fiesta_skeleton **out);
void fiesta_skeleton_destroy(fiesta_skeleton *f);
int fiesta_skeleton_compute(fiesta_skeleton *f, const int box_lo[3], const int box_hi[3], double clearance, int flags, double max_cos,
                            int64_t min_branch, fiesta_skeleton_stats *stats /* nullable */);
int fiesta_skeleton_vertices(const fiesta_skeleton *f, int64_t cap, int64_t *size, int32_t *rep_xyz /* cap * 3 */,
                             double *centroid_xyz /* cap * 3 */, int32_t *degree);
int fiesta_skeleton_edges(const fiesta_skeleton *f, int64_t cap, int32_t *uv /* cap * 2 */, int64_t *n_vox, double *length,
                          double *min_dist);
int fiesta_skeleton_edge_voxels(const fiesta_skeleton *f, int64_t cap, int32_t *vox_xyz /* cap * 3 */);
int fiesta_skeleton_export(const fiesta_skeleton *f, uint8_t *mask /* box_voxels, nullable */, int32_t *label /* box_voxels, nullable */);

/* ---- surface meshes (viewers, simulators, other collision libraries: the map, or what the planners treat as blocked, as geometry) ----
 * The triangle mesh of the boundary of the voxels that block at a clearance in an inclusive voxel box [box_lo, box_hi]
 * (0 <= lo <= hi < grid size on every axis).  A snapshot of the integrated records at the time of the call; nothing in the map or in
 * any other result changes.
 *   blocking     a box voxel that blocks at the clearance and flags in the sense of fiesta_check_segments (GetDistance(Vector3i) <=
 *                clearance; with FIESTA_SEGMENT_UNKNOWN_BLOCKS also a never-observed voxel).  Voxels outside the box never block, so
 *                every mesh is closed and caps the box faces.
 *   distance     a box voxel whose record holds an obstacle not under an EXACT local-map reset has d(v) = GetDistance(Vector3i).
 *   E            the extended box [lo - 1, hi] on every axis, indexed ((x-lo.x+1)*(By+1) + (y-lo.y+1))*(Bz+1) + (z-lo.z+1).
 *   crossing     on a grid edge (u, w = u + e_a) with exactly one blocking endpoint: t = (clearance - d(u)) / (d(w) - d(u)) in fp64
 *                when both have a distance, else 0.5; the point u + t e_a (voxel units).
 *   vertices     one per active cell c in E (its corners c + {0,1}^3 neither all block nor all fail to), numbered in E-index order:
 *                the fp64 mean of the crossing points on its sign-changing edges (x-edges, then y-edges, then z-edges, each axis'
 *                four ordered lexicographically by the other offsets), in metres as ((m + 0.5) * resolution) + origin, rounded to
 *                float32.
 *   triangles    one quad per sign-changing grid edge (v, v + e_a), v in E: with (a, b, c) cyclic, the cells v + (0,-1,-1),
 *                v + (0,0,-1), v, v + (0,-1,0) (offsets along a, b, c) in that order when v blocks and reversed after the first
 *                otherwise, so normals point from blocking to free space; split along p0-p2 when |p0-p2|^2 <= |p1-p3|^2 (fp64 on the
 *                float32 positions) into (p0,p1,p2), (p0,p2,p3), else into (p1,p2,p3), (p1,p3,p0).  Written in order of (v's E-index,
 *                axis x, y, z), two per quad, as int32 vertex ids.
 * The mesh is closed (every directed edge meets its reverse) and combinatorially the boundary of the union of the blocking voxels'
 * cubes; voxels touching only along an edge or a corner share vertices there.  Clearance 0 puts the surface through obstacle voxel
 * centres, 0.5 * resolution on the obstacle cubes' faces.  A vertex depends only on its cell's 8 corners, so adjacent boxes agree bit
 * for bit on the cells whose corners both boxes hold.  Every output is one fixed fp64 expression rounded once: the same bits on every
 * run and as the sequential definition (tests/meshref.py; fiesta_b200/csrc/fb_mesh.h, DESIGN.md §3.15).  The reads write the first
 * min(cap, n) entries (n = stats.vertices / triangles).  The object owns its device buffers, which grow to the largest box and
 * result used: about 1 byte per extended-box position, plus 12 bytes per vertex and 12 per triangle, with the library's 50 % growth
 * headroom.  It runs on the map's stream; the calls are synchronous.  Destroy it before the map.  Errors: FIESTA_ERR_INVALID for a
 * box outside the grid or inverted, a clearance or flags fiesta_check_segments rejects, a null buffer with cap > 0, a negative cap,
 * or reads before a compute; nothing is written then.  FIESTA_ERR_LIMIT when the mesh would have more than 2^31 - 1 vertices (only
 * possible for boxes near the largest grid; mesh them in chunks).  FIESTA_ERR_CUDA when the buffers cannot be allocated.  After
 * either of the last two a new compute is needed before the results can be read. */
typedef struct fiesta_mesh fiesta_mesh;
typedef struct fiesta_mesh_stats {
  int64_t box_voxels, blocking;           /* voxels of the box, and those that block */
  int64_t vertices, quads, triangles;     /* triangles = 2 * quads */
  float ms_compute;                       /* device time of the compute, and of its three stages: */
  float ms_classify, ms_vertices, ms_faces;   /* bitmap, cell and edge counts and their scans; vertices; triangles */
} fiesta_mesh_stats;
int fiesta_mesh_create(fiesta_map *m, fiesta_mesh **out);
void fiesta_mesh_destroy(fiesta_mesh *f);
int fiesta_mesh_compute(fiesta_mesh *f, const int box_lo[3], const int box_hi[3], double clearance, int flags,
                        fiesta_mesh_stats *stats /* nullable */);
int fiesta_mesh_vertices(const fiesta_mesh *f, int64_t cap, float *xyz /* cap * 3 */);
int fiesta_mesh_triangles(const fiesta_mesh *f, int64_t cap, int32_t *ijk /* cap * 3 */);

/* ---- safe flight corridors (corridor-based trajectory planners: free convex regions around a path) ----
 * Free axis-aligned voxel boxes, inflated face by face, and chains of them along paths in which consecutive boxes share a voxel.
 * All boxes are inclusive voxel boxes; the limit box L = [box_lo, box_hi] satisfies 0 <= lo <= hi < grid size on every axis.
 *   traversable  a voxel of L that does not block at `clearance` with `flags` in the sense of fiesta_check_segments
 *                (GetDistance(Vector3i) <= clearance blocks; with FIESTA_SEGMENT_UNKNOWN_BLOCKS a never-observed voxel blocks too):
 *                the traversable voxels of a cost-to-go field over L.
 *   inflation    of a seed box S whose voxels are all traversable: B = S, all six faces active; rounds visit the faces in the
 *                order -x, +x, -y, +y, -z, +z.  An active face that has reached L or max_steps[axis] (>= 0) layers beyond S's face
 *                is deactivated; otherwise the one-voxel layer just outside it, spanning B's current extent on the other two
 *                axes, is tested: if every voxel is traversable B grows by it, else the face is deactivated for good.  Stops when
 *                no face is active.  The result is traversable and maximal: each face sits on L or its max_steps, or its next
 *                layer holds a non-traversable voxel.  The face order is part of the definition.
 *   corridor     of a path P[0..n-1] (grid voxels): status 2 and no boxes if some P[i] lies outside L.  Otherwise box 0 inflates
 *                {P[0]}; after a box whose seed index is j, let i be the first index > j with P[i] outside it: none -> status
 *                0; else the next box inflates AABB(P[i-1], P[i]) with seed index i, so consecutive boxes share P[i-1].  A seed
 *                that holds a non-traversable voxel ends the corridor with status 1 and blocked_at = its seed index; the boxes
 *                before it are kept.  An empty path has status 0 and no boxes; a path of n voxels has at most n boxes.  The
 *                path of a cost-to-go field over the same L at the same clearance and flags, on unchanged records, never gets
 *                status 1 (each of its moves spans a traversable box).
 * The records are read as they are at the time of the call.  Every output is an integer: the same on every run and as the
 * sequential rule (tests/corridorref.py).  Memory on the map, grown as needed: 2 bits per limit-box voxel (32 MB for a 512^3 box),
 * 52 bytes per seed, or 40 per path voxel and 20 per path.  Host pointers, the map's stream, synchronous.  Errors (nothing is
 * written): FIESTA_ERR_INVALID for a box outside the grid or inverted, a clearance or flags that fiesta_check_segments rejects, a
 * negative max_steps entry, n or n_paths, offsets that do not start at 0 or that decrease, or null buffers where work exists
 * (box_lo, box_hi and max_steps are always needed); FIESTA_ERR_LIMIT when n or the number of path voxels is >= 2^31 - 1;
 * FIESTA_ERR_CUDA when the buffers cannot be allocated. */
typedef struct fiesta_corridor_stats {
  int64_t boxes;                          /* boxes written (corridors) or seeds inflated (inflate) */
  int64_t layers_tested;                  /* layer tests of the sequential rule (grown + refused); schedule-independent */
  int64_t layers_grown;
  int64_t mask_voxels;                    /* limit-box voxels evaluated (0 when there is no seed or path voxel) */
  float ms_compute;                       /* device time of the whole call */
  float reserved_f[1];
} fiesta_corridor_stats;
/* Independent seeds: n inclusive seed boxes -> inflated boxes.  status 0 ok; 1 the seed holds a non-traversable voxel; 2 the seed
 * is inverted or not inside L.  out_lo / out_hi are -1 for status 1 and 2. */
int fiesta_inflate_boxes(fiesta_map *m, const int box_lo[3], const int box_hi[3], const int32_t *seed_lo_xyz, const int32_t *seed_hi_xyz,
                         int64_t n, const int32_t max_steps[3], double clearance, int flags, int32_t *status, int32_t *out_lo_xyz,
                         int32_t *out_hi_xyz, fiesta_corridor_stats *stats /* nullable */);
/* n_paths paths, their grid voxels (xyz int32) concatenated, with offsets path_off[0] = 0 <= ... <= path_off[n_paths] = total.
 * Box k of path p is written to slot path_off[p] + k (k < n_boxes[p]) of box_lo_xyz / box_hi_xyz / first (total slots each);
 * every other slot is -1.  first[slot] = the box's seed index within its path; blocked_at[p] = that index for status 1, else -1. */
int fiesta_corridors(fiesta_map *m, const int box_lo[3], const int box_hi[3], const int32_t *path_vox_xyz, const int64_t *path_off,
                     int64_t n_paths, const int32_t max_steps[3], double clearance, int flags, int32_t *status, int32_t *n_boxes,
                     int32_t *blocked_at, int32_t *box_lo_xyz, int32_t *box_hi_xyz, int32_t *first,
                     fiesta_corridor_stats *stats /* nullable */);

/* ---- stream-ordered queries on DEVICE buffers (GPU planners whose positions already live in HBM) ----
 * The same queries on device pointers valid on the map's device, enqueued on `stream` (a cudaStream_t; 0 = the legacy default
 * stream); they return without synchronising the host.  Ordering: the query sees every map update issued before the call (the
 * stream first waits for the work enqueued on the map's stream), and every map update issued after the call (ray casting,
 * UpdateOccupancy, UpdateESDF, ...) waits for the query to finish reading.  The query writes only the caller's buffers.  The point
 * queries run the kernel of the host batch forms and return the same bits.  CUDA-graph capture is not supported: a capturing
 * stream is rejected with FIESTA_ERR_INVALID. */
int fiesta_check_segments_device(fiesta_map *m, const double *d_ab, int64_t n, double clearance, int flags, int32_t *d_status,
                                 int64_t *d_hit_idx, double *d_hit_t, double *d_min_dist, void *stream);
/* Robot-shaped collision checks on device poses (n * 12 doubles); half_extents is a HOST array.  The work list and scan storage
 * are the map's own (queries are ordered through the map's stream, so two of them never share them at once). */
int fiesta_check_poses_device(fiesta_map *m, const double *d_poses, int64_t n, const double half_extents[3] /* host */,
                              double clearance, int flags, int32_t *d_status, int32_t *d_n_blocked, int64_t *d_hit_idx, void *stream);
int fiesta_get_distance_batch_device(fiesta_map *m, const double *d_pos_xyz, int64_t n, double *d_dist, void *stream);
int fiesta_get_dist_grad_trilinear_batch_device(fiesta_map *m, const double *d_pos_xyz, int64_t n, double *d_dist, double *d_grad_xyz,
                                                void *stream);

/* ---- state dumps in the reference's own representation (parity harness; host pointers, grid_total_size entries) ---- */
int fiesta_export_distance(fiesta_map *m, double *out);             /* distance_buffer_: -10000 unknown, +10000 unreached */
int fiesta_export_closest_obstacle(fiesta_map *m, int *out_xyz);    /* closest_obstacle_: 3 ints, -10000 = none */
int fiesta_export_occupancy(fiesta_map *m, double *out);            /* occupancy_buffer_ log-odds */
int fiesta_export_counters(fiesta_map *m, int *num_hit, int *num_total); /* num_hit_, num_miss_ (all observations) */

/* ---- map snapshots: save a map to bytes and load it into a new map that continues bit for bit (DESIGN.md §3.12) ----
 * fiesta_snapshot_save serialises the map into a self-describing, versioned little-endian byte stream; fiesta_snapshot_load
 * creates a NEW map from one on `device`.  Continuation guarantee: feed the saved map A and the loaded map B the same calls
 * afterwards (frames, update boxes, UpdateOccupancy, UpdateESDF, SetParameters, filtered depth frames) and after every call
 * the exports, every query, GetPointCloud / GetSliceMarker and every fiesta_stats field except kernel_launches, the ms_*
 * timings and raycast_rounds are equal bit for bit, in both modes (raycast_rounds counts stamp-resolution rounds, which depend
 * on the order in which concurrent rays claim voxels: two maps fed the same frames can differ in it, so it is not stored); an EXACT map therefore stays bit-identical to the reference.  The stream
 * carries the mode, and load creates the map in that mode: FIESTA_B200_MODE is ignored by load.  Objects attached to a map
 * (host mirror, nav fields, frontiers, query plans, shard settings) are not saved; create them again on the loaded map.  The
 * stream depends only on the map's state: saving a loaded map gives the same bytes.
 *
 * Save.  Only a quiescent map can be saved, as it stands after UpdateESDF in the per-frame driver: FIESTA_ERR_INVALID, with
 * nothing written, while SetOccupancy events are staged, while the occupancy queue is not empty (fiesta_check_update() == 1),
 * while inserts or deletes are pending (UpdateOccupancy returned 1 and UpdateESDF has not run), and for an x-slab shard
 * (fiesta_set_shard with world > 1).  *size always receives the stream size when the map can be saved; buf == NULL with cap == 0
 * only queries it; cap < *size returns FIESTA_ERR_LIMIT and writes nothing.  The source map is not changed.
 * Load.  FIESTA_ERR_INVALID for anything malformed: a truncated or oversized stream, a bad magic, version or checksum, a
 * config whose grid differs from the stored one, an update box outside the grid, tiles not strictly ascending or past the grid,
 * or a voxel word that is not a valid state (a closest-obstacle record outside the grid, bit 31 in a FAST snapshot, a non-finite
 * log-odds, a relink time not below the stored relink clock); every word is checked on the device before any other kernel can
 * read it.  FIESTA_ERR_NO_DEVICE / FIESTA_ERR_LIMIT as fiesta_create.  On any failure the new map is destroyed, *out is NULL
 * and fiesta_last_error() names the reason.
 * Size.  Only the 8^3 tiles holding anything but the never-observed state are stored: per voxel 20 bytes (FAST) or 28 bytes
 * (EXACT) plus 8 bytes per stored tile; a map that has seen little of its volume is small, a fully observed 512^3 grid is about
 * 2.7 GB (FAST) or 3.8 GB (EXACT).
 * Memory.  Both run through two 16 MB device and two 16 MB pinned staging buffers whatever the grid size, plus per-tile arrays
 * of at most 8 bytes per 8^3 tile of the grid; neither needs a copy of the grid.  Synchronous. */
int fiesta_snapshot_save(fiesta_map *m, void *buf, int64_t cap, int64_t *size);
int fiesta_snapshot_load(const void *buf, int64_t size, int32_t device, fiesta_map **out);
/* The configuration the map was created with: origin, resolution and map_size as given, the device, and the mode in force. */
int fiesta_get_config(const fiesta_map *m, fiesta_config *out);

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
