// fiesta_b200 -- header-compatible C++ facade for the reference class `fiesta::ESDFMap`.
//
// Put this directory BEFORE the reference's include/ on the include path and `#include "ESDFMap.h"` in Fiesta.h
// resolves here: same namespace, class name, constructor and public methods as FIESTA include/ESDFMap.h:111-164
// (dense-array + PROBABILISTIC build, the shipped configuration: parameters.h:9-14), same public field
// `grid_total_size_`, same sentinel returns.  Every method forwards 1:1 to the C ABI in include/fiesta_b200.h, which runs
// on the H100.  Ownership matches the reference (Fiesta.h:96,137): `new ESDFMap(...)` / `delete`.
//
// Differences a maintainer should know (see INTEGRATION.md):
//  * RaycastFrame() is an ADDITION: one call replaces the whole Fiesta::RaycastMultithread loop (Fiesta.h:281-303) and is
//    the fast path.  The per-call SetOccupancy() path still works unchanged (events are staged and applied on the device
//    at the next UpdateOccupancy), so Fiesta.h compiles and runs without edits.
//  * SetOccupancy() is not thread-safe; the reference's threaded ray casting (ray_cast_num_thread > 0) is itself racy
//    (Fiesta.h:294-300, ESDFMap.cpp:430-433).  Use RaycastFrame() instead of host threads.
//  * A failed construction (no sm_90 GPU, out of memory) throws std::runtime_error -- there is no CPU fallback.
#ifndef ESDF_MAP_H
#define ESDF_MAP_H

#include <Eigen/Eigen>
#include <cmath>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>
#include <visualization_msgs/Marker.h>
#include <sensor_msgs/PointCloud.h>
#if defined(__has_include)
#if __has_include("parameters.h")
#include "parameters.h"   // the reference's own header (macros, dirs_, Parameters) when built inside the FIESTA tree
#endif
#endif
#include "../fiesta_b200.h"

namespace fiesta {

class ESDFMap {
  fiesta_map *h_ = nullptr;
  double resolution_;
  Eigen::Vector3d origin_;
  Eigen::Vector3i grid_size_;

  static void check(int rc, const char *what) {
    if (rc != FIESTA_OK) throw std::runtime_error(std::string(what) + ": " + fiesta_last_error());
  }
  // a map the library created (Load): the geometry comes from the map itself
  explicit ESDFMap(fiesta_map *h) : h_(h) {
    fiesta_config cfg;
    check(fiesta_get_config(h_, &cfg), "fiesta_get_config");
    resolution_ = cfg.resolution;
    origin_ = Eigen::Vector3d(cfg.origin[0], cfg.origin[1], cfg.origin[2]);
    grid_total_size_ = fiesta_grid_total_size(h_);
    int gs[3];
    fiesta_grid_size(h_, gs);
    grid_size_ = Eigen::Vector3i(gs[0], gs[1], gs[2]);
  }
  void Pos2VoxHost(const Eigen::Vector3d &pos, Eigen::Vector3i &vox) const {   // ESDFMap.cpp:74-77
    for (int i = 0; i < 3; ++i) vox(i) = (int)std::floor((pos(i) - origin_(i)) / resolution_);
  }

 public:
  int grid_total_size_;   // ESDFMap.h:115, read by Fiesta.h:107-108

  // ESDFMap(origin, resolution, map_size) -- ESDFMap.h:116, ESDFMap.cpp:171-213
  // `mode`: FIESTA_MODE_EXACT (default) reproduces the reference's distance_ / closest_obstacle_ bit for bit;
  // FIESTA_MODE_FAST is the faster order-free wavefront whose distances differ slightly on ray-cast maps (fiesta_b200.h).
  // FIESTA_B200_MODE=exact|fast in the environment overrides it without a rebuild.
  ESDFMap(Eigen::Vector3d origin, double resolution, Eigen::Vector3d map_size, int device = 0, int mode = FIESTA_MODE_EXACT)
      : resolution_(resolution), origin_(origin) {
    fiesta_config cfg = {};
    for (int i = 0; i < 3; ++i) { cfg.origin[i] = origin(i); cfg.map_size[i] = map_size(i); }
    cfg.resolution = resolution;
    cfg.device = device;
    cfg.mode = mode;
    check(fiesta_create(&cfg, &h_), "fiesta_create");
    grid_total_size_ = fiesta_grid_total_size(h_);
    int gs[3];
    fiesta_grid_size(h_, gs);
    grid_size_ = Eigen::Vector3i(gs[0], gs[1], gs[2]);
  }
  ~ESDFMap() { fiesta_destroy(h_); }
  ESDFMap(const ESDFMap &) = delete;
  ESDFMap &operator=(const ESDFMap &) = delete;
  fiesta_map *handle() { return h_; }

  // Map snapshots (fiesta_snapshot_save / fiesta_snapshot_load): a loaded map continues bit for bit like the saved one.  Save
  // needs a quiescent map (after UpdateESDF in the per-frame driver); Load creates the map in the snapshot's mode.
  std::vector<uint8_t> Save() {
    int64_t size = 0;
    check(fiesta_snapshot_save(h_, nullptr, 0, &size), "Save");
    std::vector<uint8_t> out((size_t)size);
    check(fiesta_snapshot_save(h_, out.data(), size, &size), "Save");
    return out;
  }
  static std::unique_ptr<ESDFMap> Load(const void *data, size_t size, int device = 0) {
    fiesta_map *h = nullptr;
    check(fiesta_snapshot_load(data, (int64_t)size, device, &h), "Load");
    return std::unique_ptr<ESDFMap>(new ESDFMap(h));
  }

  // ESDFMap.h:124
  void SetParameters(double p_hit, double p_miss, double p_min, double p_max, double p_occ) {
    check(fiesta_set_parameters(h_, p_hit, p_miss, p_min, p_max, p_occ), "SetParameters");
  }

  // ESDFMap.h:128-130 -- the per-frame driver calls (Fiesta.h:507-514)
  bool CheckUpdate() { return fiesta_check_update(h_) != 0; }
  bool UpdateOccupancy(bool global_map) {
    int r = fiesta_update_occupancy(h_, global_map ? 1 : 0);
    if (r < 0) check(-r, "UpdateOccupancy");
    return r > 0;
  }
  void UpdateESDF() { check(fiesta_update_esdf(h_), "UpdateESDF"); }

  // ESDFMap.h:133-136
  int SetOccupancy(Eigen::Vector3d pos, int occ) { double p[3] = {pos(0), pos(1), pos(2)}; return fiesta_set_occupancy_pos(h_, p, occ); }
  int SetOccupancy(Eigen::Vector3i vox, int occ) { int v[3] = {vox(0), vox(1), vox(2)}; return fiesta_set_occupancy_vox(h_, v, occ); }
  int GetOccupancy(Eigen::Vector3d pos) { double p[3] = {pos(0), pos(1), pos(2)}; return fiesta_get_occupancy_pos(h_, p); }
  int GetOccupancy(Eigen::Vector3i vox) { int v[3] = {vox(0), vox(1), vox(2)}; return fiesta_get_occupancy_vox(h_, v); }

  // ESDFMap.h:139-141
  double GetDistance(Eigen::Vector3d pos) { double p[3] = {pos(0), pos(1), pos(2)}; return fiesta_get_distance_pos(h_, p); }
  double GetDistance(Eigen::Vector3i vox) { int v[3] = {vox(0), vox(1), vox(2)}; return fiesta_get_distance_vox(h_, v); }
  double GetDistWithGradTrilinear(Eigen::Vector3d pos, Eigen::Vector3d &grad) {
    double p[3] = {pos(0), pos(1), pos(2)}, g[3] = {0, 0, 0};
    double d = fiesta_get_dist_grad_trilinear(h_, p, g);
    grad(0) = g[0]; grad(1) = g[1]; grad(2) = g[2];
    return d;
  }

  // ESDFMap.h:148-149
  void SetUpdateRange(Eigen::Vector3d min_pos, Eigen::Vector3d max_pos, bool new_vec = true) {
    double a[3] = {min_pos(0), min_pos(1), min_pos(2)}, b[3] = {max_pos(0), max_pos(1), max_pos(2)};
    check(fiesta_set_update_range(h_, a, b, new_vec ? 1 : 0), "SetUpdateRange");
  }
  void SetOriginalRange() { check(fiesta_set_original_range(h_), "SetOriginalRange"); }

  // ---- additions (fast paths; not in the reference class) ----
  // One call for Fiesta::RaycastMultithread (Fiesta.h:281-303): `cloud` holds n points as packed float xyz in the sensor
  // frame, `transform` is Fiesta's transform_ (row-major 4x4).  Serial-mode semantics, computed on the GPU.
  void RaycastFrame(const float *cloud_xyz, long n, const double transform_row_major[16], double min_ray_length, double max_ray_length) {
    fiesta_raycast_params p = {min_ray_length, max_ray_length};
    check(fiesta_raycast_frame(h_, cloud_xyz, n, transform_row_major, &p), "RaycastFrame");
  }
  void GetDistWithGradTrilinearBatch(const double *pos_xyz, long n, double *dist, double *grad_xyz) {
    check(fiesta_get_dist_grad_trilinear_batch(h_, pos_xyz, n, dist, grad_xyz), "GetDistWithGradTrilinearBatch");
  }
  // Fixed-size variant for optimiser loops: pinned buffers + one CUDA-graph launch per call (fiesta_query_plan_* in
  // fiesta_b200.h): fill fiesta_query_plan_positions(p), fiesta_query_plan_run(p), read distances / gradients.
  fiesta_query_plan *MakeQueryPlan(long n) {
    fiesta_query_plan *p = nullptr;
    check(fiesta_query_plan_create(h_, n, &p), "MakeQueryPlan");
    return p;
  }

  // Per-call host consumers: a pinned host mirror of the distance records (fiesta_host_mirror_* in fiesta_b200.h).  Call
  // fiesta_host_mirror_refresh(p, nullptr) after UpdateESDF(); fiesta_host_mirror_get_distance_pos /
  // fiesta_host_mirror_get_dist_grad_trilinear then answer from host memory with the bits GetDistance /
  // GetDistWithGradTrilinear return.
  fiesta_host_mirror *MakeHostMirror() {
    fiesta_host_mirror *p = nullptr;
    check(fiesta_host_mirror_create(h_, &p), "MakeHostMirror");
    return p;
  }

  // Segment clearance for planners (fiesta_check_segments in fiesta_b200.h): n segments {ax, ay, az, bx, by, bz}; per segment
  // status (0 clear, 1 blocked, 2 outside the map), the first blocking voxel's linear index and entry parameter, and the minimum
  // distance walked.  flags: FIESTA_SEGMENT_UNKNOWN_BLOCKS.  Host pointers, synchronous.
  void CheckSegments(const double *ab, long n, double clearance, int flags, int32_t *status, int64_t *hit_idx, double *hit_t,
                     double *min_dist) {
    check(fiesta_check_segments(h_, ab, n, clearance, flags, status, hit_idx, hit_t, min_dist), "CheckSegments");
  }
  // The same queries on DEVICE buffers, enqueued on `stream` (a cudaStream_t) without synchronising the host; ordered after every
  // earlier map update and before every later one (fiesta_b200.h).
  void CheckSegmentsDevice(const double *d_ab, long n, double clearance, int flags, int32_t *d_status, int64_t *d_hit_idx,
                           double *d_hit_t, double *d_min_dist, void *stream) {
    check(fiesta_check_segments_device(h_, d_ab, n, clearance, flags, d_status, d_hit_idx, d_hit_t, d_min_dist, stream),
          "CheckSegmentsDevice");
  }
  // Robot-shaped collision checks (fiesta_check_poses in fiesta_b200.h): an oriented box of half extents h (metres) at n poses
  // {px, py, pz, R00 .. R22} (R world-to-body, rows = box axes); per pose status (0 clear, 1 blocked, 2 invalid pose, 3 leaves the
  // map), the number of touched blocking voxels and the least linear index among them.  flags: FIESTA_SEGMENT_UNKNOWN_BLOCKS.
  // Host pointers, synchronous.
  void CheckPoses(const double *poses, long n, const double half_extents[3], double clearance, int flags, int32_t *status,
                  int32_t *n_blocked, int64_t *hit_idx) {
    check(fiesta_check_poses(h_, poses, n, half_extents, clearance, flags, status, n_blocked, hit_idx), "CheckPoses");
  }
  // The same on DEVICE poses and outputs (half_extents stays on the host), enqueued on `stream` without synchronising the host.
  void CheckPosesDevice(const double *d_poses, long n, const double half_extents[3], double clearance, int flags, int32_t *d_status,
                        int32_t *d_n_blocked, int64_t *d_hit_idx, void *stream) {
    check(fiesta_check_poses_device(h_, d_poses, n, half_extents, clearance, flags, d_status, d_n_blocked, d_hit_idx, stream),
          "CheckPosesDevice");
  }
  // The same from a host mirror's pinned records (pure host code, as of its last refresh).
  void CheckPosesMirror(const fiesta_host_mirror *p, const double *poses, long n, const double half_extents[3], double clearance,
                        int flags, int32_t *status, int32_t *n_blocked, int64_t *hit_idx) {
    check(fiesta_host_mirror_check_poses(p, poses, n, half_extents, clearance, flags, status, n_blocked, hit_idx), "CheckPosesMirror");
  }
  // Cost-to-go field for planners (fiesta_nav_* in fiesta_b200.h): geodesic distance from every voxel of a box to the nearest
  // goal through free space at a clearance, and paths down it.  Destroy the field with fiesta_nav_destroy before the map.
  fiesta_nav_field *MakeNavField() {
    fiesta_nav_field *f = nullptr;
    check(fiesta_nav_create(h_, &f), "MakeNavField");
    return f;
  }
  fiesta_nav_stats ComputeNavField(fiesta_nav_field *f, const int box_lo[3], const int box_hi[3], const double *goals_xyz, long n_goals,
                                   double clearance, int flags) {
    fiesta_nav_stats st = {};
    check(fiesta_nav_compute(f, box_lo, box_hi, goals_xyz, n_goals, clearance, flags, &st), "ComputeNavField");
    return st;
  }
  // Repair the field after map updates (fiesta_nav_update): the bits ComputeNavField would give now with the same box, goals,
  // clearance and flags, at the cost of the region the changes affect.
  fiesta_nav_update_stats UpdateNavField(fiesta_nav_field *f) {
    fiesta_nav_update_stats st = {};
    check(fiesta_nav_update(f, &st), "UpdateNavField");
    return st;
  }
  // Cost matrix (fiesta_nav_matrix): cost[i * n_tgt + j] = the field of source i alone read at target j, NaN where either point is
  // blocked or outside the box.  Leaves the last ComputeNavField result as it was.
  fiesta_nav_matrix_stats NavCostMatrix(fiesta_nav_field *f, const int box_lo[3], const int box_hi[3], const double *sources_xyz, long n_src,
                                        const double *targets_xyz, long n_tgt, double clearance, int flags, int32_t *src_status,
                                        int32_t *tgt_status, double *cost) {
    fiesta_nav_matrix_stats st = {};
    check(fiesta_nav_matrix(f, box_lo, box_hi, sources_xyz, n_src, targets_xyz, n_tgt, clearance, flags, src_status, tgt_status, cost, &st),
          "NavCostMatrix");
    return st;
  }
  void ExportNavField(const fiesta_nav_field *f, double *out) { check(fiesta_nav_export(f, out), "ExportNavField"); }
  void NavPaths(fiesta_nav_field *f, const double *starts_xyz, long n, int max_len, int32_t *status, int32_t *len, double *cost,
                int32_t *vox_xyz) {
    check(fiesta_nav_paths(f, starts_xyz, n, max_len, status, len, cost, vox_xyz), "NavPaths");
  }
  // Signed distance of a box for trajectory optimisers (fiesta_signed_* in fiesta_b200.h): FIESTA's distance outside obstacles,
  // minus the exact depth inside them.  Compute again after UpdateOccupancy / UpdateESDF.  Destroy with fiesta_signed_destroy
  // before the map.
  fiesta_signed_field *MakeSignedField() {
    fiesta_signed_field *f = nullptr;
    check(fiesta_signed_create(h_, &f), "MakeSignedField");
    return f;
  }
  fiesta_signed_stats ComputeSignedField(fiesta_signed_field *f, const int box_lo[3], const int box_hi[3]) {
    fiesta_signed_stats st = {};
    check(fiesta_signed_compute(f, box_lo, box_hi, &st), "ComputeSignedField");
    return st;
  }
  void ExportSignedField(const fiesta_signed_field *f, double *out) { check(fiesta_signed_export(f, out), "ExportSignedField"); }
  // GetDistWithGradTrilinear on the signed field: S inside the box, the map's distance outside it (host pointers).
  void SignedDistWithGradTrilinearBatch(fiesta_signed_field *f, const double *pos_xyz, long n, double *dist, double *grad_xyz) {
    check(fiesta_signed_get_dist_grad_trilinear_batch(f, pos_xyz, n, dist, grad_xyz), "SignedDistWithGradTrilinearBatch");
  }
  // Frontier extraction for exploration planners (fiesta_frontiers_* in fiesta_b200.h): the free voxels of a box that border
  // unknown space, in 26-connected clusters with statistics and member lists.  Destroy with fiesta_frontiers_destroy before the map.
  fiesta_frontiers *MakeFrontiers() {
    fiesta_frontiers *f = nullptr;
    check(fiesta_frontiers_create(h_, &f), "MakeFrontiers");
    return f;
  }
  fiesta_frontier_stats ComputeFrontiers(fiesta_frontiers *f, const int box_lo[3], const int box_hi[3], double clearance,
                                         long min_cluster_size) {
    fiesta_frontier_stats st = {};
    check(fiesta_frontiers_compute(f, box_lo, box_hi, clearance, min_cluster_size, &st), "ComputeFrontiers");
    return st;
  }
  void FrontierClusters(const fiesta_frontiers *f, long cap, int64_t *size, int32_t *rep_xyz, int32_t *bbox_lo_xyz, int32_t *bbox_hi_xyz,
                        double *centroid_xyz) {
    check(fiesta_frontiers_clusters(f, cap, size, rep_xyz, bbox_lo_xyz, bbox_hi_xyz, centroid_xyz), "FrontierClusters");
  }
  void FrontierVoxels(const fiesta_frontiers *f, long cap, int32_t *vox_xyz) { check(fiesta_frontiers_voxels(f, cap, vox_xyz), "FrontierVoxels"); }
  void ExportFrontierLabels(const fiesta_frontiers *f, int32_t *labels) { check(fiesta_frontiers_export(f, labels), "ExportFrontierLabels"); }
  fiesta_viewpoint_stats ScoreViewpoints(fiesta_frontiers *f, const int32_t *cluster, const double *pos_xyz, long n, const double *orient,
                                         int n_orient, const fiesta_sensor_model &sensor, double clearance, int flags, int32_t *status,
                                         int32_t *score) {
    fiesta_viewpoint_stats st = {};
    check(fiesta_frontiers_score_viewpoints(f, cluster, pos_xyz, n, orient, n_orient, &sensor, clearance, flags, status, score, &st), "ScoreViewpoints");
    return st;
  }
  // Topological roadmaps (fiesta_skeleton_* in fiesta_b200.h): the skeleton of a box's free space on the generalized Voronoi diagram
  // of the obstacles, as a graph of vertices and edges.  Destroy with fiesta_skeleton_destroy before the map.
  fiesta_skeleton *MakeSkeleton() {
    fiesta_skeleton *f = nullptr;
    check(fiesta_skeleton_create(h_, &f), "MakeSkeleton");
    return f;
  }
  fiesta_skeleton_stats ComputeSkeleton(fiesta_skeleton *f, const int box_lo[3], const int box_hi[3], double clearance, int flags,
                                        double max_cos, long min_branch) {
    fiesta_skeleton_stats st = {};
    check(fiesta_skeleton_compute(f, box_lo, box_hi, clearance, flags, max_cos, min_branch, &st), "ComputeSkeleton");
    return st;
  }
  void SkeletonVertices(const fiesta_skeleton *f, long cap, int64_t *size, int32_t *rep_xyz, double *centroid_xyz, int32_t *degree) {
    check(fiesta_skeleton_vertices(f, cap, size, rep_xyz, centroid_xyz, degree), "SkeletonVertices");
  }
  void SkeletonEdges(const fiesta_skeleton *f, long cap, int32_t *uv, int64_t *n_vox, double *length, double *min_dist) {
    check(fiesta_skeleton_edges(f, cap, uv, n_vox, length, min_dist), "SkeletonEdges");
  }
  void SkeletonEdgeVoxels(const fiesta_skeleton *f, long cap, int32_t *vox_xyz) {
    check(fiesta_skeleton_edge_voxels(f, cap, vox_xyz), "SkeletonEdgeVoxels");
  }
  void ExportSkeleton(const fiesta_skeleton *f, uint8_t *mask, int32_t *label) { check(fiesta_skeleton_export(f, mask, label), "ExportSkeleton"); }
  // Surface meshes (fiesta_mesh_* in fiesta_b200.h): the triangle mesh of the boundary of what blocks at a clearance in a box, float32
  // vertices in metres and int32 triangles.  Destroy with fiesta_mesh_destroy before the map.
  fiesta_mesh *MakeMesh() {
    fiesta_mesh *f = nullptr;
    check(fiesta_mesh_create(h_, &f), "MakeMesh");
    return f;
  }
  fiesta_mesh_stats ComputeMesh(fiesta_mesh *f, const int box_lo[3], const int box_hi[3], double clearance, int flags) {
    fiesta_mesh_stats st = {};
    check(fiesta_mesh_compute(f, box_lo, box_hi, clearance, flags, &st), "ComputeMesh");
    return st;
  }
  void MeshVertices(const fiesta_mesh *f, long cap, float *xyz) { check(fiesta_mesh_vertices(f, cap, xyz), "MeshVertices"); }
  void MeshTriangles(const fiesta_mesh *f, long cap, int32_t *ijk) { check(fiesta_mesh_triangles(f, cap, ijk), "MeshTriangles"); }
  // Safe flight corridors (fiesta_inflate_boxes / fiesta_corridors in fiesta_b200.h): free axis-aligned voxel boxes in a limit box,
  // and chains of them along paths in which consecutive boxes share a voxel.
  fiesta_corridor_stats InflateBoxes(const int box_lo[3], const int box_hi[3], const int32_t *seed_lo_xyz, const int32_t *seed_hi_xyz,
                                     long n, const int32_t max_steps[3], double clearance, int flags, int32_t *status, int32_t *out_lo_xyz,
                                     int32_t *out_hi_xyz) {
    fiesta_corridor_stats st = {};
    check(fiesta_inflate_boxes(h_, box_lo, box_hi, seed_lo_xyz, seed_hi_xyz, n, max_steps, clearance, flags, status, out_lo_xyz, out_hi_xyz, &st),
          "InflateBoxes");
    return st;
  }
  fiesta_corridor_stats Corridors(const int box_lo[3], const int box_hi[3], const int32_t *path_vox_xyz, const int64_t *path_off, long n_paths,
                                  const int32_t max_steps[3], double clearance, int flags, int32_t *status, int32_t *n_boxes, int32_t *blocked_at,
                                  int32_t *box_lo_xyz, int32_t *box_hi_xyz, int32_t *first) {
    fiesta_corridor_stats st = {};
    check(fiesta_corridors(h_, box_lo, box_hi, path_vox_xyz, path_off, n_paths, max_steps, clearance, flags, status, n_boxes, blocked_at,
                           box_lo_xyz, box_hi_xyz, first, &st), "Corridors");
    return st;
  }
  void GetDistanceBatchDevice(const double *d_pos_xyz, long n, double *d_dist, void *stream) {
    check(fiesta_get_distance_batch_device(h_, d_pos_xyz, n, d_dist, stream), "GetDistanceBatchDevice");
  }
  void GetDistWithGradTrilinearBatchDevice(const double *d_pos_xyz, long n, double *d_dist, double *d_grad_xyz, void *stream) {
    check(fiesta_get_dist_grad_trilinear_batch_device(h_, d_pos_xyz, n, d_dist, d_grad_xyz, stream), "GetDistWithGradTrilinearBatchDevice");
  }

  // ---- visualisation (ESDFMap.h:144-145): flag pass + ordered stream compaction on the device, only the selected points
  // cross PCIe (fiesta_get_point_cloud / fiesta_get_slice_marker) ----
  void GetPointCloud(sensor_msgs::PointCloud &m, int vis_lower_bound, int vis_upper_bound) {
    m.header.frame_id = "world";
    m.points.clear();
    int64_t n = 0;
    check(fiesta_get_point_cloud(h_, vis_lower_bound, vis_upper_bound, nullptr, 0, &n), "GetPointCloud");
    std::vector<float> xyz((size_t)n * 3 + 3);
    if (n) check(fiesta_get_point_cloud(h_, vis_lower_bound, vis_upper_bound, xyz.data(), n, &n), "GetPointCloud");
    m.points.resize((size_t)n);
    for (int64_t i = 0; i < n; ++i) { m.points[i].x = xyz[3 * i]; m.points[i].y = xyz[3 * i + 1]; m.points[i].z = xyz[3 * i + 2]; }
  }
  void GetSliceMarker(visualization_msgs::Marker &m, int slice, int id, Eigen::Vector4d /*color*/, double max_dist) {
    m.header.frame_id = "world";
    m.id = id;
    m.type = visualization_msgs::Marker::POINTS;
    m.action = visualization_msgs::Marker::MODIFY;
    m.scale.x = m.scale.y = m.scale.z = resolution_;
    m.pose.orientation.w = 1; m.pose.orientation.x = m.pose.orientation.y = m.pose.orientation.z = 0;
    m.points.clear();
    m.colors.clear();
    int64_t n = 0;
    check(fiesta_get_slice_marker(h_, slice, max_dist, nullptr, nullptr, 0, &n), "GetSliceMarker");
    std::vector<double> xyz((size_t)n * 3 + 3);
    std::vector<float> rgba((size_t)n * 4 + 4);
    if (n) check(fiesta_get_slice_marker(h_, slice, max_dist, xyz.data(), rgba.data(), n, &n), "GetSliceMarker");
    m.points.resize((size_t)n);
    m.colors.resize((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
      m.points[i].x = xyz[3 * i]; m.points[i].y = xyz[3 * i + 1]; m.points[i].z = xyz[3 * i + 2];
      m.colors[i].r = rgba[4 * i]; m.colors[i].g = rgba[4 * i + 1]; m.colors[i].b = rgba[4 * i + 2]; m.colors[i].a = rgba[4 * i + 3];
    }
  }
};

}  // namespace fiesta
#endif  // ESDF_MAP_H
