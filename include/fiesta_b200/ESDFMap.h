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
