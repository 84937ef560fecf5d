// TEST INFRASTRUCTURE ONLY -- never linked into, imported by or called from the product path.
//
// C API around the UNMODIFIED reference class fiesta::ESDFMap (compiled in place from
// FIESTA src/ESDFMap.cpp + src/raycast.cpp against oracle/shims) so that tests/, bench.py's
// cpu_baseline / --impl reference legs and __graft_entry__.smoke() can drive the real reference
// through ctypes.  Built by oracle/Makefile into oracle/_ref/libfiesta_ref.so (git-ignored).
//
// The only logic restated here is Fiesta::RaycastProcess / RaycastMultithread
// (FIESTA include/Fiesta.h:194-303): it lives in a header that needs ROS/OpenCV/PCL and
// cannot be compiled in this image.  The restatement follows that text in serial mode
// (ray_cast_num_thread == 0, the only deterministic mode; launch/*.launch:23) and calls the
// compiled reference Raycast() and ESDFMap::SetOccupancy().
#include <sstream>
#include <iostream>
#include <cstring>
#include <cstdio>
#include <cmath>
#include <vector>

#define private public  // inspect reference state (distance_buffer_, closest_obstacle_, ...) from tests
#include "ESDFMap.h"
#undef private
#include "raycast.h"
#include "depth_restated.h"

namespace {

struct RefMap {
  fiesta::ESDFMap *map;
  Eigen::Vector3d l_cornor, r_cornor;
  double resolution;
  // Fiesta.h:59-64,107-110 -- per-frame stamp arrays owned by the Fiesta node
  std::vector<int> set_free, set_occ;
  unsigned tot;
  long hung;  // rays dropped by the hang guard
  // numbers the reference only prints (ESDFMap.cpp:237,277,394)
  long last_occupancy_updates, last_insert, last_delete, last_expansions, last_change_num;
};

// Run f() with std::cout captured; the reference prints inside its hot path.
template <typename F>
std::string captured(F f) {
  std::ostringstream oss;
  std::streambuf *old = std::cout.rdbuf(oss.rdbuf());
  f();
  std::cout.rdbuf(old);
  return oss.str();
}

long number_after(const std::string &s, const char *key) {
  std::size_t p = s.find(key);
  if (p == std::string::npos) return -1;
  return std::strtol(s.c_str() + p + std::strlen(key), nullptr, 10);
}

// Hang guard (test infrastructure, not reference code): the reference Raycast() loop (raycast.cpp:116-158) only
// returns from inside the box, so it spins forever once the walk has overshot the end voxel on some axis and has
// left the box for good (e.g. a start exactly on a lattice plane heading in a negative direction -- intbound quirk).
// This replays the same stepping arithmetic WITHOUT emitting anything and reports whether the call would hang.
double gb_mod(double a, double b) { return std::fmod(std::fmod(a, b) + b, b); }
double gb_intbound(double s, double ds) { if (ds < 0) { s = -s; ds = -ds; } s = gb_mod(s, 1); return (1 - s) / ds; }
bool raycast_would_hang(const Eigen::Vector3d &start, const Eigen::Vector3d &end, const Eigen::Vector3d &mn,
                        const Eigen::Vector3d &mx) {
  int c[3], e[3], step[3];
  double delta[3], tmax[3], tdelta[3];
  for (int i = 0; i < 3; ++i) { c[i] = (int)std::floor(start(i)); e[i] = (int)std::floor(end(i)); }
  const double maxd = (end - start).squaredNorm();
  for (int i = 0; i < 3; ++i) {
    delta[i] = e[i] - c[i];
    step[i] = delta[i] == 0 ? 0 : (delta[i] < 0 ? -1 : 1);
    tmax[i] = gb_intbound(start(i), delta[i]);
    tdelta[i] = ((double)step[i]) / delta[i];
  }
  if (!step[0] && !step[1] && !step[2]) return false;
  for (;;) {
    if (c[0] >= mn(0) && c[0] < mx(0) && c[1] >= mn(1) && c[1] < mx(1) && c[2] >= mn(2) && c[2] < mx(2)) {
      double a = c[0] - start(0), b = c[1] - start(1), g = c[2] - start(2);
      if ((a * a + b * b) + g * g > maxd) return false;
    }
    if (c[0] == e[0] && c[1] == e[1] && c[2] == e[2]) return false;
    bool overshot = false, gone = false;
    for (int i = 0; i < 3; ++i) {
      if ((step[i] > 0 && c[i] > e[i]) || (step[i] < 0 && c[i] < e[i]) || (step[i] == 0 && c[i] != e[i])) overshot = true;
      if ((step[i] >= 0 && !(c[i] < mx(i))) || (step[i] <= 0 && !(c[i] >= mn(i)))) gone = true;
    }
    if (overshot && gone) return true;
    if (tmax[0] < tmax[1]) {
      if (tmax[0] < tmax[2]) { c[0] += step[0]; tmax[0] += tdelta[0]; } else { c[2] += step[2]; tmax[2] += tdelta[2]; }
    } else {
      if (tmax[1] < tmax[2]) { c[1] += step[1]; tmax[1] += tdelta[1]; } else { c[2] += step[2]; tmax[2] += tdelta[2]; }
    }
  }
}

Eigen::Vector3d v3(const double *p) { return Eigen::Vector3d(p[0], p[1], p[2]); }
Eigen::Vector3i v3i(const int *p) { return Eigen::Vector3i(p[0], p[1], p[2]); }

}  // namespace

extern "C" {

void *fiesta_ref_create(const double origin[3], double resolution, const double map_size[3]) {
  RefMap *r = new RefMap();
  captured([&] { r->map = new fiesta::ESDFMap(v3(origin), resolution, v3(map_size)); });  // ctor prints grid_total_size_
  r->l_cornor = v3(origin);
  r->r_cornor = v3(origin) + v3(map_size);
  r->resolution = resolution;
  r->set_free.assign(r->map->grid_total_size_, 0);  // Fiesta.h:107-110
  r->set_occ.assign(r->map->grid_total_size_, 0);
  r->tot = 0;
  r->hung = 0;
  r->last_occupancy_updates = r->last_insert = r->last_delete = r->last_expansions = r->last_change_num = 0;
  return r;
}

void fiesta_ref_destroy(void *h) {
  RefMap *r = (RefMap *)h;
  delete r->map;
  delete r;
}

void fiesta_ref_set_parameters(void *h, double p_hit, double p_miss, double p_min, double p_max, double p_occ) {
  ((RefMap *)h)->map->SetParameters(p_hit, p_miss, p_min, p_max, p_occ);
}

int fiesta_ref_grid_total_size(void *h) { return ((RefMap *)h)->map->grid_total_size_; }

void fiesta_ref_grid_size(void *h, int out[3]) {
  fiesta::ESDFMap *m = ((RefMap *)h)->map;
  for (int i = 0; i < 3; ++i) out[i] = m->grid_size_(i);
}

int fiesta_ref_set_occupancy_pos(void *h, const double pos[3], int occ) {
  RefMap *r = (RefMap *)h;
  int ret = 0;
  if (occ != 0 && occ != 1) { captured([&] { ret = r->map->SetOccupancy(v3(pos), occ); }); return ret; }
  return r->map->SetOccupancy(v3(pos), occ);
}

int fiesta_ref_set_occupancy_vox(void *h, const int vox[3], int occ) {
  return ((RefMap *)h)->map->SetOccupancy(v3i(vox), occ);
}

void fiesta_ref_set_occupancy_batch_pos(void *h, const double *pos, const unsigned char *occ, long n, int *out_idx) {
  fiesta::ESDFMap *m = ((RefMap *)h)->map;
  for (long i = 0; i < n; ++i) {
    int idx = m->SetOccupancy(v3(pos + 3 * i), (int)occ[i]);
    if (out_idx) out_idx[i] = idx;
  }
}

void fiesta_ref_set_occupancy_batch_vox(void *h, const int *vox, const unsigned char *occ, long n, int *out_idx) {
  fiesta::ESDFMap *m = ((RefMap *)h)->map;
  for (long i = 0; i < n; ++i) {
    int idx = m->SetOccupancy(v3i(vox + 3 * i), (int)occ[i]);
    if (out_idx) out_idx[i] = idx;
  }
}

int fiesta_ref_check_update(void *h) { return ((RefMap *)h)->map->CheckUpdate() ? 1 : 0; }

int fiesta_ref_update_occupancy(void *h, int global_map) {
  RefMap *r = (RefMap *)h;
  bool ret = false;
  std::string s = captured([&] { ret = r->map->UpdateOccupancy(global_map != 0); });
  r->last_occupancy_updates = number_after(s, "Occupancy Update ");
  return ret ? 1 : 0;
}

void fiesta_ref_update_esdf(void *h) {
  RefMap *r = (RefMap *)h;
  std::string s = captured([&] { r->map->UpdateESDF(); });
  r->last_insert = number_after(s, "Insert ");
  r->last_delete = number_after(s, "Delete ");
  r->last_expansions = number_after(s, "Expanding ");
  r->last_change_num = number_after(s, "change_num = ");
}

void fiesta_ref_set_update_range(void *h, const double mn[3], const double mx[3], int new_vec) {
  ((RefMap *)h)->map->SetUpdateRange(v3(mn), v3(mx), new_vec != 0);
}

void fiesta_ref_set_original_range(void *h) { ((RefMap *)h)->map->SetOriginalRange(); }

double fiesta_ref_get_distance_pos(void *h, const double pos[3]) { return ((RefMap *)h)->map->GetDistance(v3(pos)); }
double fiesta_ref_get_distance_vox(void *h, const int vox[3]) { return ((RefMap *)h)->map->GetDistance(v3i(vox)); }
int fiesta_ref_get_occupancy_pos(void *h, const double pos[3]) { return ((RefMap *)h)->map->GetOccupancy(v3(pos)); }
int fiesta_ref_get_occupancy_vox(void *h, const int vox[3]) { return ((RefMap *)h)->map->GetOccupancy(v3i(vox)); }

double fiesta_ref_get_dist_grad_trilinear(void *h, const double pos[3], double grad[3]) {
  Eigen::Vector3d g(0.0, 0.0, 0.0);
  double d = ((RefMap *)h)->map->GetDistWithGradTrilinear(v3(pos), g);
  grad[0] = g(0); grad[1] = g(1); grad[2] = g(2);
  return d;
}

void fiesta_ref_get_distance_batch_pos(void *h, const double *pos, long n, double *out) {
  fiesta::ESDFMap *m = ((RefMap *)h)->map;
  for (long i = 0; i < n; ++i) out[i] = m->GetDistance(v3(pos + 3 * i));
}

void fiesta_ref_get_dist_grad_trilinear_batch(void *h, const double *pos, long n, double *dist, double *grad) {
  for (long i = 0; i < n; ++i) dist[i] = fiesta_ref_get_dist_grad_trilinear(h, pos + 3 * i, grad + 3 * i);
}

// ---- raw state dumps (reference-private arrays; ESDFMap.h:83-91) ----
void fiesta_ref_export_distance(void *h, double *out) {
  fiesta::ESDFMap *m = ((RefMap *)h)->map;
  std::memcpy(out, m->distance_buffer_.data(), sizeof(double) * m->grid_total_size_);
}
void fiesta_ref_export_occupancy(void *h, double *out) {
  fiesta::ESDFMap *m = ((RefMap *)h)->map;
  std::memcpy(out, m->occupancy_buffer_.data(), sizeof(double) * m->grid_total_size_);
}
void fiesta_ref_export_closest_obstacle(void *h, int *out3) {
  fiesta::ESDFMap *m = ((RefMap *)h)->map;
  for (int i = 0; i < m->grid_total_size_; ++i)
    for (int k = 0; k < 3; ++k) out3[3 * i + k] = m->closest_obstacle_[i](k);
}
void fiesta_ref_export_counters(void *h, int *hit, int *total) {
  fiesta::ESDFMap *m = ((RefMap *)h)->map;
  std::memcpy(hit, m->num_hit_.data(), sizeof(int) * m->grid_total_size_);
  std::memcpy(total, m->num_miss_.data(), sizeof(int) * m->grid_total_size_);  // num_miss_ counts ALL observations
}

long fiesta_ref_hung_rays(void *h) { return ((RefMap *)h)->hung; }

long fiesta_ref_pending_occupancy(void *h) { return (long)((RefMap *)h)->map->occupancy_queue_.size(); }

void fiesta_ref_get_stats(void *h, long out[6]) {
  RefMap *r = (RefMap *)h;
  out[0] = r->last_occupancy_updates; out[1] = r->last_insert; out[2] = r->last_delete;
  out[3] = r->last_expansions; out[4] = r->last_change_num; out[5] = r->map->total_time_;
}

// ESDFMap::GetPointCloud / GetSliceMarker (ESDFMap.cpp:544-582, 639-699) -- the reference's own code, results flattened.
long fiesta_ref_get_point_cloud(void *h, int lo, int hi, float *out, long cap) {
  sensor_msgs::PointCloud pc;
  ((RefMap *)h)->map->GetPointCloud(pc, lo, hi);
  long n = (long)pc.points.size();
  for (long i = 0; i < n && i < cap; ++i) { out[3 * i] = pc.points[i].x; out[3 * i + 1] = pc.points[i].y; out[3 * i + 2] = pc.points[i].z; }
  return n;
}
long fiesta_ref_get_slice_marker(void *h, int slice, double max_dist, double *xyz, float *rgba, long cap) {
  visualization_msgs::Marker mk;
  ((RefMap *)h)->map->GetSliceMarker(mk, slice, 100, Eigen::Vector4d(0, 1.0, 0, 1), max_dist);
  long n = (long)mk.points.size();
  for (long i = 0; i < n && i < cap; ++i) {
    xyz[3 * i] = mk.points[i].x; xyz[3 * i + 1] = mk.points[i].y; xyz[3 * i + 2] = mk.points[i].z;
    rgba[4 * i] = mk.colors[i].r; rgba[4 * i + 1] = mk.colors[i].g; rgba[4 * i + 2] = mk.colors[i].b; rgba[4 * i + 3] = mk.colors[i].a;
  }
  return n;
}

long fiesta_ref_depth_conversion(const uint16_t *img, const uint16_t *last, int rows, int cols, unsigned image_cnt,
                                 const oracle_depth_params *p, const double *m_rel, float *cloud) {
  return oracle_depth_conversion(img, last, rows, cols, image_cnt, p, m_rel, cloud);
}

int fiesta_ref_check_consistency(void *h) {
  RefMap *r = (RefMap *)h;
  bool ok = false;
  captured([&] { ok = r->map->CheckConsistency(); });
  return ok ? 1 : 0;
}

// Reference Raycast() (raycast.cpp:56-158) exposed for direct DDA parity tests.
// Returns the number of voxels, -1 if the reference threw (more than 1500 voxels), -2 if it would never return.
long fiesta_ref_raycast(const double start[3], const double end[3], const double mn[3], const double mx[3],
                        double *out_xyz, long cap) {
  std::vector<Eigen::Vector3d> out;
  if (raycast_would_hang(v3(start), v3(end), v3(mn), v3(mx))) return -2;
  try {
    std::streambuf *old = std::cerr.rdbuf(nullptr);
    try { Raycast(v3(start), v3(end), v3(mn), v3(mx), &out); } catch (...) { std::cerr.rdbuf(old); throw; }
    std::cerr.rdbuf(old);
  } catch (const std::out_of_range &) { return -1; }
  long n = (long)out.size();
  for (long i = 0; i < n && i < cap; ++i) for (int k = 0; k < 3; ++k) out_xyz[3 * i + k] = out[i](k);
  return n;
}

// Restatement of Fiesta::RaycastMultithread + RaycastProcess, serial mode (Fiesta.h:194-303).
// xyz: n points (pcl::PointXYZ floats) in the sensor frame; T: row-major 4x4 transform_ (Fiesta.h:415-419);
// raycast_origin_ = T[:3,3]/T[3,3] (Fiesta.h:420).  Returns the number of rays actually cast, or -1 when the
// reference Raycast() threw.
long fiesta_ref_raycast_frame(void *h, const float *xyz, long n, const double T[16], double min_ray_length,
                              double max_ray_length) {
  RefMap *r = (RefMap *)h;
  fiesta::ESDFMap *map = r->map;
  const double res = r->resolution;
  const Eigen::Vector3d origin(T[3] / T[15], T[7] / T[15], T[11] / T[15]);
  const Eigen::Vector3d half(0.5, 0.5, 0.5);
  const int tt = (int)(++r->tot);                                       // Fiesta.h:287
  long cast = 0;
  std::vector<Eigen::Vector3d> output;
  for (long idx = 0; idx < n; ++idx) {                                  // Fiesta.h:196 (serial: one part = all points)
    const float px = xyz[3 * idx], py = xyz[3 * idx + 1], pz = xyz[3 * idx + 2];
    if (std::isnan(px) || std::isnan(py) || std::isnan(pz)) continue;  // :202
    double tmp[4];
    for (int row = 0; row < 4; ++row)                                   // :204  transform_ * (x,y,z,1)
      tmp[row] = ((T[4 * row] * (double)px + T[4 * row + 1] * (double)py) + T[4 * row + 2] * (double)pz) + T[4 * row + 3] * 1.0;
    Eigen::Vector3d point = Eigen::Vector3d(tmp[0], tmp[1], tmp[2]) / tmp[3];  // :205
    int tmp_idx;
    double length = (point - origin).norm();                            // :208
    if (length < min_ray_length) continue;                              // :209
    else if (length > max_ray_length) {                                 // :211-213
      point = (point - origin) / length * max_ray_length + origin;
      tmp_idx = map->SetOccupancy(point, 0);
    } else {
      tmp_idx = map->SetOccupancy(point, 1);                            // :215
    }
    if (tmp_idx != -10000 && tmp_idx >= 0 && tmp_idx < map->grid_total_size_) {  // :221-231 endpoint dedupe (+ index guard)
      if (r->set_occ[tmp_idx] == tt) continue;
      else r->set_occ[tmp_idx] = tt;
    }
    if (raycast_would_hang(origin / res, point / res, r->l_cornor / res, r->r_cornor / res)) { ++r->hung; continue; }
    try {
      std::streambuf *old = std::cerr.rdbuf(nullptr);
      try { Raycast(origin / res, point / res, r->l_cornor / res, r->r_cornor / res, &output); }  // :233-237
      catch (...) { std::cerr.rdbuf(old); throw; }
      std::cerr.rdbuf(old);
    } catch (const std::out_of_range &) { return -1; }
    ++cast;
    int cnt = 0;
    for (int i = (int)output.size() - 2; i >= 0; i--) {                 // :239 skips the last voxel
      Eigen::Vector3d c = (output[i] + half) * res;                     // :240
      length = (c - origin).norm();
      if (length < min_ray_length) break;                               // :243
      if (length > max_ray_length) continue;                            // :245
      int fi = map->SetOccupancy(c, 0);                                 // :248
      if (fi != -10000 && fi >= 0 && fi < map->grid_total_size_) {     // :253-275
        if (r->set_free[fi] == tt) {
          if (++cnt >= 1) { cnt = 0; break; }
        } else {
          r->set_free[fi] = tt;
          cnt = 0;
        }
      }
    }
  }
  return cast;
}

}  // extern "C"
