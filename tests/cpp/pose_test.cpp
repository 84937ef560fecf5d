// CPU driver of fiesta_b200/csrc/fb_pose.h for tests/test_pose_oracle.py (floats as hex, so that Python compares bits).
//
// stdin starts with a mode word:
//   touch  res / origin[3] / min_range[3] max_range[3] / h[3] / margin / n / per pose: 12 entries
//          -> per pose "valid lo0 lo1 lo2 hi0 hi1 hi2 count x y z ...": the candidate range and every voxel of the range widened by
//          `margin` on each side that fb_pose_touches accepts, in x, y, z loop order (only "0" for an invalid pose)
//   check  gx gy gz / origin[3] res / min_range[3] max_range[3] / nrec rec... (device layout) / h[3] / clearance flags / n /
//          per pose: 12 entries  -> per pose "status n_blocked hit_idx" from fb_pose_check
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../fiesta_b200/csrc/fb_pose.h"

static double rd() {
  char buf[64];
  if (std::scanf("%63s", buf) != 1) std::exit(3);
  return std::strtod(buf, nullptr);   // hex floats, nan, inf: exact
}
static long long rdi() {
  long long v;
  if (std::scanf("%lld", &v) != 1) std::exit(3);
  return v;
}
static void rd_ranges(FbGeom &g) {
  for (int k = 0; k < 3; ++k) g.min_range[k] = rd();
  for (int k = 0; k < 3; ++k) g.max_range[k] = rd();
}

static int touch() {
  FbGeom g = {};
  g.res = rd();
  for (int k = 0; k < 3; ++k) g.origin[k] = rd();
  rd_ranges(g);
  double h[3];
  for (double &x : h) x = rd();
  const int margin = (int)rdi();
  const long long n = rdi();
  for (long long i = 0; i < n; ++i) {
    double pose[12];
    for (double &x : pose) x = rd();
    if (!fb_pose_valid(g, pose)) { std::printf("0\n"); continue; }
    FbPose P;
    fb_pose_setup(g, pose, h, P);
    std::vector<int> hits;
    int v[3];
    for (v[0] = P.lo[0] - margin; v[0] < P.lo[0] + P.n[0] + margin; ++v[0])
      for (v[1] = P.lo[1] - margin; v[1] < P.lo[1] + P.n[1] + margin; ++v[1])
        for (v[2] = P.lo[2] - margin; v[2] < P.lo[2] + P.n[2] + margin; ++v[2])
          if (fb_pose_touches(g, P, v)) hits.insert(hits.end(), v, v + 3);
    std::printf("1 %d %d %d %d %d %d %zu", P.lo[0], P.lo[1], P.lo[2], P.lo[0] + P.n[0] - 1, P.lo[1] + P.n[1] - 1, P.lo[2] + P.n[2] - 1,
                hits.size() / 3);
    for (int x : hits) std::printf(" %d", x);
    std::printf("\n");
  }
  return 0;
}

static int check() {
  FbGeom g = {};
  g.gx = (int)rdi(); g.gy = (int)rdi(); g.gz = (int)rdi();
  g.pz = (g.gz + 3) & ~3; g.gyz = g.gy * g.gz;
  for (int k = 0; k < 3; ++k) g.origin[k] = rd();
  g.res = rd(); g.res_inv = 1 / g.res;
  rd_ranges(g);
  const long long nrec = rdi();
  std::vector<uint32_t> rec((size_t)nrec);
  for (uint32_t &r : rec) r = (uint32_t)rdi();
  double h[3];
  for (double &x : h) x = rd();
  const double clearance = rd();
  const bool unk = (rdi() & 1) != 0;
  const long long n = rdi();
  for (long long i = 0; i < n; ++i) {
    double pose[12];
    for (double &x : pose) x = rd();
    int32_t st, nb;
    int64_t idx;
    fb_pose_check(g, rec.data(), pose, h, clearance, unk, &st, &nb, &idx);
    std::printf("%d %d %lld\n", st, nb, (long long)idx);
  }
  return 0;
}

int main() {
  char mode[16];
  if (std::scanf("%15s", mode) != 1) return 3;
  if (!std::strcmp(mode, "touch")) return touch();
  if (!std::strcmp(mode, "check")) return check();
  return 3;
}
