// CPU driver of fiesta_b200/csrc/fb_frontier.h for tests/test_frontier_oracle.py: reads a grid's records and log-odds on stdin,
// evaluates the frontier predicate the kernel evaluates (fb_fr_is_frontier) for every voxel of a box, prints the distances
// export_distance() would read, and evaluates the centroid expression (floats as hex, so that Python compares bits).
//
// stdin:  gx gy gz res / origin xyz / l_occ r / box lo xyz hi xyz / gx*gy*gz records (reference order) / as many log-odds /
//         n / n lines "s n" (sum, count) for the centroid on axis 0
// stdout: one line of gx*gy*gz distances, one line of box-order 0/1 flags, n centroid lines
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../fiesta_b200/csrc/fb_frontier.h"

static double rd() {
  char buf[64];
  if (std::scanf("%63s", buf) != 1) std::exit(3);
  return std::strtod(buf, nullptr);   // hex floats: exact
}
static long long rdi() {
  long long v;
  if (std::scanf("%lld", &v) != 1) std::exit(3);
  return v;
}

int main() {
  FbGeom g{};
  g.gx = (int)rdi(); g.gy = (int)rdi(); g.gz = (int)rdi();
  g.pz = (g.gz + 3) / 4 * 4;                       // the device's padded pitch
  g.gyz = g.gy * g.gz;
  g.res = rd();
  for (int k = 0; k < 3; ++k) g.origin[k] = rd();
  const double l_occ = rd(), r = rd();
  int lo[3], hi[3];
  for (int k = 0; k < 3; ++k) lo[k] = (int)rdi();
  for (int k = 0; k < 3; ++k) hi[k] = (int)rdi();
  const size_t P = (size_t)g.gx * g.gy * g.pz;
  std::vector<uint32_t> rec(P, 0u);
  std::vector<double> occ(P, 0.0);
  for (int x = 0; x < g.gx; ++x)
    for (int y = 0; y < g.gy; ++y)
      for (int z = 0; z < g.gz; ++z) rec[fb_ii(g, x, y, z)] = (uint32_t)rdi();
  for (int x = 0; x < g.gx; ++x)
    for (int y = 0; y < g.gy; ++y)
      for (int z = 0; z < g.gz; ++z) occ[fb_ii(g, x, y, z)] = rd();
  for (int x = 0; x < g.gx; ++x)
    for (int y = 0; y < g.gy; ++y)
      for (int z = 0; z < g.gz; ++z) std::printf("%a ", fb_record_distance(rec[fb_ii(g, x, y, z)], x, y, z, g.res));
  std::printf("\n");
  for (int x = lo[0]; x <= hi[0]; ++x)
    for (int y = lo[1]; y <= hi[1]; ++y)
      for (int z = lo[2]; z <= hi[2]; ++z) {
        const int v[3] = {x, y, z};
        std::printf("%d", fb_fr_is_frontier(g, rec.data(), occ.data(), l_occ, v, r) ? 1 : 0);
      }
  std::printf("\n");
  const long long n = rdi();
  for (long long i = 0; i < n; ++i) {
    const long long s = rdi(), c = rdi();
    std::printf("%a\n", fb_fr_centroid(s, c, g.res, g.origin[0]));
  }
  return 0;
}
