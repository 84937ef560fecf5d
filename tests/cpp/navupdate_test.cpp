// CPU driver of the field update's support predicate in fiesta_b200/csrc/fb_nav.h for tests/test_nav_update_oracle.py: reads an
// old box field and prints, per voxel, the tight-support mask fb_nav_support_bits gives from its 3x3x3 neighbourhood (-1 outside
// the box, as the kernel stages it).
//
// stdin:  Bx By Bz / w1 w2 w3 / Bx*By*Bz field values (hex floats, inf)
// stdout: one line per voxel in box order: the 27-bit mask (bit k: neighbour fb_nav_dir(k) is a tight support)
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../fiesta_b200/csrc/fb_nav.h"

static double rd() {
  char buf[64];
  if (std::scanf("%63s", buf) != 1) std::exit(3);
  return std::strtod(buf, nullptr);
}

int main() {
  FbNavBox b{};
  for (int k = 0; k < 3; ++k) b.n[k] = (int)rd();
  double w[3];
  for (int k = 0; k < 3; ++k) w[k] = rd();
  std::vector<double> D((size_t)b.n[0] * b.n[1] * b.n[2]);
  for (double &d : D) d = rd();
  for (int x = 0; x < b.n[0]; ++x)
    for (int y = 0; y < b.n[1]; ++y)
      for (int z = 0; z < b.n[2]; ++z) {
        double d27[27];
        for (int e = 0; e < 27; ++e) {
          int d[3];
          fb_nav_dir(e, d);
          d27[e] = fb_nav_in_box(b, x + d[0], y + d[1], z + d[2]) ? D[fb_nav_idx(b, x + d[0], y + d[1], z + d[2])] : FB_NAV_BLOCKED;
        }
        std::printf("%u\n", fb_nav_support_bits(d27, w));
      }
  return 0;
}
