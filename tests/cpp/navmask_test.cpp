// CPU driver of fb_nav_move_bits (fiesta_b200/csrc/fb_nav.h) for tests/test_nav_matrix_oracle.py: reads a box's traversable flags
// on stdin and prints each voxel's move mask as k_navm_mask computes it (neighbours outside the box count as blocked).
//
// stdin:  Bx By Bz / Bx*By*Bz flags (0 / 1, box index order)
// stdout: one mask per voxel, box index order
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../fiesta_b200/csrc/fb_nav.h"

int main() {
  FbNavBox b{};
  for (int k = 0; k < 3; ++k)
    if (std::scanf("%d", &b.n[k]) != 1) return 3;
  std::vector<int> T((size_t)b.n[0] * b.n[1] * b.n[2]);
  for (int &t : T)
    if (std::scanf("%d", &t) != 1) return 3;
  for (int x = 0; x < b.n[0]; ++x)
    for (int y = 0; y < b.n[1]; ++y)
      for (int z = 0; z < b.n[2]; ++z) {
        unsigned nb = 0;
        for (int e = 0; e < 27; ++e) {
          int d[3];
          fb_nav_dir(e, d);
          if (fb_nav_in_box(b, x + d[0], y + d[1], z + d[2]) && T[fb_nav_idx(b, x + d[0], y + d[1], z + d[2])]) nb |= 1u << e;
        }
        std::printf("%u\n", fb_nav_move_bits(nb));
      }
  return 0;
}
