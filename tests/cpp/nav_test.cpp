// CPU driver of fiesta_b200/csrc/fb_nav.h for tests/test_nav_oracle.py: reads a box field and starts on stdin, runs the path rule
// the kernel runs (fb_nav_path) and prints each result (floats as hex, so that Python compares bits).
//
// stdin:  Bx By Bz lox loy loz / w1 w2 w3 / Bx*By*Bz field values / nstart max_len / 3 box-local ints per start
// stdout: per start "status len cost" then len lines "x y z" (grid voxels)
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../fiesta_b200/csrc/fb_nav.h"

static double rd() {
  char buf[64];
  if (std::scanf("%63s", buf) != 1) std::exit(3);
  return std::strtod(buf, nullptr);   // hex floats and "inf": exact
}

int main() {
  FbNavBox b;
  for (int k = 0; k < 3; ++k) b.n[k] = (int)rd();
  for (int k = 0; k < 3; ++k) b.lo[k] = (int)rd();
  double w[3];
  for (int k = 0; k < 3; ++k) w[k] = rd();
  std::vector<double> D((size_t)b.n[0] * b.n[1] * b.n[2]);
  for (double &d : D) d = rd();
  const int n = (int)rd(), max_len = (int)rd();
  std::vector<int32_t> vox((size_t)max_len * 3);
  for (int i = 0; i < n; ++i) {
    int v[3];
    for (int k = 0; k < 3; ++k) v[k] = (int)rd();
    int32_t len;
    double cost;
    const int st = fb_nav_path(b, D.data(), w, v, max_len, vox.data(), &len, &cost);
    std::printf("%d %d %a\n", st, (int)len, cost);
    for (int j = 0; j < len; ++j) std::printf("%d %d %d\n", vox[3 * j], vox[3 * j + 1], vox[3 * j + 2]);
  }
  return 0;
}
