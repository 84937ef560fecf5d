// CPU driver of fiesta_b200/csrc/fb_mesh.h for tests/test_mesh_oracle.py.  Floating-point values are read and written as hex floats.
//
// `mesh_test order`: the 12 cell edges (fb_mesh_cell_edge: axis, lower corner, upper corner) on one line, then for a = 0..2 and
//   v_blocks = 0, 1 the quad's four cell offsets (fb_mesh_quad) on one line each.
// `mesh_test t`: reads n, then n lines "has_u du has_w dw r"; prints fb_mesh_t for each, one per line.
// `mesh_test vertex`: reads n, then n lines "cx cy cz blk0..blk7 has0..has7 d0..d7 r res ox oy oz"; prints the three float32
//   coordinates of fb_mesh_vertex, one vertex per line.
// `mesh_test split`: reads n, then n lines of 12 float32 coordinates p0 p1 p2 p3 and 4 vertex ids; prints fb_mesh_split02 and the six
//   ids of fb_mesh_tris, one quad per line.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../../fiesta_b200/csrc/fb_mesh.h"

static bool rd(double *x) {
  char buf[64];
  if (std::scanf("%63s", buf) != 1) return false;
  *x = std::strtod(buf, nullptr);
  return true;
}
static bool rdi(int *x) { return std::scanf("%d", x) == 1; }

int main(int argc, char **argv) {
  if (argc < 2) return 2;
  if (!std::strcmp(argv[1], "order")) {
    for (int e = 0; e < 12; ++e) {
      int a, k0, k1;
      fb_mesh_cell_edge(e, &a, &k0, &k1);
      std::printf("%d %d %d ", a, k0, k1);
    }
    std::printf("\n");
    for (int a = 0; a < 3; ++a)
      for (int vb = 0; vb < 2; ++vb) {
        int off[4][3];
        fb_mesh_quad(a, vb != 0, off);
        for (int i = 0; i < 4; ++i) std::printf("%d %d %d ", off[i][0], off[i][1], off[i][2]);
        std::printf("\n");
      }
    return 0;
  }
  long long n;
  if (std::scanf("%lld", &n) != 1) return 3;
  if (!std::strcmp(argv[1], "t")) {
    for (long long i = 0; i < n; ++i) {
      int hu, hw;
      double du, dw, r;
      if (!rdi(&hu) || !rd(&du) || !rdi(&hw) || !rd(&dw) || !rd(&r)) return 3;
      std::printf("%a\n", fb_mesh_t(hu != 0, du, hw != 0, dw, r));
    }
    return 0;
  }
  if (!std::strcmp(argv[1], "vertex")) {
    for (long long i = 0; i < n; ++i) {
      int c[3], b;
      bool blk[8], has[8];
      double d[8], r, res, org[3];
      for (int k = 0; k < 3; ++k) if (!rdi(&c[k])) return 3;
      for (int k = 0; k < 8; ++k) { if (!rdi(&b)) return 3; blk[k] = b != 0; }
      for (int k = 0; k < 8; ++k) { if (!rdi(&b)) return 3; has[k] = b != 0; }
      for (int k = 0; k < 8; ++k) if (!rd(&d[k])) return 3;
      if (!rd(&r) || !rd(&res) || !rd(&org[0]) || !rd(&org[1]) || !rd(&org[2])) return 3;
      float p[3];
      fb_mesh_vertex(c, blk, has, d, r, res, org, p);
      std::printf("%a %a %a\n", (double)p[0], (double)p[1], (double)p[2]);
    }
    return 0;
  }
  if (!std::strcmp(argv[1], "split")) {
    for (long long i = 0; i < n; ++i) {
      float p[4][3];
      int32_t q[4], t[6];
      for (int j = 0; j < 4; ++j)
        for (int k = 0; k < 3; ++k) {
          double x;
          if (!rd(&x)) return 3;
          p[j][k] = (float)x;                                               // exact: the values are float32
        }
      for (int j = 0; j < 4; ++j) if (!rdi(&q[j])) return 3;
      const bool s = fb_mesh_split02(p[0], p[1], p[2], p[3]);
      fb_mesh_tris(q, s, t);
      std::printf("%d %d %d %d %d %d %d\n", (int)s, t[0], t[1], t[2], t[3], t[4], t[5]);
    }
    return 0;
  }
  return 2;
}
