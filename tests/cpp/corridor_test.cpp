// CPU driver of fiesta_b200/csrc/fb_corridor.h for tests/test_corridor_oracle.py: the sequential rule with the traversability of
// fb_seg_blocks evaluated voxel by voxel.
//
// stdin: gx gy gz / origin[3] res (hex floats) / nrec rec... (device layout, z pitch rounded up to 4) / clearance flags /
// L lo[3] hi[3] / max_steps[3] / then a mode word:
//   inflate  n / per seed: lo[3] hi[3]          -> per seed "status lo[3] hi[3]"
//   paths    n_paths / per path: len and len * 3 ints -> per path "status n_boxes blocked_at" and then per box "lo[3] hi[3] first"
// and finally "stats boxes tested grown".
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../fiesta_b200/csrc/fb_corridor.h"

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

struct Seq {
  const FbGeom *g;
  const uint32_t *rec;
  double r;
  bool unk;
  int L_lo[3], L_hi[3];
  const int *P = nullptr;
  int n = 0;
  std::vector<int> out;        // per box: lo[3] hi[3] first

  bool traversable(int x, int y, int z) const {
    const int v[3] = {x, y, z};
    if (!fb_corr_inside(v, L_lo, L_hi)) return false;
    double d;
    return !fb_seg_blocks(*g, rec, v, r, unk, d);
  }
  bool box_free(const int *lo, const int *hi) const {
    for (int x = lo[0]; x <= hi[0]; ++x)
      for (int y = lo[1]; y <= hi[1]; ++y)
        for (int z = lo[2]; z <= hi[2]; ++z)
          if (!traversable(x, y, z)) return false;
    return true;
  }
  void vox(int i, int *v) const { for (int k = 0; k < 3; ++k) v[k] = P[3 * i + k]; }
  bool any_outside(const int *lo, const int *hi) const {
    for (int i = 0; i < n; ++i)
      if (!fb_corr_inside(P + 3 * i, lo, hi)) return true;
    return false;
  }
  int next_outside(int j, const int *lo, const int *hi) const {
    for (int i = j + 1; i < n; ++i)
      if (!fb_corr_inside(P + 3 * i, lo, hi)) return i;
    return n;
  }
  void emit(int, const int *lo, const int *hi, int j) {
    for (int k = 0; k < 3; ++k) out.push_back(lo[k]);
    for (int k = 0; k < 3; ++k) out.push_back(hi[k]);
    out.push_back(j);
  }
};

int main() {
  FbGeom g = {};
  g.gx = (int)rdi(); g.gy = (int)rdi(); g.gz = (int)rdi();
  g.pz = (g.gz + 3) & ~3; g.gyz = g.gy * g.gz;
  for (int k = 0; k < 3; ++k) g.origin[k] = rd();
  g.res = rd(); g.res_inv = 1 / g.res;
  const long long nrec = rdi();
  std::vector<uint32_t> rec((size_t)nrec);
  for (uint32_t &x : rec) x = (uint32_t)rdi();
  Seq acc;
  acc.g = &g; acc.rec = rec.data();
  acc.r = rd();
  acc.unk = (rdi() & 1) != 0;
  for (int k = 0; k < 3; ++k) acc.L_lo[k] = (int)rdi();
  for (int k = 0; k < 3; ++k) acc.L_hi[k] = (int)rdi();
  int ms[3];
  for (int k = 0; k < 3; ++k) ms[k] = (int)rdi();
  char mode[16];
  if (std::scanf("%15s", mode) != 1) return 3;
  FbCorrCount c{0, 0};
  unsigned long long boxes = 0;
  if (!std::strcmp(mode, "inflate")) {
    const long long n = rdi();
    for (long long i = 0; i < n; ++i) {
      int lo[3], hi[3];
      for (int k = 0; k < 3; ++k) lo[k] = (int)rdi();
      for (int k = 0; k < 3; ++k) hi[k] = (int)rdi();
      const int st = fb_corr_seed(acc, acc.L_lo, acc.L_hi, ms, lo, hi, c);
      boxes += st == FB_CORR_OK;
      if (st != FB_CORR_OK) for (int k = 0; k < 3; ++k) lo[k] = hi[k] = -1;
      std::printf("%d %d %d %d %d %d %d\n", st, lo[0], lo[1], lo[2], hi[0], hi[1], hi[2]);
    }
  } else if (!std::strcmp(mode, "paths")) {
    const long long np = rdi();
    for (long long p = 0; p < np; ++p) {
      std::vector<int> P((size_t)(3 * rdi()));
      for (int &x : P) x = (int)rdi();
      acc.P = P.data();
      acc.n = (int)(P.size() / 3);
      acc.out.clear();
      int nb, bl;
      const int st = fb_corr_chain(acc, acc.n, acc.L_lo, acc.L_hi, ms, &nb, &bl, c);
      boxes += (unsigned long long)nb;
      std::printf("%d %d %d\n", st, nb, bl);
      for (int k = 0; k < nb; ++k) {
        const int *b = &acc.out[(size_t)(7 * k)];
        std::printf("%d %d %d %d %d %d %d\n", b[0], b[1], b[2], b[3], b[4], b[5], b[6]);
      }
    }
  } else {
    return 3;
  }
  std::printf("stats %llu %lld %lld\n", boxes, c.tested, c.grown);
  return 0;
}
