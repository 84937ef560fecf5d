// CPU driver of fiesta_b200/csrc/fb_segment.h for tests/test_segment_traversal.py.  Reads a grid, its packed records (device layout)
// and segments on stdin, and prints for every segment the lattice endpoints, the sequential walk (voxel and entry parameter), whether
// the slab-by-slab walks the kernel's lanes take concatenate to the same sequence, whether the kernel's sweep-of-32 combination of
// per-slab results gives fb_seg_check's result, and that result (floats as hex, so that Python compares bits).
//
// stdin:  gx gy gz / origin[3] res / min_range[3] max_range[3] / nrec rec... / nseg clearance flags / 6 values per segment
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../fiesta_b200/csrc/fb_segment.h"

struct Collect {
  std::vector<long long> out;   // x y z tn td per voxel
  bool operator()(const int *v, long long tn, long long td) {
    out.insert(out.end(), {(long long)v[0], (long long)v[1], (long long)v[2], tn, td});
    return false;
  }
};

// same voxels entered at the same parameters (a parameter may come as n / den of different axes: compare the rationals)
static bool same_walk(const std::vector<long long> &a, const std::vector<long long> &b) {
  if (a.size() != b.size()) return false;
  for (size_t k = 0; k < a.size(); k += 5)
    if (a[k] != b[k] || a[k + 1] != b[k + 1] || a[k + 2] != b[k + 2] || a[k + 3] * b[k + 4] != b[k + 3] * a[k + 4]) return false;
  return true;
}

static double rd() {
  char buf[64];
  if (std::scanf("%63s", buf) != 1) std::exit(3);
  return std::strtod(buf, nullptr);   // hex floats: exact
}

int main() {
  FbGeom g = {};
  g.gx = (int)rd(); g.gy = (int)rd(); g.gz = (int)rd();
  g.pz = (g.gz + 3) & ~3; g.gyz = g.gy * g.gz;
  for (int k = 0; k < 3; ++k) g.origin[k] = rd();
  g.res = rd(); g.res_inv = 1 / g.res;
  for (int k = 0; k < 3; ++k) g.min_range[k] = rd();
  for (int k = 0; k < 3; ++k) g.max_range[k] = rd();
  const long long nrec = (long long)rd();
  std::vector<uint32_t> rec((size_t)nrec);
  for (long long i = 0; i < nrec; ++i) { unsigned long u; if (std::scanf("%lu", &u) != 1) return 3; rec[(size_t)i] = (uint32_t)u; }
  const long long nseg = (long long)rd();
  const double r = rd();
  const bool unk = ((int)rd() & 1) != 0;
  for (long long i = 0; i < nseg; ++i) {
    double ab[6];
    for (int k = 0; k < 6; ++k) ab[k] = rd();
    int32_t st; int64_t idx; double t, md;
    fb_seg_check(g, rec.data(), ab, r, unk, &st, &idx, &t, &md);
    FbSeg s;
    if (!fb_seg_setup(g, ab, s)) {
      std::printf("seg out\n");
    } else {
      Collect seq, slabs;
      fb_seg_walk(s, 0, s.nslabs, seq);
      for (int j = 0; j < s.nslabs; ++j) fb_seg_walk(s, j, j + 1, slabs);
      // the kernel's combination: sweeps of 32 slabs, first blocking slab, minimum over the slabs up to it
      double run = FIESTA_INFINITY;
      int32_t kst = 0; int64_t kidx = -1; double kt = nan(""), kmd = 0;
      bool blocked = false;
      for (int base = 0; base < s.nslabs && !blocked; base += 32) {
        std::vector<FbSegScan> lanes;
        int first = 32;
        for (int l = 0; l < 32; ++l) {
          FbSegScan sc = fb_seg_scan(g, rec.data(), r, unk);
          if (base + l < s.nslabs) fb_seg_walk(s, base + l, base + l + 1, sc);
          if (sc.hit && first == 32) first = l;
          lanes.push_back(sc);
        }
        for (int l = 0; l <= first && l < 32; ++l) run = std::fmin(run, lanes[(size_t)l].min_d);
        blocked = first < 32;
        if (blocked) fb_seg_store(g, lanes[(size_t)first], run, &kst, &kidx, &kt, &kmd);
      }
      if (!blocked) fb_seg_store(g, fb_seg_scan(g, rec.data(), r, false), run, &kst, &kidx, &kt, &kmd);
      const bool kernel_equal = kst == st && kidx == idx && (kt == t || (kt != kt && t != t)) && kmd == md;
      std::printf("seg ok %lld %lld %lld %lld %lld %lld %d %d %d %zu\n", s.qa[0], s.qa[1], s.qa[2], s.qb[0], s.qb[1], s.qb[2], s.nslabs,
                  (int)same_walk(slabs.out, seq.out), (int)kernel_equal, seq.out.size() / 5);
      for (size_t k = 0; k < seq.out.size(); k += 5)
        std::printf("v %lld %lld %lld %lld %lld\n", seq.out[k], seq.out[k + 1], seq.out[k + 2], seq.out[k + 3], seq.out[k + 4]);
    }
    std::printf("res %d %lld %a %a\n", (int)st, (long long)idx, t, md);
  }
  return 0;
}
