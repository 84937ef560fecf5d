// CPU driver of fiesta_b200/csrc/fb_view.h for tests/test_viewpoint_oracle.py (floats as hex, so that Python compares bits).
//
// stdin starts with a mode word:
//   pairs   res / origin[3] / n_orient / 9 * n_orient matrix entries / max_range tan_h tan_v / npairs / per pair: vx vy vz px py pz
//           -> per pair "in_range mask" (the mask is printed whether or not the pair is in range)
//   chunks  n / n chunk sizes (members of the candidate's cluster, 0 for a candidate that is not scored)
//           -> the total, then per chunk w "i lo hi": the candidate fb_view_find gives and the member range [lo, hi) of its lanes
//   score   gx gy gz / origin[3] res / min_range[3] max_range[3] / nrec rec... (device layout) / clearance flags /
//           n_orient / 9 * n_orient entries / max_range tan_h tan_v / K / K cluster sizes / the members, 3 ints each, cluster by
//           cluster / n / per candidate: cluster px py pz
//           -> per candidate "status score_0 .. score_{n_orient-1}", then "stats scored walked visible": the kernel's per-lane
//           logic run sequentially over the chunk list
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../fiesta_b200/csrc/fb_view.h"

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

static void read_sensor(std::vector<double> &R, int &n_orient, double &range, double &tan_h, double &tan_v) {
  n_orient = (int)rdi();
  R.resize((size_t)9 * n_orient);
  for (double &x : R) x = rd();
  range = rd(); tan_h = rd(); tan_v = rd();
}

static int pairs() {
  FbGeom g = {};
  g.res = rd();
  for (int k = 0; k < 3; ++k) g.origin[k] = rd();
  std::vector<double> R;
  int n_orient;
  double range, tan_h, tan_v;
  read_sensor(R, n_orient, range, tan_h, tan_v);
  const long long np = rdi();
  for (long long i = 0; i < np; ++i) {
    int v[3];
    double p[3], c[3], d[3];
    for (int k = 0; k < 3; ++k) v[k] = (int)rdi();
    for (int k = 0; k < 3; ++k) p[k] = rd();
    fb_view_offset(g, v, p, c, d);
    std::printf("%d %u\n", (int)fb_view_in_range(d, range * range), fb_view_mask(R.data(), n_orient, d, tan_h, tan_v));
  }
  return 0;
}

static void scan(const std::vector<long long> &work, std::vector<long long> &first) {
  first.assign(work.size() + 1, 0);
  for (size_t i = 0; i < work.size(); ++i) first[i + 1] = first[i] + work[i];
}

static int chunks() {
  const long long n = rdi();
  std::vector<long long> size((size_t)n), work((size_t)n), first;
  for (long long i = 0; i < n; ++i) { size[(size_t)i] = rdi(); work[(size_t)i] = fb_view_chunks(size[(size_t)i]); }
  scan(work, first);
  const long long total = first[(size_t)n];
  std::printf("%lld\n", total);
  for (long long w = 0; w < total; ++w) {
    const long long i = fb_view_find(first.data(), n, w);
    const long long lo = (w - first[(size_t)i]) * FB_VIEW_CHUNK, hi = lo + FB_VIEW_CHUNK;
    std::printf("%lld %lld %lld\n", i, lo, hi < size[(size_t)i] ? hi : size[(size_t)i]);
  }
  return 0;
}

static int score() {
  FbGeom g = {};
  g.gx = (int)rdi(); g.gy = (int)rdi(); g.gz = (int)rdi();
  g.pz = (g.gz + 3) & ~3; g.gyz = g.gy * g.gz;
  for (int k = 0; k < 3; ++k) g.origin[k] = rd();
  g.res = rd(); g.res_inv = 1 / g.res;
  for (int k = 0; k < 3; ++k) g.min_range[k] = rd();
  for (int k = 0; k < 3; ++k) g.max_range[k] = rd();
  const long long nrec = rdi();
  std::vector<uint32_t> rec((size_t)nrec);
  for (uint32_t &r : rec) r = (uint32_t)rdi();
  const double clearance = rd();
  const bool unk = (rdi() & 1) != 0;
  std::vector<double> R;
  int n_orient;
  double range, tan_h, tan_v;
  read_sensor(R, n_orient, range, tan_h, tan_v);
  const long long K = rdi();
  std::vector<long long> size((size_t)K), moff((size_t)K + 1, 0);
  for (long long k = 0; k < K; ++k) { size[(size_t)k] = rdi(); moff[(size_t)k + 1] = moff[(size_t)k] + size[(size_t)k]; }
  std::vector<int> mem((size_t)(3 * moff[(size_t)K]));
  for (int &x : mem) x = (int)rdi();
  const long long n = rdi();
  std::vector<int> cl((size_t)n), status((size_t)n);
  std::vector<double> pos((size_t)(3 * n));
  std::vector<long long> work((size_t)n), first;
  unsigned long long scored = 0, walked = 0, visible = 0;
  for (long long i = 0; i < n; ++i) {
    cl[(size_t)i] = (int)rdi();
    for (int k = 0; k < 3; ++k) pos[(size_t)(3 * i + k)] = rd();
    status[(size_t)i] = fb_view_status(g, rec.data(), &pos[(size_t)(3 * i)], clearance);
    scored += status[(size_t)i] == 0;
    work[(size_t)i] = status[(size_t)i] == 0 ? fb_view_chunks(size[(size_t)cl[(size_t)i]]) : 0;
  }
  scan(work, first);
  std::vector<int> sc((size_t)(n * n_orient), 0);
  for (long long w = 0; w < first[(size_t)n]; ++w) {
    const long long i = fb_view_find(first.data(), n, w);
    const int c = cl[(size_t)i];
    for (int lane = 0; lane < FB_VIEW_CHUNK; ++lane) {
      const long long j = (w - first[(size_t)i]) * FB_VIEW_CHUNK + lane;
      if (j >= size[(size_t)c]) continue;
      const double *p = &pos[(size_t)(3 * i)];
      const int *v = &mem[(size_t)(3 * (moff[(size_t)c] + j))];
      double cc[3], d[3];
      fb_view_offset(g, v, p, cc, d);
      const unsigned mask = fb_view_in_range(d, range * range) ? fb_view_mask(R.data(), n_orient, d, tan_h, tan_v) : 0u;
      if (!mask) continue;
      ++walked;
      if (!fb_view_visible(g, rec.data(), p, cc, unk)) continue;
      ++visible;
      for (int o = 0; o < n_orient; ++o) sc[(size_t)(i * n_orient + o)] += (mask >> o) & 1u;
    }
  }
  for (long long i = 0; i < n; ++i) {
    std::printf("%d", status[(size_t)i]);
    for (int o = 0; o < n_orient; ++o) std::printf(" %d", sc[(size_t)(i * n_orient + o)]);
    std::printf("\n");
  }
  std::printf("stats %llu %llu %llu\n", scored, walked, visible);
  return 0;
}

int main() {
  char mode[16];
  if (std::scanf("%15s", mode) != 1) return 3;
  if (!std::strcmp(mode, "pairs")) return pairs();
  if (!std::strcmp(mode, "chunks")) return chunks();
  if (!std::strcmp(mode, "score")) return score();
  return 3;
}
