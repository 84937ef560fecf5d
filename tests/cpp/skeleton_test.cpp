// CPU driver of fiesta_b200/csrc/fb_skel.h for tests/test_skeleton_oracle.py.
//
// `skeleton_test simple`: fb_sk_simple against an independent breadth-first search on every one of the 2^26 neighbourhoods: T26
//   counts the 26-components of the foreground neighbours, T6 the 6-components of the background in N18 that hold a face neighbour,
//   both from explicit coordinates.  Prints "configs <n> simple <k> mismatches <m>".
// `skeleton_test anchor`: reads n, then n lines "vx vy vz ox oy oz ux uy uz px py pz max_cos" (max_cos as a hex float) and prints
//   fb_sk_anchor_pair for each as one line of 0/1 characters.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include "../../fiesta_b200/csrc/fb_skel.h"

static int cx[27], cy[27], cz[27];
static unsigned adj26[27], adj6[27];

// Components of `set` (a 27-bit mask) under the adjacency table, counting only those that meet `must` (all when must == set).
static int components(unsigned set, const unsigned *adj, unsigned must) {
  int n = 0;
  unsigned left = set;
  int queue[27];
  while (left) {
    const int s = __builtin_ctz(left);
    unsigned comp = 1u << s;
    left &= ~comp;
    int head = 0, tail = 0;
    queue[tail++] = s;
    while (head < tail) {
      const int u = queue[head++];
      unsigned nb = adj[u] & left;
      while (nb) {
        const int w = __builtin_ctz(nb);
        nb &= nb - 1;
        left &= ~(1u << w);
        comp |= 1u << w;
        queue[tail++] = w;
      }
    }
    if (comp & must) ++n;
  }
  return n;
}

int main(int argc, char **argv) {
  if (argc < 2) return 2;
  for (int e = 0; e < 27; ++e) { cx[e] = e / 9 - 1; cy[e] = e / 3 % 3 - 1; cz[e] = e % 3 - 1; }
  for (int a = 0; a < 27; ++a)
    for (int b = 0; b < 27; ++b) {
      if (a == b) continue;
      const int dx = std::abs(cx[a] - cx[b]), dy = std::abs(cy[a] - cy[b]), dz = std::abs(cz[a] - cz[b]);
      if (dx <= 1 && dy <= 1 && dz <= 1) adj26[a] |= 1u << b;
      if (dx + dy + dz == 1) adj6[a] |= 1u << b;
    }
  if (!std::strcmp(argv[1], "simple")) {
    unsigned n18 = 0, n6 = 0;
    for (int e = 0; e < 27; ++e) {
      const int k = std::abs(cx[e]) + std::abs(cy[e]) + std::abs(cz[e]);
      if (k >= 1 && k <= 2) n18 |= 1u << e;
      if (k == 1) n6 |= 1u << e;
    }
    long long simple = 0, bad = 0;
    for (unsigned c = 0; c < (1u << 26); ++c) {
      const unsigned code = (c & 0x1fffu) | ((c >> 13) << 14);           // the 26 neighbours around bit 13
      const unsigned fg = code, bg = ~code & n18;
      const bool want = components(fg, adj26, fg) == 1 && components(bg, adj6, n6 & bg) == 1;
      const bool got = fb_sk_simple(code | FB_SK_CENTER) && fb_sk_simple(code);   // the centre bit is ignored
      simple += want;
      if (want != got && bad++ < 5) std::fprintf(stderr, "mismatch at code %07x: want %d\n", code, (int)want);
    }
    std::printf("configs %lld simple %lld mismatches %lld\n", 1ll << 26, simple, bad);
    return bad != 0;
  }
  if (!std::strcmp(argv[1], "anchor")) {
    long long n;
    if (std::scanf("%lld", &n) != 1) return 3;
    for (long long i = 0; i < n; ++i) {
      int v[3], o[3], u[3], p[3];
      char buf[64];
      for (int *a : {v, o, u, p})
        for (int k = 0; k < 3; ++k)
          if (std::scanf("%d", &a[k]) != 1) return 3;
      if (std::scanf("%63s", buf) != 1) return 3;
      std::putchar(fb_sk_anchor_pair(v, o, u, p, std::strtod(buf, nullptr)) ? '1' : '0');
    }
    std::putchar('\n');
    return 0;
  }
  return 2;
}
