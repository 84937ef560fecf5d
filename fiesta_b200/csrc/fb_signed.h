// fiesta_b200 -- signed distance of a voxel box (include/fiesta_b200.h, DESIGN.md §3.13): the per-voxel classification, the
// signed value S, the 1-D distance of the first pass and one line of the lower-envelope passes.  Plain C++: fb_signed.cu runs it
// on the device and tests/cpp/signed_test.cpp compiles the same source with g++.
//
// Box layout: as fb_nav.h, index ((x-lo.x)*By + (y-lo.y))*Bz + (z-lo.z), z fastest.  The field keeps one int32 q per box voxel:
// 0 on a non-obstacle, the exact squared Euclidean distance (voxel units) to the nearest non-obstacle voxel of the box on an
// obstacle, FB_SIGNED_NONE on an obstacle when the box holds no non-obstacle voxel.  q <= 2045^2 + 2 * 1023^2 < 2^31.
#ifndef FB_SIGNED_H_
#define FB_SIGNED_H_
#include <math.h>
#include <stdint.h>
#include "fb_record.h"

#define FB_SIGNED_NONE 0x7fffffff      // no non-obstacle voxel in reach: the line (passes 1, 2) or the box (final q)
#define FB_SIGNED_SBITS 11             // envelope stack entry: F << 11 | s, s < 2046 (FB_MAX_GX), F < 2^21 (see fb_signed_envelope)

struct FbSignedBox {
  int lo[3], n[3];
};

// An obstacle voxel is one whose distance reads exactly 0: its closest obstacle is itself.  The record then is fb_pack of the
// voxel's own coordinates with bit 31 clear (bit 31 set is EXACT mode's local-map reset, which reads +10000).
FB_HD bool fb_signed_obstacle(uint32_t c, int x, int y, int z) { return c == fb_pack(x, y, z); }

// S of an obstacle voxel with q > 0; each fp64 operation rounded on its own.  q == 1 (a surface voxel) gives +0.0.
FB_HD double fb_signed_depth(int32_t q, double res) {
  return q == FB_SIGNED_NONE ? -INFINITY : (1.0 - sqrt((double)q)) * res;
}

FB_HD int32_t fb_signed_ld(const int32_t *p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// The corner read of the signed queries (fb_query_distance / fb_query_trilinear, fb_record.h): S inside the box, the records'
// GetDistance(Vector3i) outside it and on the box's non-obstacles.
struct FbSignedRead {
  const FbGeom &g;
  const uint32_t *cobs;
  const int32_t *q;
  FbSignedBox b;
  FB_HD double operator()(int x, int y, int z) const {
    const int bx = x - b.lo[0], by = y - b.lo[1], bz = z - b.lo[2];
    if (bx >= 0 && bx < b.n[0] && by >= 0 && by < b.n[1] && bz >= 0 && bz < b.n[2]) {
      const int32_t v = fb_signed_ld(&q[((long long)bx * b.n[1] + by) * b.n[2] + bz]);
      if (v != 0) return fb_signed_depth(v, g.res);
    }
    return fb_get_distance_vox(g, cobs, x, y, z);
  }
};

// Pass 1, along z.  A line is cut into 32-voxel chunks; `mask` has bit l set when voxel 32 c + l of chunk c is a non-obstacle,
// prev_end is the last non-obstacle before chunk c (-1 if none) and next_start the first one after it (FB_SIGNED_NONE if none).
// Returns the squared distance from voxel 32 c + l to the nearest non-obstacle of the line, or FB_SIGNED_NONE.
FB_HD int32_t fb_signed_1d(uint32_t mask, int c, int l, int prev_end, int next_start) {
  const int z = 32 * c + l;
  const uint32_t below = mask & (0xffffffffu >> (31 - l));               // bits 0..l
  const uint32_t above = mask >> l;                                      // bits l..31, shifted to 0
  int p = prev_end, n = next_start;
  if (below) {
    int hb = 31;
    while (!((below >> hb) & 1u)) --hb;
    p = 32 * c + hb;
  }
  if (above) {
    int lb = 0;
    while (!((above >> lb) & 1u)) ++lb;
    n = z + lb;
  }
  int d = FB_SIGNED_NONE;
  if (p >= 0) d = z - p;
  if (n != FB_SIGNED_NONE && n - z < d) d = n - z;
  return d == FB_SIGNED_NONE ? FB_SIGNED_NONE : d * d;
}

// floor((u^2 - s^2 + Fu - Fs) / (2 (u - s))) for s < u: the last position at which the parabola of s is not above that of u.
FB_HD int fb_signed_sep(int s, int32_t Fs, int u, int32_t Fu) {
  const int num = (u * u - s * s) + (Fu - Fs), den = 2 * (u - s);
  return num >= 0 ? num / den : -((-num + den - 1) / den);
}
FB_HD uint32_t fb_signed_entry(int s, int32_t F) { return ((uint32_t)F << FB_SIGNED_SBITS) | (uint32_t)s; }

// Per-voxel totals of the last pass (fiesta_signed_stats).
struct FbSignedAcc {
  unsigned long long obstacles, interior;
  int32_t max_q;                                                          // largest finite q
};
FB_HD void fb_signed_count(FbSignedAcc &a, int32_t v) {
  if (v > 0) a.obstacles++;
  if (v > 1) a.interior++;
  if (v != FB_SIGNED_NONE && v > a.max_q) a.max_q = v;
}

// Passes 2 and 3: one line of m voxels.  out[u] = min over i with F[i] != FB_SIGNED_NONE of (u - i)^2 + F[i] (FB_SIGNED_NONE when
// there is no such i), in exact integers (Meijster et al.'s lower envelope of parabolas).  F[i] is read at F[i * fs]; the
// envelope stack lives in buf[k * bs] (entry k = F << 11 | s) and out[u] is written to buf[u * bs] over it: the backward sweep
// only reads entries k <= u - 1 after writing position u (the stack's boundaries t[k] are strictly increasing from t[0] = 0, so
// k <= t[k] <= u while entry k is in use), and it holds the top two entries in registers.  Every F read must be < 2^21: 1023^2 in
// the y pass, 2 * 1023^2 in the x pass.  With acc, every value written is counted into it.
FB_HD void fb_signed_envelope(const int32_t *F, long long fs, int32_t *buf, long long bs, int m, FbSignedAcc *acc) {
  uint32_t *st = (uint32_t *)buf;
  int k = -1;                                                             // stack top
  int s = 0, t = 0, s2 = 0;                                               // top entry: position, start of its region; entry k - 1
  int32_t Fs = 0, F2 = 0;
  for (int u = 0; u < m; ++u) {
    const int32_t Fu = F[u * fs];
    if (Fu == FB_SIGNED_NONE) continue;
    while (k >= 0) {
      const int32_t a = (t - s) * (t - s) + Fs, b = (t - u) * (t - u) + Fu;
      if (a <= b) break;
      if (--k < 0) break;                                                 // pop: entry k - 1 becomes the top
      s = s2; Fs = F2;
      if (k > 0) {
        const uint32_t e = st[(k - 1) * bs];
        s2 = (int)(e & ((1u << FB_SIGNED_SBITS) - 1u)); F2 = (int32_t)(e >> FB_SIGNED_SBITS);
        t = 1 + fb_signed_sep(s2, F2, s, Fs);
      } else {
        t = 0;
      }
    }
    if (k < 0) {
      k = 0; s = u; Fs = Fu; t = 0;
      st[0] = fb_signed_entry(u, Fu);
    } else {
      const int w = 1 + fb_signed_sep(s, Fs, u, Fu);
      if (w < m) {
        ++k;
        st[k * bs] = fb_signed_entry(u, Fu);
        s2 = s; F2 = Fs; s = u; Fs = Fu; t = w;
      }
    }
  }
  if (k < 0) {                                                            // no finite value on the line
    for (int u = m - 1; u >= 0; --u) {
      buf[u * bs] = FB_SIGNED_NONE;
      if (acc) fb_signed_count(*acc, FB_SIGNED_NONE);
    }
    return;
  }
  for (int u = m - 1; u >= 0; --u) {
    while (k > 0 && (u - s2) * (u - s2) + F2 <= (u - s) * (u - s) + Fs) {  // u is left of the top entry's region
      --k;
      s = s2; Fs = F2;
      if (k > 0) {
        const uint32_t e = st[(k - 1) * bs];
        s2 = (int)(e & ((1u << FB_SIGNED_SBITS) - 1u)); F2 = (int32_t)(e >> FB_SIGNED_SBITS);
      }
    }
    const int32_t v = (u - s) * (u - s) + Fs;
    buf[u * bs] = v;
    if (acc) fb_signed_count(*acc, v);
  }
}
#endif
