// CPU driver of fiesta_b200/csrc/fb_signed.h for tests/test_signed_oracle.py.  Reads commands from stdin until EOF:
//   line x y m r_0 .. r_{m-1}   records of the z-line at (x, y, 0..m-1): classify each voxel (fb_signed_obstacle), form the
//                               32-voxel chunk masks and their neighbours as k_signed_z does, and print fb_signed_1d per voxel
//   env m F_0 .. F_{m-1}        one line of the lower envelope (fb_signed_envelope, F strided by 2, stack / output by 3): prints the
//                               m outputs, then "acc obstacles interior max_q"
// Values FB_SIGNED_NONE (2147483647) mean "no non-obstacle in reach".
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../fiesta_b200/csrc/fb_signed.h"

static long long rd() {
  long long v;
  if (std::scanf("%lld", &v) != 1) std::exit(3);
  return v;
}

int main() {
  char cmd[16];
  while (std::scanf("%15s", cmd) == 1) {
    if (!std::strcmp(cmd, "line")) {
      const int x = (int)rd(), y = (int)rd(), m = (int)rd();
      std::vector<uint32_t> mask((m + 31) / 32, 0u);
      for (int z = 0; z < m; ++z) {
        const uint32_t c = (uint32_t)rd();
        if (!fb_signed_obstacle(c, x, y, z)) mask[z / 32] |= 1u << (z % 32);
      }
      const int nch = (int)mask.size();
      std::vector<int> last(nch), first(nch);                             // the warp's inclusive max / suffix-min scans
      for (int c = 0; c < nch; ++c) {
        int l = -1;
        for (int b = 31; b >= 0 && mask[c]; --b) if ((mask[c] >> b) & 1u) { l = 32 * c + b; break; }
        last[c] = l > -1 ? l : (c > 0 ? last[c - 1] : -1);
      }
      for (int c = nch - 1; c >= 0; --c) {
        int f = FB_SIGNED_NONE;
        for (int b = 0; b < 32 && mask[c]; ++b) if ((mask[c] >> b) & 1u) { f = 32 * c + b; break; }
        first[c] = f != FB_SIGNED_NONE ? f : (c + 1 < nch ? first[c + 1] : FB_SIGNED_NONE);
      }
      for (int z = 0; z < m; ++z) {
        const int c = z / 32;
        std::printf("%d\n", fb_signed_1d(mask[c], c, z % 32, c > 0 ? last[c - 1] : -1, c + 1 < nch ? first[c + 1] : FB_SIGNED_NONE));
      }
    } else if (!std::strcmp(cmd, "env")) {
      const int m = (int)rd();
      std::vector<int32_t> F(2 * (size_t)m + 1, -7), buf(3 * (size_t)m + 1, -9);
      for (int i = 0; i < m; ++i) F[2 * (size_t)i] = (int32_t)rd();
      FbSignedAcc acc{0, 0, 0};
      fb_signed_envelope(F.data(), 2, buf.data(), 3, m, &acc);
      for (int u = 0; u < m; ++u) std::printf("%d\n", buf[3 * (size_t)u]);
      std::printf("acc %llu %llu %d\n", acc.obstacles, acc.interior, acc.max_q);
    } else {
      return 2;
    }
  }
  return 0;
}
