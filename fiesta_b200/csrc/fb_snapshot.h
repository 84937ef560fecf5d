// fiesta_b200 -- the map snapshot format (fiesta_snapshot_save / fiesta_snapshot_load, DESIGN.md §3.12).  All knowledge of
// the byte layout is here.  Plain C++ (no CUDA, no torch): compiled by nvcc for the library and the device kernels
// (fb_snapshot.cu), and by g++ for the CPU tests (tests/cpp/snapshot_test.cpp).
//
// One versioned little-endian stream, every section a multiple of 8 bytes:
//   header   FB_SNAP_HDR bytes at fixed offsets (FbSnapHeader; offsets in fb_snap_encode), the last 8 its checksum
//   tiles    n_tiles u32 indices of the stored 8^3 tiles, strictly ascending, zero-padded to 8 bytes
//   payload  per stored tile, its in-grid voxels in (x, y, z) order, z fastest, one plain array per field:
//            occ f64[n], cnt u64[n], LS u64[n] (EXACT only), cobs u32[n], a zero u32 when n is odd, then the u64 checksum of
//            the tile's words before it.  Voxels outside the grid (z padding, the far edges) are not stored.
//   depth    depth_pixels u16 of the depth front end's last image, zero-padded to 8 bytes (absent when depth_pixels == 0)
// A tile is stored when any of its voxels differs from the default state (cobs 0, occ +0.0, cnt 0, LS 0).
#ifndef FB_SNAPSHOT_H_
#define FB_SNAPSHOT_H_
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#ifdef __CUDACC__
#define FB_SNAP_HD __host__ __device__ __forceinline__
#else
#define FB_SNAP_HD inline
#endif

#define FB_SNAP_MAGIC "FIESTASN"
#define FB_SNAP_VERSION 1u
#define FB_SNAP_HDR 384                       // header bytes; its checksum covers the first FB_SNAP_HDR - 8
#define FB_SNAP_NSTATS 13                     // fiesta_stats fields occupancy_updates .. touched_voxels
#define FB_SNAP_STAT_ROUNDS 11                // ... of which raycast_rounds is not stored (always 0): it depends on the order in
                                              // which concurrent rays claim voxels, not on the map's state
#define FB_SNAP_LOCAL_BOX_SEEN 1u             // flags: FAST mode's sticky pull-all flag (DESIGN.md §3.3)
#define FB_SNAP_MAX_GX 2046                   // the grid limits of fiesta_create (FB_MAX_* in fb_common.cuh)
#define FB_SNAP_MAX_GY 1024
#define FB_SNAP_MAX_GZ 1024
#define FB_SNAP_MAX_PTOTAL 0x3fffffffLL       // padded voxels (FB_LIST_IDX_MASK)
#define FB_SNAP_MAX_DEPTH (1LL << 28)         // depth pixels

// ---- checksum: 64-bit words w_0 .. w_{n-1} -> mix(n + sum_j mix(w_j ^ (j * K))) mod 2^64, with mix the splitmix64 finaliser.
// A sum of independent terms, so a warp or a CTA can add its words in any order and get the same bits.
FB_SNAP_HD uint64_t fb_snap_mix(uint64_t z) {
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
FB_SNAP_HD uint64_t fb_snap_term(uint64_t w, uint64_t j) { return fb_snap_mix(w ^ (j * 0xd1b54a32d192ed03ull)); }
FB_SNAP_HD uint64_t fb_snap_final(uint64_t sum, uint64_t n) { return fb_snap_mix(sum + n); }
FB_SNAP_HD uint64_t fb_snap_ld64(const uint8_t *p) {
  uint64_t v = 0;
  for (int k = 7; k >= 0; --k) v = (v << 8) | p[k];
  return v;
}
// checksum of n little-endian words at p
inline uint64_t fb_snap_checksum(const uint8_t *p, uint64_t n) {
  uint64_t s = 0;
  for (uint64_t j = 0; j < n; ++j) s += fb_snap_term(fb_snap_ld64(p + 8 * j), j);
  return fb_snap_final(s, n);
}

// ---- geometry
// grid_size_ of ESDFMap's constructor (ESDFMap.cpp:171-186), the expression fiesta_create uses; 0 when not representable
inline int fb_snap_grid_dim(double map_size, double resolution) {
  const double v = ceil(map_size / resolution);
  return (v >= 1.0 && v <= 1e9) ? (int)v : 0;
}
FB_SNAP_HD int fb_snap_ext(int g, int t) { const int r = g - 8 * t; return r < 8 ? r : 8; }
// in-grid voxels of 8^3 tile `tile` (tiles numbered (tx * ty_n + ty) * tz_n + tz, as the device arrays)
FB_SNAP_HD void fb_snap_tile_dims(int gx, int gy, int gz, uint32_t tile, int *tc, int *n) {
  const int tyn = (gy + 7) / 8, tzn = (gz + 7) / 8;
  tc[2] = (int)(tile % (uint32_t)tzn); tc[1] = (int)((tile / (uint32_t)tzn) % (uint32_t)tyn); tc[0] = (int)(tile / (uint32_t)(tzn * tyn));
  n[0] = fb_snap_ext(gx, tc[0]); n[1] = fb_snap_ext(gy, tc[1]); n[2] = fb_snap_ext(gz, tc[2]);
}
// 64-bit words of a tile's payload before its checksum: 2 or 3 8-byte fields and the cobs words
FB_SNAP_HD uint32_t fb_snap_tile_words(int nvox, int exact) { return (uint32_t)((exact ? 3 : 2) * nvox + (nvox + 1) / 2); }
inline uint64_t fb_snap_tile_bytes(int gx, int gy, int gz, int exact, uint32_t tile) {
  int tc[3], n[3];
  fb_snap_tile_dims(gx, gy, gz, tile, tc, n);
  return 8ull * (fb_snap_tile_words(n[0] * n[1] * n[2], exact) + 1);
}
inline uint64_t fb_snap_pad8(uint64_t b) { return (b + 7) & ~7ull; }

// ---- header
struct FbSnapHeader {
  uint32_t version, mode;                       // FIESTA_MODE_EXACT / FIESTA_MODE_FAST
  double origin[3], resolution, map_size[3];    // the fiesta_config doubles as given at create
  int32_t grid[3];                              // grid_size_, checked against the one the config gives
  int32_t params_set;
  double l_hit, l_miss, l_min, l_max, l_occ;    // derived log-odds, bit for bit
  int32_t min_vec[3], max_vec[3], last_min_vec[3], last_max_vec[3];   // the update box and the previous one
  uint32_t flags;                               // FB_SNAP_LOCAL_BOX_SEEN
  uint32_t image_cnt;                           // depth front end: images seen (Fiesta.h:321-323)
  uint64_t tclock, key_base;                    // EXACT: relink clock, observation clock of the integration epoch; FAST: 0
  int64_t stats[FB_SNAP_NSTATS];                // fiesta_stats, occupancy_updates .. touched_voxels (raycast_rounds: 0)
  int64_t depth_pixels;                         // pixels of the stored depth image
  uint64_t n_tiles;                             // stored tiles
  uint64_t list_sum, depth_sum;                 // checksums of the tile list and the depth section
};
// byte offsets of the header fields
enum {
  FB_SNAP_O_VERSION = 8, FB_SNAP_O_MODE = 12, FB_SNAP_O_ORIGIN = 16, FB_SNAP_O_RES = 40, FB_SNAP_O_SIZE = 48, FB_SNAP_O_GRID = 72,
  FB_SNAP_O_PARAMS = 84, FB_SNAP_O_L = 88, FB_SNAP_O_BOX = 128, FB_SNAP_O_FLAGS = 176, FB_SNAP_O_IMGCNT = 180, FB_SNAP_O_TCLOCK = 184,
  FB_SNAP_O_KEYBASE = 192, FB_SNAP_O_STATS = 200, FB_SNAP_O_DEPTH = 304, FB_SNAP_O_NTILES = 312, FB_SNAP_O_LISTSUM = 320,
  FB_SNAP_O_DEPTHSUM = 328, FB_SNAP_O_RESERVED = 336, FB_SNAP_O_HDRSUM = FB_SNAP_HDR - 8
};
inline void fb_snap_st32(uint8_t *p, uint32_t v) { for (int k = 0; k < 4; ++k) p[k] = (uint8_t)(v >> (8 * k)); }
inline void fb_snap_st64(uint8_t *p, uint64_t v) { for (int k = 0; k < 8; ++k) p[k] = (uint8_t)(v >> (8 * k)); }
inline uint32_t fb_snap_ld32(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
inline void fb_snap_stf(uint8_t *p, double d) { uint64_t v; memcpy(&v, &d, 8); fb_snap_st64(p, v); }
inline double fb_snap_ldf(const uint8_t *p) { const uint64_t v = fb_snap_ld64(p); double d; memcpy(&d, &v, 8); return d; }

// FB_SNAP_HDR bytes, checksum included
inline void fb_snap_encode(const FbSnapHeader &h, uint8_t *p) {
  memset(p, 0, FB_SNAP_HDR);
  memcpy(p, FB_SNAP_MAGIC, 8);
  fb_snap_st32(p + FB_SNAP_O_VERSION, h.version);
  fb_snap_st32(p + FB_SNAP_O_MODE, h.mode);
  for (int i = 0; i < 3; ++i) {
    fb_snap_stf(p + FB_SNAP_O_ORIGIN + 8 * i, h.origin[i]);
    fb_snap_stf(p + FB_SNAP_O_SIZE + 8 * i, h.map_size[i]);
    fb_snap_st32(p + FB_SNAP_O_GRID + 4 * i, (uint32_t)h.grid[i]);
    fb_snap_st32(p + FB_SNAP_O_BOX + 4 * i, (uint32_t)h.min_vec[i]);
    fb_snap_st32(p + FB_SNAP_O_BOX + 12 + 4 * i, (uint32_t)h.max_vec[i]);
    fb_snap_st32(p + FB_SNAP_O_BOX + 24 + 4 * i, (uint32_t)h.last_min_vec[i]);
    fb_snap_st32(p + FB_SNAP_O_BOX + 36 + 4 * i, (uint32_t)h.last_max_vec[i]);
  }
  fb_snap_stf(p + FB_SNAP_O_RES, h.resolution);
  fb_snap_st32(p + FB_SNAP_O_PARAMS, (uint32_t)h.params_set);
  const double l[5] = {h.l_hit, h.l_miss, h.l_min, h.l_max, h.l_occ};
  for (int i = 0; i < 5; ++i) fb_snap_stf(p + FB_SNAP_O_L + 8 * i, l[i]);
  fb_snap_st32(p + FB_SNAP_O_FLAGS, h.flags);
  fb_snap_st32(p + FB_SNAP_O_IMGCNT, h.image_cnt);
  fb_snap_st64(p + FB_SNAP_O_TCLOCK, h.tclock);
  fb_snap_st64(p + FB_SNAP_O_KEYBASE, h.key_base);
  for (int i = 0; i < FB_SNAP_NSTATS; ++i) fb_snap_st64(p + FB_SNAP_O_STATS + 8 * i, (uint64_t)h.stats[i]);
  fb_snap_st64(p + FB_SNAP_O_DEPTH, (uint64_t)h.depth_pixels);
  fb_snap_st64(p + FB_SNAP_O_NTILES, h.n_tiles);
  fb_snap_st64(p + FB_SNAP_O_LISTSUM, h.list_sum);
  fb_snap_st64(p + FB_SNAP_O_DEPTHSUM, h.depth_sum);
  fb_snap_st64(p + FB_SNAP_O_HDRSUM, fb_snap_checksum(p, FB_SNAP_O_HDRSUM / 8));
}
inline void fb_snap_decode(const uint8_t *p, FbSnapHeader *h) {
  h->version = fb_snap_ld32(p + FB_SNAP_O_VERSION);
  h->mode = fb_snap_ld32(p + FB_SNAP_O_MODE);
  for (int i = 0; i < 3; ++i) {
    h->origin[i] = fb_snap_ldf(p + FB_SNAP_O_ORIGIN + 8 * i);
    h->map_size[i] = fb_snap_ldf(p + FB_SNAP_O_SIZE + 8 * i);
    h->grid[i] = (int32_t)fb_snap_ld32(p + FB_SNAP_O_GRID + 4 * i);
    h->min_vec[i] = (int32_t)fb_snap_ld32(p + FB_SNAP_O_BOX + 4 * i);
    h->max_vec[i] = (int32_t)fb_snap_ld32(p + FB_SNAP_O_BOX + 12 + 4 * i);
    h->last_min_vec[i] = (int32_t)fb_snap_ld32(p + FB_SNAP_O_BOX + 24 + 4 * i);
    h->last_max_vec[i] = (int32_t)fb_snap_ld32(p + FB_SNAP_O_BOX + 36 + 4 * i);
  }
  h->resolution = fb_snap_ldf(p + FB_SNAP_O_RES);
  h->params_set = (int32_t)fb_snap_ld32(p + FB_SNAP_O_PARAMS);
  double *l[5] = {&h->l_hit, &h->l_miss, &h->l_min, &h->l_max, &h->l_occ};
  for (int i = 0; i < 5; ++i) *l[i] = fb_snap_ldf(p + FB_SNAP_O_L + 8 * i);
  h->flags = fb_snap_ld32(p + FB_SNAP_O_FLAGS);
  h->image_cnt = fb_snap_ld32(p + FB_SNAP_O_IMGCNT);
  h->tclock = fb_snap_ld64(p + FB_SNAP_O_TCLOCK);
  h->key_base = fb_snap_ld64(p + FB_SNAP_O_KEYBASE);
  for (int i = 0; i < FB_SNAP_NSTATS; ++i) h->stats[i] = (int64_t)fb_snap_ld64(p + FB_SNAP_O_STATS + 8 * i);
  h->depth_pixels = (int64_t)fb_snap_ld64(p + FB_SNAP_O_DEPTH);
  h->n_tiles = fb_snap_ld64(p + FB_SNAP_O_NTILES);
  h->list_sum = fb_snap_ld64(p + FB_SNAP_O_LISTSUM);
  h->depth_sum = fb_snap_ld64(p + FB_SNAP_O_DEPTHSUM);
}

// Where the sections of a stream lie.
struct FbSnapLayout {
  uint64_t list_off, payload_off, payload_bytes, depth_off, depth_bytes, total;
};
inline void fb_snap_layout(uint64_t n_tiles, uint64_t payload_bytes, int64_t depth_pixels, FbSnapLayout *L) {
  L->list_off = FB_SNAP_HDR;
  L->payload_off = L->list_off + fb_snap_pad8(4 * n_tiles);
  L->payload_bytes = payload_bytes;
  L->depth_off = L->payload_off + payload_bytes;
  L->depth_bytes = fb_snap_pad8(2 * (uint64_t)depth_pixels);
  L->total = L->depth_off + L->depth_bytes;
}

// Every host-side rule of a stream of `size` bytes: header, tile list, section sizes and the depth checksum (the tile payloads
// are checked by the unpack kernel).  0 and *h / *L filled when it passes, else -1 with the reason in err.
inline int fb_snap_parse(const uint8_t *p, int64_t size, FbSnapHeader *h, FbSnapLayout *L, char *err, int errlen) {
#define FB_SNAP_FAIL(...) do { snprintf(err, (size_t)errlen, __VA_ARGS__); return -1; } while (0)
  if (size < FB_SNAP_HDR) FB_SNAP_FAIL("truncated: %lld bytes, the header alone is %d", (long long)size, FB_SNAP_HDR);
  if (memcmp(p, FB_SNAP_MAGIC, 8) != 0) FB_SNAP_FAIL("not a map snapshot (bad magic)");
  if (fb_snap_ld32(p + FB_SNAP_O_VERSION) != FB_SNAP_VERSION) FB_SNAP_FAIL("unsupported snapshot version %u", fb_snap_ld32(p + FB_SNAP_O_VERSION));
  if (fb_snap_checksum(p, FB_SNAP_O_HDRSUM / 8) != fb_snap_ld64(p + FB_SNAP_O_HDRSUM)) FB_SNAP_FAIL("header checksum mismatch");
  for (int o = FB_SNAP_O_RESERVED; o < FB_SNAP_O_HDRSUM; ++o)
    if (p[o]) FB_SNAP_FAIL("reserved header bytes are not zero");
  fb_snap_decode(p, h);
  if (h->mode > 1u) FB_SNAP_FAIL("unknown mode %u", h->mode);
  if (!(h->resolution > 0) || !isfinite(h->resolution)) FB_SNAP_FAIL("resolution must be finite and > 0");
  const int gmax[3] = {FB_SNAP_MAX_GX, FB_SNAP_MAX_GY, FB_SNAP_MAX_GZ};
  for (int i = 0; i < 3; ++i) {
    if (!isfinite(h->origin[i]) || !isfinite(h->map_size[i])) FB_SNAP_FAIL("origin and map size must be finite");
    const int gi = fb_snap_grid_dim(h->map_size[i], h->resolution);
    if (gi < 1 || gi > gmax[i]) FB_SNAP_FAIL("grid exceeds the supported 2046 x 1024 x 1024 voxels");
    if (gi != h->grid[i]) FB_SNAP_FAIL("stored grid %d x %d x %d differs from the one its config gives", h->grid[0], h->grid[1], h->grid[2]);
  }
  const int gx = h->grid[0], gy = h->grid[1], gz = h->grid[2];
  if ((long long)gx * gy * ((gz + 3) & ~3) > FB_SNAP_MAX_PTOTAL) FB_SNAP_FAIL("grid exceeds 2^30 voxels");
  for (int i = 0; i < 3; ++i)
    if (h->min_vec[i] < 0 || h->last_min_vec[i] < 0 || h->max_vec[i] > h->grid[i] - 1 || h->last_max_vec[i] > h->grid[i] - 1)
      FB_SNAP_FAIL("update box outside the grid");
  if (h->params_set != 0 && h->params_set != 1) FB_SNAP_FAIL("bad params_set %d", h->params_set);
  if (h->flags & ~FB_SNAP_LOCAL_BOX_SEEN) FB_SNAP_FAIL("unknown flag bits 0x%x", h->flags);
  if (h->mode == 0 && (h->tclock < 1 || (h->flags & FB_SNAP_LOCAL_BOX_SEEN))) FB_SNAP_FAIL("EXACT snapshot with a zero relink clock or FAST state");
  if (h->mode == 1 && (h->tclock != 0 || h->key_base != 0)) FB_SNAP_FAIL("FAST snapshot with EXACT clocks");
  for (int i = 0; i < FB_SNAP_NSTATS; ++i)
    if (h->stats[i] < 0 || (i == FB_SNAP_STAT_ROUNDS && h->stats[i] != 0)) FB_SNAP_FAIL("bad statistic %d", i);
  if (h->depth_pixels < 0 || h->depth_pixels > FB_SNAP_MAX_DEPTH || (h->depth_pixels > 0 && h->image_cnt == 0))
    FB_SNAP_FAIL("bad depth image size %lld", (long long)h->depth_pixels);
  const uint64_t ntiles = (uint64_t)((gx + 7) / 8) * ((gy + 7) / 8) * ((gz + 7) / 8);
  if (h->n_tiles > ntiles) FB_SNAP_FAIL("%llu stored tiles, the grid has %llu", (unsigned long long)h->n_tiles, (unsigned long long)ntiles);
  const uint64_t list_bytes = fb_snap_pad8(4 * h->n_tiles);
  if ((uint64_t)size < FB_SNAP_HDR + list_bytes) FB_SNAP_FAIL("truncated tile list");
  const uint8_t *lp = p + FB_SNAP_HDR;
  if (fb_snap_checksum(lp, list_bytes / 8) != h->list_sum) FB_SNAP_FAIL("tile list checksum mismatch");
  uint64_t payload = 0;
  for (uint64_t t = 0; t < h->n_tiles; ++t) {
    const uint32_t tile = fb_snap_ld32(lp + 4 * t);
    if (tile >= ntiles) FB_SNAP_FAIL("tile index %u past the grid's %llu tiles", tile, (unsigned long long)ntiles);
    if (t > 0 && tile <= fb_snap_ld32(lp + 4 * (t - 1))) FB_SNAP_FAIL("tile list not strictly ascending at entry %llu", (unsigned long long)t);
    payload += fb_snap_tile_bytes(gx, gy, gz, h->mode == 0, tile);
  }
  if ((h->n_tiles & 1) && fb_snap_ld32(lp + 4 * h->n_tiles) != 0) FB_SNAP_FAIL("tile list padding is not zero");
  fb_snap_layout(h->n_tiles, payload, h->depth_pixels, L);
  if ((uint64_t)size != L->total) FB_SNAP_FAIL("stream is %lld bytes, its header describes %llu", (long long)size, (unsigned long long)L->total);
  if (fb_snap_checksum(p + L->depth_off, L->depth_bytes / 8) != h->depth_sum) FB_SNAP_FAIL("depth image checksum mismatch");
  for (uint64_t b = L->depth_off + 2 * (uint64_t)h->depth_pixels; b < L->total; ++b)
    if (p[b]) FB_SNAP_FAIL("depth image padding is not zero");
  return 0;
#undef FB_SNAP_FAIL
}

// Per-tile reasons the unpack kernel reports (bits)
#define FB_SNAP_BAD_SUM 1u        // payload checksum mismatch
#define FB_SNAP_BAD_COBS 2u       // a record is neither 0, 1 nor an obstacle coordinate inside the grid, or padding not zero
#define FB_SNAP_BAD_BIT31 4u      // bit 31 in a FAST snapshot, or without an obstacle
#define FB_SNAP_BAD_OCC 8u        // a log-odds value is not finite
#define FB_SNAP_BAD_LS 16u        // a relink time is not below the stored relink clock
#define FB_SNAP_BAD_CNT 32u       // more hits than observations
#endif
