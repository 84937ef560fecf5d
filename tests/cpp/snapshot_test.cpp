// CPU checks of the map snapshot format (fiesta_b200/csrc/fb_snapshot.h), built with g++ by tests/test_snapshot_format.py, and
// the stream editor the GPU tests use to make well-checksummed malformed snapshots.
//   snapshot_test selftest                 header round trips and every host-side rejection rule
//   snapshot_test sum <file>               checksum of the file's little-endian 64-bit words, in hex
//   snapshot_test edit <in> <out> <op>     apply op to a valid snapshot, then recompute every checksum:
//       zero_ls       EXACT: every relink time 0 and the relink clock at its initial value 1
//       obstacle_out  first record of the first stored tile -> an obstacle at x = grid x (outside the grid)
//       bit31         first record of the first stored tile -> an obstacle with bit 31 set
//       nan_occ       first log-odds of the first stored tile -> NaN
//       ls_ge_tclock  EXACT: first relink time of the first stored tile -> the relink clock
//       tile_past     last stored tile index -> the number of tiles in the grid
//       refix         nothing (only the checksums)
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../fiesta_b200/csrc/fb_record.h"
#include "../../fiesta_b200/csrc/fb_snapshot.h"

static int fails = 0, checks = 0;
#define EXPECT(c, ...) do { ++checks; if (!(c)) { ++fails; fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); } } while (0)

// The stream's tiles: (index, byte offset of the payload, in-grid voxels).
struct Tile { uint32_t idx; uint64_t off; int nv; };
static std::vector<Tile> tiles_of(const std::vector<uint8_t> &s, const FbSnapHeader &h) {
  std::vector<Tile> t;
  uint64_t off = FB_SNAP_HDR + fb_snap_pad8(4 * h.n_tiles);
  for (uint64_t i = 0; i < h.n_tiles; ++i) {
    const uint32_t idx = fb_snap_ld32(&s[FB_SNAP_HDR + 4 * i]);
    int tc[3], n[3];
    fb_snap_tile_dims(h.grid[0], h.grid[1], h.grid[2], idx, tc, n);
    t.push_back({idx, off, n[0] * n[1] * n[2]});
    off += fb_snap_tile_bytes(h.grid[0], h.grid[1], h.grid[2], h.mode == 0, idx);
  }
  return t;
}
// Recompute the tile, list, depth and header checksums of s (whose header h describes it).
static void refix(std::vector<uint8_t> &s, FbSnapHeader h) {
  uint64_t end = FB_SNAP_HDR + fb_snap_pad8(4 * h.n_tiles);
  for (const Tile &t : tiles_of(s, h)) {
    const uint32_t W = fb_snap_tile_words(t.nv, h.mode == 0);
    fb_snap_st64(&s[t.off + 8ull * W], fb_snap_checksum(&s[t.off], W));
    end = t.off + 8ull * (W + 1);
  }
  h.list_sum = fb_snap_checksum(&s[FB_SNAP_HDR], fb_snap_pad8(4 * h.n_tiles) / 8);
  h.depth_sum = fb_snap_checksum(s.data() + end, (s.size() - end) / 8);
  fb_snap_encode(h, s.data());
}

// Recompute only the tile list and header checksums (after an edit of the list, whose tiles can then not be walked).
static void refix_list(std::vector<uint8_t> &s, FbSnapHeader h) {
  h.list_sum = fb_snap_checksum(&s[FB_SNAP_HDR], fb_snap_pad8(4 * h.n_tiles) / 8);
  fb_snap_encode(h, s.data());
}

// A valid stream: grid 20 x 16 x 30 (edge tiles and z padding), `tiles` stored with simple contents.
static std::vector<uint8_t> make_stream(int mode, const std::vector<uint32_t> &tiles, int64_t depth_pixels) {
  FbSnapHeader h{};
  h.version = FB_SNAP_VERSION; h.mode = (uint32_t)mode;
  const double size[3] = {2.0, 1.6, 3.0};
  for (int i = 0; i < 3; ++i) { h.origin[i] = -1.0 + 0.25 * i; h.map_size[i] = size[i]; }
  h.resolution = 0.1;
  for (int i = 0; i < 3; ++i) h.grid[i] = fb_snap_grid_dim(h.map_size[i], h.resolution);
  h.params_set = 1; h.l_hit = 0.85; h.l_miss = -0.4; h.l_min = -2.0; h.l_max = 3.5; h.l_occ = 0.8;
  for (int i = 0; i < 3; ++i) { h.min_vec[i] = 1; h.max_vec[i] = h.grid[i] - 2; h.last_min_vec[i] = 0; h.last_max_vec[i] = h.grid[i] - 1; }
  h.flags = mode == 1 ? FB_SNAP_LOCAL_BOX_SEEN : 0u;
  h.image_cnt = depth_pixels ? 3 : 0;
  h.tclock = mode == 0 ? 1000 : 0; h.key_base = 0;
  for (int i = 0; i < FB_SNAP_NSTATS; ++i) h.stats[i] = i == FB_SNAP_STAT_ROUNDS ? 0 : 10 * i;
  h.depth_pixels = depth_pixels;
  h.n_tiles = tiles.size();
  uint64_t payload = 0;
  for (uint32_t t : tiles) payload += fb_snap_tile_bytes(h.grid[0], h.grid[1], h.grid[2], mode == 0, t);
  FbSnapLayout L;
  fb_snap_layout(h.n_tiles, payload, depth_pixels, &L);
  std::vector<uint8_t> s(L.total, 0);
  for (size_t i = 0; i < tiles.size(); ++i) fb_snap_st32(&s[FB_SNAP_HDR + 4 * i], tiles[i]);
  fb_snap_encode(h, s.data());
  for (const Tile &t : tiles_of(s, h)) {
    for (int k = 0; k < t.nv; ++k) fb_snap_stf(&s[t.off + 8ull * k], 0.5);
    const uint64_t cobs = t.off + 8ull * (mode == 0 ? 3 : 2) * t.nv;
    for (int k = 0; k < t.nv; ++k) fb_snap_st32(&s[cobs + 4ull * k], 1u);
  }
  for (int64_t k = 0; k < depth_pixels; ++k) { s[L.depth_off + 2 * k] = (uint8_t)k; s[L.depth_off + 2 * k + 1] = (uint8_t)(k >> 8); }
  refix(s, h);
  return s;
}

static bool parses(const std::vector<uint8_t> &s, std::string *why = nullptr, int64_t size = -1) {
  FbSnapHeader h;
  FbSnapLayout L;
  char err[256] = "";
  const int r = fb_snap_parse(s.data(), size < 0 ? (int64_t)s.size() : size, &h, &L, err, sizeof(err));
  if (why) *why = err;
  return r == 0;
}
static FbSnapHeader header_of(const std::vector<uint8_t> &s) { FbSnapHeader h; fb_snap_decode(s.data(), &h); return h; }
// s with its header changed by f and every checksum fixed
template <class F> static std::vector<uint8_t> with_header(std::vector<uint8_t> s, F f) {
  FbSnapHeader h = header_of(s);
  f(h);
  fb_snap_encode(h, s.data());
  return s;
}
static void expect_reject(const std::vector<uint8_t> &s, const char *what, const char *needle) {
  std::string why;
  const bool ok = parses(s, &why);
  EXPECT(!ok, "%s: accepted", what);
  EXPECT(why.find(needle) != std::string::npos, "%s: rejected for '%s', expected '%s'", what, why.c_str(), needle);
}

static int selftest() {
  // header round trip, every field
  for (int mode = 0; mode < 2; ++mode) {
    const std::vector<uint8_t> s = make_stream(mode, {0, 5, 17, 23}, mode ? 0 : 77);
    std::string why;
    EXPECT(parses(s, &why), "valid mode %d stream rejected: %s", mode, why.c_str());
    const FbSnapHeader h = header_of(s);
    std::vector<uint8_t> e(FB_SNAP_HDR);
    fb_snap_encode(h, e.data());
    EXPECT(memcmp(e.data(), s.data(), FB_SNAP_HDR) == 0, "encode(decode(header)) differs");
    FbSnapHeader h2;
    fb_snap_decode(e.data(), &h2);
    EXPECT(memcmp(&h, &h2, sizeof(h)) == 0, "decode(encode(h)) differs");
    EXPECT(h.grid[0] == 20 && h.grid[1] == 16 && h.grid[2] == 30 && h.n_tiles == 4 && h.stats[12] == 120, "fields");
  }
  // the layout: payload sizes of edge tiles (grid 20 x 16 x 30 = tiles 3 x 2 x 4; tile 23 = (2, 1, 3): 4 x 8 x 6 voxels)
  EXPECT(fb_snap_tile_bytes(20, 16, 30, 1, 0) == 8ull * (3 * 512 + 256 + 1), "full EXACT tile bytes");
  EXPECT(fb_snap_tile_bytes(20, 16, 30, 0, 23) == 8ull * (2 * 192 + 96 + 1), "edge FAST tile bytes");
  EXPECT(fb_snap_tile_bytes(3, 3, 3, 0, 0) == 8ull * (2 * 27 + 14 + 1), "odd tile bytes");
  const std::vector<uint8_t> good = make_stream(0, {0, 5, 17, 23}, 77);
  // truncation at every length below the header, and anywhere below the total
  for (int64_t n = 0; n < FB_SNAP_HDR; ++n) EXPECT(!parses(good, nullptr, n), "truncated to %lld accepted", (long long)n);
  for (int64_t n = FB_SNAP_HDR; n < (int64_t)good.size(); n += 7) EXPECT(!parses(good, nullptr, n), "truncated to %lld accepted", (long long)n);
  { std::vector<uint8_t> s = good; s.push_back(0); s.resize(s.size() + 7); expect_reject(s, "longer stream", "header describes"); }
  { std::vector<uint8_t> s = good; s[0] ^= 1; expect_reject(s, "bad magic", "magic"); }
  { std::vector<uint8_t> s = good; fb_snap_st32(&s[FB_SNAP_O_VERSION], 2); expect_reject(s, "bad version", "version"); }
  for (int o : std::initializer_list<int>{FB_SNAP_O_MODE, FB_SNAP_O_RES + 3, FB_SNAP_O_BOX, FB_SNAP_O_TCLOCK, FB_SNAP_O_NTILES, FB_SNAP_O_RESERVED + 5, FB_SNAP_O_HDRSUM}) {
    std::vector<uint8_t> s = good;
    s[o] ^= 0x10;
    expect_reject(s, "header byte flipped", "header checksum");
  }
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.grid[2] = 31; }), "grid differs from config", "differs");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.map_size[1] = 1.71; }), "config gives another grid", "differs");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.map_size[0] = 300.0; h.grid[0] = 3000; }), "grid over the x limit", "exceeds");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.map_size[2] = 102.5; h.grid[2] = 1025; }), "grid over the z limit", "exceeds");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.resolution = 0.0; }), "zero resolution", "resolution");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.max_vec[1] = h.grid[1]; }), "box past the grid", "update box");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.last_min_vec[0] = -1; }), "previous box below the grid", "update box");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.mode = 2; }), "unknown mode", "mode");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.tclock = 0; }), "EXACT with a zero relink clock", "relink clock");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.flags = 4; }), "unknown flags", "flag");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.stats[FB_SNAP_STAT_ROUNDS] = 1; }), "raycast_rounds stored", "statistic");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.stats[0] = -1; }), "negative statistic", "statistic");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.depth_pixels = 81; }), "depth size", "header describes");
  {
    std::vector<uint8_t> s = good;
    s[s.size() - 8 + 1] ^= 1;                                 // depth pixel bytes (77 pixels: the last word holds pixels 76..79)
    expect_reject(s, "depth image flipped", "depth image checksum");
  }
  {
    std::vector<uint8_t> s = good;
    s[FB_SNAP_HDR + 4] ^= 1;
    expect_reject(s, "tile list flipped", "tile list checksum");
  }
  {                                                           // not ascending / repeated / past the grid, each with fixed checksums
    const uint32_t lists[3][4] = {{0, 17, 5, 23}, {0, 5, 5, 23}, {0, 5, 17, 24}};
    const char *needle[3] = {"ascending", "ascending", "past the grid"};
    for (int c = 0; c < 3; ++c) {
      std::vector<uint8_t> s = good;
      for (int i = 0; i < 4; ++i) fb_snap_st32(&s[FB_SNAP_HDR + 4 * i], lists[c][i]);
      refix_list(s, header_of(s));
      expect_reject(s, "bad tile list", needle[c]);
    }
  }
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.n_tiles = 3; }), "fewer tiles than stored", "");
  expect_reject(with_header(good, [](FbSnapHeader &h) { h.n_tiles = 1000; }), "more tiles than the grid", "stored tiles");
  // an empty map: header, nothing else
  {
    const std::vector<uint8_t> s = make_stream(1, {}, 0);
    EXPECT(s.size() == FB_SNAP_HDR && parses(s), "empty FAST snapshot");
  }
  printf("ok %d checks\n", checks);
  return fails ? 1 : 0;
}

static std::vector<uint8_t> read_file(const char *path) {
  FILE *f = fopen(path, "rb");
  if (!f) { perror(path); exit(2); }
  std::vector<uint8_t> s;
  uint8_t b[1 << 16];
  size_t n;
  while ((n = fread(b, 1, sizeof(b), f)) > 0) s.insert(s.end(), b, b + n);
  fclose(f);
  return s;
}

static int edit(const char *in, const char *out, const std::string &op) {
  std::vector<uint8_t> s = read_file(in);
  FbSnapHeader h = header_of(s);
  const std::vector<Tile> T = tiles_of(s, h);
  if (T.empty() && op != "refix") { fprintf(stderr, "no stored tiles\n"); return 2; }
  const bool exact = h.mode == 0;
  auto cobs_at = [&](const Tile &t) { return t.off + 8ull * (exact ? 3 : 2) * t.nv; };
  if (op == "zero_ls") {
    if (!exact) { fprintf(stderr, "zero_ls: not an EXACT snapshot\n"); return 2; }
    for (const Tile &t : T) memset(&s[t.off + 16ull * t.nv], 0, 8ull * t.nv);
    h.tclock = 1;
  } else if (op == "obstacle_out") {
    fb_snap_st32(&s[cobs_at(T[0])], fb_pack(h.grid[0], 0, 0));
  } else if (op == "bit31") {
    fb_snap_st32(&s[cobs_at(T[0])], fb_pack(0, 0, 0) | 0x80000000u);
  } else if (op == "nan_occ") {
    fb_snap_st64(&s[T[0].off], 0x7ff8000000000000ull);
  } else if (op == "ls_ge_tclock") {
    if (!exact) { fprintf(stderr, "ls_ge_tclock: not an EXACT snapshot\n"); return 2; }
    fb_snap_st64(&s[T[0].off + 16ull * T[0].nv], h.tclock);
  } else if (op == "tile_past") {
    fb_snap_st32(&s[FB_SNAP_HDR + 4 * (T.size() - 1)], (uint32_t)(((h.grid[0] + 7) / 8) * ((h.grid[1] + 7) / 8) * ((h.grid[2] + 7) / 8)));
  } else if (op != "refix") {
    fprintf(stderr, "unknown op %s\n", op.c_str());
    return 2;
  }
  if (op == "tile_past") {
    refix_list(s, h);
  } else {
    refix(s, h);
  }
  FILE *f = fopen(out, "wb");
  if (!f || fwrite(s.data(), 1, s.size(), f) != s.size()) { perror(out); return 2; }
  fclose(f);
  return 0;
}

int main(int argc, char **argv) {
  if (argc >= 2 && !strcmp(argv[1], "selftest")) return selftest();
  if (argc == 3 && !strcmp(argv[1], "sum")) {
    const std::vector<uint8_t> s = read_file(argv[2]);
    printf("%016llx\n", (unsigned long long)fb_snap_checksum(s.data(), s.size() / 8));
    return 0;
  }
  if (argc == 5 && !strcmp(argv[1], "edit")) return edit(argv[2], argv[3], argv[4]);
  fprintf(stderr, "usage: snapshot_test selftest | sum <file> | edit <in> <out> <op>\n");
  return 2;
}
