/* TEST INFRASTRUCTURE ONLY -- never linked into, imported by or executed from the product path.
 *
 * CPU model of fiesta_b200's FAST-mode UpdateESDF (fiesta_b200/csrc/fb_esdf.cu): the order-free tile wavefront that
 * replaces ESDFMap::UpdateESDF (FIESTA src/ESDFMap.cpp:273-398) on the throughput path.  It restates, sequentially
 * and without any CUDA, exactly the schedule-independent semantics of the kernels:
 *   E1  insert seeds            record := self | FRESH, tiles within reach 2 queued           (k_seed_inserts)
 *   E2  delete scan             records whose obstacle no longer exists := INF | FRESH         (k_delete_scan)
 *   E3  generations of 8^3 tile visits, each a local Jacobi fixpoint over the 24-neighbourhood dirs_ (parameters.h:55-68)
 *       with the strict-improvement rule, unknown-voxel barriers, FRESH = "is in the queue" frontier semantics, ties to
 *       the smallest packed obstacle coordinate, Jacobi between tiles (a generation only reads the previous one), bounding
 *       box driven neighbour activation, flag-retire visits                                    (k_wavefront)
 * (Tiles are 8^3 like the kernels'; fm_create_tiled(.., 16) exists only to study a 16^3 variant offline.)
 * The GPU result does not depend on thread or CTA scheduling, so the kernels must reproduce this model bit for bit
 * (tests/test_gpu_fast_model.py); the model itself is checked against the reference build on CPU (tests/test_fast_model.py).
 * Two switches exist to study variants offline: FM_FULL_PULL (every queued voxel pulls, the literal reading of
 * ESDFMap.cpp:349-367) and FM_EXIT_TEST (a visiting tile decides exactly whether its changes can improve a neighbour's
 * border before queueing it).  Both must leave the arrays unchanged.
 * Also modelled: the local-map reset of UpdateOccupancy(false) (fm_local_reset) and the x-slab sharded UpdateESDF
 * (fm_set_slab / fm_pack / fm_halo_ingest / fm_relax, tests/test_fast_model_boxes.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define FM_UNKNOWN 0u
#define FM_INF 1u
#define FM_FRESH 0x80000000u
#define FM_MASK 0x7fffffffu
#define FM_FULL_PULL 1
#define FM_EXIT_TEST 2
#define FM_UNDEFINED (-10000)
#define FM_INFINITY 10000

typedef struct fm {
  int gx, gy, gz, tx, ty, tz;
  int T, lg;                   /* tile edge (8 like the kernels; 16 for offline studies) and its log2 */
  long long total;
  int lo[3], hi[3];            /* update box, inclusive (ESDFMap::VoxInRange, ESDFMap.cpp:63-72) */
  uint32_t *code, *stage;      /* records {0 unknown | 1 no obstacle | packed obstacle} + FRESH bit; staging copy */
  uint32_t *tile_flag, *nb_flag;
  uint32_t *list[2], *changed, *changed_bb, *changed_need;
  unsigned n_list[2], n_changed, stamp;
  int pull_all;                /* sticky: some UpdateESDF / relax ran under a box that is not the whole grid */
  int slab_lo, slab_hi;        /* tile columns [lo, hi) this map relaxes (x-slab sharding; all of them when unsharded) */
} fm;

static const int KD[24][3] = {{-1, 0, 0}, {1, 0, 0}, {0, -1, 0}, {0, 1, 0}, {0, 0, -1}, {0, 0, 1},
                              {-1, -1, 0}, {1, 1, 0}, {0, -1, -1}, {0, 1, 1}, {-1, 0, -1}, {1, 0, 1},
                              {-1, 1, 0}, {1, -1, 0}, {0, -1, 1}, {0, 1, -1}, {1, 0, -1}, {-1, 0, 1},
                              {-2, 0, 0}, {2, 0, 0}, {0, -2, 0}, {0, 2, 0}, {0, 0, -2}, {0, 0, 2}};

static uint32_t pack(int x, int y, int z) { return ((uint32_t)(x + 1) << 20) | ((uint32_t)y << 10) | (uint32_t)z; }
static void unpack(uint32_t c, int *x, int *y, int *z) { *x = (int)((c & FM_MASK) >> 20) - 1; *y = (int)((c >> 10) & 1023u); *z = (int)(c & 1023u); }
static long long lin(const fm *m, int x, int y, int z) { return ((long long)x * m->gy + y) * m->gz + z; }
static int in_grid(const fm *m, int x, int y, int z) { return x >= 0 && x < m->gx && y >= 0 && y < m->gy && z >= 0 && z < m->gz; }
static int in_range(const fm *m, int x, int y, int z) {
  return x >= m->lo[0] && x <= m->hi[0] && y >= m->lo[1] && y <= m->hi[1] && z >= m->lo[2] && z <= m->hi[2];
}
static int box_is_full(const fm *m) {
  return m->lo[0] == 0 && m->lo[1] == 0 && m->lo[2] == 0 && m->hi[0] == m->gx - 1 && m->hi[1] == m->gy - 1 && m->hi[2] == m->gz - 1;
}
static unsigned dist2(uint32_t c, int x, int y, int z) {
  int ox, oy, oz;
  unpack(c, &ox, &oy, &oz);
  ox -= x; oy -= y; oz -= z;
  return (unsigned)(ox * ox + oy * oy + oz * oz);
}

fm *fm_create_tiled(int gx, int gy, int gz, int tile) {
  fm *m = (fm *)calloc(1, sizeof(fm));
  if (!m || (tile != 8 && tile != 16)) { free(m); return NULL; }
  m->gx = gx; m->gy = gy; m->gz = gz;
  m->T = tile; m->lg = tile == 8 ? 3 : 4;
  m->tx = (gx + tile - 1) / tile; m->ty = (gy + tile - 1) / tile; m->tz = (gz + tile - 1) / tile;
  m->total = (long long)gx * gy * gz;
  const size_t nt = (size_t)m->tx * m->ty * m->tz;
  m->code = (uint32_t *)calloc((size_t)m->total, 4);
  m->stage = (uint32_t *)calloc((size_t)m->total, 4);
  m->tile_flag = (uint32_t *)calloc(nt, 4);
  m->nb_flag = (uint32_t *)calloc(nt, 4);
  m->list[0] = (uint32_t *)calloc(nt, 4);
  m->list[1] = (uint32_t *)calloc(nt, 4);
  m->changed = (uint32_t *)calloc(nt, 4);
  m->changed_bb = (uint32_t *)calloc(nt, 4);
  m->changed_need = (uint32_t *)calloc(nt, 4);
  m->lo[0] = m->lo[1] = m->lo[2] = 0;
  m->hi[0] = gx - 1; m->hi[1] = gy - 1; m->hi[2] = gz - 1;
  m->stamp = 1;
  m->slab_lo = 0; m->slab_hi = m->tx;
  return m;
}
fm *fm_create(int gx, int gy, int gz) { return fm_create_tiled(gx, gy, gz, 8); }
void fm_destroy(fm *m) {
  if (!m) return;
  free(m->code); free(m->stage); free(m->tile_flag); free(m->nb_flag); free(m->list[0]); free(m->list[1]);
  free(m->changed); free(m->changed_bb); free(m->changed_need); free(m);
}
void fm_set_range(fm *m, const int lo[3], const int hi[3]) {
  for (int k = 0; k < 3; ++k) { m->lo[k] = lo[k]; m->hi[k] = hi[k]; }
}
/* first observation of a voxel (k_integrate: `if (cobs == UNKNOWN) cobs = INF`, ESDFMap.cpp:246-249): not queued */
void fm_observe(fm *m, const uint32_t *idx, long long n) {
  for (long long i = 0; i < n; ++i)
    if (m->code[idx[i]] == FM_UNKNOWN) m->code[idx[i]] = FM_INF;
}

/* fb_activate: queue tile t for the generation `stamp`; work = a neighbour / seed / reset asks for a full visit.
 * Tiles outside this map's x-slab belong to another rank and are never queued here. */
static void activate(fm *m, unsigned t, unsigned stamp, int which, int work) {
  const int txc = (int)(t / ((unsigned)m->ty * (unsigned)m->tz));
  if (txc < m->slab_lo || txc >= m->slab_hi) return;
  if (work) m->nb_flag[t] = stamp;
  if (m->tile_flag[t] != stamp) { m->tile_flag[t] = stamp; m->list[which][m->n_list[which]++] = t; }
}

#define MAXT 16
#define MAXBOX (MAXT + 4)
#define BIDX(bx, by, bz) (((bx) * BOX + (by)) * BOX + (bz))
#define VIDX(lx, ly, lz) (((lx) * T + (ly)) * T + (lz))

/* k_halo_retire: FRESH flags that E1 / E2 / E3 left in the ghost layers of a sharded map */
static void retire_halos(fm *m) {
  const long long per = (long long)m->gy * m->gz;
  const int x0 = m->slab_lo * m->T, x1 = m->slab_hi * m->T < m->gx ? m->slab_hi * m->T : m->gx;
  if (m->slab_lo > 0)
    for (long long k = (long long)(x0 - 2) * per; k < (long long)x0 * per; ++k) m->code[k] &= FM_MASK;
  if (m->slab_hi < m->tx)
    for (long long k = (long long)x1 * per; k < (long long)(x1 + 2) * per; ++k) m->code[k] &= FM_MASK;
}

/* E3 (k_wavefront): generations over the tiles queued for generation m->stamp in list 0 */
static void wavefront(fm *m, int flags, long long *st) {
  const int T = m->T, BOX = T + 4;
  const unsigned stamp0 = m->stamp;
  /* A queued voxel may skip its pull only while every value a neighbour holds has been offered to it.  That holds for a
   * map whose update box has always been the whole grid; once a relaxation ran under a smaller box, VoxInRange(new_pos)
   * (ESDFMap.cpp:351) withheld pushes to the voxels outside it, and from then on every queued voxel pulls. */
  const int pull_all = (flags & FM_FULL_PULL) || m->pull_all;
  unsigned cur = 0, gen = 0;
  static uint32_t V[MAXBOX * MAXBOX * MAXBOX], orig[MAXBOX * MAXBOX * MAXBOX], nv[MAXT * MAXT * MAXT];
  static unsigned char fresh[MAXBOX * MAXBOX * MAXBOX], upd[MAXT * MAXT * MAXT], pulls[MAXT * MAXT * MAXT], chg[MAXBOX * MAXBOX * MAXBOX];
  while (m->n_list[cur]) {
    const unsigned nwork = m->n_list[cur], stamp_cur = stamp0 + gen;
    m->n_changed = 0;
    for (unsigned w = 0; w < nwork; ++w) {
      const unsigned tile = m->list[cur][w];
      const int tzc = (int)(tile % (unsigned)m->tz), tyc = (int)((tile / (unsigned)m->tz) % (unsigned)m->ty), txc = (int)(tile / ((unsigned)m->tz * (unsigned)m->ty));
      const int x0 = txc * T, y0 = tyc * T, z0 = tzc * T;
      if (m->nb_flag[tile] != stamp_cur) {
        /* queued only by itself: retire the FRESH flags (through the staging copy) */
        for (int lx = 0; lx < T; ++lx)
          for (int ly = 0; ly < T; ++ly)
            for (int lz = 0; lz < T; ++lz)
              if (in_grid(m, x0 + lx, y0 + ly, z0 + lz)) { const long long ii = lin(m, x0 + lx, y0 + ly, z0 + lz); m->stage[ii] = m->code[ii] & FM_MASK; }
        m->changed[m->n_changed] = tile; m->changed_bb[m->n_changed] = 0; m->changed_need[m->n_changed] = 0; ++m->n_changed;
        ++st[2];
        continue;
      }
      ++st[1];
      for (int bx = 0; bx < BOX; ++bx)
        for (int by = 0; by < BOX; ++by)
          for (int bz = 0; bz < BOX; ++bz) {
            const int x = x0 - 2 + bx, y = y0 - 2 + by, z = z0 - 2 + bz;
            const uint32_t c = in_grid(m, x, y, z) ? m->code[lin(m, x, y, z)] : 0u;   /* outside the grid = never observed */
            V[BIDX(bx, by, bz)] = c & FM_MASK; orig[BIDX(bx, by, bz)] = c; fresh[BIDX(bx, by, bz)] = (unsigned char)(c >> 31);
          }
      for (int lx = 0; lx < T; ++lx)
        for (int ly = 0; ly < T; ++ly)
          for (int lz = 0; lz < T; ++lz) {
            const int v = VIDX(lx, ly, lz);
            const uint32_t c = V[BIDX(lx + 2, ly + 2, lz + 2)];
            /* unknown voxels are barriers (distance_ = -10000 is never > tmp, ESDFMap.cpp:382); only in-box voxels are queued */
            upd[v] = (unsigned char)(c != FM_UNKNOWN && in_range(m, x0 + lx, y0 + ly, z0 + lz));
            pulls[v] = (unsigned char)(pull_all || c == FM_INF);
          }
      for (;;) {                                          /* local Jacobi iterations */
        ++st[7];
        int listed = 0, any = 0;
        for (int lx = 0; lx < T; ++lx)
          for (int ly = 0; ly < T; ++ly)
            for (int lz = 0; lz < T; ++lz) {
              const int v = VIDX(lx, ly, lz), b = BIDX(lx + 2, ly + 2, lz + 2);
              nv[v] = V[b];
              if (!upd[v]) continue;
              const int x = x0 + lx, y = y0 + ly, z = z0 + lz;
              const int pull = pulls[v] && fresh[b];
              uint32_t best = V[b];
              unsigned bestd = best >= 2u ? dist2(best, x, y, z) : 0xffffffffu;
              int considered = 0;
              for (int k = 0; k < 24; ++k) {
                const int nb = BIDX(lx + 2 + KD[k][0], ly + 2 + KD[k][1], lz + 2 + KD[k][2]);
                if (!(pull || fresh[nb])) continue;       /* the neighbour's push (ESDFMap.cpp:375-391) or this voxel's pull (:349-367) */
                if (!in_range(m, x + KD[k][0], y + KD[k][1], z + KD[k][2])) continue;   /* VoxInRange(new_pos), :351 */
                considered = 1;
                ++st[9];
                const uint32_t c = V[nb];
                if (c >= 2u && c != best) {
                  const unsigned d = dist2(c, x, y, z);
                  if (d < bestd || (d == bestd && c < best)) { bestd = d; best = c; }   /* strict improvement; ties -> smallest coordinate */
                }
              }
              listed |= considered;
              st[8] += considered;
              nv[v] = best;
            }
        if (!listed) break;
        for (int lx = 0; lx < T; ++lx)
          for (int ly = 0; ly < T; ++ly)
            for (int lz = 0; lz < T; ++lz) {
              const int v = VIDX(lx, ly, lz), b = BIDX(lx + 2, ly + 2, lz + 2);
              const int c = nv[v] != V[b];
              any |= c;
              chg[b] = (unsigned char)c;
            }
        if (!any) break;
        for (int lx = 0; lx < T; ++lx)
          for (int ly = 0; ly < T; ++ly)
            for (int lz = 0; lz < T; ++lz) {
              const int v = VIDX(lx, ly, lz), b = BIDX(lx + 2, ly + 2, lz + 2);
              V[b] = nv[v]; fresh[b] = chg[b];             /* the queue of the next iteration */
            }
      }
      /* epilogue: what changed during this generation is FRESH for the next one */
      int nch = 0, dirty = 0, bb[6] = {T, -1, T, -1, T, -1};
      memset(chg, 0, sizeof(chg));
      for (int lx = 0; lx < T; ++lx)
        for (int ly = 0; ly < T; ++ly)
          for (int lz = 0; lz < T; ++lz) {
            const int b = BIDX(lx + 2, ly + 2, lz + 2);
            const int changed = V[b] != (orig[b] & FM_MASK);
            const uint32_t outw = V[b] | (changed ? FM_FRESH : 0u);
            if (changed) {
              ++nch; chg[b] = 1;
              bb[0] = lx < bb[0] ? lx : bb[0]; bb[1] = lx > bb[1] ? lx : bb[1];
              bb[2] = ly < bb[2] ? ly : bb[2]; bb[3] = ly > bb[3] ? ly : bb[3];
              bb[4] = lz < bb[4] ? lz : bb[4]; bb[5] = lz > bb[5] ? lz : bb[5];
            }
            if (outw != orig[b]) dirty = 1;
          }
      if (dirty) {
        for (int lx = 0; lx < T; ++lx)
          for (int ly = 0; ly < T; ++ly)
            for (int lz = 0; lz < T; ++lz)
              if (in_grid(m, x0 + lx, y0 + ly, z0 + lz)) {
                const int b = BIDX(lx + 2, ly + 2, lz + 2);
                m->stage[lin(m, x0 + lx, y0 + ly, z0 + lz)] = V[b] | (chg[b] ? FM_FRESH : 0u);
              }
        uint32_t need = 0;
        if (nch && (flags & FM_EXIT_TEST)) {
          /* Would any border voxel of a neighbouring tile (the halo of this box) improve from a record changed here?  Only
           * those records are in the queue next generation, the halo holds the neighbour's values, records only improve,
           * and a queued neighbour voxel is visited anyway -- so "no" is exact, not a heuristic. */
          for (int bx = 0; bx < BOX; ++bx)
            for (int by = 0; by < BOX; ++by)
              for (int bz = 0; bz < BOX; ++bz) {
                const int ox = bx < 2 ? -1 : bx > T + 1 ? 1 : 0, oy = by < 2 ? -1 : by > T + 1 ? 1 : 0, oz = bz < 2 ? -1 : bz > T + 1 ? 1 : 0;
                if (!ox && !oy && !oz) continue;
                const int dirbit = ((ox + 1) * 3 + (oy + 1)) * 3 + (oz + 1);
                if ((need >> dirbit) & 1u) continue;
                const int x = x0 - 2 + bx, y = y0 - 2 + by, z = z0 - 2 + bz;
                const uint32_t cy = V[BIDX(bx, by, bz)];
                if (cy == FM_UNKNOWN || !in_grid(m, x, y, z) || !in_range(m, x, y, z)) continue;
                const unsigned dy = cy >= 2u ? dist2(cy, x, y, z) : 0xffffffffu;
                for (int k = 0; k < 24; ++k) {
                  const int nx = bx + KD[k][0], ny = by + KD[k][1], nz = bz + KD[k][2];
                  if (nx < 2 || nx > T + 1 || ny < 2 || ny > T + 1 || nz < 2 || nz > T + 1) continue;      /* candidates: this tile's records */
                  if (!chg[BIDX(nx, ny, nz)]) continue;
                  const uint32_t c = V[BIDX(nx, ny, nz)];
                  if (c >= 2u && c != cy) {
                    const unsigned d = dist2(c, x, y, z);
                    if (d < dy || (d == dy && c < cy)) { need |= 1u << dirbit; break; }
                  }
                }
              }
        }
        m->changed[m->n_changed] = tile;
        m->changed_bb[m->n_changed] = nch ? ((unsigned)bb[0] | ((unsigned)bb[1] << 5) | ((unsigned)bb[2] << 10) | ((unsigned)bb[3] << 15) |
                                             ((unsigned)bb[4] << 20) | ((unsigned)bb[5] << 25) | (1u << 30)) : 0u;
        m->changed_need[m->n_changed] = need;
        ++m->n_changed;
        st[3] += nch;
      }
    }
    /* phase 2: commit, queue the neighbours for the next generation */
    m->n_list[cur] = 0;
    const unsigned stamp = stamp0 + gen + 1u;
    for (unsigned w = 0; w < m->n_changed; ++w) {
      const unsigned tile = m->changed[w], bbw = m->changed_bb[w];
      const int tzc = (int)(tile % (unsigned)m->tz), tyc = (int)((tile / (unsigned)m->tz) % (unsigned)m->ty), txc = (int)(tile / ((unsigned)m->tz * (unsigned)m->ty));
      for (int lx = 0; lx < T; ++lx)
        for (int ly = 0; ly < T; ++ly)
          for (int lz = 0; lz < T; ++lz)
            if (in_grid(m, txc * T + lx, tyc * T + ly, tzc * T + lz)) { const long long ii = lin(m, txc * T + lx, tyc * T + ly, tzc * T + lz); m->code[ii] = m->stage[ii]; }
      if (!(bbw >> 30)) continue;
      const int mnx = bbw & 31, mxx = (bbw >> 5) & 31, mny = (bbw >> 10) & 31, mxy = (bbw >> 15) & 31, mnz = (bbw >> 20) & 31, mxz = (bbw >> 25) & 31;
      for (int ox = -1; ox <= 1; ++ox)
        for (int oy = -1; oy <= 1; ++oy)
          for (int oz = -1; oz <= 1; ++oz) {
            const int nz = (ox != 0) + (oy != 0) + (oz != 0);
            if (nz == 0) activate(m, tile, stamp, (int)(cur ^ 1u), 0);       /* once more, only to retire the FRESH flags */
            if (nz != 1 && nz != 2) continue;                                /* no 3-D corner directions in dirs_ */
            int need = 1;
            if (ox < 0) need = need && (mnx < 2);
            if (ox > 0) need = need && (mxx > T - 3);
            if (oy < 0) need = need && (mny < 2);
            if (oy > 0) need = need && (mxy > T - 3);
            if (oz < 0) need = need && (mnz < 2);
            if (oz > 0) need = need && (mxz > T - 3);
            const int ax = txc + ox, ay = tyc + oy, az = tzc + oz;
            if (!(need && ax >= 0 && ax < m->tx && ay >= 0 && ay < m->ty && az >= 0 && az < m->tz)) continue;
            ++st[5];
            if ((flags & FM_EXIT_TEST) && !((m->changed_need[w] >> (((ox + 1) * 3 + (oy + 1)) * 3 + (oz + 1))) & 1u)) { ++st[6]; continue; }
            activate(m, (unsigned)((ax * m->ty + ay) * m->tz + az), stamp, (int)(cur ^ 1u), 1);
          }
    }
    cur ^= 1u;
    ++gen;
  }
  st[0] = gen;
  m->stamp = stamp0 + gen + 1u;
}

/* stats: 0 generations, 1 full visits, 2 retire-only visits, 3 changed records, 4 reset records, 5 neighbour activations
 * asked for by the bounding-box rule, 6 of those suppressed by the exit test, 7 local iterations, 8 voxel evaluations
 * (listed voxels summed over the iterations), 9 candidate records compared */
void fm_update(fm *m, const uint8_t *exist, const uint32_t *ins, long long n_ins, int have_del, int flags, long long *stats) {
  const int lg = m->lg;
  long long st[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  const unsigned stamp0 = m->stamp;
  m->n_list[0] = m->n_list[1] = 0;
  if ((n_ins > 0 || have_del) && !box_is_full(m)) m->pull_all = 1;   /* the box in force when the relaxation runs */
  /* E1 (ESDFMap.cpp:278-291) */
  for (long long i = 0; i < n_ins; ++i) {
    const uint32_t ii = ins[i];
    if (!exist[ii]) continue;
    const int z = (int)(ii % (unsigned)m->gz), y = (int)((ii / (unsigned)m->gz) % (unsigned)m->gy), x = (int)(ii / ((unsigned)m->gz * (unsigned)m->gy));
    m->code[ii] = pack(x, y, z) | FM_FRESH;
    const int tx0 = (x - 2 > 0 ? x - 2 : 0) >> lg, tx1 = (x + 2 < m->gx - 1 ? x + 2 : m->gx - 1) >> lg;
    const int ty0 = (y - 2 > 0 ? y - 2 : 0) >> lg, ty1 = (y + 2 < m->gy - 1 ? y + 2 : m->gy - 1) >> lg;
    const int tz0 = (z - 2 > 0 ? z - 2 : 0) >> lg, tz1 = (z + 2 < m->gz - 1 ? z + 2 : m->gz - 1) >> lg;
    for (int a = tx0; a <= tx1; ++a)
      for (int b = ty0; b <= ty1; ++b)
        for (int c = tz0; c <= tz1; ++c) activate(m, (unsigned)((a * m->ty + b) * m->tz + c), stamp0, 0, 1);
  }
  /* E2 (ESDFMap.cpp:292-337): dependants of deleted obstacles, found by a scan instead of the linked lists */
  if (have_del)
    for (int x = 0; x < m->gx; ++x)
      for (int y = 0; y < m->gy; ++y)
        for (int z = 0; z < m->gz; ++z) {
          const long long ii = lin(m, x, y, z);
          const uint32_t c = m->code[ii] & FM_MASK;
          if (c >= 2u) {
            int ox, oy, oz;
            unpack(c, &ox, &oy, &oz);
            if (!exist[lin(m, ox, oy, oz)]) {
              m->code[ii] = FM_INF | FM_FRESH;
              ++st[4];
              activate(m, (unsigned)(((x >> lg) * m->ty + (y >> lg)) * m->tz + (z >> lg)), stamp0, 0, 1);
            }
          }
        }
  wavefront(m, flags, st);
  retire_halos(m);
  if (stats) memcpy(stats, st, sizeof(st));
}

/* UpdateOccupancy(false) of a voxel outside the previous update box (ESDFMap.cpp:256-259, k_integrate<false>): distance_
 * +infinity_, not queued */
void fm_local_reset(fm *m, const uint32_t *idx, long long n) {
  for (long long i = 0; i < n; ++i) m->code[idx[i]] = FM_INF;
}

/* ---- x-slab sharding (fiesta_set_shard / fiesta_shard_pack / fiesta_shard_ingest / fiesta_shard_relax).  Layers are
 * gy*gz records in this model's own (unpadded) layout; only model instances exchange them. */
void fm_set_slab(fm *m, int tile_x_lo, int tile_x_hi) { m->slab_lo = tile_x_lo; m->slab_hi = tile_x_hi; }
void fm_pack(const fm *m, int x_first, int nlayers, uint32_t *out) {
  memcpy(out, m->code + (long long)x_first * m->gy * m->gz, (size_t)nlayers * m->gy * m->gz * 4);
}
/* k_halo_ingest: a received ghost record that differs from the local copy is taken over, marked FRESH (it pushes into the
 * slab next generation) and the own tiles of column own_tile_x within reach are queued.  Returns the changed records. */
long long fm_halo_ingest(fm *m, const uint32_t *recv, int x_first, int nlayers, int own_tile_x) {
  const long long per = (long long)m->gy * m->gz;
  long long n = 0;
  for (long long k = 0; k < per * nlayers; ++k) {
    const int y = (int)((k % per) / m->gz), z = (int)(k % m->gz);
    const long long ii = (long long)x_first * per + k;
    const uint32_t nw = recv[k] & FM_MASK;
    if (nw == (m->code[ii] & FM_MASK)) continue;
    m->code[ii] = nw | FM_FRESH;
    ++n;
    const int ty0 = (y - 2 > 0 ? y - 2 : 0) >> m->lg, ty1 = (y + 2 < m->gy - 1 ? y + 2 : m->gy - 1) >> m->lg;
    const int tz0 = (z - 2 > 0 ? z - 2 : 0) >> m->lg, tz1 = (z + 2 < m->gz - 1 ? z + 2 : m->gz - 1) >> m->lg;
    for (int b = ty0; b <= ty1; ++b)
      for (int c = tz0; c <= tz1; ++c) activate(m, (unsigned)((own_tile_x * m->ty + b) * m->tz + c), m->stamp, 0, 1);
  }
  return n;
}
/* fiesta_shard_relax: E3 over the tiles the ingests queued, then the ghost flags are retired */
void fm_relax(fm *m, int flags, long long *stats) {
  long long st[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (!box_is_full(m)) m->pull_all = 1;
  wavefront(m, flags, st);
  retire_halos(m);
  if (stats) memcpy(stats, st, sizeof(st));
}

/* closest_obstacle_ / distance_ in the reference's layout and value conventions (-10000 unknown, +10000 no obstacle) */
void fm_export(const fm *m, int32_t *cobs, double *dist, double res) {
  for (int x = 0; x < m->gx; ++x)
    for (int y = 0; y < m->gy; ++y)
      for (int z = 0; z < m->gz; ++z) {
        const long long ii = lin(m, x, y, z);
        const uint32_t c = m->code[ii] & FM_MASK;
        int ox = FM_UNDEFINED, oy = FM_UNDEFINED, oz = FM_UNDEFINED;
        double d = c == FM_UNKNOWN ? (double)FM_UNDEFINED : (double)FM_INFINITY;
        if (c >= 2u) {
          unpack(c, &ox, &oy, &oz);
          const double dx = (double)(ox - x), dy = (double)(oy - y), dz = (double)(oz - z);
          d = sqrt((dx * dx + dy * dy) + dz * dz) * res;
        }
        if (cobs) { cobs[3 * ii] = ox; cobs[3 * ii + 1] = oy; cobs[3 * ii + 2] = oz; }
        if (dist) dist[ii] = d;
      }
}
/* number of records of the slab and its ghost layers still carrying the FRESH bit (must be 0 between updates; records
 * further out are neither relaxed nor read by this map) */
long long fm_fresh_left(const fm *m) {
  const long long per = (long long)m->gy * m->gz;
  const int x0 = m->slab_lo * m->T - 2, x1 = m->slab_hi * m->T + 2;
  long long n = 0;
  for (long long i = (x0 > 0 ? x0 : 0) * per; i < (x1 < m->gx ? x1 : m->gx) * per; ++i) n += (m->code[i] >> 31);
  return n;
}
