// TEST INFRASTRUCTURE ONLY (design model, not shipped, not called by the product).
// CPU model of k_x_reseed (fiesta_b200/csrc/fb_xrelax.cu): the re-seeding of the dependants of deleted obstacles in four
// stages -- A classify, B validity closure, C choose, D resolve by pointer jumping.  It runs on every delete of every replay
// of oracle/exact_model.c (used as it stands) and is checked there against ONE sequential sweep of the reference's rule in
// dependant order (ESDFMap.cpp:308-321) and against exact_model.c's own re-seeding, which continues the replay:
//   gcc -O2 -ffp-contract=off -o /tmp/reseed_model scripts/reseed_model.c -lm
//   /tmp/reseed_model G obs rounds nops seed [small [local]]      (exact_model.c's arguments)
//   /tmp/reseed_model block G seed order local
// The random replays delete scattered obstacles, whose dependants lie within a few voxels of a static source: the closure
// rarely needs more than two rounds there.  `block` checks the stages alone on one synthetic delete that needs many: a
// G^3 grid, a wall of existing obstacles at x = G-3, and a block of dependants whose inside is more than two voxels from any
// non-dependant (5 % of the non-dependants hold no valid code).  order 0: the dependants from the block's surface inwards
// (deep closure, long parent chains), 1: from the inside out (the inner ones first), 2: random.  local 1: an update box
// that cuts the block.
// The hook into exact_model.c needs its main() to hold the dependants, their count, the voxel -> position array and its
// re-seeded codes in locals named deps, ndep, ord and nc0 at the call of fiesta_oracle_update_esdf(O); a rename there is a
// compile error here, and a replay in which the hook no longer runs reports "deletes 0", which tests/test_reseed_model.py
// rejects.
// The items of a stage run one after the other in a random order and update the arrays in place, which is one legal
// interleaving of the kernel's threads.  The last line is "reseed OK" or "reseed FAIL" with the totals over the replay.
// Built with one of these, the model is wrong in a way the replays must catch:
//   -DMUT_B_ANY_ORDER  B also marks the dependant neighbours that come BEFORE the newly valid one
//   -DMUT_C_LAST       C takes the last masked valid neighbour instead of the first in dirs_ order
//   -DMUT_C_STATIC     C keeps the static source even where an earlier direction holds a valid dependant
//   -DMUT_D_SHORT      D stops one pass early
#include <stdio.h>
#include <stdlib.h>
static void reseed_check(const void *deps, long ndep, const unsigned *ord, const unsigned *nc);
// exact_model.c's main() becomes exact_model_main(); its call of fiesta_oracle_update_esdf(O), which follows its own
// re-seeding, first runs reseed_check() on that delete's dependants (the macro sees main's locals); the definition of the
// oracle function becomes fiesta_oracle_update_esdf_real()
#define main exact_model_main
#define fiesta_oracle_update_esdf(...) FOUE_##__VA_ARGS__)
#define FOUE_void fiesta_oracle_update_esdf_real(void
#define FOUE_O reseed_check(deps, ndep, ord, nc0), fiesta_oracle_update_esdf_real(O
#include "../oracle/exact_model.c"
#undef main

#define R_STATIC 0x20000000u
#define R_VALID 0x40000000u
#define R_PAR 0x80000000u
static const u32 *RORD;                // voxel -> dependant position, or NONE
static long rs_deletes = 0, rs_deps = 0, rs_final_a = 0, rs_rounds_max = 0, rs_passes_max = 0, rs_bad = 0;

static void shuffle_l(long *a, long n) { for (long i = n - 1; i > 0; i--) { long j = rand() % (i + 1), t = a[i]; a[i] = a[j]; a[j] = t; } }
// the dependant at the in-grid, in-box neighbour k of voxel u, else NONE (*n: the voxel, -1 outside)
static u32 dep_at(long u, int k, long *n) {
  int x, y, z; vxyz(u, &x, &y, &z);
  int nx = x + DIRS[k][0], ny = y + DIRS[k][1], nz = z + DIRS[k][2];
  if (!ing(nx, ny, nz) || !inb(nx, ny, nz)) { *n = -1; return NONE; }
  *n = vi(nx, ny, nz);
  return RORD[*n];
}

static void reseed_check(const void *dv, long ndep, const unsigned *ord_, const unsigned *nc_fix) {
  const dep_t *deps = dv;
  RORD = ord_;
  if (!ndep) return;
  rs_deletes++; rs_deps += ndep;
  // the reference's rule, one sweep in dependant order
  u32 *sw = malloc(4 * ndep), *nc = malloc(4 * ndep), *M = malloc(4 * ndep);
  for (long i = 0; i < ndep; i++) {
    u32 res = CI;
    for (int k = 0; k < 24; k++) {
      long n; u32 o = dep_at(deps[i].v, k, &n), c;
      if (n < 0) continue;
      if (o != NONE) { if (o < (u32)i) c = sw[o]; else continue; } else c = C[n];
      if (c >= 2 && existc(c)) { res = c; break; }
    }
    sw[i] = res;
  }
  long *L = malloc(sizeof(long) * ndep), *L2 = malloc(sizeof(long) * ndep), nl = 0, nl2;
  for (long i = 0; i < ndep; i++) L[i] = i;
  shuffle_l(L, ndep);
  // A classify
  for (long q = 0; q < ndep; q++) {
    long i = L[q]; u32 mask = 0, sc = CI; int st = 0;
    for (int k = 0; k < 24 && !st; k++) {
      long n; u32 o = dep_at(deps[i].v, k, &n);
      if (n < 0) continue;
      if (o != NONE) { if (o < (u32)i) mask |= 1u << k; }
      else if (C[n] >= 2 && existc(C[n])) { sc = C[n]; st = 1; }
    }
    nc[i] = sc; M[i] = mask | (st ? R_STATIC | R_VALID : 0u);
    if (!mask) rs_final_a++;
  }
  // B closure: round 1 pulls, later rounds push from the dependants made valid in the round before
  nl = 0;
  for (long i = 0; i < ndep; i++) if (!(M[i] & R_STATIC) && (M[i] & 0xffffffu)) L[nl++] = i;
  long rounds = 0;
  for (int r = 1; nl; r++) {
    rounds++; shuffle_l(L, nl); nl2 = 0;
    for (long q = 0; q < nl; q++) {
      long i = L[q];
      if (r == 1) {
        int any = 0;
        for (int k = 0; k < 24; k++) if ((M[i] >> k) & 1u) { long n; u32 o = dep_at(deps[i].v, k, &n); if (M[o] & R_VALID) any = 1; }
        if (any) { M[i] |= R_VALID; L2[nl2++] = i; }
      } else {
        int x, y, z; vxyz(deps[i].v, &x, &y, &z);
        if (!inb(x, y, z)) continue;                           // later dependants see i only inside the box
        for (int k = 0; k < 24; k++) {
          int nx = x + DIRS[k][0], ny = y + DIRS[k][1], nz = z + DIRS[k][2];
          if (!ing(nx, ny, nz)) continue;
          u32 j = RORD[vi(nx, ny, nz)];
#ifdef MUT_B_ANY_ORDER
          int later = j != NONE && j != (u32)i;
#else
          int later = j != NONE && j > (u32)i;
#endif
          if (later && !(M[j] & (R_STATIC | R_VALID))) { M[j] |= R_VALID; L2[nl2++] = j; }
        }
      }
    }
    long *t = L; L = L2; L2 = t; nl = nl2;
  }
  // C choose
  nl = 0;
  for (long i = 0; i < ndep; i++) L[i] = i;
  shuffle_l(L, ndep);
  for (long q = 0; q < ndep; q++) {
    long i = L[q];
    if (!(M[i] & R_VALID) || !(M[i] & 0xffffffu)) continue;
#ifdef MUT_C_STATIC
    if (M[i] & R_STATIC) continue;
#endif
    for (int k = 0; k < 24; k++) if ((M[i] >> k) & 1u) {
      long n; u32 o = dep_at(deps[i].v, k, &n);
      if (M[o] & R_VALID) {
        nc[i] = R_PAR | o;
#ifndef MUT_C_LAST
        break;
#endif
      }
    }
  }
  for (long i = 0; i < ndep; i++) if (nc[i] & R_PAR) L[nl++] = i;
  // D resolve, in place
  long passes = 0;
  u32 *before = malloc(4 * ndep);
  while (nl) {
    passes++; shuffle_l(L, nl); nl2 = 0;
    memcpy(before, nc, 4 * ndep);
    for (long q = 0; q < nl; q++) { long i = L[q]; nc[i] = nc[nc[i] & ~R_PAR]; if (nc[i] & R_PAR) L2[nl2++] = i; }
    long *t = L; L = L2; L2 = t; nl = nl2;
  }
#ifdef MUT_D_SHORT
  if (passes) memcpy(nc, before, 4 * ndep);
#endif
  if (rounds > rs_rounds_max) rs_rounds_max = rounds;
  if (passes > rs_passes_max) rs_passes_max = passes;
  long bad = 0, bad_fix = 0;
  for (long i = 0; i < ndep; i++) { bad += nc[i] != sw[i]; bad_fix += nc_fix && nc_fix[i] != sw[i]; }
  if (bad || bad_fix) { printf("reseed mismatch: %ld dependants, %ld differ from the sweep (fixpoint: %ld)\n", ndep, bad, bad_fix); rs_bad++; }
  free(sw); free(nc); free(M); free(L); free(L2); free(before);
}

// one synthetic delete (see the header): returns what exact_model_main() would for a replay without mismatches
static int block_main(int G, int seed, int order, int local) {
  srand(seed);
  double org[3] = {0, 0, 0}, sz[3] = {G * 0.1 - 0.05, G * 0.1 - 0.05, G * 0.1 - 0.05};
  O = fiesta_oracle_create(org, 0.1, sz); fiesta_oracle_set_parameters(O, 0.97, 0.03, 0.30, 0.90, 0.80);
  GX = O->gs[0]; GY = O->gs[1]; GZ = O->gs[2]; N = (long)GX * GY * GZ; C = calloc(N, 4);
  u32 *ordv = malloc(4 * N);
  dep_t *deps = malloc(sizeof(dep_t) * N);
  double *key = malloc(sizeof(double) * N);
  long ndep = 0;
  const int lo[3] = {4, 6, 6}, hi[3] = {G - 10, G - 7, G - 7};
  for (long v = 0; v < N; v++) {
    int x, y, z; vxyz(v, &x, &y, &z);
    O->occ[v] = x == GX - 3 ? 5.0 : -5.0;                     // occupied iff above l_occ
    ordv[v] = NONE;
    if (x >= lo[0] && x <= hi[0] && y >= lo[1] && y <= hi[1] && z >= lo[2] && z <= hi[2]) {
      int d = x - lo[0], t;
      const int e[5] = {hi[0] - x, y - lo[1], hi[1] - y, z - lo[2], hi[2] - z};
      for (t = 0; t < 5; t++) if (e[t] < d) d = e[t];
      key[ndep] = (order == 2 ? 0 : order == 0 ? d : -d) + (rand() % 1000) / 1000.0;   // random within a shell
      deps[ndep].v = (u32)v; deps[ndep].k1 = deps[ndep].k2 = 0; ndep++;
      C[v] = CI;
    } else {
      const int u = rand() % 40;
      C[v] = u == 0 ? CU : u == 1 ? CI : pack(GX - 3, y, z);
    }
  }
  for (long i = 0; i < ndep; i++) deps[i].k1 = (u64)((key[i] + 1000.0) * 1e6);
  qsort(deps, ndep, sizeof(dep_t), cmpdep);
  for (long i = 0; i < ndep; i++) ordv[deps[i].v] = (u32)i;
  if (local) { O->max_vec[0] = (lo[0] + hi[0]) / 2; O->min_vec[1] = lo[1] + 3; }
  reseed_check(deps, ndep, ordv, NULL);
  free(ordv); free(deps); free(key); free(C);
  return 0;
}

int main(int argc, char **argv) {
  int rc = argc > 5 && !strcmp(argv[1], "block") ? block_main(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5])) : exact_model_main(argc, argv);
  printf("reseed %s: deletes %ld dependants %ld final after classify %ld closure rounds max %ld resolve passes max %ld\n",
         rs_bad ? "FAIL" : "OK", rs_deletes, rs_deps, rs_final_a, rs_rounds_max, rs_passes_max);
  return rc || rs_bad;
}
