// TEST INFRASTRUCTURE ONLY (design model, not shipped, not called by the product).
// The CPU model of k_x_relax (oracle/exact_model.c) with the asynchronous schedule of fb_xrelax.cu's x_async added: the
// same replays, checked against the sequential oracle in the same process, voxel for voxel and expansion for expansion.
//   gcc -O2 -ffp-contract=off -o /tmp/exact_async_model scripts/exact_async_model.c -lm
//   /tmp/exact_async_model WORKERS G obs rounds nops seed [small [local [dense_min]]]
// (the arguments after WORKERS are exact_model.c's).  WORKERS = 0 runs exact_model.c's round schedule unchanged.
// Built with -DNO_DIRTY_RULE, a running element that gets marked is not evaluated again (a mutation the replays must catch).
//
// In BIG generations the first work list of at most dense_min entries after round 1 is not evaluated in rounds: it seeds a
// queue; every later round before it is dense.  SMALL generations keep their rounds.  Each element is IDLE, PENDING
// (queued), RUNNING or DIRTY (running, and an input flipped since it was marked running).  WORKERS simulated workers take
// steps, one at a time, chosen at random:
//   pop    take a random queued element, PENDING -> RUNNING;
//   read   evaluate it from the current words (the kernel's stage);
//   store  write its word if it flipped, and record the flip;
//   list   for every later element it can touch: IDLE -> PENDING and push, RUNNING -> DIRTY, otherwise nothing;
//   finish DIRTY -> RUNNING and read again, else RUNNING -> IDLE.
// Other workers' steps fall between a read and its store, so evaluations from stale words happen and must be repaired
// by the DIRTY rule.  Once the queue is empty and every worker waits, the generation refreshes the summaries of every flip
// since the last refresh (last round's and every flip of the queue, repeats included) with exact_model.c's
// refresh_targets rule, in random order, exactly once each; the commit then reads the summaries.  The run prints, over
// all queue phases, evaluations per seeded entry, dirty re-runs and the longest chain of dependent evaluations (an
// evaluation's depth is one more than the deepest evaluation whose word it read).
#include <stdlib.h>
static void relax_dispatch(void);
// exact_model.c is used as it stands: its main() becomes exact_model_main(), and its relax() becomes relax_void(), while
// the call inside exact_model_main() becomes relax_dispatch()
#define main exact_model_main
#define relax(...) relax_##__VA_ARGS__(void)
#define relax_(x) relax_dispatch()
#include "../oracle/exact_model.c"
#undef main
#undef relax

static int WORKERS = 8;
static long a_phases = 0, a_seeds = 0, a_evals = 0, a_dirty = 0, a_maxchain = 0, a_refreshed = 0;
enum { A_IDLE = 0, A_PEND, A_RUN, A_DIRTY };
static unsigned char *astate; static u32 *adepth; static u32 *bag; static long nbag;
typedef struct { int step; u32 i, depth; u64 nb, old; } worker_t;
#define MAXW 64

static void a_mark(u32 j) {
  if (astate[j] == A_IDLE) { astate[j] = A_PEND; bag[nbag++] = j; }
#ifndef NO_DIRTY_RULE
  else if (astate[j] == A_RUN) astate[j] = A_DIRTY;
#endif
}
// depth of an evaluation of element i from the current words: one more than the deepest earlier element it reads
static u32 a_depth(u32 i) {
  long p = E[cur][i]; int x, y, z; vxyz(p, &x, &y, &z); u32 d = 0;
  for (int o = 0; o < nOFF; o++) {
    int nx = x + OFF[o][0], ny = y + OFF[o][1], nz = z + OFF[o][2]; if (!ing(nx, ny, nz)) continue;
    u64 w = MB[vi(nx, ny, nz)]; if (w == MB_NONE) continue; u32 j = mb_idx(w);
    if (j < i && adepth[j] > d) d = adepth[j];
  }
  return d + 1;
}
// the rest of a BIG generation's fixpoint from the nw elements of wl; every flip is recorded in F[fout]
static void async_phase(u32 *wl, long nw, int fout) {
  a_phases++; a_seeds += nw;
  memset(astate, 0, (size_t)nE); memset(adepth, 0, 4 * (size_t)nE); nbag = 0;
  for (long q = 0; q < nw; q++) a_mark(wl[q]);
  int nwk = 1 + rand() % WORKERS; worker_t wk[MAXW];
  for (int k = 0; k < nwk; k++) wk[k].step = 0;
  for (;;) {
    int en[MAXW], ne = 0;
    for (int k = 0; k < nwk; k++) if (wk[k].step != 0 || nbag > 0) en[ne++] = k;
    if (!ne) break;                                            // queue empty and every worker waiting: quiescence
    worker_t *w = &wk[en[rand() % ne]];
    for (int t = 0; t < 8 && w->step == 2; t++) w = &wk[en[rand() % ne]];   // stores lag behind: more reads of stale words
    long p;
    switch (w->step) {
      case 0:
        if (nbag == 0) break;                                                           // waits for the queue
        { long q = rand() % nbag; w->i = bag[q]; bag[q] = bag[--nbag]; astate[w->i] = A_RUN; w->step = 1; }
        break;
      case 1: w->nb = eval(w->i, 0); w->depth = a_depth(w->i); a_evals++; totevals++; w->step = 2; break;
      case 2:
        p = E[cur][w->i]; w->old = MB[p];
        if (w->nb != w->old) {
          MB[p] = w->nb; adepth[w->i] = w->depth; if (w->depth > a_maxchain) a_maxchain = w->depth;
          if (nF[fout] < N) F[fout][nF[fout]] = w->i;
          nF[fout]++;
          w->step = 3;
        } else w->step = 4;
        break;
      case 3: {
        int wide = mb_kind(w->old) == K_PUSH || mb_kind(w->nb) == K_PUSH; int x, y, z; vxyz(E[cur][w->i], &x, &y, &z);
        for (int o = 0; o < (wide ? nOFF : 25); o++) {
          int nx = x + OFF[o][0], ny = y + OFF[o][1], nz = z + OFF[o][2]; if (!ing(nx, ny, nz)) continue;
          u64 ww = MB[vi(nx, ny, nz)]; if (ww == MB_NONE) continue; u32 j = mb_idx(ww);
          if (j > w->i) a_mark(j);
        }
        w->step = 4; break;
      }
      case 4:
        if (astate[w->i] == A_DIRTY) { astate[w->i] = A_RUN; a_dirty++; w->step = 1; }
        else { astate[w->i] = A_IDLE; w->step = 0; }
        break;
    }
  }
}
static void relax_async(void) {
  int big = nE > SMALL;
  for (long i = 0; i < nE; i++) MB[E[cur][i]] = mbw((u32)i, K_PUSH, C[E[cur][i]]);
  while (nE) {
    totgens++;
    if (big) { sclock++; u32 *ord = malloc(4 * (nE + 1)); for (long i = 0; i < nE; i++) ord[i] = (u32)i; shuffle(ord, nE); for (long q = 0; q < nE; q++) claim_summaries(ord[q]); free(ord); }
    int rounds = 0; nW[0] = nW[1] = nW[2] = 0; nF[0] = nF[1] = nF[2] = 0;
    for (int r = 1;; r++) {
      int in = r % 3, out = (r + 1) % 3; nW[(r + 2) % 3] = 0; nF[(r + 2) % 3] = 0; wclock++;
      long nw; u32 *wl = W[in];
      if (r == 1) { nw = nE; for (long i = 0; i < nE; i++) wl[i] = (u32)i; } else nw = nW[in];
      long nf = (big && r > 1) ? nF[in] : 0;
      if (r > 1 && nw == 0 && nf == 0) break;
      rounds++;
      if (big && r > 1 && nw <= DENSE_MIN) {
        async_phase(wl, nw, out);
        long nfa = nF[out];                                    // one refresh of every flip since the last one, in random order
        if (nfa > N) { sclock++; for (long i = 0; i < nE; i++) claim_summaries(i); }
        else {
          u32 *ord = malloc(4 * (nf + nfa + 1)); for (long q = 0; q < nf; q++) ord[q] = F[in][q]; for (long q = 0; q < nfa; q++) ord[nf + q] = F[out][q];
          shuffle(ord, nf + nfa); for (long q = 0; q < nf + nfa; q++) refresh_targets(ord[q]); a_refreshed += nf + nfa; free(ord);
        }
        break;
      }
      int dense = big && r > 1;
      if (dense) { totdense++;
        if (nf < nE / 4) { for (long q = 0; q < nf; q++) refresh_targets(F[in][q]); } else { sclock++; for (long i = 0; i < nE; i++) claim_summaries(i); } }
      u32 *ord = malloc(4 * (nw + 1)); for (long q = 0; q < nw; q++) ord[q] = (u32)q; shuffle(ord, nw);
      for (long q = 0; q < nw; q++) {
        long i = wl[ord[q]]; totevals++;
        u64 nb = eval(i, big); long p = E[cur][i];
        if (nb != MB[p]) { int wide = mb_kind(MB[p]) == K_PUSH || mb_kind(nb) == K_PUSH;
          MB[p] = nb; if (big) F[out][nF[out]++] = (u32)i;
          int x, y, z; vxyz(p, &x, &y, &z);
          for (int o = 0; o < (wide ? nOFF : 25); o++) { int nx = x + OFF[o][0], ny = y + OFF[o][1], nz = z + OFF[o][2]; if (!ing(nx, ny, nz)) continue; u64 w = MB[vi(nx, ny, nz)]; if (w == MB_NONE) continue; u32 j = mb_idx(w);
            if (j > (u32)i && wstamp[j] != wclock) { wstamp[j] = wclock; W[out][nW[out]++] = j; } } } }
      free(ord);
      if (rounds > 100000) { printf("no convergence\n"); exit(1); } }
    totrounds += rounds; if (rounds > maxrounds) maxrounds = rounds;
    // commit and apply: as exact_model.c's relax()
    long total = 0;
    for (long i = 0; i < nE; i++) { u64 b = MB[E[cur][i]]; u32 m = 0; long p = E[cur][i]; int x, y, z; vxyz(p, &x, &y, &z);
      if (mb_kind(b) != K_DEAD) expansions++;
      if (mb_kind(b) == K_PUSH) { for (int k = 0; k < 24; k++) { int nx = x + DIRS[k][0], ny = y + DIRS[k][1], nz = z + DIRS[k][2]; if (!ing(nx, ny, nz) || !inb(nx, ny, nz)) continue; u32 ts = (u32)i * 32 + k;
          if (big) { sum_t u = SUM[vi(nx, ny, nz)]; if (u.best_ts == ts) m |= 1u << k; } else { st_t f = gather(nx, ny, nz, NONE, NULL); if (f.ts == ts) { m |= 1u << k; slotc[i * 32 + k] = f.c; } } } }
      else if (mb_kind(b) == K_PULL) { u32 ts = (u32)i * 32 + 24; if (big) { sum_t u = SUM[p]; if (u.best_ts == ts) m |= 1u << 24; } else { st_t f = gather(x, y, z, NONE, NULL); if (f.ts == ts) { m |= 1u << 24; slotc[i * 32 + 24] = f.c; } } }
      emask[i] = m; total += __builtin_popcount(m); }
    for (long i = 0; i < nE; i++) MB[E[cur][i]] = MB_NONE;
    int big2 = total > SMALL; long r = 0;
    for (long i = 0; i < nE; i++) { long p = E[cur][i]; int x, y, z; vxyz(p, &x, &y, &z); u32 m = emask[i];
      for (int k = 0; k < 25; k++) if (m >> k & 1) { int nx = k < 24 ? x + DIRS[k][0] : x, ny = k < 24 ? y + DIRS[k][1] : y, nz = k < 24 ? z + DIRS[k][2] : z; long v = vi(nx, ny, nz);
          u32 c = big ? SUM[v].best_c : slotc[i * 32 + k]; C[v] = c; LS[v] = tclock + (u64)i * 32 + k; E[cur ^ 1][r] = (u32)v; MB[v] = mbw((u32)r, K_PUSH, c); r++; } }
    tclock += (u64)nE * 32 + 1; nE = r; cur ^= 1; big = big2;
  }
}
static void relax_dispatch(void) {
  if (!WORKERS) { relax_void(); return; }
  if (!astate) { astate = calloc((size_t)N, 1); adepth = calloc((size_t)N, 4); bag = malloc(4 * (size_t)N); }
  relax_async();
}
int main(int argc, char **argv) {
  if (argc < 2) { fprintf(stderr, "usage: %s WORKERS [exact_model.c arguments]\n", argv[0]); return 2; }
  WORKERS = atoi(argv[1]);
  if (WORKERS < 0 || WORKERS > MAXW) { fprintf(stderr, "WORKERS: 0..%d\n", MAXW); return 2; }
  argv[1] = argv[0];
  const int rc = exact_model_main(argc - 1, argv + 1);
  printf("async: workers <= %d, phases %ld, seeded entries %ld, evaluations %ld (%.2f per seeded entry), dirty re-runs %ld, "
         "longest chain of dependent evaluations %ld, flips refreshed %ld\n", WORKERS, a_phases, a_seeds, a_evals,
         a_seeds ? (double)a_evals / a_seeds : 0.0, a_dirty, a_maxchain, a_refreshed);
  return rc;
}
