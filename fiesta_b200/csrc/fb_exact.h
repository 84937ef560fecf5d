// fiesta_b200 -- host interface of the order-exact mode (fb_exact.cu: ordered UpdateOccupancy, insert / delete seeding;
// fb_xrelax.cu: the persistent relaxation kernel).
#pragma once
#include "fb_common.cuh"

#define FB_X_MAX_BLOCKS 256
#define FB_X_SMALL_DEFAULT 32768u   // (from a sweep on the 512^3 LIDAR frames; FIESTA_X_SMALL / FIESTA_X_DENSE override)
// Trace layout of k_x_reseed and k_x_relax (FIESTA_DEBUG_X): [3 * FB_XDBG_GENS] per generation {nE, rounds, cycles};
// FB_XDBG_NCAT x {cycles, count} per phase category (re-seeding: 12 classify, 20 closure, 21 choose, 22 resolve, 13 assemble;
// the counts of 20 and 22 are the closure rounds and the resolve passes; 15 holds the dependants final after the
// classification and the summed closure list lengths instead); 2 x 512 work-list sizes per round (first two generations);
// 4096 per-round slots for the longest CTA work time of the round (cycles, reset once added up); FB_XDBG_NCAT x {summed longest CTA work time, summed list
// length} per round category; 2 x 32 log2 histograms of the list lengths of later rounds (the first retired, the second
// SMALL generations'); FB_XDBG_NQ counters of the asynchronous schedule.  Categories 2 and 19 are retired (BIG short-list
// rounds, SMALL generations from the work queue); their slots stay so that the offsets do not move.
#define FB_XDBG_GENS 1024
#define FB_XDBG_NCAT 24
#define FB_XDBG_NQ 8
#define FB_XDBG_PHASE (3 * FB_XDBG_GENS)
#define FB_XDBG_ROUNDS (FB_XDBG_PHASE + 2 * FB_XDBG_NCAT)
#define FB_XDBG_WMAX (FB_XDBG_ROUNDS + 2 * 512)
#define FB_XDBG_WORK (FB_XDBG_WMAX + 4096)
#define FB_XDBG_NWH (FB_XDBG_WORK + 2 * FB_XDBG_NCAT)
#define FB_XDBG_Q (FB_XDBG_NWH + 2 * 32)
#define FB_X_DBG_WORDS (FB_XDBG_Q + FB_XDBG_NQ)

struct FbExactStats {
  unsigned long long expansions;      // == the reference's "Expanding N nodes" (ESDFMap.cpp:347,394)
  unsigned long long voxels_changed;  // accepted final writes over all generations
  unsigned generations, eval_rounds, dense_rounds, dependants;
  unsigned reseed_rounds;             // re-seeding of the dependants (k_x_reseed): closure rounds + pointer-jumping passes
};

// Control block of k_x_relax (device memory; the host writes it before and reads it after every launch).
struct FbXCtl {
  unsigned bar, err;                  // grid barrier arrivals; 1 = a generation exceeded 2^27 entries
  unsigned sclock;                    // stamp of the last summary pass (SUMg dedupe; persists across launches)
  unsigned rbar;                      // grid barrier arrivals of k_x_reseed
  unsigned nE0;                       // entries of generation 0: the insert seeds, plus the re-seeded dependants k_x_reseed appends
  unsigned nW[3], nF[3];              // work / flip list lengths, rotating per round
  unsigned gen_id, wclock;            // stamps for SUMg / wstamp dedupe (persist across launches)
  unsigned generations, rounds, dense_rounds, reseed_rounds;
  unsigned long long tclock, expansions, voxels_changed;
  unsigned partial[FB_X_MAX_BLOCKS];  // winners per CTA range (ordered hand-over)
  // work queue of the asynchronous schedule (one line each: the first two take every push / pop, the third is polled)
  alignas(128) unsigned long long qtail;  // {outstanding items + warps still seeding : 32 | pushes so far : 32}
  alignas(128) unsigned qhead;            // pops reserved so far
  alignas(128) unsigned qdone;            // 1 once the outstanding count reached zero (or a wait exceeded its bound)
};

// Order-exact state of one map.  Zero until fb_exact_init; freed with the map.
struct FbExact {
  FbDevBuf<unsigned long long> MB;    // per voxel: {parity | queue position | behaviour | code} of its live entry in the current generation
  FbDevBuf<unsigned long long> LS;    // per voxel: time of the last relink into a dependant list
  FbDevBuf<unsigned long long> tkey;  // per voxel: epoch-coded serial time of the first pending observation (fb_touch, fb_common.cuh)
  FbDevBuf<uint32_t> touched;         // [ptotal] staging of the voxels whose occupancy crossed the threshold (inserts; deletes use emask)
  unsigned long long tclock = 0;      // relink clock
  unsigned long long key_base = 0;    // observation clock within the current integration epoch
  unsigned long long key_hi = 0;      // key_epoch << FB_KEY_BITS
  unsigned key_epoch = 0;             // integration epoch (one per UpdateOccupancy)
  FbDevBuf<unsigned> d_count, d_flag;
  FbHostBuf<unsigned> h_count;
  bool scratch_clean = false;         // the per-voxel scratch word array of UpdateESDF is all-XNONE
  FbDevBuf<uint4> SUM;                // per voxel offer summary of the current generation: {first ts, best ts, best code, snapshot code}
  FbDevBuf<uint32_t> SUMg;            // per voxel: summary pass for which SUM was computed (each target is claimed once per pass)
  unsigned gen_id = 0, wclock = 0, sclock = 0;
  FbDevBuf<uint32_t> emask;           // per entry: slots it owns in the next generation
  FbDevBuf<uint32_t> W[3], F[3];      // work lists / flip lists, rotating per round
  FbDevBuf<uint32_t> wstamp;          // per entry: round for which it is already in a work list
  FbDevBuf<uint32_t> slotc;           // SMALL generations: codes of the owned slots
  unsigned dense_min = 0;             // work lists longer than this are evaluated through refreshed summaries (one wave of warps)
  unsigned small_max = 0;             // generations up to this many entries run without summaries
  FbDevBuf<FbXCtl> d_ctl;
  FbHostBuf<FbXCtl> h_ctl;
  FbDevBuf<unsigned long long> d_dbg;
  int relax_blocks = 0;
  FbDevBuf<uint32_t> E[2], sel;
  FbDevBuf<unsigned long long> k1, k2, k1b, k2b;
  FbDevBuf<uint32_t> dv, idx[2], deps, nc[2];
  FbDevBuf<uint8_t> flags;
  FbDevBuf<char> cub_tmp;
};

// Host functions return FIESTA_OK or a FIESTA_ERR_* code and set fiesta_last_error().
int fb_exact_init(FbExact *X, const FbGeom &g, int device, cudaStream_t s);
int fb_exact_queue_crossings(FbExact *X, const unsigned long long *ins_key, const uint32_t *ins_vox, const unsigned long long *del_key,
                             const uint32_t *del_vox, FbDevBuf<uint32_t> &ins, unsigned *n_ins, FbDevBuf<uint32_t> &del, unsigned *n_del,
                             cudaStream_t s, int *launches);
int fb_exact_next_epoch(FbExact *X, const FbGeom &g, cudaStream_t s);
int fb_exact_update_esdf(FbExact *X, const FbGeom &g, uint32_t *cobs, uint32_t *scratch, const double *occ, const uint32_t *occbits, double l_occ,
                         const uint32_t *ins, unsigned n_ins, const uint32_t *del, unsigned n_del, cudaStream_t s, FbExactStats *st, int *launches);
// fb_xrelax.cu
cudaError_t fb_xrelax_init();
int fb_xrelax_blocks(int device);
cudaError_t fb_xrelax_launch(FbExact *X, const FbGeom &g, uint32_t *cobs, const uint32_t *deps, unsigned ndep, uint32_t *ord, uint32_t *nc, uint32_t *M,
                             const uint32_t *occbits, unsigned long long ls_deps, unsigned long long *dbg, cudaStream_t s);
