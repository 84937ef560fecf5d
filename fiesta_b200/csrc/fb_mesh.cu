// fiesta_b200 -- surface mesh kernels (definition: fb_mesh.h, DESIGN.md §3.15).
//
// Everything runs on a bitmap over the extended box E = [lo - 1, hi]: z-rows of W = ceil((Bz+1) / 32) words, word j = (ex *
// (By+1) + ey) * W + k holding the positions ez = 32k .. 32k + 31 (ex, ey, ez: E-local coordinates).  The virtual layer (ex, ey or
// ez = 0) and the padding bits past ez = Bz are zeros, and rows past E read as zeros, which is the "outside B never blocks" rule.
// k_mesh_classify : one warp per word, one lane per position: fb_seg_blocks on B's records, __ballot_sync -> bits.  Lanes read
//                   consecutive records of one z-row: a coalesced streaming pass.
// k_mesh_count    : one thread per word, from that word and the words at z+1, y+1, x+1 (and x+1, y+1): the active-cell bits (kept,
//                   for the vertex ranks of the faces), the vertex count and the quad count (the three sign-changing-edge bit sets).
// (CUB)           : exclusive scans of the counts (uint32 vertex ranks, int64 quad ranks) over nw + 1 words: the totals at [nw].
// k_mesh_vertices : one warp per word, one lane per active cell: the 8 corner records -> fb_mesh_vertex -> float32 xyz at its rank.
// k_mesh_faces    : one warp per word, one lane per position, up to three sign-changing edges per lane: the four cells' vertex ids
//                   (the word's prefix plus the popcount of the masked active word), their positions, fb_mesh_split02 -> two
//                   triangles at 2 * the quad's rank.
// Every output position is a rank given by scans and popcounts: no atomic decides anything, and the bits are the same on every run.
#include <cub/cub.cuh>
#include "fb_map.h"
#include "fb_mesh.h"
#include "fb_nav.h"       // FbNavBox: the box layout of the other planner handles
#include "fb_segment.h"   // fb_seg_blocks

struct FbMeshCtr {
  unsigned long long blocking;
  unsigned vertices;              // vpre[nw]
  unsigned pad;
  long long quads;                // qpre[nw]
};
struct FbMeshBufs {               // device buffers of one fiesta_mesh object, grown by fiesta_mesh_compute
  // per bitmap word (nw, the count and rank arrays nw + 1): blocking bits, active-cell bits, counts and their exclusive scans
  FbDevBuf<uint32_t> bits, act, vcnt, vpre;
  FbDevBuf<long long> qcnt, qpre;
  FbDevBuf<float> xyz;            // outputs: [3 V] float32 positions, [6 Q] int32 vertex ids (2 triangles per quad)
  FbDevBuf<int32_t> ijk;
  FbDevBuf<char> tmp;             // CUB temporary storage
  FbDevBuf<FbMeshCtr> ctr;
  FbHostBuf<FbMeshCtr> h_ctr;
};
struct fiesta_mesh {
  fiesta_map *m = nullptr;
  FbMeshBufs B;
  cudaEvent_t ev[4] = {};           // start, after the scans, after the vertices, end
  fiesta_mesh_stats st{};
  bool valid = false;               // B holds the result of a compute
  ~fiesta_mesh() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
  }
};

struct MeshGeom {                 // the bitmap layout of one compute
  FbNavBox b;
  int ny;                         // By + 1
  int nx;                         // Bx + 1
  int W;                          // words per z-row
  long long nw;                   // words
};

// Word (ex, ey, k) of the bitmap; zero outside E (and past the last word of a row).
__device__ __forceinline__ uint32_t mesh_word(const MeshGeom &M, const uint32_t *__restrict__ bits, int ex, int ey, int k) {
  if (ex >= M.nx || ey >= M.ny || k >= M.W) return 0u;
  return __ldg(&bits[((long long)ex * M.ny + ey) * M.W + k]);
}
// The row word shifted so that bit i holds position ez + 1.
__device__ __forceinline__ uint32_t mesh_up(const MeshGeom &M, const uint32_t *__restrict__ bits, int ex, int ey, int k, uint32_t w) {
  return (w >> 1) | (mesh_word(M, bits, ex, ey, k + 1) << 31);
}
__device__ __forceinline__ void mesh_coords(const MeshGeom &M, long long j, int &ex, int &ey, int &k) {
  k = (int)(j % M.W);
  const long long r = j / M.W;
  ey = (int)(r % M.ny);
  ex = (int)(r / M.ny);
}
// The three sign-changing-edge bit sets of word (ex, ey, k) whose blocking bits are w: edges (v, v + e_x), (v, v + e_y), (v, v + e_z).
__device__ __forceinline__ void mesh_edges(const MeshGeom &M, const uint32_t *__restrict__ bits, int ex, int ey, int k, uint32_t w,
                                           uint32_t *e) {
  e[0] = w ^ mesh_word(M, bits, ex + 1, ey, k);
  e[1] = w ^ mesh_word(M, bits, ex, ey + 1, k);
  e[2] = w ^ mesh_up(M, bits, ex, ey, k, w);
}
// Vertex id of cell (ex, ey, ez) (an active cell).
__device__ __forceinline__ int32_t mesh_vid(const MeshGeom &M, const uint32_t *__restrict__ act, const uint32_t *__restrict__ vpre,
                                            int ex, int ey, int ez) {
  const long long j = ((long long)ex * M.ny + ey) * M.W + (ez >> 5);
  return (int32_t)(__ldg(&vpre[j]) + __popc(__ldg(&act[j]) & ((1u << (ez & 31)) - 1u)));
}

__global__ void k_mesh_classify(FbGeom g, const uint32_t *__restrict__ cobs, MeshGeom M, double r, int unk, uint32_t *bits) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long j = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < M.nw; j += warps) {
    int ex, ey, k;
    mesh_coords(M, j, ex, ey, k);
    const int ez = 32 * k + lane;
    bool blk = false;
    if (ex >= 1 && ey >= 1 && ez >= 1 && ez < M.b.n[2] + 1) {
      const int v[3] = {M.b.lo[0] - 1 + ex, M.b.lo[1] - 1 + ey, M.b.lo[2] - 1 + ez};
      double d;
      blk = fb_seg_blocks(g, cobs, v, r, unk != 0, d);
    }
    const uint32_t w = __ballot_sync(0xffffffffu, blk);
    if (lane == 0) bits[j] = w;
  }
}

__global__ void k_mesh_count(MeshGeom M, const uint32_t *__restrict__ bits, uint32_t *act, uint32_t *vcnt, long long *qcnt,
                             FbMeshCtr *ctr) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned nb = 0;
  if (j < M.nw) {
    int ex, ey, k;
    mesh_coords(M, j, ex, ey, k);
    const uint32_t w00 = __ldg(&bits[j]), w10 = mesh_word(M, bits, ex + 1, ey, k), w01 = mesh_word(M, bits, ex, ey + 1, k),
                   w11 = mesh_word(M, bits, ex + 1, ey + 1, k);
    const uint32_t u00 = mesh_up(M, bits, ex, ey, k, w00), u10 = mesh_up(M, bits, ex + 1, ey, k, w10),
                   u01 = mesh_up(M, bits, ex, ey + 1, k, w01), u11 = mesh_up(M, bits, ex + 1, ey + 1, k, w11);
    const uint32_t all = w00 & w10 & w01 & w11 & u00 & u10 & u01 & u11, any = w00 | w10 | w01 | w11 | u00 | u10 | u01 | u11;
    const uint32_t a = any & ~all;                                           // past E every corner reads 0: never active
    act[j] = a;
    vcnt[j] = __popc(a);
    qcnt[j] = __popc(w00 ^ w10) + __popc(w00 ^ w01) + __popc(w00 ^ u00);
    nb = __popc(w00);
  } else if (j == M.nw) {
    vcnt[j] = 0;
    qcnt[j] = 0;
  }
  nb = __reduce_add_sync(0xffffffffu, nb);
  if ((threadIdx.x & 31) == 0 && nb) atomicAdd(&ctr->blocking, (unsigned long long)nb);
}

__global__ void k_mesh_vertices(FbGeom g, const uint32_t *__restrict__ cobs, MeshGeom M, double r, int unk,
                                const uint32_t *__restrict__ act, const uint32_t *__restrict__ vpre, float *xyz) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  const int hi[3] = {M.b.lo[0] + M.b.n[0] - 1, M.b.lo[1] + M.b.n[1] - 1, M.b.lo[2] + M.b.n[2] - 1};
  for (long long j = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < M.nw; j += warps) {
    const uint32_t a = __ldg(&act[j]);
    if (!((a >> lane) & 1u)) continue;
    int ex, ey, k;
    mesh_coords(M, j, ex, ey, k);
    const int c[3] = {M.b.lo[0] - 1 + ex, M.b.lo[1] - 1 + ey, M.b.lo[2] - 1 + 32 * k + lane};
    bool blk[8], has[8];
    double d[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int v[3] = {c[0] + (q >> 2), c[1] + ((q >> 1) & 1), c[2] + (q & 1)};
      blk[q] = has[q] = false;
      d[q] = 0.0;
      if (v[0] < M.b.lo[0] || v[0] > hi[0] || v[1] < M.b.lo[1] || v[1] > hi[1] || v[2] < M.b.lo[2] || v[2] > hi[2]) continue;
      double dd;
      blk[q] = fb_seg_blocks(g, cobs, v, r, unk != 0, dd);
      const uint32_t rec = fb_ld_record(&cobs[fb_ii(g, v[0], v[1], v[2])]);
      has[q] = fb_mesh_has_distance(rec);
      if (has[q]) d[q] = fb_record_distance(rec, v[0], v[1], v[2], g.res);
    }
    const long long id = (long long)__ldg(&vpre[j]) + __popc(a & ((1u << lane) - 1u));
    float p[3];
    fb_mesh_vertex(c, blk, has, d, r, g.res, g.origin, p);
    xyz[3 * id] = p[0];
    xyz[3 * id + 1] = p[1];
    xyz[3 * id + 2] = p[2];
  }
}

__global__ void k_mesh_faces(MeshGeom M, const uint32_t *__restrict__ bits, const uint32_t *__restrict__ act,
                             const uint32_t *__restrict__ vpre, const long long *__restrict__ qpre, const float *__restrict__ xyz,
                             int32_t *ijk) {
  const int lane = threadIdx.x & 31;
  const uint32_t below = (1u << lane) - 1u;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long j = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < M.nw; j += warps) {
    int ex, ey, k;
    mesh_coords(M, j, ex, ey, k);
    const uint32_t w = __ldg(&bits[j]);
    uint32_t e[3];
    mesh_edges(M, bits, ex, ey, k, w, e);
    if (!((e[0] | e[1] | e[2]) >> lane & 1u)) continue;
    long long q = __ldg(&qpre[j]) + __popc(e[0] & below) + __popc(e[1] & below) + __popc(e[2] & below);
    const int v[3] = {ex, ey, 32 * k + lane};
    const bool vb = (w >> lane) & 1u;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!((e[a] >> lane) & 1u)) continue;
      int off[4][3];
      fb_mesh_quad(a, vb, off);
      int32_t id[4];
      float p[4][3];
      for (int i = 0; i < 4; ++i) {
        id[i] = mesh_vid(M, act, vpre, v[0] + off[i][0], v[1] + off[i][1], v[2] + off[i][2]);
        for (int t = 0; t < 3; ++t) p[i][t] = __ldg(&xyz[3ll * id[i] + t]);
      }
      int32_t tri[6];
      fb_mesh_tris(id, fb_mesh_split02(p[0], p[1], p[2], p[3]), tri);
      for (int t = 0; t < 6; ++t) ijk[6 * q + t] = tri[t];
      ++q;
    }
  }
}

// ---------------------------------------------------------------- host side
static unsigned mesh_warp_blocks(long long words) {            // 8 warps per block, one warp per word, grid-stride beyond
  const long long want = (words + 7) / 8;
  return (unsigned)(want < FB_SMS * 64ll ? (want < 1 ? 1 : want) : FB_SMS * 64ll);
}

#define MESH_GROW(buf, n)                                                                                                 \
  do {                                                                                                                 \
    const cudaError_t e_ = (buf).grow((size_t)(n), s);                                                                 \
    if (e_ != cudaSuccess) return alloc_failed(e_, "fiesta_mesh_compute: cannot allocate %zu elements", (size_t)(n));  \
  } while (0)

template <class Call>
static int mesh_cub(FbMeshBufs &B, cudaStream_t s, Call call) {
  size_t bytes = 0;
  CK(call((void *)nullptr, bytes));
  MESH_GROW(B.tmp, bytes ? bytes : 16);
  bytes = B.tmp.cap;
  CK(call((void *)B.tmp.p, bytes));
  return FIESTA_OK;
}

static int mesh_compute(fiesta_mesh *f, const MeshGeom &M, double r, int unk, fiesta_mesh_stats &st, int *launches) {
  fiesta_map *m = f->m;
  FbMeshBufs &B = f->B;
  const cudaStream_t s = m->stream;
  const long long nw = M.nw;
  int rc;
  MESH_GROW(B.bits, nw); MESH_GROW(B.act, nw);
  MESH_GROW(B.vcnt, nw + 1); MESH_GROW(B.vpre, nw + 1); MESH_GROW(B.qcnt, nw + 1); MESH_GROW(B.qpre, nw + 1);
  CK(cudaMemsetAsync(B.ctr, 0, sizeof(FbMeshCtr), s));
  k_mesh_classify<<<mesh_warp_blocks(nw), 256, 0, s>>>(m->g, m->cobs, M, r, unk, B.bits);
  k_mesh_count<<<(unsigned)((nw + 1 + 255) / 256), 256, 0, s>>>(M, B.bits, B.act, B.vcnt, B.qcnt, B.ctr);
  CK(cudaGetLastError());
  *launches += 2;
  const uint32_t *vc = B.vcnt.p;
  uint32_t *vp = B.vpre.p;
  const long long *qc = B.qcnt.p;
  long long *qp = B.qpre.p;
  const int n = (int)(nw + 1);
  if ((rc = mesh_cub(B, s, [&](void *t, size_t &nb) { return cub::DeviceScan::ExclusiveSum(t, nb, vc, vp, n, s); }))) return rc;
  if ((rc = mesh_cub(B, s, [&](void *t, size_t &nb) { return cub::DeviceScan::ExclusiveSum(t, nb, qc, qp, n, s); }))) return rc;
  *launches += 2;
  CK(cudaMemcpyAsync(&B.ctr->vertices, vp + nw, sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CK(cudaMemcpyAsync(&B.ctr->quads, qp + nw, sizeof(long long), cudaMemcpyDeviceToDevice, s));
  CK(cudaEventRecord(f->ev[1], s));
  CK(cudaMemcpyAsync(B.h_ctr, B.ctr, sizeof(FbMeshCtr), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  const unsigned long long V = B.h_ctr->vertices;
  const long long Q = B.h_ctr->quads;
  st.blocking = (int64_t)B.h_ctr->blocking;
  if (V > 0x7fffffffull) {
    fb_set_error("fiesta_mesh_compute: the mesh has %llu vertices, more than 2^31 - 1; mesh the box in smaller chunks", V);
    return FIESTA_ERR_LIMIT;
  }
  st.vertices = (int64_t)V;
  st.quads = Q;
  st.triangles = 2 * Q;
  MESH_GROW(B.xyz, 3 * V);
  MESH_GROW(B.ijk, 6 * Q);
  if (V) {
    k_mesh_vertices<<<mesh_warp_blocks(nw), 256, 0, s>>>(m->g, m->cobs, M, r, unk, B.act, B.vpre, B.xyz);
    CK(cudaGetLastError());
    *launches += 1;
  }
  CK(cudaEventRecord(f->ev[2], s));
  if (Q) {
    k_mesh_faces<<<mesh_warp_blocks(nw), 256, 0, s>>>(M, B.bits, B.act, B.vpre, B.qpre, B.xyz, B.ijk);
    CK(cudaGetLastError());
    *launches += 1;
  }
  return FIESTA_OK;
}

// ---------------------------------------------------------------- entry points (include/fiesta_b200.h)
void fiesta_mesh_destroy(fiesta_mesh *f) { handle_destroy(f); }
int fiesta_mesh_create(fiesta_map *m, fiesta_mesh **out) {
  if (!m || !out) { fb_set_error("fiesta_mesh_create: null argument"); return FIESTA_ERR_INVALID; }
  *out = nullptr;
  FbHandle<fiesta_mesh> f;
  int r;
  if ((r = handle_new(m, f))) return r;
  if (!f) { fb_set_error("out of host memory"); return FIESTA_ERR_INVALID; }
  for (cudaEvent_t &e : f->ev) CK(cudaEventCreate(&e));
  CK(f->B.ctr.alloc(1));
  CK(f->B.h_ctr.alloc(1));
  *out = f.release();
  return FIESTA_OK;
}
int fiesta_mesh_compute(fiesta_mesh *f, const int box_lo[3], const int box_hi[3], double clearance, int flags, fiesta_mesh_stats *stats) {
  const char *fn = "fiesta_mesh_compute";
  if (!f || !box_lo || !box_hi) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  if (!clearance_flags_ok(fn, clearance, flags)) return FIESTA_ERR_INVALID;
  fiesta_map *m = f->m;
  MeshGeom M{};
  if (!box_arg(fn, m->g, box_lo, box_hi, &M.b)) return FIESTA_ERR_INVALID;
  M.nx = M.b.n[0] + 1;
  M.ny = M.b.n[1] + 1;
  M.W = (M.b.n[2] + 1 + 31) / 32;
  M.nw = (long long)M.nx * M.ny * M.W;
  CK(cudaSetDevice(m->device));
  f->valid = false;
  CK(cudaEventRecord(f->ev[0], m->stream));
  fiesta_mesh_stats st{};
  st.box_voxels = (int64_t)M.b.n[0] * M.b.n[1] * M.b.n[2];
  int launches = 0;
  const int r = mesh_compute(f, M, clearance, flags & FIESTA_SEGMENT_UNKNOWN_BLOCKS, st, &launches);
  m->st.kernel_launches += launches;
  if (r != FIESTA_OK) return r;
  CK(cudaEventRecord(f->ev[3], m->stream));
  CK(cudaStreamSynchronize(m->stream));
  CK(cudaEventElapsedTime(&st.ms_compute, f->ev[0], f->ev[3]));
  CK(cudaEventElapsedTime(&st.ms_classify, f->ev[0], f->ev[1]));
  CK(cudaEventElapsedTime(&st.ms_vertices, f->ev[1], f->ev[2]));
  CK(cudaEventElapsedTime(&st.ms_faces, f->ev[2], f->ev[3]));
  f->st = st;
  f->valid = true;
  if (stats) *stats = f->st;
  return FIESTA_OK;
}
static bool mesh_read_ok(const fiesta_mesh *f, const char *fn, int64_t cap, bool buffer) {
  if (!f || cap < 0 || (cap > 0 && !buffer)) { fb_set_error("%s: null buffer or negative capacity", fn); return false; }
  if (!f->valid) { fb_set_error("%s: no mesh has been computed", fn); return false; }
  return true;
}
int fiesta_mesh_vertices(const fiesta_mesh *f, int64_t cap, float *xyz) {
  if (!mesh_read_ok(f, "fiesta_mesh_vertices", cap, xyz != nullptr)) return FIESTA_ERR_INVALID;
  const size_t n = (size_t)(cap < f->st.vertices ? cap : f->st.vertices);
  if (n == 0) return FIESTA_OK;
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  CK(cudaMemcpyAsync(xyz, f->B.xyz, n * 12, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
int fiesta_mesh_triangles(const fiesta_mesh *f, int64_t cap, int32_t *ijk) {
  if (!mesh_read_ok(f, "fiesta_mesh_triangles", cap, ijk != nullptr)) return FIESTA_ERR_INVALID;
  const size_t n = (size_t)(cap < f->st.triangles ? cap : f->st.triangles);
  if (n == 0) return FIESTA_OK;
  const fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  CK(cudaMemcpyAsync(ijk, f->B.ijk, n * 12, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
