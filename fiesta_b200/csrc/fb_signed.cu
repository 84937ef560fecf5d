// fiesta_b200 -- signed distance of a voxel box (include/fiesta_b200.h, DESIGN.md §3.13): FIESTA's distance outside obstacles,
// minus the exact Euclidean depth inside them, with GetDistance / GetDistWithGradTrilinear queries on it.
//
// q (the squared depth) is an exact separable Euclidean distance transform of the box's obstacle mask in three passes:
//   k_signed_z  one warp per z-line: classify from the records, ballot each 32-voxel chunk, 1-D distance along z -> q
//   k_signed_y  one thread per (x, z) line, neighbouring threads on neighbouring z: lower envelope along y, q -> scratch [y][x][z]
//   k_signed_x  one thread per (y, z) line: lower envelope along x, scratch -> q in box layout, with the statistics
// Every load and store of a line step is coalesced across the warp; only the envelope stacks' pops read scattered words.
#include <math.h>
#include "fb_map.h"
#include "fb_signed.h"

struct FbSignedCtr {
  unsigned long long obstacles, interior;
  int max_q, pad;
};

struct fiesta_signed_field {
  fiesta_map *m = nullptr;
  FbDevBuf<int32_t> q, scratch;     // q per box voxel; scratch: the y pass's output and stacks
  FbDevBuf<FbSignedCtr> ctr;
  FbHostBuf<FbSignedCtr> h_ctr;
  cudaEvent_t ev[2] = {};
  FbSignedBox box{};
  unsigned long long epoch = 0;     // the map's records epoch at the last compute
  bool valid = false;               // q holds the field of `box`
  ~fiesta_signed_field() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
  }
};

// ---------------------------------------------------------------- kernels
__global__ void __launch_bounds__(256) k_signed_z(FbGeom g, const uint32_t *cobs, FbSignedBox b, int32_t *q) {
  const int lane = threadIdx.x & 31;
  const long long nlines = (long long)b.n[0] * b.n[1];
  const int nch = (b.n[2] + 31) >> 5;                                     // <= 32 chunks: Bz <= 1024
  for (long long line = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; line < nlines;
       line += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int bx = (int)(line / b.n[1]), by = (int)(line % b.n[1]);
    const int x = b.lo[0] + bx, y = b.lo[1] + by;
    const uint32_t *rec = cobs + fb_ii(g, x, y, b.lo[2]);
    uint32_t mine = 0;                                                    // lane c: the non-obstacle mask of chunk c
    for (int c = 0; c < nch; ++c) {
      const int bz = 32 * c + lane;
      const bool nonobs = bz < b.n[2] && !fb_signed_obstacle(__ldg(rec + bz), x, y, b.lo[2] + bz);
      const uint32_t msk = __ballot_sync(0xffffffffu, nonobs);
      if (lane == c) mine = msk;
    }
    int last = mine ? 32 * lane + 31 - __clz(mine) : -1;                  // last non-obstacle up to the end of chunk `lane`
    int first = mine ? 32 * lane + __ffs(mine) - 1 : FB_SIGNED_NONE;      // first one from the start of chunk `lane`
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, last, d), f = __shfl_down_sync(0xffffffffu, first, d);
      if (lane >= d && a > last) last = a;
      if (lane + d < 32 && f < first) first = f;
    }
    int32_t *out = q + line * b.n[2];
    for (int c = 0; c < nch; ++c) {
      const uint32_t msk = __shfl_sync(0xffffffffu, mine, c);
      const int prev_end = __shfl_sync(0xffffffffu, last, c > 0 ? c - 1 : 0);
      const int next_start = __shfl_sync(0xffffffffu, first, c + 1 < 32 ? c + 1 : 31);
      const int bz = 32 * c + lane;
      if (bz < b.n[2]) out[bz] = fb_signed_1d(msk, c, lane, c > 0 ? prev_end : -1, c + 1 < nch ? next_start : FB_SIGNED_NONE);
    }
  }
}

// y pass: line (x, z) reads q[(x*By + y)*Bz + z] and leaves its output at scratch[y * (Bx*Bz) + x*Bz + z]
__global__ void __launch_bounds__(128) k_signed_y(FbSignedBox b, const int32_t *q, int32_t *scratch) {
  const long long nl = (long long)b.n[0] * b.n[2];
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nl) return;
  const long long x = t / b.n[2], z = t % b.n[2];
  fb_signed_envelope(q + x * b.n[1] * b.n[2] + z, b.n[2], scratch + t, nl, b.n[1], nullptr);
}

// x pass: line (y, z) reads scratch[y * (Bx*Bz) + x*Bz + z] and leaves q[(x*By + y)*Bz + z] (box layout)
__global__ void __launch_bounds__(128) k_signed_x(FbSignedBox b, const int32_t *scratch, int32_t *q, FbSignedCtr *ctr) {
  const long long nl = (long long)b.n[1] * b.n[2];
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  FbSignedAcc acc{0, 0, 0};
  if (t < nl) {
    const long long y = t / b.n[2], z = t % b.n[2];
    fb_signed_envelope(scratch + y * b.n[0] * b.n[2] + z, b.n[2], q + t, nl, b.n[0], &acc);
  }
  const unsigned long long o = __reduce_add_sync(0xffffffffu, (unsigned)acc.obstacles), i = __reduce_add_sync(0xffffffffu, (unsigned)acc.interior);
  const int mq = __reduce_max_sync(0xffffffffu, acc.max_q);
  if ((threadIdx.x & 31) == 0) {
    if (o) atomicAdd(&ctr->obstacles, o);
    if (i) atomicAdd(&ctr->interior, i);
    if (mq) atomicMax(&ctr->max_q, mq);
  }
}

__global__ void k_signed_export(FbGeom g, const uint32_t *cobs, FbSignedBox b, const int32_t *q, double *out) {
  const long long n = (long long)b.n[0] * b.n[1] * b.n[2];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int bz = (int)(i % b.n[2]), by = (int)(i / b.n[2] % b.n[1]), bx = (int)(i / ((long long)b.n[2] * b.n[1]));
    out[i] = FbSignedRead{g, cobs, q, b}(b.lo[0] + bx, b.lo[1] + by, b.lo[2] + bz);
  }
}

// mode 0: GetDistance(Vector3d); mode 1: GetDistWithGradTrilinear -- the map's query expressions with the signed corner read
__global__ void k_signed_query(FbGeom g, const uint32_t *cobs, FbSignedBox b, const int32_t *q, const double *pos, long long n, int mode,
                               double *out, double *grad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
  const FbSignedRead rd{g, cobs, q, b};
  if (mode == 0) { out[i] = fb_query_distance(g, rd, p); return; }
  double gr[3];
  out[i] = fb_query_trilinear(g, rd, p, gr);
  grad[3 * i] = gr[0]; grad[3 * i + 1] = gr[1]; grad[3 * i + 2] = gr[2];
}

static unsigned grid_for(long long threads, int block) {
  const long long want = (threads + block - 1) / block;
  return (unsigned)(want < FB_SMS * 32ll ? want : FB_SMS * 32ll);
}

// ---------------------------------------------------------------- entry points (include/fiesta_b200.h)
// Export and queries: FIESTA_OK, or FIESTA_ERR_INVALID with the message set when there is nothing current to read.
static int readable(const fiesta_signed_field *f, const char *fn) {
  if (!f->valid) { fb_set_error("%s: no field has been computed", fn); return FIESTA_ERR_INVALID; }
  if (f->epoch != f->m->records_epoch) { fb_set_error("%s: the map's records changed after the compute; compute again", fn); return FIESTA_ERR_INVALID; }
  return FIESTA_OK;
}

void fiesta_signed_destroy(fiesta_signed_field *f) { handle_destroy(f); }
int fiesta_signed_create(fiesta_map *m, fiesta_signed_field **out) {
  if (!m || !out) { fb_set_error("fiesta_signed_create: null argument"); return FIESTA_ERR_INVALID; }
  *out = nullptr;
  FbHandle<fiesta_signed_field> f;
  int r;
  if ((r = handle_new(m, f))) return r;
  if (!f) { fb_set_error("out of host memory"); return FIESTA_ERR_INVALID; }
  for (cudaEvent_t &e : f->ev) CK(cudaEventCreate(&e));
  CK(f->ctr.alloc(1));
  CK(f->h_ctr.alloc(1));
  *out = f.release();
  return FIESTA_OK;
}

int fiesta_signed_compute(fiesta_signed_field *f, const int box_lo[3], const int box_hi[3], fiesta_signed_stats *stats) {
  const char *fn = "fiesta_signed_compute";
  if (!f || !box_lo || !box_hi) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  fiesta_map *m = f->m;
  const FbGeom &g = m->g;
  if (!box_arg(fn, g, box_lo, box_hi, nullptr)) return FIESTA_ERR_INVALID;
  FbSignedBox b;
  for (int k = 0; k < 3; ++k) { b.lo[k] = box_lo[k]; b.n[k] = box_hi[k] - box_lo[k] + 1; }
  const size_t nv = (size_t)b.n[0] * b.n[1] * b.n[2];
  CK(cudaSetDevice(m->device));
  cudaError_t e = f->q.grow(nv, m->stream);
  if (e == cudaSuccess) e = f->scratch.grow(nv, m->stream);
  f->valid = false;                                                       // from here on the old field is gone (grow keeps no contents)
  if (e != cudaSuccess) return alloc_failed(e, "%s: cannot allocate the field of %zu voxels", fn, nv);
  CK(cudaMemsetAsync(f->ctr, 0, sizeof(FbSignedCtr), m->stream));
  CK(cudaEventRecord(f->ev[0], m->stream));
  k_signed_z<<<grid_for((long long)b.n[0] * b.n[1] * 32, 256), 256, 0, m->stream>>>(g, m->cobs, b, f->q);
  k_signed_y<<<(unsigned)(((long long)b.n[0] * b.n[2] + 127) / 128), 128, 0, m->stream>>>(b, f->q, f->scratch);
  k_signed_x<<<(unsigned)(((long long)b.n[1] * b.n[2] + 127) / 128), 128, 0, m->stream>>>(b, f->scratch, f->q, f->ctr);
  m->st.kernel_launches += 3;
  CK(cudaGetLastError());
  CK(cudaEventRecord(f->ev[1], m->stream));
  CK(cudaMemcpyAsync(f->h_ctr, f->ctr, sizeof(FbSignedCtr), cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  f->box = b;
  f->epoch = m->records_epoch;
  f->valid = true;
  if (stats) {
    const FbSignedCtr &c = *f->h_ctr;
    *stats = fiesta_signed_stats{};
    stats->box_voxels = (int64_t)nv;
    stats->obstacles = (int64_t)c.obstacles;
    stats->interior = (int64_t)c.interior;
    stats->max_depth_sq = c.obstacles == nv ? -1 : (int64_t)c.max_q;
    CK(cudaEventElapsedTime(&stats->ms_compute, f->ev[0], f->ev[1]));
  }
  return FIESTA_OK;
}

int fiesta_signed_export(const fiesta_signed_field *f, double *out) {
  const char *fn = "fiesta_signed_export";
  if (!f || !out) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  int r;
  if ((r = readable(f, fn))) return r;
  fiesta_map *m = f->m;
  const size_t nv = (size_t)f->box.n[0] * f->box.n[1] * f->box.n[2];
  CK(cudaSetDevice(m->device));
  FbDevBuf<double> d_out;                                                 // staging, freed on return (as the map's exports)
  if (cudaError_t e = d_out.alloc(nv)) return alloc_failed(e, "%s: cannot allocate the staging of %zu voxels", fn, nv);
  k_signed_export<<<grid_for((long long)nv, 256), 256, 0, m->stream>>>(m->g, m->cobs, f->box, f->q, d_out);
  m->st.kernel_launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, d_out, nv * 8, cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}

static void launch_query(const fiesta_signed_field *f, const double *pos, int64_t n, int mode, double *out, double *grad, cudaStream_t s) {
  const fiesta_map *m = f->m;
  k_signed_query<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(m->g, m->cobs, f->box, f->q, pos, n, mode, out, grad);
}
// host buffers: staged through the map's query buffers on the map's stream, as fiesta_get_dist_grad_trilinear_batch
static int host_query(fiesta_signed_field *f, const char *fn, const double *pos, int64_t n, int mode, double *out, double *grad) {
  if (!f) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  if (!count_buffers_ok(fn, n, pos && out && (mode == 0 || grad))) return FIESTA_ERR_INVALID;
  int r;
  if ((r = readable(f, fn))) return r;
  if (n == 0) return FIESTA_OK;
  fiesta_map *m = f->m;
  CK(cudaSetDevice(m->device));
  cudaError_t e = m->d_qin.grow((size_t)n * 3, m->stream);
  if (e == cudaSuccess) e = m->d_qout.grow((size_t)n * 4, m->stream);   // [dist n][grad 3n]
  if (e != cudaSuccess) return alloc_failed(e, "%s: cannot allocate the staging of %lld positions", fn, (long long)n);
  CK(cudaMemcpyAsync(m->d_qin, pos, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, m->stream));
  launch_query(f, m->d_qin, n, mode, m->d_qout, m->d_qout + n, m->stream);
  m->st.kernel_launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, m->d_qout, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
  if (grad) CK(cudaMemcpyAsync(grad, m->d_qout + n, (size_t)n * 3 * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
  CK(cudaStreamSynchronize(m->stream));
  return FIESTA_OK;
}
int fiesta_signed_get_distance_batch(fiesta_signed_field *f, const double *pos_xyz, int64_t n, double *out_dist) {
  return host_query(f, "fiesta_signed_get_distance_batch", pos_xyz, n, 0, out_dist, nullptr);
}
int fiesta_signed_get_dist_grad_trilinear_batch(fiesta_signed_field *f, const double *pos_xyz, int64_t n, double *out_dist, double *out_grad_xyz) {
  return host_query(f, "fiesta_signed_get_dist_grad_trilinear_batch", pos_xyz, n, 1, out_dist, out_grad_xyz);
}

// device buffers, ordered on the caller's stream (device_query_begin / _end, fb_map.cu)
static int device_query(fiesta_signed_field *f, const char *fn, const double *d_pos, int64_t n, int mode, double *d_out, double *d_grad, void *stream) {
  if (!f) { fb_set_error("%s: null argument", fn); return FIESTA_ERR_INVALID; }
  if (!count_buffers_ok(fn, n, d_pos && d_out && (mode == 0 || d_grad))) return FIESTA_ERR_INVALID;
  int r;
  if ((r = readable(f, fn))) return r;
  fiesta_map *m = f->m;
  const cudaStream_t s = (cudaStream_t)stream;
  if ((r = device_query_begin(m, fn, s))) return r;
  if (n > 0) {
    launch_query(f, d_pos, n, mode, d_out, d_grad, s);
    m->st.kernel_launches++;
  }
  return device_query_end(m, s);
}
int fiesta_signed_get_distance_batch_device(fiesta_signed_field *f, const double *d_pos_xyz, int64_t n, double *d_dist, void *stream) {
  return device_query(f, "fiesta_signed_get_distance_batch_device", d_pos_xyz, n, 0, d_dist, nullptr, stream);
}
int fiesta_signed_get_dist_grad_trilinear_batch_device(fiesta_signed_field *f, const double *d_pos_xyz, int64_t n, double *d_dist,
                                                        double *d_grad_xyz, void *stream) {
  return device_query(f, "fiesta_signed_get_dist_grad_trilinear_batch_device", d_pos_xyz, n, 1, d_dist, d_grad_xyz, stream);
}
