// api.cu — C-ABI implementation (include/rayn_b200.h): context, scene upload, the tile-pass
// scheduler that drives the wavefront kernels, the NCCL film gather and the known-answer
// entry points.  No torch types, no exceptions across the boundary.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <limits.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <string>
#include <vector>

#include "rt_accum.cuh"
#include "rt_denoise.cuh"
#include "rt_first_hit.cuh"
#include "rt_kernels.cuh"
#include "rt_temporal.cuh"
#ifdef RAYN_LEGACY_KERNELS
#include "rt_legacy.cuh"
#endif

using namespace rt;

static thread_local std::string g_last_error;

struct TimedLaunch {
  int kernel;
  cudaEvent_t a, b;
};

// ---- NCCL, resolved at run time (no link-time dependency: the library must load on a box without NCCL) ----
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[RAYN_COMM_ID_BYTES]; } ncclUniqueId;
struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static const int kNcclFloat = 7;  // ncclFloat32

struct RaynComm {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 0;
  // shard tables of the last geometry gathered
  int W = 0, H = 0, tw = 0, th = 0, per_rank = 0;
  std::vector<std::vector<int>> shards;
  int* d_table = nullptr;   // [world * per_rank], -1 padded
  float* d_slabs = nullptr; // [world * per_rank * 10 * tw * th]
  size_t cap_slabs = 0;
};

// One entry of the pass-buffer table (pass_table): a buffer and its size in bytes, per_path * paths + per_slot * shading
// slots + per_tile * tiles + fixed.  An entry whose size is 0 (its condition does not hold) is not allocated.
struct PassBuf {
  void** ptr;
  size_t per_path, per_slot, per_tile, fixed;
};
static const int N_PASS_BUFS = 23;

// One host-space output plane of a job (job_stage): the caller's pointer (NULL: not asked for) and its floats per pixel.
struct JobPlane {
  float* user;
  int floats;
};

// The state of one pass in flight: its buffers, the work counters of its persistent kernels and the stream it runs on.  A
// render of several passes alternates them between two such sets, so that one pass's kernel tails, drains and single-CTA
// scans overlap the other pass's work (render_enqueue).  The passes cover disjoint tiles and share only the stats counters.
struct PassSet {
  cudaStream_t stream = nullptr;      // set 0: the context's stream
  size_t cap[N_PASS_BUFS] = {};       // bytes allocated per pass_table entry
  PassBufs pb;                        // pb.counters: the context's stats counters, shared by both sets
  int* d_tile_ids = nullptr;
  int* d_batch_prefix = nullptr;  // [tiles per pass + 1]
  int* d_work_ctr = nullptr;      // [WC_TOTAL] global work counters of the persistent kernels
};

struct RaynContext {
  int device = 0;
  int flags = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  bool has_scene = false;
  DevScene scene;
  int64_t cap_paths = 0;  // requested paths per pass
  PassSet ps[2];          // pass buffers; ps[1] only for renders of several passes (size_pass)
  unsigned long long* d_counters = nullptr;  // [CNT_TOTAL] stats counters of the job, order-free atomics
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;  // ps[1].stream forks from and joins back into the context's stream
  int n_sm = 148;
  int occ_ext[2][SDFV_COUNT], occ_shd[SDFV_COUNT], occ_nrm[SDFV_COUNT], occ_nrm_trap[SDFV_COUNT];  // occ_ext[constant threshold][variant]
  int occ_pre = 8, occ_post = 8, occ_sph = 8;  // resident CTAs per SM of the work-list kernels
  int occ_pre_trap = 8, occ_post_trap = 8;     // ... of the shading kernels of scenes with orbit-trap albedos
  int sdf_var[RAYN_MAX_HITABLES];  // march-kernel variant of every SDF hitable of the uploaded scene (rt_sdf2.cuh::sdf_variant)
  struct Div3Check { float min_r2, fixed_r2; bool ok; };
  std::vector<Div3Check> div3_cache;  // exhaustive fastdiv2_3 checks already run on this device
  // staging for host-space inputs / outputs
  float *d_s1 = nullptr, *d_s2 = nullptr, *d_scr = nullptr, *d_fis = nullptr;
  size_t cap_s1 = 0, cap_s2 = 0, cap_scr = 0;
  float* d_planes = nullptr;
  size_t cap_planes = 0;
  int* d_pack_ids = nullptr;
  size_t cap_pack_ids = 0;
  unsigned char* d_post = nullptr;
  size_t cap_post = 0;
  unsigned long long* d_kat = nullptr;
  DevPrev* d_prev = nullptr;  // rayn_b200_render_motion_prev's previous scene, allocated by its first call
  RaynStats stats;
  bool qlog_enabled = false;
  std::vector<int32_t> qlog;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::vector<TimedLaunch> timed;
  size_t timed_used = 0;
  // a render that has been enqueued but not finished
  bool pending = false;
  std::vector<int> job_tiles;
  std::vector<JobPlane> job_out;  // the job's host-space outputs, staged back to back in d_planes in this order (job_stage)
  int job_w = 0, job_h = 0, job_tw = 0, job_th = 0, job_spp = 0, job_nty = 0;
  unsigned long long h_counters[CNT_TOTAL];
  RaynComm comm;
  // CUDA graph of the last small single-pass frame (launch-bound frames: the whole per-depth kernel sequence replays as one launch)
  cudaGraphExec_t graph_exec = nullptr;
  uint64_t graph_key = 0;
  RaynStats graph_stats;  // launch counts recorded while capturing
};

static uint64_t fnv1a(uint64_t h, const void* data, size_t n) {
  const unsigned char* p = (const unsigned char*)data;
  for (size_t i = 0; i < n; ++i) h = (h ^ p[i]) * 1099511628211ull;
  return h;
}

static int32_t fail(RaynContext* ctx, int32_t code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_last_error = buf;
  if (ctx) ctx->err = buf;
  return code;
}
// a failing runtime call leaves a sticky per-thread "last error": clear it when reporting, or the next valid call's
// cudaGetLastError() check would fail spuriously
#define CU(call)                                                                                     \
  do {                                                                                               \
    cudaError_t e_ = (call);                                                                         \
    if (e_ != cudaSuccess) {                                                                         \
      cudaGetLastError();                                                                            \
      return fail(ctx, e_ == cudaErrorMemoryAllocation ? RAYN_ERR_OOM : RAYN_ERR_CUDA, "%s: %s (%s:%d)", #call, \
                  cudaGetErrorString(e_), __FILE__, __LINE__);                                       \
    }                                                                                                \
  } while (0)
#define NC(call)                                                                                     \
  do {                                                                                               \
    int r_ = (call);                                                                                 \
    if (r_ != 0)                                                                                     \
      return fail(ctx, RAYN_ERR_NCCL, "%s: %s (%s:%d)", #call, g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "?", __FILE__, __LINE__); \
  } while (0)

template <class T>
static cudaError_t regrow(T** p, size_t* cap, size_t need) {
  if (need <= *cap && *p) return cudaSuccess;
  if (*p) cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  cudaError_t e = cudaMalloc((void**)p, std::max<size_t>(need, 1) * sizeof(T));
  if (e == cudaSuccess) *cap = need;
  return e;
}

// Every pass buffer, in allocation order.  seg_per_path: shadow segments per path and depth over all SDF queues; lc_ns: light
// samples per path and depth; trap: the scene has orbit-trap albedos (PassBufs::trap_s).
static std::array<PassBuf, N_PASS_BUFS> pass_table(PassSet* c, int QS, int seg_per_path, int lc_ns, bool trap) {
  PassBufs& p = c->pb;
  const size_t nseg = (QS + SEG_SLOTS - 1) / SEG_SLOTS;  // segments per tile of the queue kernels
  return {{
      {(void**)&p.o_time, sizeof(float4), 0, 0, 0},
      {(void**)&p.d_t, sizeof(float4), 0, 0, 0},
      {(void**)&p.rad, sizeof(float4), 0, 0, 0},
      {(void**)&p.thr, sizeof(float4), 0, 0, 0},
      {(void**)&p.nrm0, sizeof(float4), 0, 0, 0},
      {(void**)&p.term, sizeof(uint32_t), 0, 0, 0},
      {(void**)&p.q_live, sizeof(int), 0, 0, 0},
      {(void**)&p.q_key, sizeof(int), 0, 0, 0},
      {(void**)&p.q_shade, 0, sizeof(int), 0, 0},
      {(void**)&p.n_live, 0, 0, sizeof(int), 0},
      {(void**)&p.n_slots, 0, 0, sizeof(int), 0},
      {(void**)&p.bin_start, 0, 0, (RAYN_MAX_HITABLES + 1) * sizeof(int), 0},
      {(void**)&c->d_tile_ids, 0, 0, sizeof(int), 0},
      {(void**)&c->d_batch_prefix, 0, 0, sizeof(int), sizeof(int)},
      {(void**)&p.seg_cnt, 0, 0, nseg * RAYN_MAX_HITABLES * sizeof(int), 0},
      {(void**)&p.slot_prefix, 0, 0, (1 + RAYN_MAX_HITABLES) * sizeof(int), (1 + RAYN_MAX_HITABLES) * sizeof(int)},
      {(void**)&p.nrm, sizeof(float4), 0, 0, 0},
      {(void**)&p.vis, sizeof(uint32_t), 0, 0, 0},
      {(void**)&p.seg_a, (size_t)seg_per_path * sizeof(float4), 0, 0, 0},
      {(void**)&p.seg_b, (size_t)seg_per_path * sizeof(float4), 0, 0, 0},
      {(void**)&p.lc_c, (size_t)lc_ns * sizeof(float4), 0, 0, 0},
      {(void**)&p.lc_t, lc_ns > 4 ? 8 * sizeof(float) : 0, 0, 0, 0},
      {(void**)&p.trap_s, trap ? sizeof(float) : 0, 0, 0, 0},
  }};
}

static void free_pass(PassSet* s) {
  for (const PassBuf& b : pass_table(s, 0, 0, 0, false)) {
    cudaFree(*b.ptr);
    *b.ptr = nullptr;
  }
  unsigned long long* counters = s->pb.counters;
  memset(&s->pb, 0, sizeof s->pb);
  s->pb.counters = counters;
  memset(s->cap, 0, sizeof s->cap);
}

static size_t pass_set_bytes(const PassSet& s) {
  size_t bytes = 0;
  for (size_t b : s.cap) bytes += b;
  return bytes;
}

// bytes of pass state per path (what ensure_pass allocates, less the per-tile buffers), used to size passes against free
// device memory
static size_t pass_bytes_per_path(PassSet* s, int R, int QS, int seg_per_path, int lc_ns, bool trap) {
  size_t bytes = 0;
  for (const PassBuf& b : pass_table(s, QS, seg_per_path, lc_ns, trap))
    bytes += b.per_path + (b.per_slot ? (size_t)(((double)QS / R) * b.per_slot + 1) : 0);
  return bytes;
}

static int32_t ensure_pass(RaynContext* ctx, PassSet* s, int n_tiles, int R, int QS, int seg_per_path, int n_sdf, int lc_ns, bool trap) {
  const int64_t need_paths = (int64_t)n_tiles * R, need_q = (int64_t)n_tiles * QS;
  const std::array<PassBuf, N_PASS_BUFS> table = pass_table(s, QS, seg_per_path, lc_ns, trap);
  size_t need[N_PASS_BUFS];
  bool fits = true;
  for (int i = 0; i < N_PASS_BUFS; ++i) {
    const PassBuf& b = table[i];
    need[i] = b.per_path * need_paths + b.per_slot * need_q + b.per_tile * n_tiles + b.fixed;
    fits = fits && need[i] <= s->cap[i];
  }
  if (fits) return RAYN_OK;
  free_pass(s);
  for (int i = 0; i < N_PASS_BUFS; ++i) {
    if (need[i] == 0) continue;
    const cudaError_t e = cudaMalloc(table[i].ptr, need[i]);
    if (e != cudaSuccess) {
      cudaGetLastError();
      free_pass(s);
      return fail(ctx, e == cudaErrorMemoryAllocation ? RAYN_ERR_OOM : RAYN_ERR_CUDA, "pass buffers (%lld paths): %s", (long long)need_paths,
                  cudaGetErrorString(e));
    }
    s->cap[i] = need[i];
  }
  s->pb.prefix_stride = n_tiles + 1;
  s->pb.seg_cap = n_sdf > 0 ? need_paths * seg_per_path / n_sdf : 0;
  return RAYN_OK;
}

static void timed_begin(RaynContext* ctx, int kernel) {
  if (!(ctx->flags & RAYN_FLAG_TIMING)) return;
  if (ctx->timed_used == ctx->timed.size()) {
    TimedLaunch t;
    t.kernel = kernel;
    cudaEventCreate(&t.a);
    cudaEventCreate(&t.b);
    ctx->timed.push_back(t);
  }
  ctx->timed[ctx->timed_used].kernel = kernel;
  cudaEventRecord(ctx->timed[ctx->timed_used].a, ctx->stream);
}
static void timed_end(RaynContext* ctx, int kernel, int launches = 1) {
  ctx->stats.launches += launches;
  ctx->stats.kernel_launches[kernel] += launches;
  if (!(ctx->flags & RAYN_FLAG_TIMING)) return;
  cudaEventRecord(ctx->timed[ctx->timed_used].b, ctx->stream);
  ctx->timed_used++;
}

struct DevTmp {
  std::vector<void*> ptrs;
  ~DevTmp() {
    for (void* p : ptrs) cudaFree(p);
  }
  template <class T>
  T* up(const T* h, size_t n, cudaError_t* e) {
    T* d = nullptr;
    if (*e != cudaSuccess) return nullptr;
    *e = cudaMalloc((void**)&d, std::max<size_t>(n, 1) * sizeof(T));
    if (*e != cudaSuccess) return nullptr;
    ptrs.push_back(d);
    if (h) *e = cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice);
    // cudaMemcpy from PAGEABLE memory returns once the data is staged; the DMA may still be in flight, and the test kernels
    // run on a non-blocking stream that does not order against the legacy stream: wait for the copy to land.
    if (h && *e == cudaSuccess) *e = cudaDeviceSynchronize();
    return d;
  }
};

// kernel launches specialised on the SDF variant (rt_sdf2.cuh)
#define DISPATCH_SDFV(v, STMT)                                                        \
  switch (v) {                                                                        \
    case SDFV_BOX_12_FAST: { constexpr int V = SDFV_BOX_12_FAST; STMT; } break;       \
    case SDFV_BOX_N_FAST: { constexpr int V = SDFV_BOX_N_FAST; STMT; } break;         \
    case SDFV_BULB: { constexpr int V = SDFV_BULB; STMT; } break;                     \
    case SDFV_BOX_12_DIV3: { constexpr int V = SDFV_BOX_12_DIV3; STMT; } break;       \
    case SDFV_BOX_N_DIV3: { constexpr int V = SDFV_BOX_N_DIV3; STMT; } break;         \
    default: { constexpr int V = SDFV_BOX_GENERIC; STMT; } break;                     \
  }

static void tile_grid_of(int W, int H, int tw, int th, int* ntx, int* nty) {
  *ntx = (W + W % tw) / tw;  // film.rs:399-404
  *nty = (H + H % th) / th;
}
static std::vector<int> shard_of(int W, int H, int tw, int th, int rank, int world) {
  int ntx, nty;
  tile_grid_of(W, H, tw, th, &ntx, &nty);
  std::vector<int> v;
  for (int tx = 0; tx < ntx; ++tx)
    for (int ty = 0; ty < nty; ++ty)
      if ((tx + ty) % world == rank) v.push_back(tx * nty + ty);  // ascending: tile index = tx * nty + ty (film.rs:401-425)
  return v;
}

static int32_t render_enqueue(RaynContext* ctx, const RaynFrameDesc* f, const RaynFilmPlanes* out, const std::vector<int>* tiles_override,
                              RaynFilmPlanes* dev_planes_out, const RaynMomentPlanes* moments = nullptr);
static int32_t render_finish(RaynContext* ctx);
static int32_t gather_enqueue(RaynContext* ctx, int W, int H, int tw, int th, const RaynFilmPlanes* pl, bool in_group);

extern "C" {

int32_t rayn_b200_abi_version(void) { return RAYN_B200_ABI_VERSION; }
int32_t rayn_b200_muladd_fused(void) { return RAYN_MULADD_FUSED; }

const char* rayn_b200_last_error(const RaynContext* ctx) { return ctx ? ctx->err.c_str() : g_last_error.c_str(); }

int32_t rayn_b200_create(const RaynConfig* cfg, RaynContext** out_ctx) {
  RaynContext* ctx = nullptr;
  if (!out_ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "out_ctx is NULL");
  *out_ctx = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(nullptr, RAYN_ERR_NO_DEVICE, "no CUDA device: the rayn_b200 render path has no CPU fallback");
  }
  const int dev = cfg ? cfg->device : 0;
  if (dev < 0 || dev >= ndev) return fail(nullptr, RAYN_ERR_INVALID_ARG, "device %d out of range (have %d)", dev, ndev);
#ifndef RAYN_LEGACY_KERNELS
  if (cfg && (cfg->flags & RAYN_FLAG_SIMPLE_MARCH))
    return fail(nullptr, RAYN_ERR_UNSUPPORTED, "RAYN_FLAG_SIMPLE_MARCH needs the test build (librayn_b200_legacy.so, -DRAYN_LEGACY_KERNELS)");
#endif
  CU(cudaSetDevice(dev));
  ctx = new RaynContext();
  ctx->device = dev;
  ctx->flags = cfg ? cfg->flags : 0;
  ctx->cap_paths = (cfg && cfg->max_paths_per_pass > 0) ? cfg->max_paths_per_pass : (int64_t)96 << 20;  // fewer passes = fewer kernel tails; clamped to free memory per frame
  memset(&ctx->stats, 0, sizeof ctx->stats);
  memset(&ctx->scene, 0, sizeof ctx->scene);
  cudaError_t e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->ps[1].stream, cudaStreamNonBlocking);
  ctx->ps[0].stream = ctx->stream;
  if (e == cudaSuccess) e = cudaMalloc(&ctx->d_counters, CNT_TOTAL * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMalloc(&ctx->d_fis, RAYN_FIS_TABLE_SIZE * sizeof(float));
  for (PassSet& s : ctx->ps) {
    memset(&s.pb, 0, sizeof s.pb);
    s.pb.counters = ctx->d_counters;
    if (e == cudaSuccess) e = cudaMalloc(&s.d_work_ctr, WC_TOTAL * sizeof(int));
  }
  if (e == cudaSuccess) e = cudaMalloc(&ctx->d_kat, sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx->n_sm, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev1);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming);
  // persistent kernels: exactly as many CTAs as can be resident (one wave), so every CTA pulls work until the pass is drained
  for (int v = 0; v < SDFV_COUNT && e == cudaSuccess; ++v) {
    DISPATCH_SDFV(v, e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_ext[0][v], k_extend_march<V, false>, EXT_T, 0);
                  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_ext[1][v], k_extend_march<V, true>, EXT_T, 0);
                  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_shd[v], k_shadow<V>, SHD_T, 0);
                  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_nrm[v], k_normals<V, false>, SLOT_BLOCK, 0);
                  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_nrm_trap[v], k_normals<V, true>, SLOT_BLOCK, 0));
  }
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_pre, k_shade_pre<false>, SLOT_BLOCK, 0);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_post, k_shade_post<false>, SLOT_BLOCK, 0);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_pre_trap, k_shade_pre<true>, SLOT_BLOCK, 0);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_post_trap, k_shade_post<true>, SLOT_BLOCK, 0);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->occ_sph, k_extend_spheres, EXT_BATCH, 0);
  if (e != cudaSuccess) {
    cudaGetLastError();
    fail(nullptr, RAYN_ERR_CUDA, "context setup: %s", cudaGetErrorString(e));
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->ps[1].stream) cudaStreamDestroy(ctx->ps[1].stream);
    cudaFree(ctx->d_counters), cudaFree(ctx->d_fis), cudaFree(ctx->ps[0].d_work_ctr), cudaFree(ctx->ps[1].d_work_ctr), cudaFree(ctx->d_kat);
    for (cudaEvent_t ev : {ctx->ev0, ctx->ev1, ctx->ev_fork, ctx->ev_join})
      if (ev) cudaEventDestroy(ev);
    delete ctx;
    return RAYN_ERR_CUDA;
  }
  *out_ctx = ctx;
  return RAYN_OK;
}

int32_t rayn_b200_comm_destroy(RaynContext* ctx) {
  if (!ctx) return RAYN_ERR_INVALID_ARG;
  RaynComm& c = ctx->comm;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (c.comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c.comm);
  cudaFree(c.d_table), cudaFree(c.d_slabs);
  c = RaynComm();
  return RAYN_OK;
}

void rayn_b200_destroy(RaynContext* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  cudaStreamSynchronize(ctx->ps[1].stream);
  rayn_b200_comm_destroy(ctx);
  for (PassSet& s : ctx->ps) {
    free_pass(&s);
    cudaFree(s.d_work_ctr);
  }
  cudaFree(ctx->d_counters);
  cudaFree(ctx->d_kat);
  cudaFree(ctx->d_pack_ids);
  cudaFree(ctx->d_post);
  cudaFree(ctx->d_s1), cudaFree(ctx->d_s2), cudaFree(ctx->d_scr), cudaFree(ctx->d_fis), cudaFree(ctx->d_planes);
  cudaFree(ctx->d_prev);
  for (auto& t : ctx->timed) cudaEventDestroy(t.a), cudaEventDestroy(t.b);
  if (ctx->graph_exec) cudaGraphExecDestroy(ctx->graph_exec);
  cudaEventDestroy(ctx->ev0), cudaEventDestroy(ctx->ev1), cudaEventDestroy(ctx->ev_fork), cudaEventDestroy(ctx->ev_join);
  cudaStreamDestroy(ctx->stream), cudaStreamDestroy(ctx->ps[1].stream);
  delete ctx;
}

static int32_t validate_scene(RaynContext* ctx, const RaynSceneDesc* s) {
  if (!s) return fail(ctx, RAYN_ERR_INVALID_ARG, "scene is NULL");
  if (s->n_hitables < 1 || s->n_hitables > RAYN_MAX_HITABLES)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "n_hitables %d not in [1,%d]", s->n_hitables, RAYN_MAX_HITABLES);
  if (s->n_materials < 1 || s->n_materials > RAYN_MAX_MATERIALS)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "n_materials %d not in [1,%d]", s->n_materials, RAYN_MAX_MATERIALS);
  if (s->n_lights < 0 || s->n_lights > RAYN_MAX_LIGHTS)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "n_lights %d not in [0,%d]", s->n_lights, RAYN_MAX_LIGHTS);
  if (!s->hitables || !s->materials || (s->n_lights && !s->lights)) return fail(ctx, RAYN_ERR_INVALID_ARG, "NULL scene array");
  for (int i = 0; i < s->n_hitables; ++i) {
    const RaynHitable& h = s->hitables[i];
    if (h.kind < 0 || h.kind > RAYN_HITABLE_MANDELBULB) return fail(ctx, RAYN_ERR_INVALID_ARG, "hitable %d: bad kind %d", i, h.kind);
    if (h.material < 0 || h.material >= s->n_materials)
      return fail(ctx, RAYN_ERR_INVALID_ARG, "hitable %d: material %d out of range", i, h.material);
    if (h.kind != RAYN_HITABLE_SPHERE && (h.iterations < 0 || h.iterations > 1024))
      return fail(ctx, RAYN_ERR_INVALID_ARG, "hitable %d: iterations %d", i, h.iterations);
    if (h.kind == RAYN_HITABLE_MANDELBULB && h.bulb_power != 8)
      return fail(ctx, RAYN_ERR_UNSUPPORTED, "hitable %d: Mandelbulb power %d (only 8 is built)", i, h.bulb_power);
  }
  for (int i = 0; i < s->n_materials; ++i)
    if (s->materials[i].kind < 0 || s->materials[i].kind > RAYN_MATERIAL_EMISSIVE)
      return fail(ctx, RAYN_ERR_INVALID_ARG, "material %d: bad kind %d", i, s->materials[i].kind);
  if (s->camera.kind < 0 || s->camera.kind > RAYN_CAMERA_ORTHOGRAPHIC) return fail(ctx, RAYN_ERR_INVALID_ARG, "bad camera kind");
  if (s->consts.max_marches < 1 || s->consts.max_vis_marches < 1) return fail(ctx, RAYN_ERR_INVALID_ARG, "march limits must be >= 1");
  return RAYN_OK;
}

// Is the three-operation sphere-fold division (rt_sdf2.cuh::fastdiv2_3) equal to IEEE division for EVERY divisor this
// Mandelbox can produce?  The divisor is clamp(r2, min_r2, fixed_r2), so the candidates are the floats of that interval: all of
// them are divided on the device, once per (min_r2, fixed_r2) pair and context.
static bool div3_verified(RaynContext* ctx, const RaynHitable& h) {
  if (!sdf_box_fast_ok(h)) return false;
  for (const auto& c : ctx->div3_cache)
    if (c.min_r2 == h.min_rad_sq && c.fixed_r2 == h.fixed_rad_sq) return c.ok;
  bool ok = false;
  uint32_t lo, hi;
  memcpy(&lo, &h.min_rad_sq, 4);
  memcpy(&hi, &h.fixed_rad_sq, 4);
  if (hi >= lo && cudaSetDevice(ctx->device) == cudaSuccess) {  // positive floats order like their bit patterns
    const unsigned long long n = (unsigned long long)(hi - lo) + 1ull;
    unsigned long long bad = 1;
    if (cudaMemsetAsync(ctx->d_kat, 0, sizeof(unsigned long long), ctx->stream) == cudaSuccess) {
      k_verify_div3<<<ctx->n_sm * 8, 256, 0, ctx->stream>>>(h.fixed_rad_sq, lo, n, ctx->d_kat);
      if (cudaMemcpyAsync(&bad, ctx->d_kat, sizeof bad, cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess &&
          cudaStreamSynchronize(ctx->stream) == cudaSuccess)
        ok = bad == 0;
    }
    cudaGetLastError();
  }
  ctx->div3_cache.push_back({h.min_rad_sq, h.fixed_rad_sq, ok});
  return ok;
}

int32_t rayn_b200_upload_scene(RaynContext* ctx, const RaynSceneDesc* s) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  int32_t rc = validate_scene(ctx, s);
  if (rc) return rc;
  DevScene& d = ctx->scene;
  memset(&d, 0, sizeof d);
  d.n_hit = s->n_hitables;
  d.n_mat = s->n_materials;
  d.n_lights = s->n_lights;
  memcpy(d.hit, s->hitables, sizeof(RaynHitable) * s->n_hitables);
  memcpy(d.mat, s->materials, sizeof(RaynMaterial) * s->n_materials);
  if (s->n_lights) memcpy(d.light, s->lights, sizeof(RaynLight) * s->n_lights);
  d.cam = s->camera;
  d.vol = s->volume;
  d.rc = s->consts;
  for (int i = 0; i < d.n_hit; ++i) {  // compact sphere / SDF lists in insertion order (DevScene)
    const RaynHitable& h = d.hit[i];
    if (h.kind == RAYN_HITABLE_SPHERE) {
      d.sph_idx[d.n_sph] = i;
      d.hit_ord[i] = d.n_sph;
      d.sph[d.n_sph] = make_float4(h.center[0], h.center[1], h.center[2], h.radius);
      d.sph_moving |= (h.center_velocity[0] != 0.0f || h.center_velocity[1] != 0.0f || h.center_velocity[2] != 0.0f) ? 1 : 0;
      ++d.n_sph;
    } else {
      d.hit_ord[i] = d.n_sdf;
      d.sdf_idx[d.n_sdf++] = i;
    }
  }
  for (int i = 0; i < d.n_hit; ++i)
    ctx->sdf_var[i] = d.hit[i].kind == RAYN_HITABLE_SPHERE ? -1 : sdf_variant(d.hit[i], !(ctx->flags & RAYN_FLAG_NO_DIV3) && div3_verified(ctx, d.hit[i]));
  ctx->has_scene = true;  // the memset above cleared the orbit-trap list (trap_mask = 0)
  return RAYN_OK;
}

int32_t rayn_b200_set_albedo_traps(RaynContext* ctx, int32_t n, const RaynAlbedoTrap* traps) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!ctx->has_scene) return fail(ctx, RAYN_ERR_NO_SCENE, "set_albedo_traps before upload_scene");
  if (n < 0 || n > RAYN_MAX_MATERIALS) return fail(ctx, RAYN_ERR_INVALID_ARG, "n = %d traps not in [0,%d]", n, RAYN_MAX_MATERIALS);
  if (n > 0 && !traps) return fail(ctx, RAYN_ERR_INVALID_ARG, "traps is NULL");
  uint32_t mask = 0;
  DevTrap tab[RAYN_MAX_MATERIALS];
  memset(tab, 0, sizeof tab);
  for (int i = 0; i < n; ++i) {
    const RaynAlbedoTrap& t = traps[i];
    const int m = t.material;
    if (m < 0 || m >= ctx->scene.n_mat) return fail(ctx, RAYN_ERR_INVALID_ARG, "trap %d: material %d out of range", i, m);
    const int mk = ctx->scene.mat[m].kind;
    if (mk != RAYN_MATERIAL_LAMBERTIAN && mk != RAYN_MATERIAL_DIELECTRIC)
      return fail(ctx, RAYN_ERR_INVALID_ARG, "trap %d: material %d is neither Lambertian nor Dielectric", i, m);
    if (mask & (1u << m)) return fail(ctx, RAYN_ERR_INVALID_ARG, "trap %d: material %d has a trap already", i, m);
    bool finite = std::isfinite(t.trap_lo) && std::isfinite(t.trap_hi);
    for (int c = 0; c < 3; ++c) finite = finite && std::isfinite(t.albedo_lo[c]) && std::isfinite(t.albedo_hi[c]);
    if (!finite) return fail(ctx, RAYN_ERR_INVALID_ARG, "trap %d: non-finite value", i);
    if (!(t.trap_lo < t.trap_hi)) return fail(ctx, RAYN_ERR_INVALID_ARG, "trap %d: trap_lo %g >= trap_hi %g", i, t.trap_lo, t.trap_hi);
    mask |= 1u << m;
    tab[m].lo = t.trap_lo, tab[m].hi = t.trap_hi;
    for (int c = 0; c < 3; ++c) tab[m].a_lo[c] = t.albedo_lo[c], tab[m].a_hi[c] = t.albedo_hi[c];
  }
  ctx->scene.trap_mask = mask;
  memcpy(ctx->scene.trap, tab, sizeof tab);
  return RAYN_OK;
}

int32_t rayn_b200_get_stats(const RaynContext* ctx, RaynStats* out) {
  if (!ctx || !out) return RAYN_ERR_INVALID_ARG;
  *out = ctx->stats;
  return RAYN_OK;
}

int32_t rayn_b200_debug_sdf_variant(const RaynContext* ctx, int32_t hitable_index) {
  if (!ctx || !ctx->has_scene || hitable_index < 0 || hitable_index >= ctx->scene.n_hit) return -2;
  return ctx->sdf_var[hitable_index];
}

int32_t rayn_b200_debug_enable_queue_log(RaynContext* ctx, int32_t enable) {
  if (!ctx) return RAYN_ERR_INVALID_ARG;
  ctx->qlog_enabled = enable != 0;
  ctx->qlog.clear();
  return RAYN_OK;
}
int64_t rayn_b200_debug_read_queue_log(RaynContext* ctx, int32_t* out, int64_t cap) {
  if (!ctx) return -1;
  const int64_t n = (int64_t)ctx->qlog.size();
  if (out && cap > 0) memcpy(out, ctx->qlog.data(), sizeof(int32_t) * (size_t)std::min(n, cap));
  return n;
}

}  // extern "C"

// ---- the stages a render and the albedo pass (rayn_b200_render_albedo) share ----------------------------------------
// What a render derives from its frame (frame_check) and from the uploaded scene (scene_plan) before it launches anything.
struct FramePlan {
  DevFrame fr;
  int R, QS, np, wpc;  // paths and shading slots per tile; k_resolve's padded spp and warps per CTA
  bool simple, traps, fold_all, volume_on;
  int fold_pre, n_fold, ns, seg_per_path, lc_ns;
};

// One render or albedo pass on a context: its plan and pass size (job_begin) and the pass being enqueued (pass_tiles).  The
// job's tiles are ctx->job_tiles.
struct Job {
  FramePlan P;
  PassBufs pb;  // pb.n_tiles: the tiles of the current pass
  int tiles_per_pass;
  int n_sets;   // pass sets in flight: 2 when the passes alternate between ctx->ps[0] and ctx->ps[1] (size_pass)
  bool paired;  // the current pass runs beside a pass of the other set (march_grid)
  // the current pass's set: its stream and the work lists and work counters of its persistent kernels
  cudaStream_t st;
  int *batch_prefix, *work_ctr;
};

// The resident grid (one wave) of a kernel that strides over a work list of the pass (k_scan_slots / k_scan_live), capped
// by the list's upper bound.
static unsigned resident(const RaynContext* ctx, const Job& J, int occ) {
  const int64_t max_blocks = (int64_t)J.pb.n_tiles * ((J.P.QS + SLOT_BLOCK - 1) / SLOT_BLOCK);
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((int64_t)ctx->n_sm * occ, max_blocks));
}

// The frame checks of render_frame and the DevFrame of the frame (tables not uploaded yet).  tiles_given: the caller picks
// the tiles itself, so tile_offset / tile_stride are not checked.
static int32_t frame_check(RaynContext* ctx, const RaynFrameDesc* f, bool tiles_given, FramePlan* P) {
  if (f->width <= 0 || f->height <= 0 || f->tile_w <= 0 || f->tile_h <= 0 || f->samples <= 0 || f->max_bounces < 0)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "bad frame geometry");
  if (f->volume_marches != 2)
    return fail(ctx, RAYN_ERR_UNSUPPORTED, "volume_marches = %d: the reference hard-wires samples_1d[3],[4] for vm = 2", f->volume_marches);
  const int spp = 4 * f->samples, vm = f->volume_marches, mb = f->max_bounces;
  const int need1 = 1 + (mb + 1) * (3 + vm), need2 = 2 + (mb + 1) * (12 + 8 * vm) / 2;
  if (f->sets_1d < need1 || f->sets_2d < need2)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "sample tables too small: have %d/%d sets, path needs %d/%d", f->sets_1d, f->sets_2d, need1, need2);
  if (!f->samples_1d || !f->samples_2d || !f->scramble || !f->fis_inverse_cdf) return fail(ctx, RAYN_ERR_INVALID_ARG, "NULL input table");
  const int stride = f->tile_stride > 0 ? f->tile_stride : 1;
  if (!tiles_given && !f->tile_list && (f->tile_offset < 0 || f->tile_offset >= stride))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "tile_offset %d not in [0,%d)", f->tile_offset, stride);
  if (mb >= TERM_MAX_DEPTH) return fail(ctx, RAYN_ERR_UNSUPPORTED, "max_bounces > %d", TERM_MAX_DEPTH - 1);
  const int64_t R64 = (int64_t)f->tile_w * f->tile_h * spp;
  const int n_hit = ctx->scene.n_hit;
  if (R64 + 4 * n_hit >= TERM_MAX_SLOTS)
    return fail(ctx, RAYN_ERR_UNSUPPORTED, "tile_w*tile_h*spp = %lld exceeds the 2^%d slot key space", (long long)R64, TERM_DEPTH_SHIFT);
  int& np = P->np;
  np = 32;
  while (np < spp) np <<= 1;
  const int wpc = P->wpc = resolve_warps_per_cta(np);
  if (wpc < 1 || np > 65536) return fail(ctx, RAYN_ERR_UNSUPPORTED, "spp = %d: the film resolve holds 6 B per sample of a pixel in shared memory (max 32768 spp)", spp);
  P->R = (int)R64, P->QS = P->R + 4 * n_hit;
  CU(cudaSetDevice(ctx->device));
  {  // a previous call that failed half way through a graph capture must not leave the stream capturing
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(ctx->stream, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone) {
      cudaGraph_t g = nullptr;
      cudaStreamEndCapture(ctx->stream, &g);
      if (g) cudaGraphDestroy(g);
    }
    cudaGetLastError();
  }

  DevFrame& fr = P->fr;
  fr.W = f->width, fr.H = f->height, fr.tile_w = f->tile_w, fr.tile_h = f->tile_h;
  fr.samples = f->samples, fr.spp = spp, fr.max_bounces = mb, fr.vm = vm;
  tile_grid_of(f->width, f->height, f->tile_w, f->tile_h, &fr.ntx, &fr.nty);
  fr.sets_1d = f->sets_1d, fr.sets_2d = f->sets_2d;
  fr.t0 = f->t0, fr.t1 = f->t1;
  return RAYN_OK;
}

// The sample tables, scramble and filter table on the device: host-space inputs are copied into the context's staging.
static int32_t upload_tables(RaynContext* ctx, const RaynFrameDesc* f, DevFrame* frp) {
  DevFrame& fr = *frp;
  const int spp = fr.spp;
  cudaStream_t st = ctx->stream;
  const size_t n1 = (size_t)spp * f->sets_1d, n2 = (size_t)2 * spp * f->sets_2d, npx = (size_t)f->width * f->height;
  if (f->input_space == RAYN_MEM_HOST) {
    CU(regrow(&ctx->d_s1, &ctx->cap_s1, n1));
    CU(regrow(&ctx->d_s2, &ctx->cap_s2, n2));
    CU(regrow(&ctx->d_scr, &ctx->cap_scr, npx));
    CU(cudaMemcpyAsync(ctx->d_s1, f->samples_1d, n1 * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(ctx->d_s2, f->samples_2d, n2 * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(ctx->d_scr, f->scramble, npx * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(ctx->d_fis, f->fis_inverse_cdf, RAYN_FIS_TABLE_SIZE * 4, cudaMemcpyHostToDevice, st));
    fr.s1 = ctx->d_s1, fr.s2 = ctx->d_s2, fr.scramble = ctx->d_scr, fr.fis = ctx->d_fis;
  } else {
    fr.s1 = f->samples_1d, fr.s2 = f->samples_2d, fr.scramble = f->scramble, fr.fis = f->fis_inverse_cdf;
  }
  return RAYN_OK;
}

// Which kernels the scene needs and how the closest-hit fold is split between them.
static int32_t scene_plan(RaynContext* ctx, FramePlan* P) {
  const int n_hit = ctx->scene.n_hit, n_sdf = ctx->scene.n_sdf, vm = P->fr.vm;
  const bool simple = P->simple = (ctx->flags & RAYN_FLAG_SIMPLE_MARCH) != 0;
  // time-varying sphere centres need the packet's lane-0 time: only the product kernels plumb it
  const bool motion = ctx->scene.sph_moving != 0;
  if (motion && simple) return fail(ctx, RAYN_ERR_UNSUPPORTED, "time-varying sphere centres are not supported by the legacy test kernels");
  const bool traps = P->traps = ctx->scene.trap_mask != 0u;
  if (traps && simple) return fail(ctx, RAYN_ERR_UNSUPPORTED, "orbit-trap albedos are not supported by the legacy test kernels");
  // leading analytic spheres run inside raygen / shade_post (rt_kernels.cuh::fold_head); -1 = not folded (moving spheres need
  // the extend packet's lane-0 time; the legacy test kernels do the whole fold themselves)
  int& fold_pre = P->fold_pre;
  fold_pre = -1;
  if (!motion && !simple) {
    fold_pre = 0;
    while (fold_pre < n_hit && ctx->scene.hit[fold_pre].kind == RAYN_HITABLE_SPHERE) ++fold_pre;
  }
  // Scenes of the shape [spheres] Mandelbox [spheres] (setup.rs) fold ALL analytic spheres into the producing kernel and march
  // the SDF last, against the nearest sphere: one gather of every live ray per depth less (no k_extend_spheres
  // launch) and shorter marches for rays that end on an emitter.  The result is the reference's fold bit for bit
  // (proof in rt_kernels.cuh at k_extend_march: it needs a distance estimator that is never negative, i.e. the Mandelbox -
  // sqrt(m) / |dr| - so that a march's t never decreases, and the first-index-wins tie rule, which the kernel applies).
  const bool fold_all = P->fold_all = fold_pre >= 0 && n_sdf == 1 && ctx->scene.hit[ctx->scene.sdf_idx[0]].kind == RAYN_HITABLE_MANDELBOX && !(ctx->flags & RAYN_FLAG_NO_FOLD_ALL);
  P->n_fold = fold_all ? ctx->scene.n_sph : fold_pre;  // leading spheres are the first fold_pre entries of the compact sphere list
  const bool volume_on = P->volume_on = ctx->scene.vol.has_scattering != 0 && ctx->scene.n_lights > 0;
  const int ns = P->ns = volume_on ? 4 * (1 + vm) : 4;               // light samples per path per depth
  P->seg_per_path = simple ? 0 : ns * n_sdf;          // worst case shadow segments per path per depth, all SDF queues
  P->lc_ns = simple ? 0 : ns;                         // stored light contributions per path per depth
  return RAYN_OK;
}

// Pass size for n_tiles tiles (as many tiles per pass as the path budget and free device memory allow), and the pass buffers.
// A job that needs several passes sizes each from half the memory budget, so that two passes fit at once; with two_sets
// (a render that may overlap its passes) it then also gets the second pass set, and *out_sets is 2.  A job that fits one
// pass, a half budget that holds no tile, or a second set that does not fit leave one set, sized as for a single stream.
static int32_t size_pass(RaynContext* ctx, const FramePlan& P, size_t n_tiles, bool two_sets, int* out_tiles_per_pass, int* out_sets) {
  const int R = P.R, QS = P.QS, n_sdf = ctx->scene.n_sdf, ns = P.ns, seg_per_path = P.seg_per_path, lc_ns = P.lc_ns;
  const bool traps = P.traps;
  const size_t bpp = pass_bytes_per_path(&ctx->ps[0], R, QS, seg_per_path, lc_ns, traps);
  size_t free_b = 0, total_b = 0;
  CU(cudaMemGetInfo(&free_b, &total_b));
  const size_t budget = (size_t)((double)(free_b + pass_set_bytes(ctx->ps[0]) + pass_set_bytes(ctx->ps[1])) * 0.90);
  auto tiles_for = [&](size_t bytes) {  // whole tiles of a pass that fits `bytes` (0: not even one)
    int64_t max_paths = std::min<int64_t>(ctx->cap_paths, (int64_t)(bytes / bpp));
    if (n_sdf > 0) max_paths = std::min<int64_t>(max_paths, ((int64_t)1 << 27) - 1);          // owner path index is packed with the sample bit (<< 4)
    if (n_sdf > 0) max_paths = std::min<int64_t>(max_paths, (int64_t)INT_MAX / std::max(ns, 1));  // 32-bit queue cursors per SDF
    return std::min<int64_t>(max_paths / R, 65535);
  };
  int64_t tiles = tiles_for(budget);
  const bool several = tiles < (int64_t)n_tiles, halves = several && tiles_for(budget / 2) >= 1;
  if (halves) tiles = tiles_for(budget / 2);
  int& tiles_per_pass = *out_tiles_per_pass;
  tiles_per_pass = (int)std::max<int64_t>(1, tiles);
  tiles_per_pass = std::min<int>(tiles_per_pass, (int)std::max<size_t>(n_tiles, 1));
  int32_t rc;
  while ((rc = ensure_pass(ctx, &ctx->ps[0], tiles_per_pass, R, QS, seg_per_path, n_sdf, lc_ns, traps)) == RAYN_ERR_OOM) {
    if (pass_set_bytes(ctx->ps[1])) {  // the second set's memory goes first
      free_pass(&ctx->ps[1]);
      continue;
    }
    if (tiles_per_pass == 1) break;
    tiles_per_pass = (tiles_per_pass + 1) / 2;  // fragmentation / another tenant: retry with half the pass
  }
  *out_sets = 1;
  if (rc || !two_sets || !halves || (size_t)tiles_per_pass >= n_tiles) return rc;
  rc = ensure_pass(ctx, &ctx->ps[1], tiles_per_pass, R, QS, seg_per_path, n_sdf, lc_ns, traps);
  if (rc == RAYN_ERR_OOM) return RAYN_OK;  // one pass at a time (ensure_pass left ps[1] empty)
  if (rc == RAYN_OK) {
    *out_sets = 2;
    // passes of equal size (the same count), so that the two streams run their passes side by side to the end
    const size_t passes = (n_tiles + tiles_per_pass - 1) / tiles_per_pass;
    tiles_per_pass = (int)((n_tiles + passes - 1) / passes);
  }
  return rc;
}

// Points J's current pass at pass set `set`: its buffers, stream, work lists and work counters.
static void pass_set_use(RaynContext* ctx, Job* J, int set) {
  PassSet& s = ctx->ps[set];
  PassBufs& pb = J->pb = s.pb;
  pb.R = J->P.R, pb.QS = J->P.QS, pb.tile_ids = s.d_tile_ids;
  pb.lc_ns = J->P.lc_ns;
  pb.seg_count = s.d_work_ctr + WC_SEG_COUNT;
  J->st = s.stream, J->batch_prefix = s.d_batch_prefix, J->work_ctr = s.d_work_ctr;
}

// The grid of a persistent march (k_extend_march, k_shadow): one resident wave of occ CTAs per SM, or half of it while two
// passes are in flight (J.paired).  Two marches then run side by side within one wave, and the other pass's short kernels (scans,
// bins, shading, compaction) find free CTA slots at once instead of waiting for this march's drain.  Either way the march's
// CTAs only take work from a global counter, so the grid size changes the schedule, never the result.
static unsigned march_grid(const RaynContext* ctx, const Job& J, int occ) {
  return (unsigned)ctx->n_sm * (J.paired ? (occ + 1) / 2 : occ);
}

// One depth's closest-hit stage (the non-legacy kernels): k_scan_live, then the fold over the live rays of the pass.
static int32_t extend_enqueue(RaynContext* ctx, const Job& J, const Thr& thr) {
  cudaStream_t st = J.st;
  const PassBufs& pb = J.pb;
  const int n_hit = ctx->scene.n_hit, fold_pre = J.P.fold_pre;
  const bool fold_all = J.P.fold_all, motion = ctx->scene.sph_moving != 0;
  const unsigned sph_grid = resident(ctx, J, ctx->occ_sph);
  timed_begin(ctx, RAYN_K_MISC);
  k_scan_live<<<1, SCAN_T, 0, st>>>(pb, J.batch_prefix, J.work_ctr);
  timed_end(ctx, RAYN_K_MISC);
  // fold order of hitable.rs:177-198: runs of spheres as coherent kernels, each SDF as a persistent march.  The
  // spheres before the first SDF were already folded in by the kernel that produced the rays (fold_pre >= 0).
  int k = fold_pre >= 0 ? fold_pre : 0, first_kernel = fold_pre >= 0 ? 0 : 1, n_march = 0;
  while (k < n_hit || first_kernel) {
    int e = k;
    while (e < n_hit && ctx->scene.hit[e].kind == RAYN_HITABLE_SPHERE) ++e;
    if ((e > k || first_kernel) && !fold_all) {
      timed_begin(ctx, RAYN_K_EXTEND_SPHERES);
      k_extend_spheres<<<sph_grid, EXT_BATCH, 0, st>>>(ctx->scene, pb, k, e, first_kernel, motion ? 1 : 0, J.batch_prefix, J.work_ctr + WC_SPHERES + k);
      timed_end(ctx, RAYN_K_EXTEND_SPHERES);
      first_kernel = 0;
    }
    if (e < n_hit) {
      if (n_march++ > 0) CU(cudaMemsetAsync(J.work_ctr + WC_EXTEND, 0, sizeof(int), st));
      const int v = ctx->sdf_var[e];
      timed_begin(ctx, RAYN_K_EXTEND);
      const int sf = fold_all ? 1 : 0;
      if (thr.is_const)
        DISPATCH_SDFV(v, (k_extend_march<V, true><<<march_grid(ctx, J, ctx->occ_ext[1][v]), EXT_T, 0, st>>>(ctx->scene, pb, thr, e, sf, J.batch_prefix, J.work_ctr + WC_EXTEND)))
      else
        DISPATCH_SDFV(v, (k_extend_march<V, false><<<march_grid(ctx, J, ctx->occ_ext[0][v]), EXT_T, 0, st>>>(ctx->scene, pb, thr, e, sf, J.batch_prefix, J.work_ctr + WC_EXTEND)))
      timed_end(ctx, RAYN_K_EXTEND);
      ++e;
    }
    k = e;
  }
  return RAYN_OK;
}

// ---- the job driver of a render (render_enqueue) and an albedo pass (rayn_b200_render_albedo) ---------------------------
// job_ready and job_begin, then per pass pass_tiles, pass_raygen and the job's own kernels; the job is then pending.

// The context checks of every job, made before the call's own argument checks.
static int32_t job_ready(RaynContext* ctx, const char* call) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (ctx->pending) return fail(ctx, RAYN_ERR_INVALID_ARG, "a render is already in flight on this context");
  if (!ctx->has_scene) return fail(ctx, RAYN_ERR_NO_SCENE, "%s before upload_scene", call);
  return RAYN_OK;
}

// The job prologue: frame checks, tile list, stats reset, fence, input tables, scene plan, pass sizing and pass buffers.
// render: a render, whose tiles are `tiles` or else the frame's own selection, and which restarts the debug queue log;
// otherwise the albedo pass, which renders the whole tile grid.  out_space: where the job's output lives.
static int32_t job_begin(RaynContext* ctx, const RaynFrameDesc* f, const std::vector<int>* tiles, bool render, int32_t out_space, Job* J) {
  FramePlan& P = J->P;
  int32_t rc = frame_check(ctx, f, tiles || !render, &P);
  if (rc) return rc;
  const DevFrame& fr = P.fr;
  const int stride = f->tile_stride > 0 ? f->tile_stride : 1;
  std::vector<int>& my_tiles = ctx->job_tiles;
  my_tiles.clear();
  if (tiles) {
    my_tiles = *tiles;
  } else if (!render) {
    for (int idx = 0; idx < fr.ntx * fr.nty; ++idx) my_tiles.push_back(idx);
  } else if (f->tile_list) {
    if (f->n_tile_list < 0) return fail(ctx, RAYN_ERR_INVALID_ARG, "n_tile_list < 0");
    for (int i = 0; i < f->n_tile_list; ++i) {
      const int idx = f->tile_list[i];
      if (idx < 0 || idx >= fr.ntx * fr.nty || (i && idx <= f->tile_list[i - 1]))
        return fail(ctx, RAYN_ERR_INVALID_ARG, "tile_list must be ascending tile indices in [0,%d)", fr.ntx * fr.nty);
      my_tiles.push_back(idx);
    }
  } else {
    for (int idx = f->tile_offset; idx < fr.ntx * fr.nty; idx += stride) my_tiles.push_back(idx);
  }
  // the job's geometry, for render_finish once the caller has marked the job pending; no host-space outputs until job_stage
  ctx->job_w = f->width, ctx->job_h = f->height, ctx->job_tw = f->tile_w, ctx->job_th = f->tile_h, ctx->job_spp = fr.spp, ctx->job_nty = fr.nty;
  ctx->job_out.clear();

  memset(&ctx->stats, 0, sizeof ctx->stats);
  ctx->timed_used = 0;
  if (render) ctx->qlog.clear();
  // Device-space pointers may have been produced on another stream (e.g. torch's): fence.
  if (f->input_space == RAYN_MEM_DEVICE || out_space == RAYN_MEM_DEVICE) CU(cudaDeviceSynchronize());
  CU(cudaEventRecord(ctx->ev0, ctx->stream));
  if ((rc = upload_tables(ctx, f, &P.fr))) return rc;
  if ((rc = scene_plan(ctx, &P))) return rc;
  // Two passes in flight only for a render whose launches are not bracketed one by one (RAYN_FLAG_TIMING) and whose
  // depths are not read back (the debug queue log)
  const bool two_sets = render && !(ctx->flags & RAYN_FLAG_TIMING) && !ctx->qlog_enabled;
  if ((rc = size_pass(ctx, P, my_tiles.size(), two_sets, &J->tiles_per_pass, &J->n_sets))) return rc;
  pass_set_use(ctx, J, 0);
  J->paired = false;
  CU(cudaMemsetAsync(ctx->d_counters, 0, CNT_TOTAL * sizeof(unsigned long long), ctx->stream));
  return RAYN_OK;
}

// Starts the pass over tiles [first, first + tiles_per_pass) of the job on pass set `set`: uploads their ids.  The upload
// reads host memory, so a render's graph capture begins after it.
static int32_t pass_tiles(RaynContext* ctx, Job* J, size_t first, int set) {
  pass_set_use(ctx, J, set);
  const int nt = J->pb.n_tiles = (int)std::min<size_t>(J->tiles_per_pass, ctx->job_tiles.size() - first);
  CU(cudaMemcpyAsync(ctx->ps[set].d_tile_ids, ctx->job_tiles.data() + first, nt * sizeof(int), cudaMemcpyHostToDevice, J->st));
  return RAYN_OK;
}

// Stages the job's n host-space outputs back to back in ctx->d_planes, in the order of `planes`, and zeroes the whole
// staging if `zero`; stage[i] receives the staging of planes[i], also of a plane whose user pointer is NULL.  The offsets,
// the staging size and job_end's copies all come from this one list.
static int32_t job_stage(RaynContext* ctx, const JobPlane* planes, int n, bool zero, float** stage) {
  const size_t npx = (size_t)ctx->job_w * ctx->job_h;
  size_t floats = 0;
  for (int i = 0; i < n; ++i) floats += planes[i].floats;
  CU(regrow(&ctx->d_planes, &ctx->cap_planes, floats * npx));
  if (zero) CU(cudaMemsetAsync(ctx->d_planes, 0, floats * npx * sizeof(float), ctx->stream));
  floats = 0;
  for (int i = 0; i < n; ++i) stage[i] = ctx->d_planes + floats * npx, floats += planes[i].floats;
  ctx->job_out.assign(planes, planes + n);
  return RAYN_OK;
}

// The pass's k_raygen, one thread per path.
static void pass_raygen(RaynContext* ctx, const Job& J) {
  ctx->stats.passes++;
  timed_begin(ctx, RAYN_K_RAYGEN);
  k_raygen<<<dim3((J.P.R + 255) / 256, J.pb.n_tiles), 256, 0, J.st>>>(ctx->scene, J.P.fr, J.pb, J.P.n_fold);
  timed_end(ctx, RAYN_K_RAYGEN);
}

// Enqueues one render on the context's stream.  Nothing here waits for the GPU (except the debug queue log), so a single
// host thread can keep several GPUs busy (render_frame_multi).  tiles_override replaces the frame's own tile selection.
// dev_planes_out (optional) receives the device-space planes the film was rendered into.  moments (optional,
// rayn_b200_render_frame_moments): the lum^2 planes, in out->space, which the k_resolve<true> instance also writes.
static int32_t render_enqueue(RaynContext* ctx, const RaynFrameDesc* f, const RaynFilmPlanes* out, const std::vector<int>* tiles_override,
                              RaynFilmPlanes* dev_planes_out, const RaynMomentPlanes* moments) {
  int32_t rc = job_ready(ctx, "render_frame");
  if (rc) return rc;
  if (!f || !out) return fail(ctx, RAYN_ERR_INVALID_ARG, "frame/out is NULL");
  Job J;
  if ((rc = job_begin(ctx, f, tiles_override, true, out->space, &J))) return rc;
  const FramePlan& P = J.P;
  const DevFrame& fr = P.fr;
  PassBufs& pb = J.pb;
  const std::vector<int>& my_tiles = ctx->job_tiles;
  const bool mom = moments != nullptr;
  const int mb = fr.max_bounces, np = P.np, wpc = mom ? resolve_warps_per_cta(np, true) : P.wpc, R = P.R, QS = P.QS, n_hit = ctx->scene.n_hit, n_sdf = ctx->scene.n_sdf, n_fold = P.n_fold;
  const int* sdf_idx = ctx->scene.sdf_idx;
  const bool simple = P.simple, motion = ctx->scene.sph_moving != 0, traps = P.traps, volume_on = P.volume_on;

  if (mom && wpc < 1) return fail(ctx, RAYN_ERR_UNSUPPORTED, "render_frame_moments: spp = %d does not fit the film resolve's shared memory", fr.spp);
  const size_t npx = (size_t)f->width * f->height;
  RaynFilmPlanes dp = *out;  // the device-space planes the film is rendered into
  float *dm_color = mom ? moments->color_lum2 : nullptr, *dm_bg = mom ? moments->background_lum2 : nullptr;  // ... and moment planes
  if (out->space == RAYN_MEM_HOST) {  // (render_frame_moments: the moment planes are in out->space too)
    // the film block (film_block_planes' layout), then with moments the two moment planes
    const JobPlane planes[6] = {{out->color, 3}, {out->alpha, 1}, {out->background, 3}, {out->normal, 3}, {dm_color, 1}, {dm_bg, 1}};
    float* stage[6];
    if ((rc = job_stage(ctx, planes, mom ? 6 : 4, true, stage))) return rc;
    dp = RaynFilmPlanes{stage[0], stage[1], stage[2], stage[3], RAYN_MEM_DEVICE};
    dm_color = dm_color ? stage[4] : nullptr, dm_bg = dm_bg ? stage[5] : nullptr;
  } else {
    const int cov_w = std::min(fr.ntx * f->tile_w, f->width), cov_h = std::min(fr.nty * f->tile_h, f->height);
    if (cov_w < f->width || cov_h < f->height) {
      k_zero_uncovered<<<(unsigned)((npx + 255) / 256), 256, 0, ctx->stream>>>(f->width, f->height, cov_w, cov_h, dp.color, dp.alpha, dp.background, dp.normal);
      for (float* m : {dm_color, dm_bg})  // the one-channel slot of k_zero_uncovered, once per plane
        if (m) k_zero_uncovered<<<(unsigned)((npx + 255) / 256), 256, 0, ctx->stream>>>(f->width, f->height, cov_w, cov_h, nullptr, m, nullptr, nullptr);
    }
  }
  dp.space = RAYN_MEM_DEVICE;
  if (dev_planes_out) *dev_planes_out = dp;

  const size_t res_smem = resolve_smem_per_warp(np, mom) * wpc;
  int slot_bits = 5, depth_bits = 1;  // significant bits of a shading slot (< QS) and of a depth (<= max_bounces): what k_resolve's radix sort walks
  while ((1 << slot_bits) < QS + 1) ++slot_bits;
  while ((1 << depth_bits) < mb + 1) ++depth_bits;
  CU(cudaFuncSetAttribute(mom ? k_resolve<true> : k_resolve<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)res_smem));

  // Small single-pass frames are launch bound (config 1: ~20 launches of a few microseconds each): capture the whole kernel
  // sequence of the pass once and replay it as ONE graph launch while nothing that is baked into the launches changes
  // (scene, frame geometry, every pointer, the tile set).
  const bool single_pass = my_tiles.size() <= (size_t)J.tiles_per_pass;
  const bool use_graph = single_pass && !my_tiles.empty() && !(ctx->flags & (RAYN_FLAG_TIMING | RAYN_FLAG_NO_GRAPH)) && !ctx->qlog_enabled &&
                         (int64_t)my_tiles.size() * R <= ((int64_t)8 << 20);
  bool capturing = false, replayed = false;
  uint64_t key = 0;
  if (use_graph) {
    PassBufs kpb = pb;
    kpb.n_tiles = (int)my_tiles.size();
    key = fnv1a(1469598103934665603ull, &ctx->scene, sizeof ctx->scene);
    key = fnv1a(key, &fr, sizeof fr);
    key = fnv1a(key, &kpb, sizeof kpb);
    // every plane pointer: host-space moment planes are staged after the film block, so the first such render may grow
    // d_planes from 10 to 12 floats per pixel and move the film block; the moved pointers give a new key, and regrow only
    // grows, so a graph is replayed only into the staging it was captured with
    float* planes6[6] = {dp.color, dp.alpha, dp.background, dp.normal, dm_color, dm_bg};
    key = fnv1a(key, planes6, sizeof planes6);
    const int misc[7] = {np, wpc, mb, n_fold, simple ? 1 : 0, motion ? 1 : 0, mom ? 1 : 0};  // mom: the k_resolve instance
    key = fnv1a(key, misc, sizeof misc);
    key = fnv1a(key, my_tiles.data(), my_tiles.size() * sizeof(int));
    if (ctx->graph_exec && ctx->graph_key == key) {
      CU(cudaMemcpyAsync(ctx->ps[0].d_tile_ids, my_tiles.data(), my_tiles.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
      CU(cudaGraphLaunch(ctx->graph_exec, ctx->stream));
      ctx->stats = ctx->graph_stats;
      replayed = true;
    }
  }
  // Several passes alternate between the two pass sets, pass k on set k % 2 and its stream: each stream runs its passes in
  // order, so a set is reused only after its previous pass, and the two streams overlap one pass's tails with the other's
  // work.  ps[1].stream starts after everything the job has enqueued so far and is joined back into the context's stream
  // when the passes are enqueued, also on an error return, so whatever follows on the context's stream (copy-out, gather,
  // render_finish, the accumulator fold, the next job) sees the whole film.
  struct Join {
    RaynContext* ctx;
    bool on;
    ~Join() {
      if (on && cudaEventRecord(ctx->ev_join, ctx->ps[1].stream) == cudaSuccess) cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0);
    }
  } join{ctx, false};
  if (J.n_sets > 1 && !replayed) {
    CU(cudaEventRecord(ctx->ev_fork, ctx->stream));
    CU(cudaStreamWaitEvent(ctx->ps[1].stream, ctx->ev_fork, 0));
    join.on = true;
  }
  std::vector<int> h_nslots, h_slots;
  const size_t n_passes = (my_tiles.size() + J.tiles_per_pass - 1) / J.tiles_per_pass;
  for (size_t first = 0, k = 0; first < my_tiles.size() && !replayed; first += J.tiles_per_pass, ++k) {
    if ((rc = pass_tiles(ctx, &J, first, (int)(k % J.n_sets)))) return rc;
    // the last pass of an odd count runs alone once its partner's pass ends: full waves
    J.paired = J.n_sets > 1 && !(n_passes % 2 == 1 && k == n_passes - 1);
    const cudaStream_t st = J.st;
    if (use_graph) {
      CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      capturing = true;
    }
    pass_raygen(ctx, J);
    const int nt = pb.n_tiles;
    const int nseg = (QS + SEG_SLOTS - 1) / SEG_SLOTS;  // segments per tile of the queue kernels
    for (int depth = 0; depth <= mb; ++depth) {
      const Thr thr = make_thr(ctx->scene.cam, depth);
      if (simple) {
#ifdef RAYN_LEGACY_KERNELS
        timed_begin(ctx, RAYN_K_EXTEND);
        k_extend<<<dim3((R + 127) / 128, nt), 128, 0, st>>>(ctx->scene, pb, thr);
        timed_end(ctx, RAYN_K_EXTEND);
#endif
      } else {
        if ((rc = extend_enqueue(ctx, J, thr))) return rc;
      }
      timed_begin(ctx, RAYN_K_BIN);
      k_bin_count<<<dim3(nseg, nt), BIN_T, 0, st>>>(pb, n_hit, nseg);
      k_bin_scatter<<<dim3(nseg, nt), BIN_T, 0, st>>>(pb, n_hit, nseg);
      if (!simple) k_scan_slots<<<1, SCAN_T, 0, st>>>(ctx->scene, pb);  // work lists of k_normals / k_shade_pre / k_shade_post
      timed_end(ctx, RAYN_K_BIN, simple ? 2 : 3);
      if (ctx->qlog_enabled) {
        h_nslots.resize(nt);
        h_slots.resize((size_t)nt * QS);
        CU(cudaMemcpyAsync(h_nslots.data(), pb.n_slots, nt * sizeof(int), cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(h_slots.data(), pb.q_shade, (size_t)nt * QS * sizeof(int), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        for (int t = 0; t < nt; ++t) {
          ctx->qlog.push_back(depth);
          ctx->qlog.push_back(my_tiles[first + t]);
          ctx->qlog.push_back(h_nslots[t]);
          for (int s = 0; s < h_nslots[t]; ++s) ctx->qlog.push_back(h_slots[(size_t)t * QS + s]);
        }
      }
      if (!simple) {
        // get_shading_info of the SDF hitables whose material is shaded (receives light, or volumetrics sample along the ray)
        for (int j = 0; j < n_sdf; ++j) {
          const RaynHitable& h = ctx->scene.hit[sdf_idx[j]];
          const int mk = ctx->scene.mat[h.material].kind;
          if (!(mk == RAYN_MATERIAL_LAMBERTIAN || mk == RAYN_MATERIAL_DIELECTRIC || volume_on)) continue;
          const int v = ctx->sdf_var[sdf_idx[j]];
          timed_begin(ctx, RAYN_K_NORMALS);
          if ((ctx->scene.trap_mask >> h.material) & 1u)  // the bin's material has an orbit-trap albedo: normals + trap
            DISPATCH_SDFV(v, (k_normals<V, true><<<resident(ctx, J, ctx->occ_nrm_trap[v]), SLOT_BLOCK, 0, st>>>(ctx->scene, pb, thr, sdf_idx[j], j, J.work_ctr + WC_NORMALS + j)))
          else
            DISPATCH_SDFV(v, (k_normals<V, false><<<resident(ctx, J, ctx->occ_nrm[v]), SLOT_BLOCK, 0, st>>>(ctx->scene, pb, thr, sdf_idx[j], j, J.work_ctr + WC_NORMALS + j)))
          timed_end(ctx, RAYN_K_NORMALS);
        }
        timed_begin(ctx, RAYN_K_SHADE_PRE);
        if (traps)
          k_shade_pre<true><<<resident(ctx, J, ctx->occ_pre_trap), SLOT_BLOCK, 0, st>>>(ctx->scene, fr, pb, depth, thr, J.work_ctr + WC_PRE);
        else
          k_shade_pre<false><<<resident(ctx, J, ctx->occ_pre), SLOT_BLOCK, 0, st>>>(ctx->scene, fr, pb, depth, thr, J.work_ctr + WC_PRE);
        timed_end(ctx, RAYN_K_SHADE_PRE);
        if (ctx->scene.n_lights > 0) {
          for (int j = 0; j < n_sdf; ++j) {
            const int v = ctx->sdf_var[sdf_idx[j]];
            timed_begin(ctx, RAYN_K_SHADOW);
            DISPATCH_SDFV(v, (k_shadow<V><<<march_grid(ctx, J, ctx->occ_shd[v]), SHD_T, 0, st>>>(ctx->scene, pb, sdf_idx[j], j, J.work_ctr + WC_SHADOW + j)));
            timed_end(ctx, RAYN_K_SHADOW);
          }
        }
        timed_begin(ctx, RAYN_K_SHADE_POST);
        if (traps)
          k_shade_post<true><<<resident(ctx, J, ctx->occ_post_trap), SLOT_BLOCK, 0, st>>>(ctx->scene, fr, pb, depth, n_fold, J.work_ctr + WC_POST);
        else
          k_shade_post<false><<<resident(ctx, J, ctx->occ_post), SLOT_BLOCK, 0, st>>>(ctx->scene, fr, pb, depth, n_fold, J.work_ctr + WC_POST);
        timed_end(ctx, RAYN_K_SHADE_POST);
      } else {
#ifdef RAYN_LEGACY_KERNELS
        timed_begin(ctx, RAYN_K_SHADE_PRE);
        k_shade<<<dim3((QS + 127) / 128, nt), 128, 0, st>>>(ctx->scene, fr, pb, depth, thr);
        timed_end(ctx, RAYN_K_SHADE_PRE);
#endif
      }
      if (depth < mb) {
        timed_begin(ctx, RAYN_K_COMPACT);
        k_compact_count<<<dim3(nseg, nt), CMP_T, 0, st>>>(pb, nseg);
        k_compact_scatter<<<dim3(nseg, nt), CMP_T, 0, st>>>(pb, nseg);
        timed_end(ctx, RAYN_K_COMPACT, 2);
      }
    }
    timed_begin(ctx, RAYN_K_RESOLVE);
    if (mom)
      k_resolve<true><<<dim3((f->tile_w * f->tile_h + wpc - 1) / wpc, nt), wpc * 32, res_smem, st>>>(fr, pb, dp.color, dp.alpha, dp.background, dp.normal, np, wpc,
                                                                                                     slot_bits, depth_bits, dm_color, dm_bg);
    else
      k_resolve<false><<<dim3((f->tile_w * f->tile_h + wpc - 1) / wpc, nt), wpc * 32, res_smem, st>>>(fr, pb, dp.color, dp.alpha, dp.background, dp.normal, np, wpc,
                                                                                                      slot_bits, depth_bits);
    timed_end(ctx, RAYN_K_RESOLVE);
    if (capturing) {
      cudaGraph_t graph = nullptr;
      CU(cudaStreamEndCapture(st, &graph));
      capturing = false;
      if (ctx->graph_exec) cudaGraphExecDestroy(ctx->graph_exec);
      ctx->graph_exec = nullptr;
      const cudaError_t ge = cudaGraphInstantiate(&ctx->graph_exec, graph, 0);
      cudaGraphDestroy(graph);
      CU(ge);
      ctx->graph_key = key;
      ctx->graph_stats = ctx->stats;
      ctx->graph_stats.reserved_ = 1;  // marks "replayed from a captured graph" for callers that look
      CU(cudaGraphLaunch(ctx->graph_exec, st));
      ctx->stats.reserved_ = 1;  // this frame, too, ran as one graph launch
    }
    CU(cudaGetLastError());
  }
  ctx->pending = true;
  return RAYN_OK;
}

// Copies the non-NULL planes of `user` between user memory and a device block of 10 floats per pixel (film_block_planes),
// on the context's stream: kind cudaMemcpyHostToDevice fills the block, cudaMemcpyDeviceToHost reads it.
static int32_t copy_planes(RaynContext* ctx, const RaynFilmPlanes& user, float* block, size_t npx, cudaMemcpyKind kind) {
  const RaynFilmPlanes dev = film_block_planes(block, npx);
  float* const u[4] = {user.color, user.alpha, user.background, user.normal};
  float* const d[4] = {dev.color, dev.alpha, dev.background, dev.normal};
  const bool h2d = kind == cudaMemcpyHostToDevice;
  for (int i = 0; i < 4; ++i) {
    if (!u[i]) continue;
    const size_t bytes = npx * (i == 1 ? 1 : 3) * sizeof(float);  // alpha has one channel
    CU(cudaMemcpyAsync(h2d ? d[i] : u[i], h2d ? u[i] : d[i], bytes, kind, ctx->stream));
  }
  return RAYN_OK;
}

// The D2H copies of the job's host-space outputs that the caller asked for, from their staging (job_stage).
static int32_t copy_out(RaynContext* ctx) {
  const size_t npx = (size_t)ctx->job_w * ctx->job_h;
  const float* stage = ctx->d_planes;
  for (const JobPlane& p : ctx->job_out) {
    if (p.user) CU(cudaMemcpyAsync(p.user, stage, npx * p.floats * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    stage += npx * p.floats;
  }
  return RAYN_OK;
}

// The tail of a pending job: copy_out unless rc is already an error, then render_finish even if that failed; the first error.
static int32_t job_end(RaynContext* ctx, int32_t rc = RAYN_OK) {
  if (!rc) rc = copy_out(ctx);
  const int32_t rc2 = render_finish(ctx);
  return rc ? rc : rc2;
}

static int32_t render_finish(RaynContext* ctx) {
  if (!ctx->pending) return RAYN_OK;
  ctx->pending = false;
  cudaStream_t st = ctx->stream;
  CU(cudaSetDevice(ctx->device));
  CU(cudaEventRecord(ctx->ev1, st));
  CU(cudaMemcpyAsync(ctx->h_counters, ctx->d_counters, sizeof ctx->h_counters, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  CU(cudaEventElapsedTime(&ctx->stats.total_ms, ctx->ev0, ctx->ev1));
  const unsigned long long* h = ctx->h_counters;
  ctx->stats.extend_rays = (int64_t)h[CNT_EXTEND_RAYS];
  ctx->stats.shade_lanes = (int64_t)h[CNT_SHADE_LANES];
  ctx->stats.shadow_rays = (int64_t)h[CNT_SHADOW_RAYS];
  ctx->stats.sdf_evals_extend = (int64_t)h[CNT_EVALS_EXTEND];
  ctx->stats.sdf_evals_shadow = (int64_t)h[CNT_EVALS_SHADOW];
  ctx->stats.sdf_evals_normals = (int64_t)h[CNT_EVALS_NORMALS];
  ctx->stats.bulb_iters_extend = (int64_t)h[CNT_BULB_ITERS_EXTEND];
  ctx->stats.bulb_iters_shadow = (int64_t)h[CNT_BULB_ITERS_SHADOW];
  ctx->stats.march_trips_extend = (int64_t)h[CNT_TRIPS_EXTEND];
  ctx->stats.march_trips_shadow = (int64_t)h[CNT_TRIPS_SHADOW];
  {
    int64_t paths = 0;
    for (int idx : ctx->job_tiles) {
      const int tx = idx / ctx->job_nty, ty = idx % ctx->job_nty;
      const int tw = std::min(tx * ctx->job_tw + ctx->job_tw, ctx->job_w) - tx * ctx->job_tw;
      const int th = std::min(ty * ctx->job_th + ctx->job_th, ctx->job_h) - ty * ctx->job_th;
      paths += (int64_t)tw * th * ctx->job_spp;
    }
    ctx->stats.paths = paths;
  }
  for (size_t i = 0; i < ctx->timed_used; ++i) {
    float ms = 0.0f;
    cudaEventElapsedTime(&ms, ctx->timed[i].a, ctx->timed[i].b);
    ctx->stats.kernel_ms[ctx->timed[i].kernel] += ms;
  }
  return RAYN_OK;
}

static int32_t check_planes(RaynContext* ctx, const RaynFilmPlanes* out, bool need_all) {
  if (!out) return fail(ctx, RAYN_ERR_INVALID_ARG, "out is NULL");
  if (!out->color && !out->alpha && !out->background && !out->normal) return fail(ctx, RAYN_ERR_INVALID_ARG, "every film plane is NULL");
  if (need_all && (!out->color || !out->alpha || !out->background || !out->normal))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "a gathered device-space film needs all four planes");
  return RAYN_OK;
}

// ---- NCCL plumbing ---------------------------------------------------------------------------------------
static int32_t nccl_load(RaynContext* ctx) {
  if (g_nccl.handle) return RAYN_OK;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);  // the copy already mapped by the host process (e.g. torch's) wins by soname
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return fail(ctx, RAYN_ERR_NCCL, "cannot load libnccl.so.2: %s", dlerror());
  NcclApi a;
  a.handle = h;
#define SYM(field, name)                                                                     \
  *(void**)(&a.field) = dlsym(h, name);                                                      \
  if (!a.field) return fail(ctx, RAYN_ERR_NCCL, "libnccl.so.2 lacks %s", name);
  SYM(GetUniqueId, "ncclGetUniqueId")
  SYM(CommInitRank, "ncclCommInitRank")
  SYM(CommInitAll, "ncclCommInitAll")
  SYM(CommDestroy, "ncclCommDestroy")
  SYM(AllGather, "ncclAllGather")
  SYM(GroupStart, "ncclGroupStart")
  SYM(GroupEnd, "ncclGroupEnd")
  SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
  g_nccl = a;
  return RAYN_OK;
}

// shard tables + slab storage for a film geometry (uploaded once per geometry, not per frame)
static int32_t comm_prepare(RaynContext* ctx, int W, int H, int tw, int th) {
  RaynComm& c = ctx->comm;
  if (c.W == W && c.H == H && c.tw == tw && c.th == th && c.d_table) return RAYN_OK;
  CU(cudaSetDevice(ctx->device));
  c.shards.clear();
  size_t per = 0;
  for (int r = 0; r < c.world; ++r) {
    c.shards.push_back(shard_of(W, H, tw, th, r, c.world));
    per = std::max(per, c.shards.back().size());
  }
  per = std::max<size_t>(per, 1);
  std::vector<int> table((size_t)c.world * per, -1);
  for (int r = 0; r < c.world; ++r) std::copy(c.shards[r].begin(), c.shards[r].end(), table.begin() + (size_t)r * per);
  CU(cudaStreamSynchronize(ctx->stream));
  cudaFree(c.d_table);
  c.d_table = nullptr;
  CU(cudaMalloc(&c.d_table, table.size() * sizeof(int)));
  CU(cudaMemcpy(c.d_table, table.data(), table.size() * sizeof(int), cudaMemcpyHostToDevice));
  CU(regrow(&c.d_slabs, &c.cap_slabs, (size_t)c.world * per * 10 * tw * th));
  c.W = W, c.H = H, c.tw = tw, c.th = th, c.per_rank = (int)per;
  return RAYN_OK;
}

// pack this rank's tiles into its slab, all-gather in place, ONE unpack kernel over the peers' slabs: all on the render
// stream, zero host synchronisation.  in_group: the caller brackets several contexts with ncclGroupStart/End.
static int32_t gather_pack(RaynContext* ctx, const RaynFilmPlanes* pl) {
  RaynComm& c = ctx->comm;
  int ntx, nty;
  tile_grid_of(c.W, c.H, c.tw, c.th, &ntx, &nty);
  k_film_slab<<<c.per_rank, 256, 0, ctx->stream>>>(c.W, c.H, c.tw, c.th, nty, c.d_table, c.per_rank, c.rank, -1, 0, c.d_slabs, pl->color, pl->alpha,
                                                   pl->background, pl->normal);
  ctx->stats.launches++;
  return RAYN_OK;
}
static int32_t gather_collective(RaynContext* ctx) {
  RaynComm& c = ctx->comm;
  const size_t count = (size_t)c.per_rank * 10 * c.tw * c.th;
  NC(g_nccl.AllGather(c.d_slabs + (size_t)c.rank * count, c.d_slabs, count, kNcclFloat, c.comm, ctx->stream));
  return RAYN_OK;
}
static int32_t gather_unpack(RaynContext* ctx, const RaynFilmPlanes* pl) {
  RaynComm& c = ctx->comm;
  int ntx, nty;
  tile_grid_of(c.W, c.H, c.tw, c.th, &ntx, &nty);
  k_film_slab<<<c.world * c.per_rank, 256, 0, ctx->stream>>>(c.W, c.H, c.tw, c.th, nty, c.d_table, c.per_rank, 0, c.rank, 1, c.d_slabs, pl->color,
                                                             pl->alpha, pl->background, pl->normal);
  ctx->stats.launches++;
  CU(cudaGetLastError());
  return RAYN_OK;
}
static int32_t gather_enqueue(RaynContext* ctx, int W, int H, int tw, int th, const RaynFilmPlanes* pl, bool in_group) {
  (void)in_group;
  if (!ctx->comm.comm) return fail(ctx, RAYN_ERR_INVALID_ARG, "no communicator: call rayn_b200_comm_init_rank / comm_init_all first");
  int32_t rc = comm_prepare(ctx, W, H, tw, th);
  if (rc) return rc;
  CU(cudaSetDevice(ctx->device));
  timed_begin(ctx, RAYN_K_GATHER);
  if ((rc = gather_pack(ctx, pl))) return rc;
  if ((rc = gather_collective(ctx))) return rc;
  if ((rc = gather_unpack(ctx, pl))) return rc;
  timed_end(ctx, RAYN_K_GATHER, 0);
  return RAYN_OK;
}

extern "C" {

int32_t rayn_b200_render_frame(RaynContext* ctx, const RaynFrameDesc* f, const RaynFilmPlanes* out) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  int32_t rc = check_planes(ctx, out, false);
  if (rc) return rc;
  if ((rc = render_enqueue(ctx, f, out, nullptr, nullptr))) return rc;
  return job_end(ctx);
}

// render_frame plus the lum^2 moment planes (statement in include/rayn_b200.h): the same job, with the k_resolve<true> instance
int32_t rayn_b200_render_frame_moments(RaynContext* ctx, const RaynFrameDesc* f, const RaynFilmPlanes* out, const RaynMomentPlanes* moments) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!out || !moments) return fail(ctx, RAYN_ERR_INVALID_ARG, "render_frame_moments: out/moments is NULL");
  if (!out->color && !out->alpha && !out->background && !out->normal && !moments->color_lum2 && !moments->background_lum2)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "render_frame_moments: every film and moment plane is NULL");
  if ((out->space != RAYN_MEM_HOST && out->space != RAYN_MEM_DEVICE) || moments->space != out->space)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "render_frame_moments: the moment planes must be in the film planes' memory space");
  if (ctx->flags & RAYN_FLAG_SIMPLE_MARCH) return fail(ctx, RAYN_ERR_UNSUPPORTED, "render_frame_moments: RAYN_FLAG_SIMPLE_MARCH (legacy test kernels)");
  int32_t rc = render_enqueue(ctx, f, out, nullptr, nullptr, moments);
  if (rc) return rc;
  return job_end(ctx);
}

// The first-hit passes (statements in include/rayn_b200.h): the albedo plane (motion == NULL), or the motion plane and
// optionally the albedo plane, against the uploaded scene run backwards (prev == NULL) or against prev.  Each pass runs the
// render's raygen and depth-0 closest-hit stage, then one k_first_hit_paths instance and the resolves (rt_first_hit.cuh),
// pass by pass over the whole tile grid.  Never captured into a graph.  The callers have made job_ready and their own
// pointer checks.
static int32_t first_hit_job(RaynContext* ctx, const char* name, const RaynFrameDesc* f, float frame_dt, const RaynSceneDesc* prev,
                             float* motion, float* albedo, int32_t space) {
  if (space != RAYN_MEM_HOST && space != RAYN_MEM_DEVICE) return fail(ctx, RAYN_ERR_INVALID_ARG, "%s: bad memory space %d", name, space);
  if (!isfinite(frame_dt)) return fail(ctx, RAYN_ERR_INVALID_ARG, "%s: frame_dt %g is not finite", name, frame_dt);
  if (ctx->flags & RAYN_FLAG_SIMPLE_MARCH) return fail(ctx, RAYN_ERR_UNSUPPORTED, "%s: RAYN_FLAG_SIMPLE_MARCH (legacy test kernels)", name);
  DevPrev dp;
  if (prev) {
    const DevScene& sc = ctx->scene;
    if (prev->n_hitables != sc.n_hit)
      return fail(ctx, RAYN_ERR_INVALID_ARG, "%s: prev has %d hitables, the uploaded scene %d", name, prev->n_hitables, sc.n_hit);
    if (!prev->hitables) return fail(ctx, RAYN_ERR_INVALID_ARG, "%s: prev->hitables is NULL", name);
    if (prev->camera.kind != sc.cam.kind)
      return fail(ctx, RAYN_ERR_INVALID_ARG, "%s: prev camera kind %d differs from the uploaded %d (a cut is a reset, not motion)", name,
                  prev->camera.kind, sc.cam.kind);
    memset(&dp, 0, sizeof dp);
    dp.cam = prev->camera;
    for (int j = 0; j < sc.n_hit; ++j) {
      const RaynHitable &p = prev->hitables[j], &h = sc.hit[j];
      if (p.kind != h.kind) return fail(ctx, RAYN_ERR_INVALID_ARG, "%s: prev hitable %d has kind %d, the uploaded one %d", name, j, p.kind, h.kind);
      memcpy(dp.center[j], p.center, sizeof dp.center[j]);
      memcpy(dp.velocity[j], p.center_velocity, sizeof dp.velocity[j]);
      const bool zero_v = !(p.center_velocity[0] != 0.0f || p.center_velocity[1] != 0.0f || p.center_velocity[2] != 0.0f) &&
                          !(h.center_velocity[0] != 0.0f || h.center_velocity[1] != 0.0f || h.center_velocity[2] != 0.0f);
      if (h.kind == RAYN_HITABLE_SPHERE && zero_v && memcmp(p.center, h.center, sizeof h.center) == 0) dp.still |= 1u << j;
    }
  }
  Job J;  // the render's own pass sizing: alternating renders and first-hit passes reuse the same pass buffers
  int32_t rc = job_begin(ctx, f, nullptr, false, space, &J);
  if (rc) return rc;
  const DevFrame& fr = J.P.fr;
  const PassBufs& pb = J.pb;
  cudaStream_t st = ctx->stream;
  const size_t npx = (size_t)f->width * f->height;
  float* dev[2] = {motion, albedo};  // the device-space planes: motion, then albedo, also in the host-space staging
  if (space == RAYN_MEM_HOST) {
    const JobPlane planes[2] = {{motion, 4}, {albedo, 3}};
    if ((rc = job_stage(ctx, planes, 2, false, dev))) return rc;
  }
  float *dm = motion ? dev[0] : nullptr, *da = albedo ? dev[1] : nullptr;
  if (prev) {  // pageable source: the copy has left dp when cudaMemcpyAsync returns
    if (!ctx->d_prev) CU(cudaMalloc(&ctx->d_prev, sizeof(DevPrev)));
    CU(cudaMemcpyAsync(ctx->d_prev, &dp, sizeof dp, cudaMemcpyHostToDevice, st));
  }
  if (dm) k_motion_clear<<<(unsigned)((npx + 255) / 256), 256, 0, st>>>((long long)npx, dm);  // pixels outside the tile grid
  if (da) CU(cudaMemsetAsync(da, 0, npx * 3 * sizeof(float), st));                          // ... which stay 0
  typedef void (*PathsKernel)(DevScene, DevFrame, PassBufs, float, const DevPrev*);
  static const PathsKernel motion_paths[2][2] = {  // [prev][albedo]
      {k_first_hit_paths<true, false, false>, k_first_hit_paths<true, true, false>},
      {k_first_hit_paths<true, false, true>, k_first_hit_paths<true, true, true>}};
  const PathsKernel paths = dm ? motion_paths[prev != nullptr][da != nullptr] : k_first_hit_paths<false, true, false>;
  const Thr thr = make_thr(ctx->scene.cam, 0);
  for (size_t first = 0; first < ctx->job_tiles.size(); first += J.tiles_per_pass) {
    if ((rc = pass_tiles(ctx, &J, first, 0))) return rc;
    pass_raygen(ctx, J);
    if ((rc = extend_enqueue(ctx, J, thr))) return rc;
    const dim3 gp((J.P.R + 255) / 256, pb.n_tiles), gr((f->tile_w * f->tile_h + 255) / 256, pb.n_tiles);
    timed_begin(ctx, RAYN_K_NORMALS);
    paths<<<gp, 256, 0, st>>>(ctx->scene, fr, pb, frame_dt, prev ? ctx->d_prev : nullptr);
    timed_end(ctx, RAYN_K_NORMALS);
    timed_begin(ctx, RAYN_K_RESOLVE);
    if (dm) k_motion_resolve<<<gr, 256, 0, st>>>(fr, pb, pb.rad, dm);
    if (da) k_albedo_resolve<<<gr, 256, 0, st>>>(fr, pb, pb.nrm, da);
    timed_end(ctx, RAYN_K_RESOLVE, (dm ? 1 : 0) + (da ? 1 : 0));
    CU(cudaGetLastError());
  }
  ctx->pending = true;
  return job_end(ctx);
}

int32_t rayn_b200_render_albedo(RaynContext* ctx, const RaynFrameDesc* f, float* albedo, int32_t space) {
  int32_t rc = job_ready(ctx, "render_albedo");
  if (rc) return rc;
  if (!f || !albedo) return fail(ctx, RAYN_ERR_INVALID_ARG, "frame/albedo is NULL");
  return first_hit_job(ctx, "render_albedo", f, 0.0f, nullptr, nullptr, albedo, space);
}

int32_t rayn_b200_render_motion(RaynContext* ctx, const RaynFrameDesc* f, float frame_dt, float* motion, float* albedo, int32_t space) {
  int32_t rc = job_ready(ctx, "render_motion");
  if (rc) return rc;
  if (!f || !motion) return fail(ctx, RAYN_ERR_INVALID_ARG, "frame/motion is NULL");
  return first_hit_job(ctx, "render_motion", f, frame_dt, nullptr, motion, albedo, space);
}

int32_t rayn_b200_render_motion_prev(RaynContext* ctx, const RaynFrameDesc* f, float frame_dt, const RaynSceneDesc* prev, float* motion,
                                     float* albedo, int32_t space) {
  int32_t rc = job_ready(ctx, "render_motion_prev");
  if (rc) return rc;
  if (!f || !motion) return fail(ctx, RAYN_ERR_INVALID_ARG, "frame/motion is NULL");
  if (!prev) return fail(ctx, RAYN_ERR_INVALID_ARG, "render_motion_prev: prev is NULL");
  return first_hit_job(ctx, "render_motion_prev", f, frame_dt, prev, motion, albedo, space);
}

int32_t rayn_b200_sync(RaynContext* ctx) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->stream));
  return RAYN_OK;
}

// ---- communicator ------------------------------------------------------------------------------------------
int32_t rayn_b200_comm_unique_id(uint8_t* out_id) {
  RaynContext* ctx = nullptr;
  if (!out_id) return fail(nullptr, RAYN_ERR_INVALID_ARG, "out_id is NULL");
  int32_t rc = nccl_load(nullptr);
  if (rc) return rc;
  ncclUniqueId id;
  NC(g_nccl.GetUniqueId(&id));
  memcpy(out_id, id.internal, RAYN_COMM_ID_BYTES);
  return RAYN_OK;
}
int32_t rayn_b200_comm_init_rank(RaynContext* ctx, const uint8_t* id_bytes, int32_t rank, int32_t world) {
  if (!ctx || !id_bytes) return fail(ctx, RAYN_ERR_INVALID_ARG, "comm_init_rank: NULL argument");
  if (world < 1 || rank < 0 || rank >= world) return fail(ctx, RAYN_ERR_INVALID_ARG, "comm_init_rank: rank %d of %d", rank, world);
  int32_t rc = nccl_load(ctx);
  if (rc) return rc;
  rayn_b200_comm_destroy(ctx);
  CU(cudaSetDevice(ctx->device));
  ncclUniqueId id;
  memcpy(id.internal, id_bytes, RAYN_COMM_ID_BYTES);
  NC(g_nccl.CommInitRank(&ctx->comm.comm, world, id, rank));
  ctx->comm.rank = rank, ctx->comm.world = world;
  return RAYN_OK;
}
int32_t rayn_b200_comm_init_all(RaynContext* const* ctxs, int32_t n) {
  RaynContext* ctx = (ctxs && n > 0) ? ctxs[0] : nullptr;
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "comm_init_all: no contexts");
  int32_t rc = nccl_load(ctx);
  if (rc) return rc;
  std::vector<int> devs(n);
  std::vector<ncclComm_t> comms(n, nullptr);
  for (int i = 0; i < n; ++i) {
    if (!ctxs[i]) return fail(ctx, RAYN_ERR_INVALID_ARG, "comm_init_all: ctxs[%d] is NULL", i);
    for (int j = 0; j < i; ++j)
      if (ctxs[j]->device == ctxs[i]->device) return fail(ctx, RAYN_ERR_INVALID_ARG, "comm_init_all: device %d used twice", ctxs[i]->device);
    rayn_b200_comm_destroy(ctxs[i]);
    devs[i] = ctxs[i]->device;
  }
  NC(g_nccl.CommInitAll(comms.data(), n, devs.data()));
  for (int i = 0; i < n; ++i) ctxs[i]->comm.comm = comms[i], ctxs[i]->comm.rank = i, ctxs[i]->comm.world = n;
  return RAYN_OK;
}
int32_t rayn_b200_comm_info(const RaynContext* ctx, int32_t* rank, int32_t* world) {
  if (!ctx) return RAYN_ERR_INVALID_ARG;
  if (rank) *rank = ctx->comm.rank;
  if (world) *world = ctx->comm.comm ? ctx->comm.world : 0;
  return RAYN_OK;
}
int32_t rayn_b200_shard_tiles(int32_t W, int32_t H, int32_t tw, int32_t th, int32_t rank, int32_t world, int32_t* out, int32_t cap) {
  if (W <= 0 || H <= 0 || tw <= 0 || th <= 0 || world < 1 || rank < 0 || rank >= world) return -1;
  const std::vector<int> v = shard_of(W, H, tw, th, rank, world);
  if (out && cap >= (int32_t)v.size()) std::copy(v.begin(), v.end(), out);
  return (int32_t)v.size();
}

int32_t rayn_b200_film_gather(RaynContext* ctx, int32_t W, int32_t H, int32_t tw, int32_t th, const RaynFilmPlanes* pl) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (W <= 0 || H <= 0 || tw <= 0 || th <= 0) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_gather: bad geometry");
  int32_t rc = check_planes(ctx, pl, true);
  if (rc) return rc;
  if (pl->space != RAYN_MEM_DEVICE) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_gather: planes must be device pointers");
  return gather_enqueue(ctx, W, H, tw, th, pl, false);
}

int32_t rayn_b200_render_frame_sharded(RaynContext* ctx, const RaynFrameDesc* f, const RaynFilmPlanes* out) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!ctx->comm.comm) return fail(ctx, RAYN_ERR_INVALID_ARG, "render_frame_sharded: no communicator on this context");
  if (!f) return fail(ctx, RAYN_ERR_INVALID_ARG, "frame is NULL");
  int32_t rc = check_planes(ctx, out, out && out->space == RAYN_MEM_DEVICE);
  if (rc) return rc;
  const std::vector<int> tiles = shard_of(f->width, f->height, f->tile_w, f->tile_h, ctx->comm.rank, ctx->comm.world);
  RaynFilmPlanes dev;
  if ((rc = render_enqueue(ctx, f, out, &tiles, &dev))) return rc;
  return job_end(ctx, gather_enqueue(ctx, f->width, f->height, f->tile_w, f->tile_h, &dev, false));
}

int32_t rayn_b200_render_frame_multi(RaynContext* const* ctxs, int32_t n, const RaynFrameDesc* f, const RaynFilmPlanes* out) {
  RaynContext* ctx = (ctxs && n > 0) ? ctxs[0] : nullptr;
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "render_frame_multi: no contexts");
  if (!f || !out) return fail(ctx, RAYN_ERR_INVALID_ARG, "frame/out is NULL");
  if (f->input_space != RAYN_MEM_HOST || out->space != RAYN_MEM_HOST)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "render_frame_multi: frame inputs and film planes must be host pointers");
  int32_t rc = check_planes(ctx, out, false);
  if (rc) return rc;
  for (int i = 0; i < n; ++i)
    if (!ctxs[i] || !ctxs[i]->comm.comm || ctxs[i]->comm.world != n || ctxs[i]->comm.rank != i)
      return fail(ctx, RAYN_ERR_INVALID_ARG, "render_frame_multi: contexts must come from comm_init_all(ctxs, %d) in the same order", n);
  std::vector<RaynFilmPlanes> dev(n);
  RaynFilmPlanes scratch = *out;  // host-space marker: every context renders into its own device planes
  int32_t first_err = RAYN_OK;
  for (int i = 0; i < n && !first_err; ++i) {
    const std::vector<int> tiles = shard_of(f->width, f->height, f->tile_w, f->tile_h, i, n);
    first_err = render_enqueue(ctxs[i], f, &scratch, &tiles, &dev[i]);
    if (first_err && ctxs[i] != ctx) fail(ctx, first_err, "GPU %d: %s", ctxs[i]->device, ctxs[i]->err.c_str());
  }
  if (!first_err) {
    for (int i = 0; i < n && !first_err; ++i) {
      first_err = comm_prepare(ctxs[i], f->width, f->height, f->tile_w, f->tile_h);
      if (!first_err) {
        cudaSetDevice(ctxs[i]->device);
        first_err = gather_pack(ctxs[i], &dev[i]);
      }
    }
    if (!first_err) {
      g_nccl.GroupStart();
      for (int i = 0; i < n && !first_err; ++i) {
        cudaSetDevice(ctxs[i]->device);
        first_err = gather_collective(ctxs[i]);
      }
      const int gr = g_nccl.GroupEnd();
      if (!first_err && gr) first_err = fail(ctx, RAYN_ERR_NCCL, "ncclGroupEnd: %s", g_nccl.GetErrorString(gr));
    }
    for (int i = 0; i < n && !first_err; ++i) {
      cudaSetDevice(ctxs[i]->device);
      first_err = gather_unpack(ctxs[i], &dev[i]);
    }
  }
  for (int i = 0; i < n; ++i) {  // the caller's planes are copied from the first context's staging
    const int32_t rc2 = i == 0 ? job_end(ctx, first_err) : render_finish(ctxs[i]);
    if (!first_err && rc2) first_err = rc2;
  }
  return first_err;
}

// ---- explicit slab helpers --------------------------------------------------------------------------------------
int64_t rayn_b200_film_slab_floats(int32_t tw, int32_t th, int32_t n_tiles) {
  if (tw <= 0 || th <= 0 || n_tiles < 0) return -1;
  return (int64_t)n_tiles * 10 * tw * th;
}
static int32_t pack_unpack(RaynContext* ctx, int W, int H, int tw, int th, const int32_t* tile_list, int n, const RaynFilmPlanes* pl,
                           float* slab, int unpack) {
  if (!ctx || !pl || !slab || n < 0 || (n && !tile_list) || W <= 0 || H <= 0 || tw <= 0 || th <= 0)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "film pack/unpack: bad argument");
  if (n == 0) return RAYN_OK;
  CU(cudaSetDevice(ctx->device));
  int ntx, nty;
  tile_grid_of(W, H, tw, th, &ntx, &nty);
  for (int i = 0; i < n; ++i)
    if (tile_list[i] < 0 || tile_list[i] >= ntx * nty) return fail(ctx, RAYN_ERR_INVALID_ARG, "film pack/unpack: tile %d out of range", tile_list[i]);
  CU(regrow(&ctx->d_pack_ids, &ctx->cap_pack_ids, (size_t)n));
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpyAsync(ctx->d_pack_ids, tile_list, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  k_film_slab<<<n, 256, 0, ctx->stream>>>(W, H, tw, th, nty, ctx->d_pack_ids, n, 0, -1, unpack, slab, pl->color, pl->alpha, pl->background, pl->normal);
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(ctx->stream));
  return RAYN_OK;
}
int32_t rayn_b200_film_pack_tiles(RaynContext* ctx, int32_t W, int32_t H, int32_t tw, int32_t th, const int32_t* tile_list, int32_t n_tiles,
                                  const RaynFilmPlanes* planes_dev, float* slab_dev) {
  return pack_unpack(ctx, W, H, tw, th, tile_list, n_tiles, planes_dev, slab_dev, 0);
}
int32_t rayn_b200_film_unpack_tiles(RaynContext* ctx, int32_t W, int32_t H, int32_t tw, int32_t th, const int32_t* tile_list, int32_t n_tiles,
                                    const float* slab_dev, const RaynFilmPlanes* planes_dev) {
  return pack_unpack(ctx, W, H, tw, th, tile_list, n_tiles, planes_dev, const_cast<float*>(slab_dev), 1);
}

// ---- film post-process (film.rs:205-377 arithmetic) -------------------------------------------------
int32_t rayn_b200_film_postprocess(RaynContext* ctx, int32_t mode, int32_t W, int32_t H, const RaynFilmPlanes* pl, uint8_t* out,
                                   int32_t out_space) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (mode < 0 || mode > RAYN_POST_ALPHA || W <= 0 || H <= 0 || !pl || !out) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_postprocess: bad argument");
  const bool need_color = mode <= RAYN_POST_COLOR_ONLY, need_bg = mode == RAYN_POST_COLOR_PLUS_BACKGROUND || mode == RAYN_POST_BACKGROUND;
  const bool need_alpha = mode == RAYN_POST_COLOR_ALPHA || mode == RAYN_POST_ALPHA, need_normal = mode == RAYN_POST_WORLD_NORMAL;
  if ((need_color && !pl->color) || (need_bg && !pl->background) || (need_alpha && !pl->alpha) || (need_normal && !pl->normal))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "Attempted to write a channel with insufficient channels");  // film.rs:294-298
  CU(cudaSetDevice(ctx->device));
  const size_t npx = (size_t)W * H, nbytes = npx * post_bytes_per_pixel(mode);
  cudaStream_t st = ctx->stream;
  RaynFilmPlanes src = *pl;
  CU(cudaDeviceSynchronize());
  if (pl->space == RAYN_MEM_HOST) {  // copies the planes the mode reads
    CU(regrow(&ctx->d_planes, &ctx->cap_planes, npx * 10));
    const RaynFilmPlanes used{need_color ? pl->color : nullptr, need_alpha ? pl->alpha : nullptr, need_bg ? pl->background : nullptr,
                              need_normal ? pl->normal : nullptr, RAYN_MEM_HOST};
    int32_t rc = copy_planes(ctx, used, ctx->d_planes, npx, cudaMemcpyHostToDevice);
    if (rc) return rc;
    src = film_block_planes(ctx->d_planes, npx);
  }
  unsigned char* dout = out;
  if (out_space == RAYN_MEM_HOST) {
    CU(regrow(&ctx->d_post, &ctx->cap_post, nbytes));
    dout = ctx->d_post;
  }
  k_postprocess<<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(mode, W, H, src.color, src.alpha, src.background, src.normal, dout);
  CU(cudaGetLastError());
  if (out_space == RAYN_MEM_HOST) CU(cudaMemcpyAsync(out, dout, nbytes, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return RAYN_OK;
}

// ---- film denoise (rt_denoise.cuh; statement in include/rayn_b200.h) ----------------------------------------------
// 1 / sigma^2 in float; +inf -> 0 (term disabled).  False for a sigma that is not > 0 or so small the factor overflows.
static bool denoise_factor(float sigma, float* f) {
  if (!(sigma > 0.0f)) return false;
  *f = 1.0f / (sigma * sigma);
  return isfinite(*f);
}

// Enqueues the whole filter on ctx->stream.  `scratch` holds guide + ping-pong planes (12 floats per pixel), then the
// device copies of host-space inputs (10) and one host-space output channel (3), as the caller sized it.
// albedo != NULL (rayn_b200_film_denoise_albedo with a finite sigma): the albedo plane in in->space and its factor il; the
// scratch then holds 4 more floats per pixel (its float4 guide) after the ping-pong planes, and 3 more for a host-space plane.
// mom != NULL (rayn_b200_film_denoise_variance with a finite sigma_luminance sl): the moment planes in in->space, 2 more
// floats per pixel of staging when that is host memory; the variance travels in the .w lane of the ping-pong planes.
// scale != NULL (rayn_b200_film_denoise_variance_scaled, with mom): the per-pixel variance scale in in->space, 1 more float per
// pixel of staging when that is host memory.
static int32_t denoise_enqueue(RaynContext* ctx, const RaynDenoiseDesc* d, int W, int H, const RaynFilmPlanes* in, const RaynFilmPlanes* out,
                               float ic0, float in_, float ia, float* scratch, const float* albedo, float il, const RaynMomentPlanes* mom, float sl,
                               int spp, const float* scale) {
  cudaStream_t st = ctx->stream;
  const size_t npx = (size_t)W * H;
  const unsigned blocks1d = (unsigned)((npx + 255) / 256);
  float4* guide = (float4*)scratch;
  float4* ping[2] = {guide + npx, guide + 2 * npx};
  float4* alb = albedo ? guide + 3 * npx : nullptr;
  float* stage = scratch + (albedo ? 16 : 12) * npx;
  const float *c_in = in->color, *b_in = in->background, *n_in = in->normal, *a_in = in->alpha;
  if (in->space == RAYN_MEM_HOST) {
    int32_t rc = copy_planes(ctx, *in, stage, npx, cudaMemcpyHostToDevice);
    if (rc) return rc;
    const RaynFilmPlanes s = film_block_planes(stage, npx);
    stage += 10 * npx;
    n_in = s.normal, a_in = s.alpha, c_in = in->color ? s.color : nullptr, b_in = in->background ? s.background : nullptr;
  }
  k_denoise_guides<<<blocks1d, 256, 0, st>>>((long long)npx, n_in, a_in, guide);
  if (albedo) {
    const float* l_in = albedo;
    if (in->space == RAYN_MEM_HOST) {
      CU(cudaMemcpyAsync(stage, albedo, npx * 12, cudaMemcpyHostToDevice, st));
      l_in = stage;
      stage += 3 * npx;
    }
    k_denoise_pack<<<blocks1d, 256, 0, st>>>((long long)npx, l_in, alb);
  }
  const float *m_c = mom ? mom->color_lum2 : nullptr, *m_b = mom ? mom->background_lum2 : nullptr;
  if (mom && in->space == RAYN_MEM_HOST) {
    if (c_in) CU(cudaMemcpyAsync(stage, m_c, npx * 4, cudaMemcpyHostToDevice, st));
    if (b_in) CU(cudaMemcpyAsync(stage + npx, m_b, npx * 4, cudaMemcpyHostToDevice, st));
    m_c = stage, m_b = stage + npx;
    stage += 2 * npx;
  }
  if (scale && in->space == RAYN_MEM_HOST) {
    CU(cudaMemcpyAsync(stage, scale, npx * 4, cudaMemcpyHostToDevice, st));
    scale = stage;
    stage += npx;
  }
  CU(cudaGetLastError());
  for (int ch = 0; ch < 2; ++ch) {
    const float* src3 = ch == 0 ? c_in : b_in;
    if (!src3) continue;
    float* dst_user = ch == 0 ? out->color : out->background;
    float* dst3 = out->space == RAYN_MEM_HOST ? stage : dst_user;
    if (mom && scale)
      k_denoise_pack_var<true><<<blocks1d, 256, 0, st>>>((long long)npx, src3, ch == 0 ? m_c : m_b, (float)spp, ping[0], scale);
    else if (mom)
      k_denoise_pack_var<<<blocks1d, 256, 0, st>>>((long long)npx, src3, ch == 0 ? m_c : m_b, (float)spp, ping[0]);
    else
      k_denoise_pack<<<blocks1d, 256, 0, st>>>((long long)npx, src3, ping[0]);
    for (int i = 0; i < d->iterations; ++i) {
      const float ic = ldexpf(ic0, i);
      const float4* src = ping[i & 1];
      float4* dst4 = ping[(i + 1) & 1];
      const bool last = i == d->iterations - 1;
      if (albedo && mom)
        denoise_level<true, true>(st, last, W, H, 1 << i, ic, in_, ia, guide, src, dst4, dst3, alb, il, sl);
      else if (albedo)
        denoise_level<true, false>(st, last, W, H, 1 << i, ic, in_, ia, guide, src, dst4, dst3, alb, il, 0.0f);
      else if (mom)
        denoise_level<false, true>(st, last, W, H, 1 << i, ic, in_, ia, guide, src, dst4, dst3, nullptr, 0.0f, sl);
      else
        denoise_level<false, false>(st, last, W, H, 1 << i, ic, in_, ia, guide, src, dst4, dst3, nullptr, 0.0f, 0.0f);
    }
    CU(cudaGetLastError());
    if (out->space == RAYN_MEM_HOST) CU(cudaMemcpyAsync(dst_user, dst3, npx * 12, cudaMemcpyDeviceToHost, st));
  }
  return RAYN_OK;
}

// rayn_b200_film_denoise and, with an albedo plane (albedo != NULL), rayn_b200_film_denoise_albedo; with moment planes
// (mom != NULL) and a finite sigma_luminance sl, rayn_b200_film_denoise_variance, and with a variance scale too (scale != NULL),
// rayn_b200_film_denoise_variance_scaled
static int32_t film_denoise(RaynContext* ctx, const RaynDenoiseDesc* d, int32_t W, int32_t H, const RaynFilmPlanes* in, const RaynFilmPlanes* out,
                            const float* albedo, float il, const RaynMomentPlanes* mom = nullptr, float sl = 0.0f, int spp = 0,
                            const float* scale = nullptr) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!d || !in || !out || W <= 0 || H <= 0) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise: bad argument");
  if (d->iterations < 1 || d->iterations > 8) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise: iterations %d not in [1,8]", d->iterations);
  if (!in->normal || !in->alpha) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise: the normal and alpha guide planes are required");
  if ((in->color && !out->color) || (in->background && !out->background))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise: every input colour plane needs its output plane");
  if ((in->space != RAYN_MEM_HOST && in->space != RAYN_MEM_DEVICE) || (out->space != RAYN_MEM_HOST && out->space != RAYN_MEM_DEVICE))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise: bad memory space");
  float ic0, in_, ia;
  if (!denoise_factor(d->sigma_color, &ic0) || !isfinite(ldexpf(ic0, d->iterations - 1)) || !denoise_factor(d->sigma_normal, &in_) ||
      !denoise_factor(d->sigma_alpha, &ia))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise: sigmas (%g, %g, %g) must be > 0 (+inf disables a term) and give finite 1/sigma^2",
                d->sigma_color, d->sigma_normal, d->sigma_alpha);
  CU(cudaSetDevice(ctx->device));
  if (!in->color && !in->background) return RAYN_OK;
  const size_t npx = (size_t)W * H;
  const size_t nfloat = npx * (12 + (in->space == RAYN_MEM_HOST ? 10 : 0) + (out->space == RAYN_MEM_HOST ? 3 : 0) +
                               (albedo ? 4 + (in->space == RAYN_MEM_HOST ? 3 : 0) : 0) + (mom && in->space == RAYN_MEM_HOST ? 2 : 0) +
                               (mom && scale && in->space == RAYN_MEM_HOST ? 1 : 0));
  cudaStream_t st = ctx->stream;
  float* scratch = nullptr;
  // stream-ordered and released below: nothing persists between calls (render-pass sizing reads cudaMemGetInfo)
  CU(cudaMallocAsync((void**)&scratch, nfloat * sizeof(float), st));
  const int32_t rc = denoise_enqueue(ctx, d, W, H, in, out, ic0, in_, ia, scratch, albedo, il, mom, sl, spp, mom ? scale : nullptr);
  const cudaError_t ef = cudaFreeAsync(scratch, st);
  if (rc) return rc;
  CU(ef);
  if (in->space == RAYN_MEM_HOST || out->space == RAYN_MEM_HOST) CU(cudaStreamSynchronize(st));
  return RAYN_OK;
}

int32_t rayn_b200_film_denoise(RaynContext* ctx, const RaynDenoiseDesc* d, int32_t W, int32_t H, const RaynFilmPlanes* in,
                               const RaynFilmPlanes* out) {
  return film_denoise(ctx, d, W, H, in, out, nullptr, 0.0f);
}

int32_t rayn_b200_film_denoise_albedo(RaynContext* ctx, const RaynDenoiseDesc* d, float sigma_albedo, const float* albedo, int32_t W, int32_t H,
                                      const RaynFilmPlanes* in, const RaynFilmPlanes* out) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!albedo) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise_albedo: the albedo plane is NULL");
  float il;
  if (!denoise_factor(sigma_albedo, &il))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise_albedo: sigma_albedo %g must be > 0 (+inf disables the term) and give a finite 1/sigma^2",
                sigma_albedo);
  // +inf: the term is not added at all (adding dl2 * 0 would turn a non-finite albedo tap into a NaN tap)
  return film_denoise(ctx, d, W, H, in, out, il == 0.0f ? nullptr : albedo, il);
}

// rayn_b200_film_denoise_variance (scale NULL) and rayn_b200_film_denoise_variance_scaled
static int32_t film_denoise_variance(RaynContext* ctx, const RaynDenoiseDesc* d, float sigma_luminance, int32_t spp, const RaynMomentPlanes* moments,
                                     const float* scale, float sigma_albedo, const float* albedo, int32_t W, int32_t H, const RaynFilmPlanes* in,
                                     const RaynFilmPlanes* out) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!moments || !in) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise_variance: moments/in is NULL");
  if ((in->color && !moments->color_lum2) || (in->background && !moments->background_lum2))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise_variance: every input colour plane needs its moment plane");
  if (moments->space != in->space) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise_variance: the moment planes must be in in->space");
  if (spp < 1) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise_variance: spp %d < 1", spp);
  if (!(sigma_luminance > 0.0f)) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise_variance: sigma_luminance %g must be > 0 (+inf disables the term)", sigma_luminance);
  float il = 0.0f;
  if (albedo && !denoise_factor(sigma_albedo, &il))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise_variance: sigma_albedo %g must be > 0 (+inf disables the term) and give a finite 1/sigma^2",
                sigma_albedo);
  // +inf: the term is not added (inf * sqrt(0) would be NaN), and the call is film_denoise / film_denoise_albedo
  const bool var = !isinf(sigma_luminance);
  return film_denoise(ctx, d, W, H, in, out, il == 0.0f ? nullptr : albedo, il, var ? moments : nullptr, sigma_luminance, spp, scale);
}

int32_t rayn_b200_film_denoise_variance(RaynContext* ctx, const RaynDenoiseDesc* d, float sigma_luminance, int32_t spp, const RaynMomentPlanes* moments,
                                        float sigma_albedo, const float* albedo, int32_t W, int32_t H, const RaynFilmPlanes* in,
                                        const RaynFilmPlanes* out) {
  return film_denoise_variance(ctx, d, sigma_luminance, spp, moments, nullptr, sigma_albedo, albedo, W, H, in, out);
}

int32_t rayn_b200_film_denoise_variance_scaled(RaynContext* ctx, const RaynDenoiseDesc* d, float sigma_luminance, int32_t spp,
                                               const RaynMomentPlanes* moments, const float* var_scale, float sigma_albedo, const float* albedo,
                                               int32_t W, int32_t H, const RaynFilmPlanes* in, const RaynFilmPlanes* out) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!var_scale) return fail(ctx, RAYN_ERR_INVALID_ARG, "film_denoise_variance_scaled: var_scale is NULL");
  return film_denoise_variance(ctx, d, sigma_luminance, spp, moments, var_scale, sigma_albedo, albedo, W, H, in, out);
}

int32_t rayn_b200_device_frame_inputs(RaynContext* ctx, int32_t W, int32_t H, int32_t spp, int32_t sets_1d, int32_t sets_2d, uint64_t offset,
                                      float* s1, float* s2, float* scramble) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (spp <= 0 || sets_1d < 0 || sets_2d < 0 || (sets_1d && !s1) || (sets_2d && !s2) || (scramble && (W <= 0 || H <= 0)))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "device_frame_inputs: bad argument");
  CU(cudaSetDevice(ctx->device));
  CU(cudaDeviceSynchronize());
  const long long n = (long long)spp * (sets_1d + sets_2d);
  if (n > 0) k_gen_rd_tables<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(spp, sets_1d, sets_2d, offset, 0ull, s1, s2);
  if (scramble) k_gen_scramble<<<(unsigned)(((long long)W * H + 255) / 256), 256, 0, ctx->stream>>>(W, H, scramble);
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(ctx->stream));
  return RAYN_OK;
}

int32_t rayn_b200_device_rd_tables_at(RaynContext* ctx, int32_t spp, int32_t sets_1d, int32_t sets_2d, uint64_t offset, uint64_t first,
                                      float* s1, float* s2) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (spp <= 0 || sets_1d < 0 || sets_2d < 0 || (sets_1d && !s1) || (sets_2d && !s2))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "device_rd_tables_at: bad argument");
  if (first > (1ull << 32) - (uint64_t)spp)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "device_rd_tables_at: first_sample + spp = %llu exceeds 2^32", (unsigned long long)first + spp);
  CU(cudaSetDevice(ctx->device));
  CU(cudaDeviceSynchronize());
  const long long n = (long long)spp * (sets_1d + sets_2d);
  if (n > 0) k_gen_rd_tables<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(spp, sets_1d, sets_2d, offset, first, s1, s2);
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(ctx->stream));
  return RAYN_OK;
}

// ---- film accumulator (rt_accum.cuh; statement in include/rayn_b200.h) ----------------------------------------------
struct RaynAccum {
  int device = 0, W = 0, H = 0, tw = 0, th = 0, ntx = 0, nty = 0, n_tiles = 0;
  int64_t rounds_run = 0;     // rounds that rendered at least one tile
  float* state = nullptr;     // S and H, 13 floats per pixel (rt_accum.cuh)
  float* planes = nullptr;    // the round's render (and resolve staging for host planes), 10 floats per pixel
  void* tile_mem = nullptr;   // AccumTiles arrays + the round's tile list
  AccumTiles dt{};
  int* d_list = nullptr;
  // host copies of the per-tile state, refreshed after every round
  std::vector<double> E;
  std::vector<long long> K, Kh;
  std::vector<int> rounds;
};

static void accum_free(RaynAccum* a) {
  cudaFree(a->state), cudaFree(a->planes), cudaFree(a->tile_mem);
  delete a;
}

int32_t rayn_b200_accum_create(RaynContext* ctx, int32_t W, int32_t H, int32_t tw, int32_t th, RaynAccum** out) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!out || W <= 0 || H <= 0 || tw <= 0 || th <= 0) return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_create: bad argument");
  *out = nullptr;
  CU(cudaSetDevice(ctx->device));
  RaynAccum* a = new RaynAccum();
  a->device = ctx->device, a->W = W, a->H = H, a->tw = tw, a->th = th;
  tile_grid_of(W, H, tw, th, &a->ntx, &a->nty);
  const int nt = a->n_tiles = a->ntx * a->nty;
  const size_t npx = (size_t)W * H;
  const size_t tile_bytes = (size_t)nt * (sizeof(double) + 2 * sizeof(long long) + 2 * sizeof(int));
  cudaError_t e = cudaMalloc((void**)&a->state, npx * 13 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc((void**)&a->planes, npx * 10 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&a->tile_mem, tile_bytes);
  a->E.assign(nt, INFINITY), a->K.assign(nt, 0), a->Kh.assign(nt, 0), a->rounds.assign(nt, 0);
  if (e == cudaSuccess) {
    char* p = (char*)a->tile_mem;
    a->dt.E = (double*)p, a->dt.K = (long long*)(p + nt * sizeof(double)), a->dt.Kh = a->dt.K + nt;
    a->dt.rounds = (int*)(a->dt.Kh + nt), a->d_list = a->dt.rounds + nt;
    e = cudaMemsetAsync(a->state, 0, npx * 13 * sizeof(float), ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(a->dt.K, 0, (size_t)nt * (2 * sizeof(long long) + sizeof(int)), ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(a->dt.E, a->E.data(), nt * sizeof(double), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  }
  if (e != cudaSuccess) {
    cudaGetLastError();
    accum_free(a);
    return fail(ctx, e == cudaErrorMemoryAllocation ? RAYN_ERR_OOM : RAYN_ERR_CUDA, "accum_create (%dx%d): %s", W, H, cudaGetErrorString(e));
  }
  *out = a;
  return RAYN_OK;
}

void rayn_b200_accum_destroy(RaynAccum* a) {
  if (!a) return;
  cudaSetDevice(a->device);
  cudaDeviceSynchronize();
  accum_free(a);
}

int32_t rayn_b200_accum_round(RaynContext* ctx, RaynAccum* a, const RaynFrameDesc* f, const RaynAdaptiveDesc* d, int32_t* out_tiles) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (out_tiles) *out_tiles = 0;
  if (!a || !f || !d) return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_round: NULL argument");
  if (a->device != ctx->device) return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_round: the accumulator lives on device %d, the context on %d", a->device, ctx->device);
  if (d->min_rounds < 2 || d->max_rounds < d->min_rounds || d->threshold != d->threshold)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_round: need 2 <= min_rounds (%d) <= max_rounds (%d) and a threshold that is not NaN", d->min_rounds,
                d->max_rounds);
  if (f->width != a->W || f->height != a->H || f->tile_w != a->tw || f->tile_h != a->th)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_round: frame %dx%d tiles %dx%d, accumulator %dx%d tiles %dx%d", f->width, f->height, f->tile_w,
                f->tile_h, a->W, a->H, a->tw, a->th);
  if (f->samples <= 0) return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_round: samples %d", f->samples);
  std::vector<int> active;
  for (int t = 0; t < a->n_tiles; ++t)
    if (a->rounds[t] < d->max_rounds && (a->rounds[t] < d->min_rounds || !(a->E[t] <= (double)d->threshold))) active.push_back(t);
  if (active.empty()) return RAYN_OK;
  const long long n_int = 4ll * f->samples;
  for (int t : active) {
    if (a->rounds[t] != a->rounds[active[0]])
      return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_round: active tiles %d and %d have rendered %d and %d rounds; a stopped tile cannot resume", active[0], t,
                  a->rounds[active[0]], a->rounds[t]);
    if (a->K[t] + n_int > (1ll << 24))
      return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_round: tile %d would hold %lld samples per pixel, more than 2^24", t, a->K[t] + n_int);
  }
  const RaynFilmPlanes dev = film_block_planes(a->planes, (size_t)a->W * a->H);
  int32_t rc = render_enqueue(ctx, f, &dev, &active, nullptr);
  if (rc) return rc;
  if ((rc = render_finish(ctx))) return rc;
  cudaStream_t st = ctx->stream;
  const int nt = a->n_tiles, na = (int)active.size();
  CU(cudaMemcpyAsync(a->d_list, active.data(), na * sizeof(int), cudaMemcpyHostToDevice, st));
  k_accum_fold<<<na, ACC_T, 0, st>>>(a->W, a->H, a->tw, a->th, a->nty, a->d_list, (float)n_int, n_int, a->planes, a->state, a->dt);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(a->E.data(), a->dt.E, nt * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(a->K.data(), a->dt.K, nt * sizeof(long long), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(a->Kh.data(), a->dt.Kh, nt * sizeof(long long), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(a->rounds.data(), a->dt.rounds, nt * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  a->rounds_run++;
  if (out_tiles) *out_tiles = na;
  return RAYN_OK;
}

int32_t rayn_b200_accum_tiles(RaynContext* ctx, const RaynAccum* a, double* err, int64_t* samples) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!a) return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_tiles: accumulator is NULL");
  if (err) std::copy(a->E.begin(), a->E.end(), err);
  if (samples) std::copy(a->K.begin(), a->K.end(), samples);
  return RAYN_OK;
}

int32_t rayn_b200_accum_resolve(RaynContext* ctx, const RaynAccum* a, const RaynFilmPlanes* out) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!a || !out) return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_resolve: NULL argument");
  if (out->space != RAYN_MEM_HOST && out->space != RAYN_MEM_DEVICE) return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_resolve: bad memory space");
  if (a->device != ctx->device) return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_resolve: the accumulator lives on device %d, the context on %d", a->device, ctx->device);
  if (a->rounds_run == 0) return fail(ctx, RAYN_ERR_INVALID_ARG, "accum_resolve: no round has been rendered");
  if (!out->color && !out->alpha && !out->background && !out->normal) return RAYN_OK;
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t npx = (size_t)a->W * a->H;
  float *c = out->color, *al = out->alpha, *b = out->background, *n = out->normal;
  if (out->space == RAYN_MEM_HOST) {  // resolve into the round's planes (free between rounds), then copy out
    const RaynFilmPlanes p = film_block_planes(a->planes, npx);
    c = c ? p.color : nullptr, al = al ? p.alpha : nullptr, b = b ? p.background : nullptr, n = n ? p.normal : nullptr;
  } else {
    CU(cudaDeviceSynchronize());  // device planes may still be in use on another stream (e.g. torch's)
  }
  k_accum_resolve<<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(a->W, a->H, a->tw, a->th, a->ntx, a->nty, a->state, a->dt.K, c, al, b, n);
  CU(cudaGetLastError());
  if (out->space == RAYN_MEM_HOST) {
    int32_t rc = copy_planes(ctx, *out, a->planes, npx, cudaMemcpyDeviceToHost);
    if (rc) return rc;
  }
  CU(cudaStreamSynchronize(st));
  return RAYN_OK;
}

// ---- temporal accumulation (rt_temporal.cuh; statement in include/rayn_b200.h) -----------------------------------------
struct RaynTemporal {
  int device = 0, W = 0, H = 0;
  float* hist[2] = {nullptr, nullptr};  // TH_PLANES planes of W*H floats each
  int cur = 0;                          // the history the next push reads
};

int32_t rayn_b200_temporal_create(RaynContext* ctx, int32_t W, int32_t H, RaynTemporal** out) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  // W, H <= 2^23: every pixel centre (float)x + 0.5f of the push is then exact
  if (!out || W <= 0 || H <= 0 || W > (1 << 23) || H > (1 << 23) || (int64_t)W * H > ((int64_t)1 << 31))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "temporal_create: bad argument");
  *out = nullptr;
  CU(cudaSetDevice(ctx->device));
  RaynTemporal* t = new RaynTemporal();
  t->device = ctx->device, t->W = W, t->H = H;
  const size_t bytes = (size_t)W * H * TH_PLANES * sizeof(float);
  cudaError_t e = cudaMalloc((void**)&t->hist[0], bytes);
  if (e == cudaSuccess) e = cudaMalloc((void**)&t->hist[1], bytes);
  if (e == cudaSuccess) e = cudaMemsetAsync(t->hist[0], 0, bytes, ctx->stream);  // n = 0: no history yet
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) {
    cudaGetLastError();
    cudaFree(t->hist[0]), cudaFree(t->hist[1]);
    delete t;
    return fail(ctx, e == cudaErrorMemoryAllocation ? RAYN_ERR_OOM : RAYN_ERR_CUDA, "temporal_create (%dx%d): %s", W, H, cudaGetErrorString(e));
  }
  *out = t;
  return RAYN_OK;
}

void rayn_b200_temporal_destroy(RaynTemporal* t) {
  if (!t) return;
  cudaSetDevice(t->device);
  cudaDeviceSynchronize();
  cudaFree(t->hist[0]), cudaFree(t->hist[1]);
  delete t;
}

int32_t rayn_b200_temporal_push(RaynContext* ctx, RaynTemporal* t, const RaynTemporalDesc* d, const RaynFilmPlanes* in, const RaynMomentPlanes* mom,
                                const float* motion, const RaynFilmPlanes* out, const RaynMomentPlanes* omom, float* scale) {
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");
  if (!t || !d || !in || !mom || !motion || !out || !omom || !scale) return fail(ctx, RAYN_ERR_INVALID_ARG, "temporal_push: NULL argument");
  if (t->device != ctx->device) return fail(ctx, RAYN_ERR_INVALID_ARG, "temporal_push: the history lives on device %d, the context on %d", t->device, ctx->device);
  if (!in->color || !in->background || !in->normal || !mom->color_lum2 || !mom->background_lum2 || !out->color || !out->background ||
      !omom->color_lum2 || !omom->background_lum2)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "temporal_push: the colour, background, normal and moment planes are required");
  const int sp = in->space;
  if ((sp != RAYN_MEM_HOST && sp != RAYN_MEM_DEVICE) || mom->space != sp || out->space != sp || omom->space != sp)
    return fail(ctx, RAYN_ERR_INVALID_ARG, "temporal_push: every plane must be in one memory space");
  if (!(d->alpha_min > 0.0f && d->alpha_min <= 1.0f) || !(d->sigma_depth > 0.0f) || !(d->normal_cos >= -1.0f && d->normal_cos <= 1.0f) ||
      (d->reset != 0 && d->reset != 1))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "temporal_push: need alpha_min in (0, 1], sigma_depth > 0, normal_cos in [-1, 1], reset 0 or 1");
  CU(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t npx = (size_t)t->W * t->H;
  TemporalIo io{in->color, in->background, in->normal, mom->color_lum2, mom->background_lum2, motion,
                out->color, out->background, omom->color_lum2, omom->background_lum2, scale};
  float* stage = nullptr;
  if (sp == RAYN_MEM_HOST) {  // stream-ordered staging, released within the call: 15 floats in, 9 out per pixel
    CU(cudaMallocAsync((void**)&stage, npx * 24 * sizeof(float), st));
    const float* src[6] = {in->color, in->background, in->normal, mom->color_lum2, mom->background_lum2, motion};
    const int nf[6] = {3, 3, 3, 1, 1, 4};
    const float** dst[6] = {&io.c, &io.b, &io.n, &io.mc, &io.mb, &io.motion};
    float* s = stage;
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 6; ++i) {
      if (e == cudaSuccess) e = cudaMemcpyAsync(s, src[i], npx * nf[i] * sizeof(float), cudaMemcpyHostToDevice, st);
      *dst[i] = s;
      s += npx * nf[i];
    }
    io.oc = s, io.ob = s + 3 * npx, io.omc = s + 6 * npx, io.omb = s + 7 * npx, io.scale = s + 8 * npx;
    if (e != cudaSuccess) {
      cudaFreeAsync(stage, st);
      CU(e);
    }
  }
  k_temporal<<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(t->W, t->H, *d, t->hist[t->cur], t->hist[t->cur ^ 1], io);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) t->cur ^= 1;
  if (sp == RAYN_MEM_HOST) {
    float* const udst[5] = {out->color, out->background, omom->color_lum2, omom->background_lum2, scale};
    const float* const ddst[5] = {io.oc, io.ob, io.omc, io.omb, io.scale};
    const int nf[5] = {3, 3, 1, 1, 1};
    for (int i = 0; i < 5 && e == cudaSuccess; ++i) e = cudaMemcpyAsync(udst[i], ddst[i], npx * nf[i] * sizeof(float), cudaMemcpyDeviceToHost, st);
    const cudaError_t ef = cudaFreeAsync(stage, st);
    if (e == cudaSuccess) e = ef;
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  }
  CU(e);
  return RAYN_OK;
}

// ---- known-answer entry points ----------------------------------------------------------------------
#define KAT_PROLOGUE                                                     \
  if (!ctx) return fail(nullptr, RAYN_ERR_INVALID_ARG, "ctx is NULL");   \
  if (n < 0) return fail(ctx, RAYN_ERR_INVALID_ARG, "n < 0");            \
  CU(cudaSetDevice(ctx->device));                                        \
  if (n == 0) return RAYN_OK;                                            \
  DevTmp tmp;                                                            \
  cudaError_t e = cudaSuccess;                                           \
  const unsigned blocks = (unsigned)((n + 127) / 128);
#define KAT_EPILOGUE(dst, src, count, T)                                              \
  CU(e);                                                                              \
  CU(cudaGetLastError());                                                             \
  CU(cudaStreamSynchronize(ctx->stream));                                             \
  CU(cudaMemcpy(dst, src, (size_t)(count) * sizeof(T), cudaMemcpyDeviceToHost));

int32_t rayn_b200_kat_detmath(RaynContext* ctx, int32_t op, int64_t n, const float* a, const float* b, float* out) {
  KAT_PROLOGUE
  if (op < 0 || op > 8 || !a || !out) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_detmath: bad argument");
  float* da = tmp.up(a, n, &e);
  float* db = tmp.up(b ? b : a, n, &e);
  float* dout = tmp.up<float>(nullptr, n, &e);
  CU(e);
  k_kat_detmath<<<blocks, 128, 0, ctx->stream>>>(op, n, da, db, dout);
  KAT_EPILOGUE(out, dout, n, float)
  return RAYN_OK;
}
int32_t rayn_b200_kat_sdf_dist(RaynContext* ctx, const RaynHitable* sdf, int64_t n, const float* points3, float* out) {
  KAT_PROLOGUE
  if (!sdf || !points3 || !out) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_sdf_dist: NULL");
  float* dp = tmp.up(points3, 3 * n, &e);
  float* dout = tmp.up<float>(nullptr, n, &e);
  CU(e);
  k_kat_sdf_dist<<<blocks, 128, 0, ctx->stream>>>(*sdf, n, dp, dout);
  KAT_EPILOGUE(out, dout, n, float)
  return RAYN_OK;
}
int32_t rayn_b200_kat_sdf_trap(RaynContext* ctx, const RaynHitable* sdf, int64_t n, const float* points3, float* out) {
  KAT_PROLOGUE
  if (!sdf || !points3 || !out) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_sdf_trap: NULL");
  if (sdf->kind != RAYN_HITABLE_MANDELBOX && sdf->kind != RAYN_HITABLE_MANDELBULB) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_sdf_trap: not an SDF");
  float* dp = tmp.up(points3, 3 * n, &e);
  float* dout = tmp.up<float>(nullptr, n, &e);
  CU(e);
  k_kat_sdf_trap<<<blocks, 128, 0, ctx->stream>>>(*sdf, n, dp, dout);
  KAT_EPILOGUE(out, dout, n, float)
  return RAYN_OK;
}
int32_t rayn_b200_kat_sdf_dist2(RaynContext* ctx, const RaynHitable* sdf, int32_t variant, int64_t n, const float* points3, float* out) {
  KAT_PROLOGUE
  if (!sdf || !points3 || !out) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_sdf_dist2: NULL");
  if (sdf->kind == RAYN_HITABLE_SPHERE) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_sdf_dist2: not an SDF");
  int v = variant < 0 ? sdf_variant(*sdf, div3_verified(ctx, *sdf)) : variant;
  const bool v_fast = v == SDFV_BOX_12_FAST || v == SDFV_BOX_N_FAST, v_div3 = v == SDFV_BOX_12_DIV3 || v == SDFV_BOX_N_DIV3;
  if (v >= SDFV_COUNT || (v == SDFV_BULB) != (sdf->kind == RAYN_HITABLE_MANDELBULB) || ((v_fast || v_div3) && !sdf_box_fast_ok(*sdf)) ||
      ((v == SDFV_BOX_12_FAST || v == SDFV_BOX_12_DIV3) && sdf->iterations != 12) || (v_div3 && !div3_verified(ctx, *sdf)))
    return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_sdf_dist2: variant %d does not fit the hitable", v);
  float* dp = tmp.up(points3, 3 * n, &e);
  float* dout = tmp.up<float>(nullptr, n, &e);
  CU(e);
  DISPATCH_SDFV(v, (k_kat_sdf_dist2<V><<<(unsigned)((n / 2 + 128) / 128), 128, 0, ctx->stream>>>(*sdf, n, dp, dout)));
  KAT_EPILOGUE(out, dout, n, float)
  return RAYN_OK;
}
int32_t rayn_b200_kat_fastdiv(RaynContext* ctx, float num, uint32_t first_bits, int64_t n, int64_t* out_mismatches) {
  if (!ctx || !out_mismatches || n < 0) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_fastdiv: bad argument");
  CU(cudaSetDevice(ctx->device));
  CU(cudaMemsetAsync(ctx->d_kat, 0, sizeof(unsigned long long), ctx->stream));
  if (n > 0) k_kat_fastdiv<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(num, first_bits, n, ctx->d_kat);
  CU(cudaGetLastError());
  unsigned long long h = 0;
  CU(cudaMemcpyAsync(&h, ctx->d_kat, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  *out_mismatches = (int64_t)h;
  return RAYN_OK;
}
int32_t rayn_b200_kat_detmath_sweep(RaynContext* ctx, int32_t op, float b, int32_t swap, uint64_t* out_hashes256) {
  if (!ctx || op < 0 || op > 8 || !out_hashes256) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_detmath_sweep: bad argument");
  CU(cudaSetDevice(ctx->device));
  DevTmp tmp;
  cudaError_t e = cudaSuccess;
  unsigned long long* dh = tmp.up<unsigned long long>(nullptr, 256, &e);
  CU(e);
  CU(cudaMemsetAsync(dh, 0, 256 * sizeof(unsigned long long), ctx->stream));
  k_kat_detmath_sweep<<<256 * KAT_SWEEP_BLOCKS, 256, 0, ctx->stream>>>(op, b, swap, dh);
  KAT_EPILOGUE(out_hashes256, dh, 256, unsigned long long)
  return RAYN_OK;
}
int32_t rayn_b200_kat_sdf_hit(RaynContext* ctx, const RaynHitable* sdf, const RaynRenderConsts* consts, int64_t n, const float* origins3,
                              const float* dirs3, const float* t_max, float thr_scale, int32_t thr_const, float* out_t) {
  KAT_PROLOGUE
  if (!sdf || !consts || !origins3 || !dirs3 || !t_max || !out_t) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_sdf_hit: NULL");
  float* dor = tmp.up(origins3, 3 * n, &e);
  float* ddi = tmp.up(dirs3, 3 * n, &e);
  float* dtm = tmp.up(t_max, n, &e);
  float* dout = tmp.up<float>(nullptr, n, &e);
  CU(e);
  Thr thr;
  thr.scale = thr_scale;
  thr.is_const = thr_const;
  k_kat_sdf_hit<<<blocks, 128, 0, ctx->stream>>>(*sdf, *consts, n, dor, ddi, dtm, thr, dout);
  KAT_EPILOGUE(out_t, dout, n, float)
  return RAYN_OK;
}
int32_t rayn_b200_kat_occluded(RaynContext* ctx, int64_t n, const float* start3, const float* end3, float* out) {
  KAT_PROLOGUE
  if (!ctx->has_scene) return fail(ctx, RAYN_ERR_NO_SCENE, "kat_occluded before upload_scene");
  if (!start3 || !end3 || !out) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_occluded: NULL");
  float* ds = tmp.up(start3, 3 * n, &e);
  float* de = tmp.up(end3, 3 * n, &e);
  float* dout = tmp.up<float>(nullptr, n, &e);
  CU(e);
  k_kat_occluded<<<blocks, 128, 0, ctx->stream>>>(ctx->scene, n, ds, de, dout);
  KAT_EPILOGUE(out, dout, n, float)
  return RAYN_OK;
}
int32_t rayn_b200_kat_closest_hit(RaynContext* ctx, int32_t depth, int64_t n, const float* origins3, const float* dirs3, float* out_t,
                                  int32_t* out_obj) {
  KAT_PROLOGUE
  if (!ctx->has_scene) return fail(ctx, RAYN_ERR_NO_SCENE, "kat_closest_hit before upload_scene");
  if (!origins3 || !dirs3 || !out_t || !out_obj) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_closest_hit: NULL");
  float* dor = tmp.up(origins3, 3 * n, &e);
  float* ddi = tmp.up(dirs3, 3 * n, &e);
  float* dt = tmp.up<float>(nullptr, n, &e);
  int* dobj = tmp.up<int>(nullptr, n, &e);
  CU(e);
  k_kat_closest_hit<<<blocks, 128, 0, ctx->stream>>>(ctx->scene, make_thr(ctx->scene.cam, depth), n, dor, ddi, dt, dobj);
  KAT_EPILOGUE(out_t, dt, n, float)
  CU(cudaMemcpy(out_obj, dobj, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
  return RAYN_OK;
}

int32_t rayn_b200_kat_light_sample(RaynContext* ctx, const RaynLight* light, int64_t n, const float* s0, const float* s1, const float* points3,
                                   float* out_point3, float* out_pdf) {
  KAT_PROLOGUE
  if (!light || !s0 || !s1 || !points3 || !out_point3 || !out_pdf) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_light_sample: NULL");
  float *d0 = tmp.up(s0, n, &e), *d1 = tmp.up(s1, n, &e), *dp = tmp.up(points3, 3 * n, &e);
  float *dpt = tmp.up<float>(nullptr, 3 * n, &e), *dpdf = tmp.up<float>(nullptr, n, &e);
  CU(e);
  k_kat_light_sample<<<blocks, 128, 0, ctx->stream>>>(*light, n, d0, d1, dp, dpt, dpdf);
  KAT_EPILOGUE(out_point3, dpt, 3 * n, float)
  CU(cudaMemcpy(out_pdf, dpdf, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  return RAYN_OK;
}
int32_t rayn_b200_kat_light_sample_volume(RaynContext* ctx, const RaynLight* light, int64_t n, const float* sample, const float* origins3,
                                          const float* dirs3, const float* t_max, float* out_t, float* out_pdf) {
  KAT_PROLOGUE
  if (!light || !sample || !origins3 || !dirs3 || !t_max || !out_t || !out_pdf) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_light_sample_volume: NULL");
  float *ds = tmp.up(sample, n, &e), *dor = tmp.up(origins3, 3 * n, &e), *ddi = tmp.up(dirs3, 3 * n, &e), *dtm = tmp.up(t_max, n, &e);
  float *dt = tmp.up<float>(nullptr, n, &e), *dpdf = tmp.up<float>(nullptr, n, &e);
  CU(e);
  k_kat_light_sample_volume<<<blocks, 128, 0, ctx->stream>>>(*light, n, ds, dor, ddi, dtm, dt, dpdf);
  KAT_EPILOGUE(out_t, dt, n, float)
  CU(cudaMemcpy(out_pdf, dpdf, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  return RAYN_OK;
}
int32_t rayn_b200_kat_bsdf(RaynContext* ctx, const RaynMaterial* mat, int64_t n, const float* normals3, const float* wo3, const float* s1d,
                           const float* u4, float* out_wi3, float* out_f3, float* out_pdf, float* out_feval3) {
  KAT_PROLOGUE
  if (!mat || !normals3 || !wo3 || !s1d || !u4 || !out_wi3 || !out_f3 || !out_pdf || !out_feval3) return fail(ctx, RAYN_ERR_INVALID_ARG, "kat_bsdf: NULL");
  float *dn = tmp.up(normals3, 3 * n, &e), *dw = tmp.up(wo3, 3 * n, &e), *ds = tmp.up(s1d, n, &e), *du = tmp.up(u4, 4 * n, &e);
  float *dwi = tmp.up<float>(nullptr, 3 * n, &e), *df = tmp.up<float>(nullptr, 3 * n, &e), *dpdf = tmp.up<float>(nullptr, n, &e),
        *dfe = tmp.up<float>(nullptr, 3 * n, &e);
  CU(e);
  k_kat_bsdf<<<blocks, 128, 0, ctx->stream>>>(*mat, n, dn, dw, ds, du, dwi, df, dpdf, dfe);
  KAT_EPILOGUE(out_wi3, dwi, 3 * n, float)
  CU(cudaMemcpy(out_f3, df, (size_t)3 * n * sizeof(float), cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(out_pdf, dpdf, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(out_feval3, dfe, (size_t)3 * n * sizeof(float), cudaMemcpyDeviceToHost));
  return RAYN_OK;
}

}  // extern "C"
