// F2: coarse-to-fine occupancy engine (replaces implicit_seg.functional.Seg3dLossless / Seg3dTopk, a third-party
// un-vendored dependency of the reference: requirements.txt:15, call sites RTL/main.py:28-29,188-195,390-395).
// PARITY UNPINNED against upstream; bit-exact against this repo's restatement oracle/spec.py (seg3d_*_ref).
//
// One level step  (coarse res_c -> fine res_f = 2*res_c-1), all HBM-bound integer/byte work:
//   upsample_kernel   trilinear 2x (align_corners=True => weights {0,1/2,1}; x then y then z, one rounding per
//                     add -> bit-identical to F.interpolate), known-mask propagation, and the *dilated* boundary
//                     test folded into one pass: a fine node is a candidate iff the coarse occupancy flags are not
//                     uniform over the coarse box covering its (2r+1)^3 fine neighbourhood (== "interpolated mask
//                     strictly between 0 and 1, box-filtered, > 0" of the upstream algorithm).  Candidate flags are
//                     written transposed ([x][y][z]) so that the ordered compaction yields upstream's x-major order.
//   mpscan::scan_emit ordered stream compaction -> node list + device-side count (no host sync needed)
//   F1 query          fused sample+MLP on the node list, scattering straight into the level volume
//   (lossless mode)   conflict detection + 27-neighbourhood re-query loop
// Top-k variant: 4-pass radix select on |occ - balance| with index-order tie break.
#include "mp_common.cuh"
#include "octree_loop.cuh"

using namespace octree_k;

namespace {

__global__ void node_points_kernel(MpPointSrc src, float* __restrict__ pts) {
  long long n = src.n;
  if (src.count_dev) { const long long c = *src.count_dev; n = c < n ? c : n; }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float x, y, z;
    mp_load_point(src, MpBatch(), 0, i, x, y, z);
    pts[3 * i + 0] = x; pts[3 * i + 1] = y; pts[3 * i + 2] = z;
  }
}

// per-level evaluated-node counters [MP_MAX_LAYERS + 4] + one slot for the non-empty flag
constexpr int kStatSlots = MP_MAX_LAYERS + 5;
// per-level pass counters of the device-driven conflict loop + one slot for the truncated level (level + 1, 0 = none)
constexpr int kLoopSlots = MP_MAX_LAYERS + 5;
// A level of `res` nodes per axis stops its device-driven conflict loop after kLoopPassesPerRes * res passes.  The loop
// walks a thin feature about one node per pass: a one-voxel rod took 0.3 * res passes, 25x below the cap.
constexpr int kLoopPassesPerRes = 8;

// ---- multi-GPU list sharding (SURVEY.md §8e): every rank keeps the whole pyramid state and runs the cheap volume passes
// itself (identical inputs => identical node lists on every rank, including the lossless conflict loop, which can walk
// across any slab boundary); only the expensive part -- the MLP evaluation of a level's node list -- is split: rank r
// evaluates the r-th window of the ordered list (balanced to one 128-point tile) and its kernel stores each value into the
// value lists of ALL ranks over NVLink peer memory.  What is left of the exchange is this barrier between the ranks'
// streams: thread p publishes "rank `rank` has finished epoch e" in peer p's flag array and waits for peer p's flag.
struct XBarrier {
  uint32_t* peer[MP_MAX_PEERS];   // flag arrays of all ranks ([MP_MAX_PEERS] words each), peer-mapped
  uint32_t* mine;
  int rank, world;
  uint32_t epoch;
};
__global__ void xgpu_barrier_kernel(XBarrier b) {
  const int p = threadIdx.x;
  if (p < b.world) {
    // (the peer stores of the preceding kernels of this stream have completed; the fence orders them before the flag)
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(b.peer[p] + b.rank), "r"(b.epoch) : "memory");
    uint32_t v;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(b.mine + p) : "memory");
    } while ((int32_t)(v - b.epoch) < 0);
  }
}

inline int grid_for(long long n, int threads = 256, int cap = 148 * 8) {
  long long b = (n + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace


// ---------------------------------------------------------------------------------------------------
struct mp_octree {
  int n_levels;
  int res[MP_MAX_LAYERS + 4];
  float bmin[3], bmax[3];
  float balance;
  int faster;
  int use_topk;
  int topk[MP_MAX_LAYERS + 4];
  int R;
  long long cap;              // node-list capacity
  long long vol_elems;        // R^3
  float* vol[2];
  uint8_t* known[2];
  uint8_t* cand_t;            // transposed candidate flags
  uint8_t* conflict;
  int32_t* idx;
  float* points;              // [cap,3]
  float* vals;                // [cap] scratch (fused path conflict detection); == vals2[0]
  // list sharding: two alternating value lists (a rank may already receive the next list while it still scatters this
  // one), the flag array of the cross-GPU barrier, and the peer mappings of all ranks' (own included)
  float* vals2[2];
  uint32_t* flags;
  float* peer_vals[2][MP_MAX_PEERS];
  uint32_t* peer_flags[MP_MAX_PEERS];
  int shard_rank, shard_world;
  uint32_t epoch;
  int vsel;
  unsigned long long* sums;   // scan block sums
  unsigned long long* total;  // scan total
  int32_t* count;             // device count of the current node list
  int* nonempty;              // device flag
  long long* stats;           // device [n_levels]
  SelectState* sel;
  // lossless handles: the device-driven conflict loop of mp_octree_run_fused_async.  `loops` holds its pass counters;
  // body_stream records the WHILE bodies, cap_stream the whole run when the caller's stream is not being captured.
  int32_t* loops;
  cudaStream_t body_stream, cap_stream;
  // stepping state
  int level;                  // level of the outstanding batch (-1 before begin)
  int cur;                    // which vol/known buffer holds `level`
  int phase;                  // 0: level-0 batch outstanding/next, 1: regular, 2: finished
  long long batch_n;
  int awaiting_commit;
  int evaluated;              // the current level received at least one committed batch
};

static int radius_for(const mp_octree* h, int level) {
  if (!h->faster) return 1;
  return level == 1 ? 4 : (level == 2 ? 3 : 1);    // box k = 9 / 7 / 3
}

extern "C" int mp_octree_destroy(mp_octree_t* h) {
  if (!h) return MP_OK;
  for (int i = 0; i < 2; ++i) { if (h->vol[i]) cudaFree(h->vol[i]); if (h->known[i]) cudaFree(h->known[i]); }
  if (h->cand_t) cudaFree(h->cand_t);
  if (h->conflict) cudaFree(h->conflict);
  if (h->idx) cudaFree(h->idx);
  if (h->points) cudaFree(h->points);
  if (h->vals) cudaFree(h->vals);
  if (h->vals2[1]) cudaFree(h->vals2[1]);
  if (h->flags) cudaFree(h->flags);
  if (h->sums) cudaFree(h->sums);
  if (h->total) cudaFree(h->total);
  if (h->count) cudaFree(h->count);
  if (h->stats) cudaFree(h->stats);
  if (h->sel) cudaFree(h->sel);
  if (h->loops) cudaFree(h->loops);
  if (h->body_stream) cudaStreamDestroy(h->body_stream);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  delete h;
  return MP_OK;
}

extern "C" int mp_octree_create(int n_levels, const int* resolutions, const float* b_min3, const float* b_max3,
                                float balance_value, int faster, const int* topk_points, mp_octree_t** out) {
  MP_REQUIRE(out != nullptr, "out is NULL");
  *out = nullptr;
  MP_REQUIRE(n_levels >= 1 && n_levels <= MP_MAX_LAYERS + 4, "n_levels=%d out of range", n_levels);
  MP_REQUIRE(resolutions && b_min3 && b_max3, "NULL argument");
  for (int l = 0; l < n_levels; ++l) {
    MP_REQUIRE(resolutions[l] >= 3 && (resolutions[l] & 1) && resolutions[l] <= 1025, "resolution[%d]=%d must be odd, 3..1025", l, resolutions[l]);
    if (l > 0) MP_REQUIRE(resolutions[l] == 2 * resolutions[l - 1] - 1, "resolutions must follow r -> 2r-1 (got %d after %d)", resolutions[l], resolutions[l - 1]);
  }
  mp_octree* h = new mp_octree();
  memset(h, 0, sizeof(*h));
  h->n_levels = n_levels;
  for (int l = 0; l < n_levels; ++l) h->res[l] = resolutions[l];
  for (int a = 0; a < 3; ++a) { h->bmin[a] = b_min3[a]; h->bmax[a] = b_max3[a]; }
  h->balance = balance_value;
  h->faster = faster ? 1 : 0;
  h->use_topk = topk_points != nullptr;
  h->R = resolutions[n_levels - 1];
  h->vol_elems = (long long)h->R * h->R * h->R;
  long long cap = (long long)h->res[0] * h->res[0] * h->res[0];
  if (h->use_topk) {
    for (int l = 0; l < n_levels; ++l) {
      h->topk[l] = topk_points[l];
      const long long r3 = (long long)h->res[l] * h->res[l] * h->res[l];
      long long k = topk_points[l] < 0 ? 0 : topk_points[l];
      if (k > r3) k = r3;
      if (l > 0 && k > cap) cap = k;
    }
  } else {
    const int last_examined = (h->faster && n_levels > 1) ? n_levels - 2 : n_levels - 1;
    const long long r = h->res[last_examined];
    if (r * r * r > cap) cap = r * r * r;
  }
  h->cap = cap;
  h->level = -1;
  h->phase = 2;
  const long long V = h->vol_elems;
  cudaError_t e = cudaSuccess;
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
    e = cudaMalloc(&h->vol[i], V * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&h->known[i], V);
  }
  if (e == cudaSuccess) e = cudaMalloc(&h->cand_t, V);
  if (e == cudaSuccess) e = cudaMalloc(&h->conflict, V);
  if (e == cudaSuccess) e = cudaMalloc(&h->idx, cap * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->points, cap * 3 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->vals, cap * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->sums, (size_t)(mpscan::num_blocks(V) + 1) * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMalloc(&h->total, 2 * sizeof(unsigned long long));                 // [0] total, [1] scan ticket
  if (e == cudaSuccess) e = cudaMemset(h->total, 0, 2 * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMalloc(&h->count, sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->stats, sizeof(long long) * kStatSlots);
  // the non-empty flag lives in the last slot of the stats buffer: one memset resets both, one copy reads both back
  if (e == cudaSuccess) h->nonempty = reinterpret_cast<int*>(h->stats + kStatSlots - 1);
  if (e == cudaSuccess) e = cudaMalloc(&h->sel, sizeof(SelectState));
  if (!h->use_topk && !h->faster) {   // (streams are created here, never while a caller's stream is being captured)
    if (e == cudaSuccess) e = cudaMalloc(&h->loops, sizeof(int32_t) * kLoopSlots);
    if (e == cudaSuccess) e = cudaMemset(h->loops, 0, sizeof(int32_t) * kLoopSlots);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->body_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking);
  }
  if (e != cudaSuccess) {
    mp_set_error("mp_octree_create: %s", cudaGetErrorString(e));
    mp_octree_destroy(h);
    return MP_E_NOMEM;
  }
  h->vals2[0] = h->vals;
  h->shard_world = 1;
  *out = h;
  return MP_OK;
}

// ---- list sharding over the GPUs of a node --------------------------------------------------------
extern "C" int mp_octree_shard_export(mp_octree_t* h, unsigned char* handles192) {
  MP_REQUIRE(h && handles192, "NULL argument");
  if (!h->vals2[1]) MP_CUDA(cudaMalloc(&h->vals2[1], h->cap * sizeof(float)));
  if (!h->flags) {
    MP_CUDA(cudaMalloc(&h->flags, MP_MAX_PEERS * sizeof(uint32_t)));
    MP_CUDA(cudaMemset(h->flags, 0, MP_MAX_PEERS * sizeof(uint32_t)));
  }
  void* ptrs[3] = {h->vals2[0], h->vals2[1], h->flags};
  for (int k = 0; k < 3; ++k) {
    cudaIpcMemHandle_t ih;
    MP_CUDA(cudaIpcGetMemHandle(&ih, ptrs[k]));
    memcpy(handles192 + 64 * k, &ih, 64);
  }
  return MP_OK;
}

extern "C" int mp_octree_shard_set(mp_octree_t* h, int rank, int world, float* const* vals0, float* const* vals1,
                                   uint32_t* const* flags) {
  MP_REQUIRE(h, "NULL handle");
  MP_REQUIRE(world >= 1 && world <= MP_MAX_PEERS && rank >= 0 && rank < world, "bad rank %d of %d (at most %d ranks)", rank, world, MP_MAX_PEERS);
  if (world == 1) { h->shard_world = 1; h->shard_rank = 0; return MP_OK; }
  MP_REQUIRE(vals0 && vals1 && flags, "NULL pointer arrays");
  MP_REQUIRE(h->vals2[1] && h->flags, "mp_octree_shard_export must run first");
  for (int p = 0; p < world; ++p) {
    h->peer_vals[0][p] = (p == rank) ? h->vals2[0] : vals0[p];
    h->peer_vals[1][p] = (p == rank) ? h->vals2[1] : vals1[p];
    h->peer_flags[p] = (p == rank) ? h->flags : flags[p];
    MP_REQUIRE(h->peer_vals[0][p] && h->peer_vals[1][p] && h->peer_flags[p], "peer %d: NULL mapping", p);
  }
  h->shard_rank = rank;
  h->shard_world = world;
  h->epoch = 0;
  h->vsel = 0;
  return MP_OK;
}

// evaluate `src` (this rank's window of it) into the value lists of all ranks, wait for everybody; returns the list to
// scatter from
static int sharded_query(mp_octree* h, mp_mlp_t* mlp, mp_feat_t* feat, MpPointSrc src, const MpCalib& cal, int mode,
                         cudaStream_t st, const float** vals_out) {
  src.shard_rank = h->shard_rank;
  src.shard_world = h->shard_world;
  MpOutDst dst;
  dst.out = nullptr; dst.ld = 0; dst.scatter_vol = nullptr;
  for (int p = 0; p < h->shard_world; ++p) dst.peer[p] = h->peer_vals[h->vsel][p];
  dst.n_peers = h->shard_world;
  dst.peer_off = 0;
  int rc = mp_query_dispatch(mlp, feat, src, cal, dst, mode, st);
  if (rc != MP_OK) return rc;
  XBarrier b;
  for (int p = 0; p < MP_MAX_PEERS; ++p) b.peer[p] = p < h->shard_world ? h->peer_flags[p] : nullptr;
  b.mine = h->flags;
  b.rank = h->shard_rank;
  b.world = h->shard_world;
  b.epoch = ++h->epoch;
  xgpu_barrier_kernel<<<1, 32, 0, st>>>(b);
  MP_CUDA(cudaGetLastError());
  *vals_out = h->vals2[h->vsel];
  h->vsel ^= 1;
  return MP_OK;
}

// ---- building blocks shared by the stepping API and the fused run ----------------------------------
static void fill_src_nodes(const mp_octree* h, int level, MpPointSrc& src, long long n_upper, bool device_count) {
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_NODES;
  const int res = h->res[level];
  mp_fill_grid_geom(src, res, (h->R - 1) / (res - 1), h->R, h->bmin, h->bmax);
  src.nodes = h->idx;
  src.count_dev = device_count ? h->count : nullptr;
  src.n = n_upper;
}

// Upsample level-1 -> level and build the (ordered) candidate list of `level`.  Leaves count on the device.
static int build_level_list(mp_octree* h, int level, cudaStream_t st) {
  const int res_c = h->res[level - 1], res_f = h->res[level];
  const long long nf = (long long)res_f * res_f * res_f;
  const int src_buf = h->cur, dst_buf = h->cur ^ 1;
  const bool last = level == h->n_levels - 1;
  const bool interp_only = h->use_topk || (h->faster && last);
  {
    const dim3 grid((unsigned)(((long long)res_c * res_c + 255) / 256), (unsigned)res_c);
    const float* vc = h->vol[src_buf];
    const uint8_t* kc = h->use_topk ? nullptr : h->known[src_buf];
    float* vf = h->vol[dst_buf];
    // (the last level of the `faster` engine is interpolation only: nothing reads its known mask afterwards)
    uint8_t* kf = (h->use_topk || (h->faster && last)) ? nullptr : h->known[dst_buf];
    const int radius = radius_for(h, level);
    // the union of the eight boxes of a cell is at most radius + 2 coarse nodes wide
    if (interp_only) upsample_kernel<0><<<grid, 256, 0, st>>>(vc, kc, vf, kf, nullptr, res_c, res_f, radius, h->balance);
    else if (radius <= 1) upsample_kernel<3><<<grid, 256, 0, st>>>(vc, kc, vf, kf, h->cand_t, res_c, res_f, radius, h->balance);
    else if (radius <= 3) upsample_kernel<5><<<grid, 256, 0, st>>>(vc, kc, vf, kf, h->cand_t, res_c, res_f, radius, h->balance);
    else if (radius <= 4) upsample_kernel<6><<<grid, 256, 0, st>>>(vc, kc, vf, kf, h->cand_t, res_c, res_f, radius, h->balance);
    else { mp_set_error("octree: box radius %d not supported", radius); return MP_E_UNSUPPORTED; }
  }
  MP_CUDA(cudaGetLastError());
  h->cur = dst_buf;
  if (h->use_topk) {
    long long k = h->topk[level] < 0 ? 0 : h->topk[level];
    if (k > nf) k = nf;
    if (k == 0) {
      MP_CUDA(cudaMemsetAsync(h->count, 0, sizeof(int32_t), st));
      return MP_OK;
    }
    select_init_kernel<<<1, 256, 0, st>>>(h->sel, (uint32_t)k);
    for (int pass = 0; pass < 4; ++pass) {
      select_hist_kernel<<<grid_for(nf), 256, 0, st>>>(h->vol[dst_buf], nf, h->balance, h->sel, pass);
      select_pick_kernel<<<1, 256, 0, st>>>(h->sel, pass);
    }
    TopkF f{h->vol[dst_buf], h->balance, h->sel};
    TopkEmit em{h->idx, h->sel};
    MP_CUDA(mpscan::scan_emit(f, em, nf, h->sums, h->total, st));
    // count = k exactly, or 0 when level 0 found nothing occupied
    topk_count_kernel<<<1, 1, 0, st>>>(h->count, h->stats + level, h->nonempty, (int32_t)k);
    MP_CUDA(cudaGetLastError());
    return MP_OK;
  }
  if (interp_only) {
    MP_CUDA(cudaMemsetAsync(h->count, 0, sizeof(int32_t), st));
    return MP_OK;
  }
  FlagF f{h->cand_t};
  EmitNodesT em{h->idx, res_f, h->cap};
  MP_CUDA(mpscan::scan_emit(f, em, nf, h->sums, h->total, st, CountPost{h->count, h->cap, h->stats + level}));
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

static int build_conflict_list(mp_octree* h, int level, cudaStream_t st) {
  const int res = h->res[level];
  const long long nf = (long long)res * res * res;
  conflict_neighbours_kernel<<<grid_for(nf), 256, 0, st>>>(h->conflict, h->known[h->cur], h->cand_t, res);
  MP_CUDA(cudaGetLastError());
  MP_CUDA(cudaMemsetAsync(h->conflict, 0, nf, st));
  FlagF f{h->cand_t};
  EmitNodesT em{h->idx, res, h->cap};
  MP_CUDA(mpscan::scan_emit(f, em, nf, h->sums, h->total, st, CountPost{h->count, h->cap, h->stats + level}));
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

static int reset_run(mp_octree* h, cudaStream_t st) {
  MP_CUDA(cudaMemsetAsync(h->stats, 0, sizeof(long long) * kStatSlots, st));   // includes the non-empty flag
  if (!h->use_topk && !h->faster) MP_CUDA(cudaMemsetAsync(h->conflict, 0, h->vol_elems, st));   // only the lossless loop reads it
  h->cur = 0;
  return MP_OK;
}

// ---- stepping API ---------------------------------------------------------------------------------
extern "C" int mp_octree_begin(mp_octree_t* h, void* stream) {
  MP_REQUIRE(h, "NULL handle");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = reset_run(h, st);
  if (rc != MP_OK) return rc;
  h->level = 0;
  h->phase = 0;
  h->awaiting_commit = 0;
  h->evaluated = 0;
  h->batch_n = 0;
  return MP_OK;
}

extern "C" int mp_octree_next(mp_octree_t* h, int64_t* n_out, int* level_out, const float** points_dev_out,
                              const int32_t** idx_dev_out, void* stream) {
  MP_REQUIRE(h && n_out, "NULL argument");
  MP_REQUIRE(h->level >= 0, "mp_octree_begin was not called");
  MP_REQUIRE(!h->awaiting_commit, "previous batch was not committed");
  cudaStream_t st = (cudaStream_t)stream;
  *n_out = 0;
  if (level_out) *level_out = h->level;
  if (points_dev_out) *points_dev_out = h->points;
  if (idx_dev_out) *idx_dev_out = h->idx;
  if (h->phase == 2) return MP_OK;
  long long n = 0;
  if (h->phase == 0) {
    const int r0 = h->res[0];
    n = (long long)r0 * r0 * r0;
    iota_kernel<<<grid_for(n), 256, 0, st>>>(h->idx, (int)n);
    const int32_t c = (int32_t)n;
    MP_CUDA(cudaMemcpyAsync(h->count, &c, sizeof(int32_t), cudaMemcpyHostToDevice, st));
    set_u8_kernel<<<grid_for(n), 256, 0, st>>>(h->known[h->cur], n, 1);
    MP_CUDA(cudaGetLastError());
  } else {
    if (h->level == 0) {   // after level 0: stop if nothing is occupied (the engine then returns None)
      int ne = 0;
      MP_CUDA(cudaMemcpyAsync(&ne, h->nonempty, sizeof(int), cudaMemcpyDeviceToHost, st));
      MP_CUDA(cudaStreamSynchronize(st));
      if (!ne) { h->phase = 2; return MP_OK; }
    }
    const bool lossless = !h->use_topk && !h->faster;
    int32_t cnt = 0;
    for (;;) {
      if (lossless && h->level > 0 && h->evaluated) {
        // conflict loop: re-query the 27-neighbourhood of sign conflicts until none remain
        int rc = build_conflict_list(h, h->level, st);
        if (rc != MP_OK) return rc;
        MP_CUDA(cudaMemcpyAsync(&cnt, h->count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        MP_CUDA(cudaStreamSynchronize(st));
        if (cnt > 0) break;
      }
      if (h->level + 1 >= h->n_levels) {
        h->phase = 2;
        if (level_out) *level_out = h->level;
        return MP_OK;
      }
      h->level += 1;
      h->evaluated = 0;
      int rc = build_level_list(h, h->level, st);
      if (rc != MP_OK) return rc;
      MP_CUDA(cudaMemcpyAsync(&cnt, h->count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      MP_CUDA(cudaStreamSynchronize(st));
      if (cnt > 0) break;
    }
    n = cnt;
  }
  MpPointSrc src;
  fill_src_nodes(h, h->level, src, n, false);
  node_points_kernel<<<grid_for(n), 256, 0, st>>>(src, h->points);
  MP_CUDA(cudaGetLastError());
  MP_CUDA(cudaStreamSynchronize(st));
  h->batch_n = n;
  h->awaiting_commit = 1;
  *n_out = n;
  if (level_out) *level_out = h->level;
  return MP_OK;
}

extern "C" int mp_octree_commit(mp_octree_t* h, const float* values_dev, void* stream) {
  MP_REQUIRE(h && values_dev, "NULL argument");
  MP_REQUIRE(h->awaiting_commit, "no outstanding batch");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = h->batch_n;
  const bool lossless = !h->use_topk && !h->faster && h->level > 0;
  scatter_kernel<<<grid_for(n), 256, 0, st>>>(h->idx, nullptr, n, values_dev, h->vol[h->cur],
                                              h->use_topk ? nullptr : h->known[h->cur],
                                              lossless ? h->conflict : nullptr, h->balance, true);
  MP_CUDA(cudaGetLastError());
  if (h->level == 0) {
    any_gt_kernel<<<grid_for(n), 256, 0, st>>>(h->vol[h->cur], n, h->balance, h->nonempty);
    MP_CUDA(cudaGetLastError());
  }
  h->phase = 1;
  h->evaluated = 1;
  h->awaiting_commit = 0;
  return MP_OK;
}

extern "C" int mp_octree_finish(mp_octree_t* h, float* out_dev, int* nonempty, void* stream) {
  MP_REQUIRE(h && nonempty, "NULL argument");
  cudaStream_t st = (cudaStream_t)stream;
  int ne = 0;
  MP_CUDA(cudaMemcpyAsync(&ne, h->nonempty, sizeof(int), cudaMemcpyDeviceToHost, st));
  MP_CUDA(cudaStreamSynchronize(st));
  *nonempty = ne;
  if (ne && out_dev) {
    MP_REQUIRE(h->level == h->n_levels - 1, "reconstruction not finished (level %d of %d)", h->level, h->n_levels);
    MP_CUDA(cudaMemcpyAsync(out_dev, h->vol[h->cur], h->vol_elems * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return MP_OK;
}

// ---- fused run --------------------------------------------------------------------------------------
// One evaluation pass of `level` over its node list (h->idx, count on the device): the query, then the scatter (lossless:
// into the value list first, with conflict detection against the interpolated volume, then the next conflict list).
static int level_pass(mp_octree* h, int level, mp_mlp_t* mlp, mp_feat_t* feat, const MpCalib& cal, const MpBatch* bt, int mode,
                      cudaStream_t st) {
  const bool lossless = !h->use_topk && !h->faster;
  int rc = MP_OK;
  MpPointSrc src;
  fill_src_nodes(h, level, src, h->cap, true);
  if (h->use_topk) {   // (the count on the device is k, or 0 after an empty level 0: build_level_list)
    long long k = h->topk[level];
    const long long nf = (long long)h->res[level] * h->res[level] * h->res[level];
    if (k > nf) k = nf;
    if (k <= 0) return MP_OK;
    src.n = k;
  }
  const float* vals = h->vals;
  const bool via_vals = lossless || h->shard_world > 1;
  if (h->shard_world > 1) {
    rc = sharded_query(h, mlp, feat, src, cal, mode, st, &vals);
    if (rc != MP_OK) return rc;
  } else {
    MpOutDst dst;
    dst.out = nullptr; dst.ld = 0; dst.scatter_vol = h->vol[h->cur];
    if (lossless) {
      // keep the interpolated values, evaluate into vals, then scatter+conflict-detect
      dst.out = h->vals; dst.ld = h->cap; dst.scatter_vol = nullptr;
    }
    rc = mp_query_dispatch(mlp, feat, src, cal, dst, mode, st, bt);
    if (rc != MP_OK) return rc;
  }
  scatter_kernel<<<grid_for(h->cap > 1 << 20 ? 1 << 20 : h->cap), 256, 0, st>>>(
      h->idx, src.count_dev, src.n, via_vals ? vals : h->vol[h->cur], h->vol[h->cur],
      h->use_topk ? nullptr : h->known[h->cur], lossless ? h->conflict : nullptr, h->balance, via_vals);
  MP_CUDA(cudaGetLastError());
  if (lossless) return build_conflict_list(h, level, st);
  return MP_OK;
}

// The conflict loop of a lossless level as a WHILE node of the graph being captured on `st`: the body is one level_pass
// followed by loop_control_kernel, which decides on the device whether the body runs again.  The condition defaults to 1
// on every launch of the graph, so the body runs at least once, as in the host-driven loop.
static int device_conflict_loop(mp_octree* h, int level, mp_mlp_t* mlp, mp_feat_t* feat, const MpCalib& cal, const MpBatch* bt,
                                int mode, cudaStream_t st) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaGraph_t graph = nullptr;
  const cudaGraphNode_t* deps = nullptr;
  size_t n_deps = 0;
  MP_CUDA(cudaStreamGetCaptureInfo(st, &cs, nullptr, &graph, &deps, &n_deps));
  if (cs != cudaStreamCaptureStatusActive) {
    mp_set_error("octree: the device-driven conflict loop needs a stream that is being captured");
    return MP_E_CUDA;
  }
  cudaGraphConditionalHandle cond;
  MP_CUDA(cudaGraphConditionalHandleCreate(&cond, graph, 1, cudaGraphCondAssignDefault));
  cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
  np.conditional.handle = cond;
  np.conditional.type = cudaGraphCondTypeWhile;
  np.conditional.size = 1;
  cudaGraphNode_t node;
  MP_CUDA(cudaGraphAddNode(&node, graph, deps, n_deps, &np));
  MP_CUDA(cudaStreamUpdateCaptureDependencies(st, &node, 1, cudaStreamSetCaptureDependencies));   // the next level waits
  MP_CUDA(cudaStreamBeginCaptureToGraph(h->body_stream, np.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                        cudaStreamCaptureModeRelaxed));
  int rc = level_pass(h, level, mlp, feat, cal, bt, mode, h->body_stream);
  if (rc == MP_OK) {
    loop_control_kernel<<<1, 1, 0, h->body_stream>>>(h->count, h->loops + level, h->loops + kLoopSlots - 1, level,
                                                     kLoopPassesPerRes * h->res[level], cond);
    const cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) {
      mp_set_error("octree: loop_control_kernel: %s", cudaGetErrorString(le));
      rc = MP_E_CUDA;
    }
  }
  cudaGraph_t body = nullptr;
  const cudaError_t e = cudaStreamEndCapture(h->body_stream, &body);   // (always: the private stream stays usable)
  if (rc != MP_OK) return rc;
  MP_CUDA(e);
  return MP_OK;
}

// device_loop: the lossless conflict loop of every level runs as a WHILE node of the graph captured on `st` (no host read);
// otherwise it is driven from the host, which reads the list length back after every pass.
static int run_fused_levels(mp_octree* h, mp_mlp_t* mlp, mp_feat_t* feat, const MpCalib& cal, const MpBatch* bt, int mode,
                            cudaStream_t st, bool device_loop = false) {
  int rc = MP_OK;
  // level 0: dense
  {
    const int r0 = h->res[0];
    const long long n = (long long)r0 * r0 * r0;
    MpPointSrc src;
    memset(&src, 0, sizeof(src));
    src.kind = MP_SRC_GRID;
    mp_fill_grid_geom(src, r0, (h->R - 1) / (r0 - 1), h->R, h->bmin, h->bmax);
    src.n = n;
    if (h->shard_world > 1) {
      const float* vals = nullptr;
      rc = sharded_query(h, mlp, feat, src, cal, mode, st, &vals);
      if (rc != MP_OK) return rc;
      MP_CUDA(cudaMemcpyAsync(h->vol[h->cur], vals, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    } else {
      MpOutDst dst;
      dst.out = h->vol[h->cur]; dst.ld = n; dst.scatter_vol = nullptr;
      rc = mp_query_dispatch(mlp, feat, src, cal, dst, mode, st, bt);
      if (rc != MP_OK) return rc;
    }
    set_u8_kernel<<<grid_for(n), 256, 0, st>>>(h->known[h->cur], n, 1);
    any_gt_kernel<<<grid_for(n), 256, 0, st>>>(h->vol[h->cur], n, h->balance, h->nonempty);
    const long long n0 = n;
    set_i64_kernel<<<1, 1, 0, st>>>(h->stats, n0);
  }
  for (int level = 1; level < h->n_levels; ++level) {
    h->level = level;
    rc = build_level_list(h, level, st);
    if (rc != MP_OK) return rc;
    const bool last = level == h->n_levels - 1;
    if (!h->use_topk && h->faster && last) break;
    const bool lossless = !h->use_topk && !h->faster;
    if (lossless && device_loop) {
      rc = device_conflict_loop(h, level, mlp, feat, cal, bt, mode, st);
      if (rc != MP_OK) return rc;
      continue;
    }
    for (;;) {
      rc = level_pass(h, level, mlp, feat, cal, bt, mode, st);
      if (rc != MP_OK) return rc;
      if (!lossless) break;
      int32_t cnt = 0;
      MP_CUDA(cudaMemcpyAsync(&cnt, h->count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      MP_CUDA(cudaStreamSynchronize(st));
      if (cnt == 0) break;
    }
  }
  h->level = h->n_levels - 1;
  return MP_OK;
}

// The enqueue sequence of mp_octree_run_fused_async on `st`.
static int enqueue_fused(mp_octree* h, mp_mlp_t* mlp, mp_feat_t* feat, const MpCalib& cal, const MpBatch* bt, int mode,
                         float* out_dev, cudaStream_t st) {
  const bool lossless = !h->use_topk && !h->faster;
  int rc = reset_run(h, st);
  if (rc != MP_OK) return rc;
  if (lossless) MP_CUDA(cudaMemsetAsync(h->loops, 0, sizeof(int32_t) * kLoopSlots, st));
  const int final_buf = (h->n_levels - 1) & 1;
  float* const own_buf = h->vol[final_buf];
  h->vol[final_buf] = out_dev;          // the last level lands in the caller's volume (see mp_octree_run_fused)
  rc = run_fused_levels(h, mlp, feat, cal, bt, mode, st, lossless);
  const bool in_place = h->cur == final_buf;
  const float* result = h->vol[h->cur];
  h->vol[final_buf] = own_buf;
  if (rc != MP_OK) return rc;
  if (!in_place) MP_CUDA(cudaMemcpyAsync(out_dev, result, h->vol_elems * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return MP_OK;
}

// The enqueue half of the fused run: everything is stream-ordered and no host memory is read, so the call can be captured
// into a CUDA graph.  Results (non-empty flag, per-level counts, conflict-loop passes) stay on the device until
// mp_octree_fetch / mp_octree_fetch_loops.  A lossless engine's conflict loop runs as a WHILE node per level; on a stream
// that is not being captured the call records its sequence into a graph of its own and launches that on the stream.
// calib_dev (the _dcal twin): the camera's 12 floats in device memory, read by the query launches when they run -- a
// captured run, the lossless WHILE bodies included, then reads the current camera at every replay.
static int run_fused_async(mp_octree* h, mp_mlp_t* mlp, mp_feat_t* feat, const float* calib12, const float* calib_dev,
                           int projection, float z_scale, int mode, float* out_dev, void* stream) {
  MP_REQUIRE(h && mlp && feat && out_dev, "NULL argument");
  MP_REQUIRE_SINGLE_MAP(feat, "the occupancy engine");
  MP_REQUIRE(mlp->cout[mlp->n_layers - 1] == 1, "the occupancy engine needs a single-channel head");
  const bool lossless = !h->use_topk && !h->faster;
  if (lossless && h->shard_world > 1) {
    // (the barrier epochs of a sharded run are counted on the host: a replayed loop body would reuse one)
    mp_set_error("a sharded lossless engine reads counts on the host; use mp_octree_run_fused");
    return MP_E_UNSUPPORTED;
  }
  // (the value lists of a sharded engine go through sharded_query, which takes the camera by value)
  MP_REQUIRE(!calib_dev || h->shard_world == 1, "a sharded engine takes its calib by value");
  MpRange nvtx("monoport_b200: F2 coarse-to-fine engine (enqueue)");
  cudaStream_t st = (cudaStream_t)stream;
  MpCalib cal;
  MpBatch one;
  const MpBatch* bt = mp_single_calib(cal, one, calib12, calib_dev, projection, z_scale);
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (lossless) MP_CUDA(cudaStreamIsCapturing(st, &cs));
  if (!lossless || cs == cudaStreamCaptureStatusActive) {
    const int rc = enqueue_fused(h, mlp, feat, cal, bt, mode, out_dev, st);
    if (rc != MP_OK) return rc;
    h->phase = 2;
    return MP_OK;
  }
  // not capturing: capture the sequence on the private stream (relaxed: the lazy allocations of a query stay legal),
  // then launch it on the caller's stream
  MP_CUDA(cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeRelaxed));
  const int rc = enqueue_fused(h, mlp, feat, cal, bt, mode, out_dev, h->cap_stream);
  cudaGraph_t graph = nullptr;
  cudaError_t e = cudaStreamEndCapture(h->cap_stream, &graph);
  if (rc != MP_OK) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  MP_CUDA(e);
  cudaGraphExec_t exec = nullptr;
  e = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  MP_CUDA(e);
  e = cudaGraphLaunch(exec, st);
  cudaGraphExecDestroy(exec);           // (released once the launch has completed)
  MP_CUDA(e);
  h->phase = 2;
  return MP_OK;
}

extern "C" int mp_octree_run_fused_async(mp_octree_t* h, mp_mlp_t* mlp, mp_feat_t* feat, const float* calib12, int projection,
                                         float z_scale, int mode, float* out_dev, void* stream) {
  return run_fused_async(h, mlp, feat, calib12, nullptr, projection, z_scale, mode, out_dev, stream);
}

extern "C" int mp_octree_run_fused_async_dcal(mp_octree_t* h, mp_mlp_t* mlp, mp_feat_t* feat, const float* calib_dev,
                                              int projection, float z_scale, int mode, float* out_dev, void* stream) {
  MP_REQUIRE(calib_dev, "NULL calib_dev");
  return run_fused_async(h, mlp, feat, nullptr, calib_dev, projection, z_scale, mode, out_dev, stream);
}

// The read-back half: non-empty flag and per-level evaluated-node counts of the last (async) run.  Synchronises.
extern "C" int mp_octree_fetch(mp_octree_t* h, int* nonempty, int64_t* stats_host, void* stream) {
  MP_REQUIRE(h && nonempty, "NULL argument");
  cudaStream_t st = (cudaStream_t)stream;
  long long stats[kStatSlots];
  MP_CUDA(cudaMemcpyAsync(stats, h->stats, sizeof(stats), cudaMemcpyDeviceToHost, st));
  MP_CUDA(cudaStreamSynchronize(st));
  *nonempty = *reinterpret_cast<const int*>(stats + kStatSlots - 1);
  if (stats_host) for (int l = 0; l < h->n_levels; ++l) stats_host[l] = stats[l];
  return MP_OK;
}

// Conflict-loop passes per level of the last mp_octree_run_fused_async (0 for level 0 and for engines without the loop).
// Synchronises.  MP_E_TRUNCATED when a level stopped at its cap with nodes still to evaluate.
extern "C" int mp_octree_fetch_loops(mp_octree_t* h, int32_t* passes_per_level, void* stream) {
  MP_REQUIRE(h && passes_per_level, "NULL argument");
  for (int l = 0; l < h->n_levels; ++l) passes_per_level[l] = 0;
  if (!h->loops) return MP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t loops[kLoopSlots];
  MP_CUDA(cudaMemcpyAsync(loops, h->loops, sizeof(loops), cudaMemcpyDeviceToHost, st));
  MP_CUDA(cudaStreamSynchronize(st));
  for (int l = 0; l < h->n_levels; ++l) passes_per_level[l] = loops[l];
  const int t = loops[kLoopSlots - 1];
  if (t > 0) {
    mp_set_error("the conflict loop of level %d (resolution %d) stopped at its cap of %d passes with nodes left to evaluate",
                 t - 1, h->res[t - 1], kLoopPassesPerRes * h->res[t - 1]);
    return MP_E_TRUNCATED;
  }
  return MP_OK;
}

extern "C" int mp_octree_run_fused(mp_octree_t* h, mp_mlp_t* mlp, mp_feat_t* feat, const float* calib12, int projection,
                                   float z_scale, int mode, float* out_dev, int* nonempty, int64_t* stats_host,
                                   void* stream) {
  MP_REQUIRE(h && mlp && feat && out_dev && nonempty, "NULL argument");
  MP_REQUIRE_SINGLE_MAP(feat, "the occupancy engine");
  MP_REQUIRE(mlp->cout[mlp->n_layers - 1] == 1, "the occupancy engine needs a single-channel head");
  MpRange nvtx("monoport_b200: F2 coarse-to-fine engine");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = reset_run(h, st);
  if (rc != MP_OK) return rc;
  MpCalib cal;
  mp_fill_calib(cal, calib12, projection, z_scale);
  // The level buffers ping-pong (level l is written to buffer l & 1), so the caller's volume stands in for the buffer
  // the last level lands in: the result is produced in place instead of being copied out (68 MB at 257^3).
  const int final_buf = (h->n_levels - 1) & 1;
  float* const own_buf = h->vol[final_buf];
  h->vol[final_buf] = out_dev;
  rc = run_fused_levels(h, mlp, feat, cal, nullptr, mode, st);
  const bool in_place = h->cur == final_buf;
  const float* result = h->vol[h->cur];
  h->vol[final_buf] = own_buf;
  if (rc != MP_OK) return rc;
  if (!in_place) MP_CUDA(cudaMemcpyAsync(out_dev, result, h->vol_elems * sizeof(float), cudaMemcpyDeviceToDevice, st));
  long long stats[kStatSlots];
  int ne = 0;
  MP_CUDA(cudaMemcpyAsync(stats, h->stats, sizeof(stats), cudaMemcpyDeviceToHost, st));
  MP_CUDA(cudaStreamSynchronize(st));
  ne = *reinterpret_cast<const int*>(stats + kStatSlots - 1);
  *nonempty = ne;
  if (stats_host) for (int l = 0; l < h->n_levels; ++l) stats_host[l] = stats[l];
  h->phase = 2;
  return MP_OK;
}
