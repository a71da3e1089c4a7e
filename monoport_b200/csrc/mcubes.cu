// F3: marching cubes on the occupancy volume (absent from the reference -- SURVEY.md finding 3; PARITY UNPINNED,
// bit-exact against oracle/spec.py:marching_cubes_ref which uses the same derived table, tools/gen_mc_table.py).
// HBM-bound byte/integer work.  Indexed, watertight mesh with deterministic ids:
//   vertex id = rank of (node, axis) among active owned edges (every grid edge is owned by its lower node);
//   face order = (cell linear index, table order).
// count:  bits_kernel (THE read of the volume: 4 B per node in, one occupancy bit per node out, streaming) ->
//         ordered scan over the 32-node words of the bit volume, (verts, tris) packed in one uint64.  Its first pass
//         (classify_sums_kernel) CLASSIFIES each word on the way (edge masks + triangle count; words with no surface inside
//         leave after a dozen cached loads), its second pass leaves the exclusive prefix per word, the totals, and an
//         unordered list of the words with a surface inside.
// emit :  mesh_emit_kernel, a warp per listed word, a lane per node: vertices from the volume (two loads per vertex); the
//         cells' triangles go through a shared-memory queue and are resolved one thread per face corner (edge -> owning
//         node -> id = the owning word's prefix + popcounts).
// mp_mcubes_run_async: the same launches without the host (graph-capturable, replayable on one workspace): the emission grid
//         is fixed at record time and reads the active-list length on the device; caller buffers with capacities, the true
//         totals and the vertex count left on the device, optional world-space vertices.
// refine: mp_mesh_refine_async moves the vertices of the last run onto the network's own iso-surface along their edges
//         (DESIGN.md §F3.1): mesh_edges_kernel (vertex -> owning node + axis, the emission's walk), refine_init_kernel, then
//         per round the query program at the candidates and refine_step_kernel (refine_kernels.cuh).
// Workspace: 1 bit + 24 B per 32 nodes (15 MB at 257^3; the round-1 byte-per-node design took 102 MB).
#include "mp_common.cuh"
#include <stdlib.h>
#include "mcubes_kernels.cuh"
#include "refine_kernels.cuh"

using namespace mcubes;


struct mp_mcubes {
  int D, H, W;
  long long n, n_words;
  uint32_t* bits;
  WordInfo* info;
  unsigned long long* prefix;
  uint32_t* active;            // words with a surface inside (unordered), filled by the scan's emit half
  uint32_t* n_active_dev;
  uint32_t n_active;
  unsigned long long* sums;
  unsigned long long* total;
  long long nv, nf;
  int counted;
  int ran;                     // a count has been enqueued: the prefixes and the active list are defined
};

extern "C" int mp_mcubes_destroy(mp_mcubes_t* h) {
  if (!h) return MP_OK;
  if (h->bits) cudaFree(h->bits);
  if (h->info) cudaFree(h->info);
  if (h->prefix) cudaFree(h->prefix);
  if (h->active) cudaFree(h->active);
  if (h->sums) cudaFree(h->sums);
  if (h->total) cudaFree(h->total);
  delete h;
  return MP_OK;
}

extern "C" int mp_mcubes_create(int D, int H, int W, mp_mcubes_t** out) {
  MP_REQUIRE(out != nullptr, "out is NULL");
  *out = nullptr;
  MP_REQUIRE(D >= 2 && H >= 2 && W >= 2 && (long long)D * H * W < (1ll << 31), "bad volume shape %dx%dx%d", D, H, W);
  mp_mcubes* h = new mp_mcubes();
  memset(h, 0, sizeof(*h));
  h->D = D; h->H = H; h->W = W;
  h->n = (long long)D * H * W;
  h->n_words = (h->n + 31) >> 5;
  const size_t bit_words = (size_t)(h->n_words + bits_pad_words(H, W));
  cudaError_t e = cudaMalloc(&h->bits, bit_words * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMemset(h->bits, 0, bit_words * sizeof(uint32_t));     // the padding stays zero for ever
  if (e == cudaSuccess) e = cudaMalloc(&h->info, (size_t)h->n_words * sizeof(WordInfo));
  if (e == cudaSuccess) e = cudaMalloc(&h->prefix, (size_t)h->n_words * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMalloc(&h->active, (size_t)h->n_words * sizeof(uint32_t));
  // chunk totals of the scan + (last entry) the length of the active list: zeroed together before every count
  if (e == cudaSuccess) e = cudaMalloc(&h->sums, (size_t)(mpscan::num_blocks(h->n_words) + 2) * sizeof(unsigned long long));
  if (e == cudaSuccess) h->n_active_dev = reinterpret_cast<uint32_t*>(h->sums + mpscan::num_blocks(h->n_words) + 1);
  if (e == cudaSuccess) e = cudaMalloc(&h->total, 2 * sizeof(unsigned long long));                 // [0] total, [1] scan ticket
  if (e == cudaSuccess) e = cudaMemset(h->total, 0, 2 * sizeof(unsigned long long));
  if (e != cudaSuccess) {
    mp_set_error("mp_mcubes_create: %s", cudaGetErrorString(e));
    mp_mcubes_destroy(h);
    return MP_E_NOMEM;
  }
  *out = h;
  return MP_OK;
}

static int sm_count() {
  static const int sms = [] {
    int dev = 0, n = 148;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
  }();
  return sms;
}

// bits_kernel -> zeroed chunk sums (and n_active_dev) -> classify_sums_kernel -> the scan's emit half: the counts, the
// prefixes and the active list on the device.  Enqueue-only; every per-run word is reset inside the sequence (the chunk
// sums and n_active_dev by the memset, the scan ticket by the scan's last CTA), so a graph can replay it.
static int enqueue_count(mp_mcubes* h, const float* vol_dev, float iso, cudaStream_t st) {
  {
    // a multiple of the SM count, 8 CTAs of 256 threads resident per SM: 8 x 128 B loads in flight per warp
    const long long warps_needed = (h->n_words + kBitsUnroll - 1) / kBitsUnroll;
    const long long blocks_needed = (warps_needed + kBitsThreads / 32 - 1) / (kBitsThreads / 32);
    const long long cap = (long long)sm_count() * 8;
    bits_kernel<<<(unsigned)(blocks_needed < cap ? blocks_needed : cap), kBitsThreads, 0, st>>>(vol_dev, h->bits, h->n, iso);
  }
  MP_CUDA(cudaGetLastError());
  // the ordered scan over the words, first pass = classify_sums_kernel (classification + chunk totals), second pass = the
  // generic emit half reading the stored info
  const int nb = mpscan::num_blocks(h->n_words);
  MP_CUDA(cudaMemsetAsync(h->sums, 0, (size_t)(nb + 2) * sizeof(unsigned long long), st));
  const unsigned n_ctas = (unsigned)((h->n_words + kClassifyWords - 1) / kClassifyWords);
  classify_sums_kernel<<<n_ctas, kClassifyThreads, 0, st>>>(h->bits, h->info, h->n, h->D, h->H, h->W, h->sums, nb, h->total);
  WordCountF f2{h->info};
  PrefixEmit em{h->prefix, h->active, h->n_active_dev};
  mpscan::emit_kernel<WordCountF, PrefixEmit><<<nb, mpscan::kThreads, 0, st>>>(f2, em, h->n_words, h->sums);
  MP_CUDA(cudaGetLastError());
  h->ran = 1;
  return MP_OK;
}

extern "C" int mp_mcubes_count(mp_mcubes_t* h, const float* vol_dev, float iso, int64_t* n_verts, int64_t* n_faces,
                               void* stream) {
  MP_REQUIRE(h && vol_dev && n_verts && n_faces, "NULL argument");
  MpRange nvtx("monoport_b200: F3 marching cubes (count)");
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = enqueue_count(h, vol_dev, iso, st);
  if (rc != MP_OK) return rc;
  unsigned long long tot = 0;
  MP_CUDA(cudaMemcpyAsync(&tot, h->total, sizeof(tot), cudaMemcpyDeviceToHost, st));
  MP_CUDA(cudaMemcpyAsync(&h->n_active, h->n_active_dev, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  MP_CUDA(cudaStreamSynchronize(st));
  h->nv = (long long)(tot & 0xffffffffull);
  h->nf = (long long)(tot >> 32);
  h->counted = 1;
  *n_verts = h->nv;
  *n_faces = h->nf;
  return MP_OK;
}

extern "C" int mp_mcubes_emit(mp_mcubes_t* h, const float* vol_dev, float iso, float* verts_dev, int32_t* faces_dev,
                              void* stream) {
  MP_REQUIRE(h && vol_dev, "NULL argument");
  MP_REQUIRE(h->counted, "mp_mcubes_count must run first");
  if (h->nv == 0 && h->nf == 0) return MP_OK;
  MP_REQUIRE(verts_dev && faces_dev, "NULL output buffers");
  MpRange nvtx("monoport_b200: F3 marching cubes (emit)");
  cudaStream_t st = (cudaStream_t)stream;
  // one warp per word with a surface inside (the active list the count pass left behind)
  const long long blocks_needed = ((long long)h->n_active + kEmitThreads / 32 - 1) / (kEmitThreads / 32);
  if (blocks_needed > 0)
    mesh_emit_kernel<<<(unsigned)blocks_needed, kEmitThreads, 0, st>>>(vol_dev, h->bits, h->info, h->prefix, h->active, h->n_active,
                                                                     verts_dev, faces_dev, h->D, h->H, h->W, h->n, iso);
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

extern "C" int mp_mcubes_run_async(mp_mcubes_t* h, const float* vol_dev, float iso, const float* world, int64_t v_cap,
                                   int64_t f_cap, float* verts_dev, int32_t* faces_dev, int64_t* counts_dev,
                                   int32_t* count32_dev, void* stream) {
  MP_REQUIRE(h && vol_dev && counts_dev && count32_dev, "NULL argument");
  MP_REQUIRE(v_cap >= 0 && f_cap >= 0 && v_cap <= INT32_MAX && f_cap <= INT32_MAX, "bad capacities v_cap=%lld f_cap=%lld",
             (long long)v_cap, (long long)f_cap);
  MP_REQUIRE((verts_dev || v_cap == 0) && (faces_dev || f_cap == 0), "NULL output buffers");
  MeshOut out;
  memset(&out, 0, sizeof(out));
  out.verts = verts_dev;
  out.faces = faces_dev;
  out.v_cap = (uint32_t)v_cap;
  out.f_cap = (uint32_t)f_cap;
  if (world) {
    const float R = world[0];
    MP_REQUIRE(R >= 1.f, "bad world mapping: R=%g", (double)R);
    out.world = 1;
    for (int a = 0; a < 3; ++a) {
      out.scale[a] = (world[4 + a] - world[1 + a]) / R;          // torch's (b_max - b_min) / R in fp32
      out.bmin[a] = world[1 + a];
    }
  }
  MpRange nvtx("monoport_b200: F3 marching cubes (enqueue-only)");
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = enqueue_count(h, vol_dev, iso, st);
  if (rc != MP_OK) return rc;
  // a persistent grid fixed at record time: 4 CTAs per SM, and no more warps than the volume has words
  const long long blocks_needed = (h->n_words + kEmitWarps - 1) / kEmitWarps;
  const long long cap = (long long)sm_count() * 4;
  mesh_emit_async_kernel<<<(unsigned)(blocks_needed < cap ? blocks_needed : cap), kEmitThreads, 0, st>>>(
      vol_dev, h->bits, h->info, h->prefix, h->active, h->n_active_dev, h->total, out,
      reinterpret_cast<long long*>(counts_dev), count32_dev, h->D, h->H, h->W, h->n, iso);
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

// ---- mesh refinement (DESIGN.md §F3.1)
// scratch layout (mrefine::State), each array 256-byte aligned: 3 + 1 + 7 float rows, the node records, the flag bytes
static size_t refine_align(size_t b) { return (b + 255) & ~(size_t)255; }

extern "C" int64_t mp_mesh_refine_scratch_bytes(int64_t v_cap) {
  if (v_cap < 0 || v_cap > INT32_MAX) return -1;
  const size_t c = (size_t)v_cap;
  return (int64_t)(11 * refine_align(c * sizeof(float)) + refine_align(c * sizeof(uint32_t)) + refine_align(c));
}

static int mesh_refine_async(mp_mlp_t* mlp, mp_feat_t* feat, mp_mcubes_t* h, const float* vol_dev, float iso, const float* world,
                             float* verts_dev, const int32_t* count32_dev, int64_t v_cap, int rounds, const float* calib12,
                             const float* calib_dev, int projection, float z_scale, int mode, void* scratch_dev, void* stream,
                             const char* what) {
  MP_REQUIRE(mlp && feat && h && vol_dev && world && count32_dev, "%s: NULL argument", what);
  MP_REQUIRE(rounds >= 0, "%s: bad rounds %d", what, rounds);
  MP_REQUIRE(v_cap >= 0 && v_cap <= INT32_MAX, "%s: bad capacity v_cap=%lld", what, (long long)v_cap);
  MP_REQUIRE((verts_dev && scratch_dev) || v_cap == 0, "%s: NULL argument", what);
  MP_REQUIRE(mlp->cout[mlp->n_layers - 1] == 1, "mesh refinement needs a head with one output (got %d)", mlp->cout[mlp->n_layers - 1]);
  MP_REQUIRE_SINGLE_MAP(feat, what);
  const float R = world[0];
  MP_REQUIRE(h->D == h->H && h->H == h->W && R == (float)h->W,
             "%s: the world mapping's R=%g is not the side of the workspace's %dx%dx%d volume", what, (double)R, h->D, h->H, h->W);
  MP_REQUIRE(h->ran, "%s: the workspace has not run marching cubes", what);
  if (rounds == 0 || v_cap == 0) return MP_OK;
  MpRange nvtx("monoport_b200: F3.1 mesh refinement (enqueue-only)");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t c = (size_t)v_cap;
  char* base = static_cast<char*>(scratch_dev);
  float* rows[11];
  for (int k = 0; k < 11; ++k) rows[k] = reinterpret_cast<float*>(base + k * refine_align(c * sizeof(float)));
  mrefine::State s;
  s.pts = rows[0];                                    // rows 0..2: the query's point rows
  s.sigma = rows[3];
  s.ta = rows[4]; s.fa = rows[5]; s.tb = rows[6]; s.fb = rows[7];
  s.tbest = rows[8]; s.fbest = rows[9]; s.tcur = rows[10];
  s.node = reinterpret_cast<uint32_t*>(base + 11 * refine_align(c * sizeof(float)));
  s.flags = reinterpret_cast<uint8_t*>(base + 11 * refine_align(c * sizeof(float)) + refine_align(c * sizeof(uint32_t)));
  s.cap = (uint32_t)v_cap;
  mrefine::Geom g;
  g.H = h->H; g.W = h->W;
  g.iso = iso;
  for (int a = 0; a < 3; ++a) {
    g.scale[a] = (world[4 + a] - world[1 + a]) / R;          // mp_mcubes_run_async's mapping
    g.bmin[a] = world[1 + a];
  }
  {
    // the emission's persistent grid: 4 CTAs per SM, and no more warps than the volume has words
    const long long blocks_needed = (h->n_words + kEdgesThreads / 32 - 1) / (kEdgesThreads / 32);
    const long long cap = (long long)sm_count() * 4;
    mesh_edges_kernel<<<(unsigned)(blocks_needed < cap ? blocks_needed : cap), kEdgesThreads, 0, st>>>(
        h->info, h->prefix, h->active, h->n_active_dev, (uint32_t)v_cap, s.node, s.flags);
  }
  MP_CUDA(cudaGetLastError());
  const long long blocks = (v_cap + mrefine::kThreads - 1) / mrefine::kThreads;
  const long long cap = (long long)sm_count() * 8;
  const unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
  mrefine::refine_init_kernel<<<grid, mrefine::kThreads, 0, st>>>(vol_dev, count32_dev, s, g);
  MP_CUDA(cudaGetLastError());
  for (int r = 0; r < rounds; ++r) {
    // the query program at the candidates: rows [3][v_cap], the count and the range guard on the device
    const int rc = calib_dev ? mp_query_points_count_dcal(mlp, feat, s.pts, v_cap, v_cap, 1, calib_dev, projection, z_scale, s.sigma,
                                                          v_cap, count32_dev, mode, stream)
                             : mp_query_points_count(mlp, feat, s.pts, v_cap, v_cap, 1, calib12, projection, z_scale, s.sigma, v_cap,
                                                     count32_dev, mode, stream);
    if (rc != MP_OK) return rc;
    mrefine::refine_step_kernel<<<grid, mrefine::kThreads, 0, st>>>(count32_dev, s, g, r == rounds - 1, verts_dev);
    MP_CUDA(cudaGetLastError());
  }
  return MP_OK;
}

extern "C" int mp_mesh_refine_async(mp_mlp_t* mlp, mp_feat_t* feat, mp_mcubes_t* ws, const float* vol_dev, float iso,
                                    const float* world, float* verts_dev, const int32_t* count32_dev, int64_t v_cap, int rounds,
                                    const float* calib12, int projection, float z_scale, int mode, void* scratch_dev, void* stream) {
  return mesh_refine_async(mlp, feat, ws, vol_dev, iso, world, verts_dev, count32_dev, v_cap, rounds, calib12, nullptr, projection,
                           z_scale, mode, scratch_dev, stream, "mp_mesh_refine_async");
}

extern "C" int mp_mesh_refine_async_dcal(mp_mlp_t* mlp, mp_feat_t* feat, mp_mcubes_t* ws, const float* vol_dev, float iso,
                                         const float* world, float* verts_dev, const int32_t* count32_dev, int64_t v_cap,
                                         int rounds, const float* calib_dev, int projection, float z_scale, int mode,
                                         void* scratch_dev, void* stream) {
  MP_REQUIRE(calib_dev, "NULL calib_dev");
  return mesh_refine_async(mlp, feat, ws, vol_dev, iso, world, verts_dev, count32_dev, v_cap, rounds, nullptr, calib_dev, projection,
                           z_scale, mode, scratch_dev, stream, "mp_mesh_refine_async_dcal");
}
