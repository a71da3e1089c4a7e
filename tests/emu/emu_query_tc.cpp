// TEST INFRASTRUCTURE ONLY: monoport_b200/csrc/query_tc.cu -- host-side weight packing, launch logic, the per-frame G0
// GEMM kernel and the fused wgmma sample+MLP kernel -- compiled UNMODIFIED for the CPU against the execution-model
// emulation (cuda_emu.h) and the functional model of the wgmma / mbarrier / bulk-copy layer (tc_ptx_emu.h).
//   emu_query_tc in.bin out.f32 program sms [grid R z0 nz | nodes R res | surface R | batch B]
// in.bin: int32 header {C, H, W, N, has_calib, perspective, res, last_op}, float z_scale, calib[12], then fp32 arrays:
//   feature map NCHW [C*H*W], points [3*N], for each of the 5 layers W_l [cout*cin] and b_l [cout].
// batch B: the batched launch (what mp_query_points_batch sets up: one launch over B images, the per-frame G0 kernel on a
//   texel-blocks x B grid, the range guard decided per tile).  in.bin then holds B feature maps [B*C*H*W] and B point sets
//   [B*3*N], and when has_calib B calibs [B*12] (rows 0..2 of [R|t]) after them instead of the header's calib;
//   out.f32 is [B][res][N], pre-filled with -4242 (the tiles a guarded launch skips keep it).
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdarg.h>

#define MP_EMU_CUDA_TYPES 1
#include <math.h>
#include "cuda_emu.h"

// ---- device intrinsics the real headers only provide to nvcc -----------------------------------------------------------
static inline __half2 __hfma2(__half2 a, __half2 b, __half2 c) {
  _Float16 av[2], bv[2], cv[2], rv[2];
  memcpy(av, &a, 4); memcpy(bv, &b, 4); memcpy(cv, &c, 4);
  for (int i = 0; i < 2; ++i) rv[i] = (_Float16)((double)av[i] * (double)bv[i] + (double)cv[i]);   // one rounding
  __half2 r;
  memcpy(&r, rv, 4);
  return r;
}
static inline float2 __fmul2_rn(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
static inline float2 __ffma2_rn(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

// ---- the dynamic shared memory of the kernels: one buffer per CTA of a (2-CTA) cluster; CTAs / clusters run one at a time ---
alignas(1024) static uint8_t g_dyn_smem[2][240 * 1024];
void* mp_emu_dyn_smem() { return g_dyn_smem[cuda_emu::t_rank]; }

// ---- a host-memory stand-in for the few CUDA runtime calls of the launcher ----------------------------------------------
static int g_fake_sms = 132;
extern "C" {
cudaError_t cudaMalloc(void** p, size_t n) { *p = aligned_alloc(256, (n + 255) / 256 * 256); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) {
  if (a == cudaDevAttrComputeCapabilityMajor) *v = 9;
  else if (a == cudaDevAttrMaxSharedMemoryPerBlockOptin) *v = 232448;
  else if (a == cudaDevAttrMultiProcessorCount) *v = g_fake_sms;
  else *v = 0;
  return cudaSuccess;
}
cudaError_t cudaFuncSetAttribute(const void*, cudaFuncAttribute, int) { return cudaSuccess; }
cudaError_t cudaGetLastError(void) { return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
}

#define MP_EMU_LAUNCH(grid, block, call) cuda_emu::launch(dim3((unsigned)(grid)), dim3((unsigned)(block)), [&] { call; })
#define MP_EMU_LAUNCH_CLUSTER2(grid, block, call) cuda_emu::launch(dim3((unsigned)(grid)), dim3((unsigned)(block)), [&] { call; }, 2)

static char g_err[512];
void mp_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
template <class T> static cudaError_t cudaFuncSetAttribute(T*, cudaFuncAttribute, int) { return cudaSuccess; }

#include "../../monoport_b200/csrc/query_tc.cu"

int mp_launch_query_fp32(const mp_mlp*, const mp_feat*, const MpPointSrc&, const MpCalib&, const MpOutDst&, cudaStream_t, int,
                         const MpBatch*) { return MP_E_UNSUPPORTED; }

// mp_api.cu's helper (that file holds <<<>>> launches and is not part of this build)
static void fill_grid_geom(MpPointSrc& s, int res, int node_stride, int r_final) {
  s.res = res;
  s.node_stride = node_stride;
  s.r_final = r_final;
  s.inv_r = 1.0f / (float)r_final;
  s.half_inv_r = (float)(1.0 / (2.0 * (double)r_final));
  for (int a = 0; a < 3; ++a) { s.bmin[a] = -1.f; s.bext[a] = 1.f - (-1.f); }
}

int main(int argc, char** argv) {
  // optional point source (default: the rows of in.bin):  grid R z0 nz   |   nodes R res   |   surface R
  //   grid : node centres of planes [z0, z0+nz) of an R^3 grid over [-1,1]^3, generated in-kernel (mp_query_grid)
  //   nodes: every third node of the res^3 level of an R^3 pyramid, through an index list + a device-side count that
  //          is smaller than the list capacity, scattered into a res^3 volume (the octree engine's fused path)
  const char* src_kind = argc >= 6 ? argv[5] : "rows";
  if (argc < 5) { fprintf(stderr, "usage: emu_query_tc in.bin out.f32 program sms [grid R z0 nz | nodes R res | surface R | batch B]\n"); return 2; }
  const bool batched = !strcmp(src_kind, "batch");
  const int B = batched ? atoi(argv[6]) : 1;
  const int program = atoi(argv[3]);
  g_fake_sms = atoi(argv[4]);
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  int32_t hd[8];
  float zs, calib[12];
  if (fread(hd, 4, 8, f) != 8 || fread(&zs, 4, 1, f) != 1 || fread(calib, 4, 12, f) != 12) { fprintf(stderr, "short header\n"); return 2; }
  const int C = hd[0], H = hd[1], W = hd[2], N = hd[3], has_calib = hd[4], persp = hd[5], res = hd[6], last_op = hd[7];
  auto rd = [&](size_t n) { std::vector<float> v(n); if (fread(v.data(), 4, n, f) != n) { fprintf(stderr, "short file\n"); exit(2); } return v; };
  const size_t per_map = (size_t)C * H * W;
  std::vector<float> nchw = rd(B * per_map), pts = rd((size_t)B * 3 * N);
  std::vector<float> calibs = batched && has_calib ? rd((size_t)B * 12) : std::vector<float>();
  const int chans[6] = {C + 1, 1024, 512, 256, 128, res};
  mp_mlp mlp;
  memset(&mlp, 0, sizeof(mlp));
  mlp.n_layers = 5; mlp.skip = 1; mlp.last_op = last_op;
  mlp.gen = 1;
  mlp.tc_amax_limit = getenv("EMU_TC_LIMIT") ? (float)atof(getenv("EMU_TC_LIMIT")) : INFINITY;      // range guard (see mp_query_dispatch)
  const int guard = getenv("EMU_TC_GUARD") ? atoi(getenv("EMU_TC_GUARD")) : MP_GUARD_NONE;
  std::vector<std::vector<float>> Ws(5), Bs(5);
  for (int l = 0; l <= 5; ++l) mlp.channels[l] = chans[l];
  for (int l = 0; l < 5; ++l) {
    mlp.cin[l] = chans[l] + (l ? chans[0] : 0);
    mlp.cout[l] = chans[l + 1];
    Ws[l] = rd((size_t)mlp.cin[l] * mlp.cout[l]);
    Bs[l] = rd(mlp.cout[l]);
    mlp.w[l] = Ws[l].data();
    mlp.bias[l] = Bs[l].data();
  }
  fclose(f);
  tc::emu::set_smem(g_dyn_smem[0], sizeof(g_dyn_smem[0]), g_dyn_smem[1]);
  if (mp_tc_prepare(&mlp) != MP_OK || !mlp.tc_ok) { fprintf(stderr, "mp_tc_prepare: %s (tc_ok=%d)\n", g_err, mlp.tc_ok); return 3; }
  if (getenv("EMU_TC_DEBUG")) {
    const TcPack* pk = static_cast<const TcPack*>(mlp.tc);
    fprintf(stderr, "d_bias0[0..3] = %g %g %g %g   d_wz0[0..1] = %g %g  h_bias[0]=%g\n", __half2float(pk->d_bias0[0]), __half2float(pk->d_bias0[1]),
            __half2float(pk->d_bias0[2]), __half2float(pk->d_bias0[3]), __half2float(pk->d_wz0[0]), __half2float(pk->d_wz0[1]), pk->h_bias[0]);
  }
  // feature handle: B channel-last maps, one after the other (what nchw_to_nhwc_kernel produces), one amax word per map
  std::vector<float> nhwc(B * per_map);
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < C; ++c)
      for (int p = 0; p < H * W; ++p) nhwc[b * per_map + (size_t)p * C + c] = nchw[b * per_map + (size_t)c * H * W + p];
  mp_feat feat;
  memset(&feat, 0, sizeof(feat));
  feat.B = B; feat.C = C; feat.H = H; feat.W = W; feat.nhwc32 = nhwc.data(); feat.version = 1;
  std::vector<unsigned> amax(B, 0u);
  feat.amax = amax.data();
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_ROWS;
  src.px = pts.data(); src.py = pts.data() + N; src.pz = pts.data() + 2 * (size_t)N;
  src.pstride = 1;
  src.n = N;
  MpCalib cal;
  memset(&cal, 0, sizeof(cal));
  cal.has = has_calib;
  memcpy(cal.m, calib, sizeof(calib));
  cal.perspective = persp && has_calib;
  cal.z_scale = zs;
  long long n_out = N;
  std::vector<int32_t> nodes;
  int32_t node_count = 0;
  std::vector<float> scatter;
  if (!strcmp(src_kind, "grid")) {
    const int R = atoi(argv[6]), z0 = atoi(argv[7]), nz = atoi(argv[8]);
    memset(&src, 0, sizeof(src));
    src.kind = MP_SRC_GRID;
    fill_grid_geom(src, R, 1, R);
    src.z0 = z0;
    src.lin0 = (long long)z0 * R * R;      // (what mp_api.cu's query_grid_range sets up)
    src.n = (long long)nz * R * R;
    n_out = src.n;
  } else if (!strcmp(src_kind, "nodes")) {
    const int R = atoi(argv[6]), lres = atoi(argv[7]);
    for (int i = 0; i < lres * lres * lres; i += 3) nodes.push_back(i);
    node_count = (int32_t)nodes.size();
    nodes.resize(nodes.size() + 300, 0);            // capacity beyond the count: must not be evaluated
    memset(&src, 0, sizeof(src));
    src.kind = MP_SRC_NODES;
    fill_grid_geom(src, lres, (R - 1) / (lres - 1), R);
    src.nodes = nodes.data();
    src.count_dev = &node_count;
    src.n = (long long)nodes.size();
    n_out = (long long)lres * lres * lres;
    scatter.assign(n_out, -4242.f);
  }
  if (!strcmp(src_kind, "surface")) {
    // surface R: the first N "points" of in.bin are visible-surface vertices (x, y integers; z float, index space);
    // the colour head renders them into an [R,R,3] canvas of ones (mp_colorize_surface)
    const int R = atoi(argv[6]);
    std::vector<long long> X(N), Y(N);
    std::vector<float> Z(N);
    for (int i = 0; i < N; ++i) { X[i] = (long long)pts[i]; Y[i] = (long long)pts[(size_t)N + i]; Z[i] = pts[2 * (size_t)N + i]; }
    std::vector<float> canvas((size_t)R * R * 3 + 1, 1.0f);
    canvas[(size_t)R * R * 3] = -4242.f;
    const float bmin[3] = {-1.f, -1.f, -1.f}, bmax[3] = {1.f, 1.f, 1.f};
    const int rc = mp_launch_colour_surface(&mlp, &feat, X.data(), Y.data(), Z.data(), N, R, bmin, bmax, cal, canvas.data(), nullptr);
    if (rc != MP_OK) { fprintf(stderr, "mp_launch_colour_surface: %s\n", g_err); return 3; }
    if (canvas[(size_t)R * R * 3] != -4242.f) { fprintf(stderr, "wrote past the canvas\n"); return 3; }
    f = fopen(argv[2], "wb");
    fwrite(canvas.data(), 4, (size_t)R * R * 3, f);
    fclose(f);
    mp_tc_release(&mlp);
    return 0;
  }
  MpBatch bt;                     // (batched: the [R|t] rows come from the device calibs)
  bt.B = B;
  bt.pt_stride = 3ll * N;
  bt.out_stride = (long long)res * N;
  bt.calibs = has_calib ? calibs.data() : nullptr;
  std::vector<float> out((size_t)B * res * n_out + 1, -4242.f);
  MpOutDst dst;
  dst.out = out.data(); dst.ld = n_out; dst.scatter_vol = nullptr;
  if (!scatter.empty()) { dst.out = nullptr; dst.ld = 0; dst.scatter_vol = scatter.data(); }
  // program 1xx: tensor-core program xx with the fused slab exchange -- three "peer volumes" (host buffers here)
  const int n_peers = program >= 100 ? 3 : 0, peer_off = 5;
  std::vector<std::vector<float>> peer(n_peers, std::vector<float>((size_t)n_out + 2 * peer_off, -4242.f));
  for (int p = 0; p < n_peers; ++p) dst.peer[p] = peer[p].data();
  dst.n_peers = n_peers;
  dst.peer_off = peer_off;
  if (program % 100 != 3 && program % 100 != 0) { fprintf(stderr, "unknown program %d (3 = the tensor-core program, 103 = with peer stores)\n", program); return 2; }
  // EMU_SHARD_WORLD=W: the query is evaluated as W launches, launch r taking the r-th window of the point list (what W
  // GPUs do with list sharding; here they share the output buffers, so together they must reproduce the unsharded result)
  const int shard_world = getenv("EMU_SHARD_WORLD") ? atoi(getenv("EMU_SHARD_WORLD")) : 1;
  int rc = MP_OK;
  for (int r = 0; r < shard_world && rc == MP_OK; ++r) {
    src.shard_rank = r;
    src.shard_world = shard_world;
    rc = mp_launch_query_tc(&mlp, &feat, src, cal, dst, nullptr, guard, batched ? &bt : nullptr);
  }
  if (getenv("EMU_TC_AMAX"))
    for (int b = 0; b < B; ++b) { float a; memcpy(&a, &amax[b], 4); fprintf(stderr, "amax[%d] %.9g\n", b, a); }
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_tc: %s\n", g_err); return 3; }
  if (out[(size_t)B * res * n_out] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  if (!scatter.empty()) out.assign(scatter.begin(), scatter.end());       // report the scattered volume
  for (int p = 0; p < n_peers; ++p)
    for (long long i = 0; i < (long long)peer[p].size(); ++i) {
      float want = -4242.f;
      if (scatter.empty()) { if (i >= peer_off && i < peer_off + n_out) want = out[i - peer_off]; }
      else if (i >= peer_off && i < peer_off + node_count) want = scatter[nodes[i - peer_off]];     // peers receive the value LIST
      if (memcmp(&peer[p][i], &want, 4) != 0) { fprintf(stderr, "peer volume %d differs at %lld\n", p, i); return 3; }
    }
  f = fopen(argv[2], "wb");
  fwrite(out.data(), 4, (size_t)B * res * n_out, f);
  fclose(f);
  if (const char* dump = getenv("EMU_TC_DUMP")) {       // per-texel products of the G0 kernel, for debugging the model
    if (feat.g0) {
      f = fopen(dump, "wb");
      fwrite(feat.g0, 2, (size_t)H * W * 1024, f);
      fwrite(feat.f16, 2, (size_t)H * W * C, f);
      fwrite(feat.s4tex, 4, (size_t)H * W, f);
      fclose(f);
    }
  }
  mp_tc_release(&mlp);
  return 0;
}
