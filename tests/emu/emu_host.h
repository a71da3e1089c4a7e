// TEST INFRASTRUCTURE ONLY: the host side of the query harnesses (emu_query_*, emu_heads_fp32, emu_colour_surface_*,
// emu_dcal_*), which compile monoport_b200/csrc/query_fp32.cu or query_tc.cu UNMODIFIED for the CPU against the
// execution-model emulation (cuda_emu.h) and, for query_tc.cu, the functional model of the wgmma / mbarrier / bulk-copy
// layer (tc_ptx_emu.h).  Include it first, then the kernel file.  It holds a host-memory stand-in for the CUDA runtime
// calls of the launchers, the models of the device intrinsics the real headers only give to nvcc, and the in.bin reader.
//
// in.bin: int32 header {C, H, W, N, has_calib, perspective, res, last_op}, float z_scale, calib[12] (rows 0..2 of [R|t]),
// then fp32 arrays: the feature maps NCHW [B*C*H*W], the points [B*3*N] (rows x, y, z of each image), when batched and
// has_calib the B calibs [B*12] (instead of the header's), and per layer W_l [cout*cin] and b_l [cout].  B is 1 unless
// the harness runs a batched launch.
#pragma once
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

// ---- a host-memory stand-in for the few CUDA runtime calls of the launchers ---------------------------------------------
static int g_fake_sms = 3;        // the simulated SM count (the launchers' grid sizes)
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
template <class T> static cudaError_t cudaFuncSetAttribute(T*, cudaFuncAttribute, int) { return cudaSuccess; }

#ifndef MP_EMU_LAUNCH
#define MP_EMU_LAUNCH(grid, block, call) cuda_emu::launch(dim3((unsigned)(grid)), dim3((unsigned)(block)), [&] { call; })
#endif
#ifndef MP_EMU_LAUNCH_CLUSTER2
#define MP_EMU_LAUNCH_CLUSTER2(grid, block, call) cuda_emu::launch(dim3((unsigned)(grid)), dim3((unsigned)(block)), [&] { call; }, 2)
#endif

static char g_err[512];
void mp_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

#include "../../monoport_b200/csrc/mp_common.cuh"

// ---- in.bin ---------------------------------------------------------------------------------------------------------------
struct EmuInput {
  int C, H, W, N, res, last_op;
  MpCalib cal;                    // the header's camera (mp_fill_calib)
  std::vector<float> nchw;        // [B][C][H][W]
  std::vector<float> pts;         // [B][3][N]
  std::vector<float> calibs;      // [B][12] (a batched input with has_calib), else empty
  FILE* f;                        // positioned at the head's weights
};

static std::vector<float> emu_read(FILE* f, size_t n) {
  std::vector<float> v(n);
  if (fread(v.data(), 4, n, f) != n) { fprintf(stderr, "short file\n"); exit(2); }
  return v;
}

// in.bin up to the head (emu_make_mlp reads that, then closes the file); a batched input holds B maps, point sets and calibs
static EmuInput emu_read_input(const char* path, int B = 1, bool batched = false) {
  EmuInput in;
  in.f = fopen(path, "rb");
  if (!in.f) { perror(path); exit(2); }
  int32_t hd[8];
  float zs, calib[12];
  if (fread(hd, 4, 8, in.f) != 8 || fread(&zs, 4, 1, in.f) != 1 || fread(calib, 4, 12, in.f) != 12) {
    fprintf(stderr, "short header\n");
    exit(2);
  }
  in.C = hd[0]; in.H = hd[1]; in.W = hd[2]; in.N = hd[3]; in.res = hd[6]; in.last_op = hd[7];
  const int has_calib = hd[4];
  mp_fill_calib(in.cal, has_calib ? calib : nullptr, hd[5] ? MP_PROJ_PERSPECTIVE : MP_PROJ_ORTHOGONAL, zs);
  in.nchw = emu_read(in.f, (size_t)B * in.C * in.H * in.W);
  in.pts = emu_read(in.f, (size_t)B * 3 * in.N);
  if (batched && has_calib) in.calibs = emu_read(in.f, (size_t)B * 12);
  return in;
}

// ---- the handles, as the library's create / upload calls leave them ------------------------------------------------------
struct EmuMlp {
  mp_mlp mlp;
  std::vector<std::vector<float>> w, wt, b;
};

// mp_mlp_create's layout for the widths after the first (channels[0] = C + 1) with the head's weights from in.bin: W [cout][cin]
// and the [cin][cout] copy transpose_w_kernel makes.  The feature limit of the range guard is EMU_TC_LIMIT (default +inf).
static EmuMlp emu_make_mlp(EmuInput& in, const std::vector<int>& widths, bool skip = true) {
  EmuMlp m;
  memset(&m.mlp, 0, sizeof(m.mlp));
  const int L = (int)widths.size();
  m.mlp.n_layers = L; m.mlp.skip = skip; m.mlp.last_op = in.last_op;
  m.mlp.gen = 1;
  m.mlp.tc_amax_limit = getenv("EMU_TC_LIMIT") ? (float)atof(getenv("EMU_TC_LIMIT")) : INFINITY;
  m.mlp.channels[0] = in.C + 1;
  for (int l = 0; l < L; ++l) m.mlp.channels[l + 1] = widths[l];
  m.w.resize(L); m.wt.resize(L); m.b.resize(L);
  for (int l = 0; l < L; ++l) {
    const int cin = m.mlp.channels[l] + (l && skip ? m.mlp.channels[0] : 0), cout = m.mlp.channels[l + 1];
    m.mlp.cin[l] = cin; m.mlp.cout[l] = cout;
    m.w[l] = emu_read(in.f, (size_t)cin * cout);
    m.b[l] = emu_read(in.f, cout);
    m.wt[l].resize((size_t)cin * cout);
    for (int o = 0; o < cout; ++o)
      for (int k = 0; k < cin; ++k) m.wt[l][(size_t)k * cout + o] = m.w[l][(size_t)o * cin + k];
    m.mlp.w[l] = m.w[l].data(); m.mlp.wt[l] = m.wt[l].data(); m.mlp.bias[l] = m.b[l].data();
  }
  fclose(in.f);
  in.f = nullptr;
  return m;
}

// the shipped widths: 1024, 512, 256, 128, res
static EmuMlp emu_make_mlp(EmuInput& in) { return emu_make_mlp(in, {1024, 512, 256, 128, in.res}); }

struct EmuFeat {
  mp_feat feat;
  std::vector<float> nhwc;
  std::vector<unsigned> amax;
};

// mp_feat_upload's result: B channel-last maps one after the other (what nchw_to_nhwc_kernel produces), one amax word per map
static EmuFeat emu_make_feat(const EmuInput& in, int B = 1) {
  EmuFeat e;
  const size_t per_map = (size_t)in.C * in.H * in.W, HW = (size_t)in.H * in.W;
  e.nhwc.resize(B * per_map);
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < in.C; ++c)
      for (size_t p = 0; p < HW; ++p) e.nhwc[b * per_map + p * in.C + c] = in.nchw[b * per_map + (size_t)c * HW + p];
  e.amax.assign(B, 0u);
  memset(&e.feat, 0, sizeof(e.feat));
  e.feat.B = B; e.feat.C = in.C; e.feat.H = in.H; e.feat.W = in.W;
  e.feat.nhwc32 = e.nhwc.data();
  e.feat.amax = e.amax.data();
  e.feat.version = 1;
  return e;
}

// ---- point sources ---------------------------------------------------------------------------------------------------------
// the N points of in.bin (image 0's; a batched launch steps by MpBatch::pt_stride)
static MpPointSrc emu_rows_src(const EmuInput& in) {
  MpPointSrc s;
  memset(&s, 0, sizeof(s));
  s.kind = MP_SRC_ROWS;
  s.px = in.pts.data(); s.py = in.pts.data() + in.N; s.pz = in.pts.data() + 2 * (size_t)in.N;
  s.pstride = 1;
  s.n = in.N;
  return s;
}

static const float kUnitMin[3] = {-1.f, -1.f, -1.f}, kUnitMax[3] = {1.f, 1.f, 1.f};

// node centres of planes [z0, z0+nz) of an R^3 grid over [-1,1]^3, generated in-kernel (what mp_api.cu's query_grid_range sets up)
static MpPointSrc emu_grid_src(int R, int z0, int nz) {
  MpPointSrc s;
  memset(&s, 0, sizeof(s));
  s.kind = MP_SRC_GRID;
  mp_fill_grid_geom(s, R, 1, R, kUnitMin, kUnitMax);
  s.z0 = z0;
  s.lin0 = (long long)z0 * R * R;
  s.n = (long long)nz * R * R;
  return s;
}

// every third node of the lres^3 level of an R^3 pyramid over [-1,1]^3, through an index list whose capacity exceeds the
// device-side count by 300 entries that must not be evaluated (the octree engine's fused path)
static MpPointSrc emu_node_src(int R, int lres, std::vector<int32_t>& nodes, int32_t& count) {
  nodes.clear();
  for (int i = 0; i < lres * lres * lres; i += 3) nodes.push_back(i);
  count = (int32_t)nodes.size();
  nodes.resize(nodes.size() + 300, 0);
  MpPointSrc s;
  memset(&s, 0, sizeof(s));
  s.kind = MP_SRC_NODES;
  mp_fill_grid_geom(s, lres, (R - 1) / (lres - 1), R, kUnitMin, kUnitMax);
  s.nodes = nodes.data();
  s.count_dev = &count;
  s.n = (long long)nodes.size();
  return s;
}

// the N "points" of in.bin read as visible-surface vertices: X, Y integers and Z a float, in index space
struct EmuVerts {
  std::vector<long long> X, Y;
  std::vector<float> Z;
};

static EmuVerts emu_vertex_rows(const EmuInput& in) {
  const int N = in.N;
  EmuVerts v{std::vector<long long>(N), std::vector<long long>(N), std::vector<float>(N)};
  for (int i = 0; i < N; ++i) {
    v.X[i] = (long long)in.pts[i]; v.Y[i] = (long long)in.pts[(size_t)N + i]; v.Z[i] = in.pts[2 * (size_t)N + i];
  }
  return v;
}

// the box [bx0 by0 bz0] .. [bx1 by1 bz1] of six command-line arguments
static void emu_box_args(char** argv, float* bmin, float* bmax) {
  for (int a = 0; a < 3; ++a) { bmin[a] = strtof(argv[a], nullptr); bmax[a] = strtof(argv[3 + a], nullptr); }
}

static void emu_write(const char* path, const float* data, size_t n) {
  FILE* f = fopen(path, "wb");
  fwrite(data, 4, n, f);
  fclose(f);
}
