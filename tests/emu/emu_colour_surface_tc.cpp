// TEST INFRASTRUCTURE ONLY: the surface render of monoport_b200/csrc/query_tc.cu (the colour head's tensor-core program
// writing the visible-surface colours into a canvas) compiled UNMODIFIED for the CPU against the execution-model emulation
// (cuda_emu.h) and the functional model of the wgmma / mbarrier / bulk-copy layer (tc_ptx_emu.h).
//   emu_colour_surface_tc in.bin out.f32 sms R count bx0 by0 bz0 bx1 by1 bz1 [host]      (the box [b_min, b_max])
// in.bin as for emu_query_tc (header, z_scale, calib[12], feature map NCHW, "points" [3*N], the 5 layers); the N points are
// the capacity of the vertex buffers: rows X, Y (integers) and Z (index space).
//   default: mp_launch_surface_tc with the vertex count on the device (`count`, an int64 that may exceed N) and the range
//            guard of EMU_TC_GUARD (limit EMU_TC_LIMIT, default +inf) -- what mp_colorize_surface_async enqueues;
//   host   : mp_launch_colour_surface with `count` vertices counted on the host -- what mp_colorize_surface runs.
// out.f32: the [R,R,3] canvas, background EMU_CANVAS_BG (default 1).
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdarg.h>

#define MP_EMU_CUDA_TYPES 1
#include <math.h>
#include "cuda_emu.h"

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

alignas(1024) static uint8_t g_dyn_smem[2][240 * 1024];
void* mp_emu_dyn_smem() { return g_dyn_smem[cuda_emu::t_rank]; }

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

int main(int argc, char** argv) {
  if (argc < 12) { fprintf(stderr, "usage: emu_colour_surface_tc in.bin out.f32 sms R count bx0 by0 bz0 bx1 by1 bz1 [host]\n"); return 2; }
  g_fake_sms = atoi(argv[3]);
  const int R = atoi(argv[4]);
  const long long count = atoll(argv[5]);
  float bmin[3], bmax[3];
  for (int a = 0; a < 3; ++a) { bmin[a] = strtof(argv[6 + a], nullptr); bmax[a] = strtof(argv[9 + a], nullptr); }
  const bool host = argc >= 13 && !strcmp(argv[12], "host");
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  int32_t hd[8];
  float zs, calib[12];
  if (fread(hd, 4, 8, f) != 8 || fread(&zs, 4, 1, f) != 1 || fread(calib, 4, 12, f) != 12) { fprintf(stderr, "short header\n"); return 2; }
  const int C = hd[0], H = hd[1], W = hd[2], N = hd[3], has_calib = hd[4], persp = hd[5], res = hd[6], last_op = hd[7];
  auto rd = [&](size_t n) { std::vector<float> v(n); if (fread(v.data(), 4, n, f) != n) { fprintf(stderr, "short file\n"); exit(2); } return v; };
  std::vector<float> nchw = rd((size_t)C * H * W), pts = rd((size_t)3 * N);
  const int chans[6] = {C + 1, 1024, 512, 256, 128, res};
  mp_mlp mlp;
  memset(&mlp, 0, sizeof(mlp));
  mlp.n_layers = 5; mlp.skip = 1; mlp.last_op = last_op;
  mlp.gen = 1;
  mlp.tc_amax_limit = getenv("EMU_TC_LIMIT") ? (float)atof(getenv("EMU_TC_LIMIT")) : INFINITY;
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
  std::vector<float> nhwc((size_t)C * H * W);
  for (int c = 0; c < C; ++c)
    for (int p = 0; p < H * W; ++p) nhwc[(size_t)p * C + c] = nchw[(size_t)c * H * W + p];
  mp_feat feat;
  memset(&feat, 0, sizeof(feat));
  feat.B = 1; feat.C = C; feat.H = H; feat.W = W; feat.nhwc32 = nhwc.data(); feat.version = 1;
  unsigned amax = 0u;
  feat.amax = &amax;
  MpCalib cal;
  memset(&cal, 0, sizeof(cal));
  cal.has = has_calib;
  memcpy(cal.m, calib, sizeof(calib));
  cal.perspective = persp && has_calib;
  cal.z_scale = zs;
  std::vector<long long> X(N), Y(N);
  std::vector<float> Z(N);
  for (int i = 0; i < N; ++i) { X[i] = (long long)pts[i]; Y[i] = (long long)pts[(size_t)N + i]; Z[i] = pts[2 * (size_t)N + i]; }
  const float bg = getenv("EMU_CANVAS_BG") ? (float)atof(getenv("EMU_CANVAS_BG")) : 1.0f;
  std::vector<float> canvas((size_t)R * R * 3 + 1, bg);
  canvas[(size_t)R * R * 3] = -4242.f;
  int rc;
  if (host) {
    rc = mp_launch_colour_surface(&mlp, &feat, X.data(), Y.data(), Z.data(), count, R, bmin, bmax, cal, canvas.data(), nullptr);
  } else {
    const MpSurfaceSrc surf = mp_surface_src(X.data(), Y.data(), Z.data(), &count, R, bmin, bmax, canvas.data());
    rc = mp_launch_surface_tc(&mlp, &feat, surf, N, cal, nullptr, guard);
  }
  if (rc != MP_OK) { fprintf(stderr, "surface render: %s (%d)\n", g_err, rc); return 3; }
  if (canvas[(size_t)R * R * 3] != -4242.f) { fprintf(stderr, "wrote past the canvas\n"); return 3; }
  float a;
  memcpy(&a, &amax, 4);
  printf("%.9g\n", a);                                   // the frame's max |feature| (the range guard's input)
  f = fopen(argv[2], "wb");
  fwrite(canvas.data(), 4, (size_t)R * R * 3, f);
  fclose(f);
  mp_tc_release(&mlp);
  return 0;
}
