// TEST INFRASTRUCTURE ONLY: the batched launch of monoport_b200/csrc/query_tc.cu (what mp_query_points_batch sets up: one
// launch over B images, the per-frame G0 kernel on a texel-blocks x B grid, the range guard decided per tile) compiled
// UNMODIFIED for the CPU against cuda_emu.h and tc_ptx_emu.h, like emu_query_tc.cpp does for the single-image launches.
//   emu_query_tc_batch in.bin out.f32 program sms B
// in.bin: int32 header {C, H, W, N, has_calib, perspective, res, last_op}, float z_scale, calib[12] (ignored), then fp32
//   arrays: B feature maps NCHW [B*C*H*W], B point sets [B*3*N], when has_calib B calibs [B*12] (rows 0..2 of [R|t]),
//   for each of the 5 layers W_l [cout*cin] and b_l [cout].  out.f32: [B][res][N], pre-filled with -4242 (the tiles a
//   guarded launch skips keep it).  EMU_TC_LIMIT / EMU_TC_GUARD / EMU_TC_ORDER as for emu_query_tc.
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
  if (argc != 6) { fprintf(stderr, "usage: emu_query_tc_batch in.bin out.f32 program sms B\n"); return 2; }
  const int program = atoi(argv[3]);
  g_fake_sms = atoi(argv[4]);
  const int B = atoi(argv[5]);
  if (program != 3 && program != 0) { fprintf(stderr, "unknown program %d (3 or 0: the tensor-core program)\n", program); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  int32_t hd[8];
  float zs, calib_unused[12];
  if (fread(hd, 4, 8, f) != 8 || fread(&zs, 4, 1, f) != 1 || fread(calib_unused, 4, 12, f) != 12) { fprintf(stderr, "short header\n"); return 2; }
  const int C = hd[0], H = hd[1], W = hd[2], N = hd[3], has_calib = hd[4], persp = hd[5], res = hd[6], last_op = hd[7];
  auto rd = [&](size_t n) { std::vector<float> v(n); if (fread(v.data(), 4, n, f) != n) { fprintf(stderr, "short file\n"); exit(2); } return v; };
  const size_t per_map = (size_t)C * H * W;
  std::vector<float> nchw = rd(B * per_map), pts = rd((size_t)B * 3 * N);
  std::vector<float> calibs = has_calib ? rd((size_t)B * 12) : std::vector<float>();
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
  // batch feature handle: B channel-last maps, one after the other (what mp_feat_upload produces), one amax word per map
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
  MpCalib cal;                    // (what mp_query_points_batch sets up: the [R|t] rows come from the device calibs)
  memset(&cal, 0, sizeof(cal));
  cal.has = has_calib;
  cal.perspective = persp && has_calib;
  cal.z_scale = zs;
  MpBatch bt;
  bt.B = B;
  bt.pt_stride = 3ll * N;
  bt.out_stride = (long long)res * N;
  bt.calibs = has_calib ? calibs.data() : nullptr;
  std::vector<float> out((size_t)B * res * N + 1, -4242.f);
  MpOutDst dst;
  dst.out = out.data(); dst.ld = N; dst.scatter_vol = nullptr;
  const int rc = mp_launch_query_tc(&mlp, &feat, src, cal, dst, nullptr, guard, &bt);
  if (getenv("EMU_TC_AMAX"))
    for (int b = 0; b < B; ++b) { float a; memcpy(&a, &amax[b], 4); fprintf(stderr, "amax[%d] %.9g\n", b, a); }
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_tc: %s\n", g_err); return 3; }
  if (out[(size_t)B * res * N] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  f = fopen(argv[2], "wb");
  fwrite(out.data(), 4, (size_t)B * res * N, f);
  fclose(f);
  mp_tc_release(&mlp);
  return 0;
}
