// TEST INFRASTRUCTURE ONLY: the surface render of monoport_b200/csrc/query_fp32.cu (the exact twin of the tensor-core colour
// render) compiled unmodified on the CPU emulation layer.
//   emu_colour_surface_fp32 in.bin out.f32 sms surface R count bx0 by0 bz0 bx1 by1 bz1
//                                                                    mp_launch_surface_fp32 over the box [b_min, b_max]: the
//                                                                    N "points" of in.bin are vertex rows X, Y, Z (capacity N,
//                                                                    count on the device); out = the [R,R,3] canvas
//                                                                    (background EMU_CANVAS_BG, default 1)
//   emu_colour_surface_fp32 in.bin out.f32 sms rows                  mp_launch_query_fp32 on the N world points of in.bin;
//                                                                    out = [res][N]
// in.bin as for emu_query_fp32.  Range guard: EMU_GUARD (sense), EMU_TC_LIMIT (the head's limit, default +inf) and
// EMU_AMAX (the frame's max |feature|, which the tensor-core program's G0 kernel would have left in the handle).
#include <cuda_runtime.h>
#include <stdarg.h>

#define MP_EMU_CUDA_TYPES 1
#include <math.h>
#include "cuda_emu.h"

alignas(1024) static float g_dyn_smem[240 * 1024 / 4];
void* mp_emu_dyn_smem() { return g_dyn_smem; }

static int g_fake_sms = 3;
extern "C" {
cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) {
  *v = a == cudaDevAttrMultiProcessorCount ? g_fake_sms : (a == cudaDevAttrMaxSharedMemoryPerBlockOptin ? 232448 : 0);
  return cudaSuccess;
}
cudaError_t cudaGetLastError(void) { return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
}
template <class T> static cudaError_t cudaFuncSetAttribute(T*, cudaFuncAttribute, int) { return cudaSuccess; }
#define MP_EMU_LAUNCH(grid, block, call) cuda_emu::launch(dim3((unsigned)(grid)), dim3((unsigned)(block)), [&] { call; })

static char g_err[512];
void mp_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

#include "../../monoport_b200/csrc/query_fp32.cu"

int main(int argc, char** argv) {
  const bool surface = argc == 13 && !strcmp(argv[4], "surface");
  if (!surface && !(argc == 5 && !strcmp(argv[4], "rows"))) {
    fprintf(stderr, "usage: emu_colour_surface_fp32 in.bin out.f32 sms (surface R count bx0 by0 bz0 bx1 by1 bz1 | rows)\n");
    return 2;
  }
  g_fake_sms = atoi(argv[3]);
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
  mlp.tc_amax_limit = getenv("EMU_TC_LIMIT") ? (float)atof(getenv("EMU_TC_LIMIT")) : INFINITY;
  const int guard = getenv("EMU_GUARD") ? atoi(getenv("EMU_GUARD")) : MP_GUARD_NONE;
  std::vector<std::vector<float>> Ws(5), Wt(5), Bs(5);
  for (int l = 0; l <= 5; ++l) mlp.channels[l] = chans[l];
  for (int l = 0; l < 5; ++l) {
    const int cin = chans[l] + (l ? chans[0] : 0), cout = chans[l + 1];
    mlp.cin[l] = cin; mlp.cout[l] = cout;
    Ws[l] = rd((size_t)cin * cout);
    Bs[l] = rd(cout);
    Wt[l].resize((size_t)cin * cout);                    // what transpose_w_kernel produces: [cin][cout]
    for (int o = 0; o < cout; ++o)
      for (int k = 0; k < cin; ++k) Wt[l][(size_t)k * cout + o] = Ws[l][(size_t)o * cin + k];
    mlp.w[l] = Ws[l].data(); mlp.wt[l] = Wt[l].data(); mlp.bias[l] = Bs[l].data();
  }
  fclose(f);
  std::vector<float> nhwc((size_t)C * H * W);
  for (int c = 0; c < C; ++c)
    for (int p = 0; p < H * W; ++p) nhwc[(size_t)p * C + c] = nchw[(size_t)c * H * W + p];
  mp_feat feat;
  memset(&feat, 0, sizeof(feat));
  feat.B = 1; feat.C = C; feat.H = H; feat.W = W; feat.nhwc32 = nhwc.data();
  const float amax_f = getenv("EMU_AMAX") ? (float)atof(getenv("EMU_AMAX")) : 0.f;
  unsigned amax;
  memcpy(&amax, &amax_f, 4);
  feat.amax = &amax;
  MpCalib cal;
  memset(&cal, 0, sizeof(cal));
  cal.has = has_calib;
  memcpy(cal.m, calib, sizeof(calib));
  cal.perspective = persp && has_calib;
  cal.z_scale = zs;
  std::vector<float> out;
  int rc;
  if (surface) {
    const int R = atoi(argv[5]);
    const long long count = atoll(argv[6]);
    std::vector<long long> X(N), Y(N);
    std::vector<float> Z(N);
    for (int i = 0; i < N; ++i) { X[i] = (long long)pts[i]; Y[i] = (long long)pts[(size_t)N + i]; Z[i] = pts[2 * (size_t)N + i]; }
    const float bg = getenv("EMU_CANVAS_BG") ? (float)atof(getenv("EMU_CANVAS_BG")) : 1.0f;
    out.assign((size_t)R * R * 3 + 1, bg);
    out.back() = -4242.f;
    float bmin[3], bmax[3];
    for (int a = 0; a < 3; ++a) { bmin[a] = strtof(argv[7 + a], nullptr); bmax[a] = strtof(argv[10 + a], nullptr); }
    const MpSurfaceSrc surf = mp_surface_src(X.data(), Y.data(), Z.data(), &count, R, bmin, bmax, out.data());
    rc = mp_launch_surface_fp32(&mlp, &feat, surf, N, cal, nullptr, guard);
  } else {
    out.assign((size_t)res * N + 1, -4242.f);
    MpPointSrc src;
    memset(&src, 0, sizeof(src));
    src.kind = MP_SRC_ROWS;
    src.px = pts.data(); src.py = pts.data() + N; src.pz = pts.data() + 2 * (size_t)N;
    src.pstride = 1;
    src.n = N;
    MpOutDst dst;
    dst.out = out.data(); dst.ld = N; dst.scatter_vol = nullptr;
    rc = mp_launch_query_fp32(&mlp, &feat, src, cal, dst, nullptr, guard);
  }
  if (rc != MP_OK) { fprintf(stderr, "fp32 launch: %s (%d)\n", g_err, rc); return 3; }
  if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  f = fopen(argv[2], "wb");
  fwrite(out.data(), 4, out.size() - 1, f);
  fclose(f);
  return 0;
}
