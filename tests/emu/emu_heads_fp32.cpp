// TEST INFRASTRUCTURE ONLY: the exact kernels of monoport_b200/csrc/query_fp32.cu -- the query, the point gradient and the
// surface render, the programs of every head the tensor-core programs do not cover -- compiled unmodified on the CPU
// emulation layer, for a head of any shape.
//   emu_heads_fp32 in.bin out.f32 widths sms query           mp_launch_query_fp32; out = [res][N]
//   emu_heads_fp32 in.bin out.f32 widths sms grad            mp_launch_query_grad (grad_output = ones); out = the value
//                                                            [res][N], then the point gradient [3][N]
//   emu_heads_fp32 in.bin out.f32 widths sms surface R bx0 by0 bz0 bx1 by1 bz1
//                                                            mp_launch_surface_fp32 over the box [b_min, b_max]: the N
//                                                            "points" of in.bin are vertex rows X, Y, Z; out = the
//                                                            [R,R,3] canvas (background 1)
//   emu_heads_fp32 limit res last_op                         prints mp_tc_default_feature_limit(res, last_op)
// widths: the head's filter_channels after the first ("64,48,1"; channels[0] = C + 1), "noskip:" in front for a
// no_residual head.  in.bin as for emu_query_fp32 (the header's res is the last width), with the weights of these widths.
// Every launch prints "launch P=<tile size>" on stdout: the instantiation the launcher's shared-memory fit chose.
#include <cuda_runtime.h>
#include <stdarg.h>

#define MP_EMU_CUDA_TYPES 1
#include <math.h>
#include "cuda_emu.h"

alignas(1024) static float g_dyn_smem[240 * 1024 / 4];        // the kernel's dynamic shared memory
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
// both launch sites (launch<P> and launch_grad<P>) expand this inside their template: P is the tile size they launch
#define MP_EMU_LAUNCH(grid, block, call)                                                                                 \
  (printf("launch P=%d\n", P), cuda_emu::launch(dim3((unsigned)(grid)), dim3((unsigned)(block)), [&] { call; }))

static char g_err[512];
void mp_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

#include "../../monoport_b200/csrc/query_fp32.cu"

int main(int argc, char** argv) {
  if (argc == 4 && !strcmp(argv[1], "limit")) {
    printf("%.9g\n", mp_tc_default_feature_limit(atoi(argv[2]), atoi(argv[3])));
    return 0;
  }
  const char* mode = argc >= 6 ? argv[5] : "";
  const bool surface = argc == 13 && !strcmp(mode, "surface");
  if (!surface && !(argc == 6 && (!strcmp(mode, "query") || !strcmp(mode, "grad")))) {
    fprintf(stderr, "usage: emu_heads_fp32 in.bin out.f32 widths sms (query | grad | surface R bx0 by0 bz0 bx1 by1 bz1)\n"
                    "       emu_heads_fp32 limit res last_op\n");
    return 2;
  }
  g_fake_sms = atoi(argv[4]);
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  int32_t hd[8];
  float zs, calib[12];
  if (fread(hd, 4, 8, f) != 8 || fread(&zs, 4, 1, f) != 1 || fread(calib, 4, 12, f) != 12) { fprintf(stderr, "short header\n"); return 2; }
  const int C = hd[0], H = hd[1], W = hd[2], N = hd[3], has_calib = hd[4], persp = hd[5], res = hd[6], last_op = hd[7];
  auto rd = [&](size_t n) { std::vector<float> v(n); if (fread(v.data(), 4, n, f) != n) { fprintf(stderr, "short file\n"); exit(2); } return v; };
  std::vector<float> nchw = rd((size_t)C * H * W), pts = rd((size_t)3 * N);

  const char* s = argv[3];
  const bool skip = strncmp(s, "noskip:", 7) != 0;
  if (!skip) s += 7;
  int chans[MP_MAX_LAYERS + 1] = {C + 1};
  int L = 0;
  for (char* e; *s && L < MP_MAX_LAYERS; s = *e ? e + 1 : e) chans[++L] = (int)strtol(s, &e, 10);
  if (L < 1 || *s || chans[L] != res) { fprintf(stderr, "bad widths %s (res %d)\n", argv[3], res); return 2; }

  mp_mlp mlp;
  memset(&mlp, 0, sizeof(mlp));
  mlp.n_layers = L; mlp.skip = skip; mlp.last_op = last_op;
  mlp.tc_amax_limit = INFINITY;
  std::vector<std::vector<float>> Ws(L), Wt(L), Bs(L);
  for (int l = 0; l <= L; ++l) mlp.channels[l] = chans[l];
  for (int l = 0; l < L; ++l) {                          // as mp_mlp_create
    const int cin = chans[l] + (l && skip ? chans[0] : 0), cout = chans[l + 1];
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
  unsigned amax = 0u;
  feat.amax = &amax;
  MpCalib cal;
  memset(&cal, 0, sizeof(cal));
  cal.has = has_calib;
  memcpy(cal.m, calib, sizeof(calib));
  cal.perspective = persp && has_calib;
  cal.z_scale = zs;
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_ROWS;
  src.px = pts.data(); src.py = pts.data() + N; src.pz = pts.data() + 2 * (size_t)N;
  src.pstride = 1;
  src.n = N;

  std::vector<float> out;
  int rc;
  if (surface) {
    const int R = atoi(argv[6]);
    const long long count = N;
    std::vector<long long> X(N), Y(N);
    std::vector<float> Z(N);
    for (int i = 0; i < N; ++i) { X[i] = (long long)pts[i]; Y[i] = (long long)pts[(size_t)N + i]; Z[i] = pts[2 * (size_t)N + i]; }
    out.assign((size_t)R * R * 3 + 1, 1.0f);
    out.back() = -4242.f;
    float bmin[3], bmax[3];
    for (int a = 0; a < 3; ++a) { bmin[a] = strtof(argv[7 + a], nullptr); bmax[a] = strtof(argv[10 + a], nullptr); }
    const MpSurfaceSrc surf = mp_surface_src(X.data(), Y.data(), Z.data(), &count, R, bmin, bmax, out.data());
    rc = mp_launch_surface_fp32(&mlp, &feat, surf, N, cal, nullptr, MP_GUARD_NONE);
  } else if (!strcmp(mode, "grad")) {
    out.assign((size_t)(res + 3) * N + 1, -4242.f);    // value [res][N], gradient [3][N], then a sentinel
    rc = mp_launch_query_grad(&mlp, &feat, src, cal, nullptr, N, out.data(), N, out.data() + (size_t)res * N, N, nullptr);
  } else {
    out.assign((size_t)res * N + 1, -4242.f);
    MpOutDst dst;
    dst.out = out.data(); dst.ld = N; dst.scatter_vol = nullptr;
    rc = mp_launch_query_fp32(&mlp, &feat, src, cal, dst, nullptr, MP_GUARD_NONE);
  }
  if (rc != MP_OK) { fprintf(stderr, "launch refused: %s (%d)\n", g_err, rc); return 3; }
  if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  f = fopen(argv[2], "wb");
  fwrite(out.data(), 4, out.size() - 1, f);
  fclose(f);
  return 0;
}
