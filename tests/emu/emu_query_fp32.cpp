// TEST INFRASTRUCTURE ONLY: monoport_b200/csrc/query_fp32.cu (the exact CUDA-core kernel: default path of the colour head
// and of every head shape the tensor-core programs do not cover) compiled unmodified on the CPU emulation layer.
//   emu_query_fp32 in.bin out.f32 [batch B]        (in.bin and out.f32 as for emu_query_tc, batch B included: one launch over
//   B images, what mp_query_points_batch sets up)
#include <cuda_runtime.h>
#include <stdarg.h>

#define MP_EMU_CUDA_TYPES 1
#include "cuda_emu.h"

alignas(1024) static float g_dyn_smem[240 * 1024 / 4];        // the kernel's dynamic shared memory
void* mp_emu_dyn_smem() { return g_dyn_smem; }

extern "C" {
cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) {
  *v = a == cudaDevAttrMultiProcessorCount ? 3 : (a == cudaDevAttrMaxSharedMemoryPerBlockOptin ? 232448 : 0);
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
  const bool batched = argc == 5 && !strcmp(argv[3], "batch");
  if (argc != 3 && !batched) { fprintf(stderr, "usage: emu_query_fp32 in.bin out.f32 [batch B]\n"); return 2; }
  const int B = batched ? atoi(argv[4]) : 1;
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
  std::vector<float> nhwc(B * per_map);
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < C; ++c)
      for (int p = 0; p < H * W; ++p) nhwc[b * per_map + (size_t)p * C + c] = nchw[b * per_map + (size_t)c * H * W + p];
  mp_feat feat;
  memset(&feat, 0, sizeof(feat));
  feat.B = B; feat.C = C; feat.H = H; feat.W = W; feat.nhwc32 = nhwc.data();
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
  MpBatch bt;                     // (batched: the [R|t] rows come from the device calibs)
  bt.B = B;
  bt.pt_stride = 3ll * N;
  bt.out_stride = (long long)res * N;
  bt.calibs = has_calib ? calibs.data() : nullptr;
  std::vector<float> out((size_t)B * res * N + 1, -4242.f);
  MpOutDst dst;
  dst.out = out.data(); dst.ld = N; dst.scatter_vol = nullptr;
  const int rc = mp_launch_query_fp32(&mlp, &feat, src, cal, dst, nullptr, MP_GUARD_NONE, batched ? &bt : nullptr);
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_fp32: %s\n", g_err); return 3; }
  if (out[(size_t)B * res * N] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  f = fopen(argv[2], "wb");
  fwrite(out.data(), 4, (size_t)B * res * N, f);
  fclose(f);
  return 0;
}
