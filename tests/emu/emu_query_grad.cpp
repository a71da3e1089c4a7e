// TEST INFRASTRUCTURE ONLY: the exact point gradient of monoport_b200/csrc/query_fp32.cu (mp_launch_query_grad: the value
// by query_fp32_kernel, d points by query_vjp_kernel) compiled unmodified on the CPU emulation layer.
//   emu_query_grad in.bin out.f32 [sms] [grad_out.f32]
// in.bin as for emu_query_fp32; grad_out.f32 (optional): [Res][N] fp32, otherwise all ones.  out.f32 = value [Res][N]
// followed by the point gradient [3][N], pre-filled with -4242 (what a guarded launch skips, and the points at or beyond the
// device-side count, keep it).  sms = simulated SM count (grid size), default 3.  Range guard: EMU_GUARD (sense),
// EMU_TC_LIMIT (the head's limit, default +inf) and EMU_AMAX (the map's max |feature|); EMU_COUNT=k: the point count on
// the device (n = N is then the capacity).
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_fp32.cu"

int main(int argc, char** argv) {
  if (argc < 3 || argc > 5) { fprintf(stderr, "usage: emu_query_grad in.bin out.f32 [sms] [grad_out.f32]\n"); return 2; }
  if (argc >= 4) g_fake_sms = atoi(argv[3]);
  EmuInput in = emu_read_input(argv[1]);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in);
  std::vector<float> gout;
  if (argc >= 5) {
    FILE* g = fopen(argv[4], "rb");
    if (!g) { perror(argv[4]); return 2; }
    gout = emu_read(g, (size_t)res * N);
    fclose(g);
  }
  EmuFeat ef = emu_make_feat(in);
  const int guard = getenv("EMU_GUARD") ? atoi(getenv("EMU_GUARD")) : MP_GUARD_NONE;
  const float amax_f = getenv("EMU_AMAX") ? (float)atof(getenv("EMU_AMAX")) : 0.f;
  memcpy(&ef.amax[0], &amax_f, 4);
  MpPointSrc src = emu_rows_src(in);
  int32_t count = 0;
  if (getenv("EMU_COUNT")) {
    count = atoi(getenv("EMU_COUNT"));
    src.count_dev = &count;
  }
  // one buffer: value [res][N], gradient [3][N], then a sentinel
  std::vector<float> out((size_t)(res + 3) * N + 1, -4242.f);
  float* dp = out.data() + (size_t)res * N;
  const int rc = mp_launch_query_grad(&m.mlp, &ef.feat, src, in.cal, gout.empty() ? nullptr : gout.data(), N, out.data(), N,
                                      dp, N, nullptr, guard);
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_grad: %s\n", g_err); return 3; }
  if (out[(size_t)(res + 3) * N] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  emu_write(argv[2], out.data(), (size_t)(res + 3) * N);
  return 0;
}
