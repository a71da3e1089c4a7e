// TEST INFRASTRUCTURE ONLY: the gradient kernel of monoport_b200/csrc/query_fp32.cu (query_grad_kernel) compiled unmodified
// on the CPU emulation layer.
//   emu_query_grad in.bin out.f32 [sms] [grad_out.f32]
// in.bin as for emu_query_fp32; grad_out.f32 (optional): [Res][N] fp32, otherwise all ones.  out.f32 = value [Res][N]
// followed by the point gradient [3][N].  sms = simulated SM count (grid size), default 3.
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
  // one buffer: value [res][N], gradient [3][N], then a sentinel
  std::vector<float> out((size_t)(res + 3) * N + 1, -4242.f);
  float* dp = out.data() + (size_t)res * N;
  const int rc = mp_launch_query_grad(&m.mlp, &ef.feat, emu_rows_src(in), in.cal, gout.empty() ? nullptr : gout.data(), N,
                                      out.data(), N, dp, N, nullptr);
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_grad: %s\n", g_err); return 3; }
  if (out[(size_t)(res + 3) * N] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  emu_write(argv[2], out.data(), (size_t)(res + 3) * N);
  return 0;
}
