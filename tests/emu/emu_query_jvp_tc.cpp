// TEST INFRASTRUCTURE ONLY: the forward-mode gradient program of monoport_b200/csrc/query_tc.cu (query_jvp_kernel, with
// the per-frame G0 kernel before it) compiled UNMODIFIED for the CPU (see emu_host.h).
//   emu_query_jvp_tc in.bin out.f32 sms [grad_out.f32]
// in.bin: the layout of emu_query_tc (one map).  out.f32: value [res][N], then dpoints [3][N], pre-filled with -4242 (what a
// guarded launch skips, and the points at or beyond the device-side count, keep it).
// EMU_TC_LIMIT / EMU_TC_GUARD: the range guard as in emu_query_tc; EMU_COUNT=k: the point count on the device (n = N is
// then the capacity).
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_tc.cu"

int mp_launch_query_fp32(const mp_mlp*, const mp_feat*, const MpPointSrc&, const MpCalib&, const MpOutDst&, cudaStream_t, int,
                         const MpBatch*) { return MP_E_UNSUPPORTED; }

int main(int argc, char** argv) {
  if (argc < 4) { fprintf(stderr, "usage: emu_query_jvp_tc in.bin out.f32 sms [grad_out.f32]\n"); return 2; }
  g_fake_sms = atoi(argv[3]);
  EmuInput in = emu_read_input(argv[1]);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in);
  mp_mlp& mlp = m.mlp;
  const int guard = getenv("EMU_TC_GUARD") ? atoi(getenv("EMU_TC_GUARD")) : MP_GUARD_NONE;
  std::vector<float> gout;
  if (argc >= 5) {
    FILE* g = fopen(argv[4], "rb");
    if (!g) { perror(argv[4]); return 2; }
    gout = emu_read(g, (size_t)res * N);
    fclose(g);
  }
  tc::emu::set_smem(g_dyn_smem[0], sizeof(g_dyn_smem[0]), g_dyn_smem[1]);
  if (mp_tc_prepare(&mlp) != MP_OK || !mlp.tc_ok) { fprintf(stderr, "mp_tc_prepare: %s (tc_ok=%d)\n", g_err, mlp.tc_ok); return 3; }
  EmuFeat ef = emu_make_feat(in);
  MpPointSrc src = emu_rows_src(in);
  int32_t count = 0;
  if (getenv("EMU_COUNT")) {
    count = atoi(getenv("EMU_COUNT"));
    src.count_dev = &count;
  }
  std::vector<float> out((size_t)(res + 3) * N + 1, -4242.f);
  const int rc = mp_launch_query_jvp_tc(&mlp, &ef.feat, src, in.cal, gout.empty() ? nullptr : gout.data(), N, out.data(), N,
                                        out.data() + (size_t)res * N, N, nullptr, guard);
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_jvp_tc: %s\n", g_err); return 3; }
  if (out[(size_t)(res + 3) * N] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  emu_write(argv[2], out.data(), (size_t)(res + 3) * N);
  mp_tc_release(&mlp);
  return 0;
}
