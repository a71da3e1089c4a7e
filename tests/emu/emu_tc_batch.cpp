// TEST INFRASTRUCTURE ONLY: emu_tc.cpp (query_tc.cu compiled UNMODIFIED on the CPU model) with the batched forward-mode
// gradient program.  Every command of emu_tc is taken as it is, and one more:
//   emu_tc_batch in.bin out.f32 jvp [grad_out.f32] --batch B
//                          mp_launch_query_jvp_tc over the B maps, point sets and calibs of a batched in.bin (grad_out
//                          [B][res][N], default ones); out = the values [B][res][N], then d points [B][3][N], pre-filled
//                          with -4242 (what a guarded launch skips keeps it).  --guard and --limit: the range guard,
//                          decided per image from the maximum the G0 kernel leaves for each map; --sms as for emu_tc.
#define main emu_tc_main
#include "emu_tc.cpp"
#undef main

int main(int argc, char** argv) {
  EmuArgs a(argc, argv);
  if (!a.get("batch") || a.pos.size() < 3 || strcmp(a.pos[2], "jvp") != 0) return emu_tc_main(argc, argv);
  if (a.pos.size() > 4) { fprintf(stderr, "usage: emu_tc_batch in.bin out.f32 jvp [grad_out.f32] --batch B [--options]\n"); return 2; }
  const int B = (int)a.num("batch", 1);
  g_fake_sms = (int)a.num("sms", 3);
  EmuInput in = emu_read_input(a.pos[0], B, true);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in, a);
  tc::emu::set_smem(g_dyn_smem[0], sizeof(g_dyn_smem[0]), g_dyn_smem[1]);
  if (mp_tc_prepare(&m.mlp) != MP_OK || !m.mlp.tc_ok) { fprintf(stderr, "mp_tc_prepare: %s\n", g_err); return 3; }
  EmuFeat ef = emu_make_feat(in, B);
  const int guard = emu_guard(a);
  const std::vector<float> gout = emu_read_file(a.arg(0), (size_t)B * res * N);
  MpBatch bt;                       // (the [R|t] rows come from the device calibs)
  bt.B = B;
  bt.pt_stride = 3ll * N;
  bt.calibs = in.calibs.empty() ? nullptr : in.calibs.data();
  const int rc = emu_output(a, in.cal, nullptr, (size_t)B * (res + 3) * N, -4242.f, [&](const MpBatch*, float* out) {
    return mp_launch_query_jvp_tc(&m.mlp, &ef.feat, emu_rows_src(in), in.cal, gout.empty() ? nullptr : gout.data(), N, out, N,
                                  out + (size_t)B * res * N, N, nullptr, guard, &bt);
  });
  mp_tc_release(&m.mlp);
  return rc;
}
