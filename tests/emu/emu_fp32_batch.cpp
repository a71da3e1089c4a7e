// TEST INFRASTRUCTURE ONLY: emu_fp32.cpp (query_fp32.cu and query_vjp.cu compiled UNMODIFIED on the CPU model) with the
// batched exact point gradient.  Every command of emu_fp32 is taken as it is, and one more:
//   emu_fp32_batch in.bin out.f32 grad [grad_out.f32] --batch B
//                          mp_launch_query_grad over the B maps, point sets and calibs of a batched in.bin (grad_out
//                          [B][res][N], default ones): the batched query_fp32_kernel for the value, query_vjp_kernel for
//                          d points.  out = the values [B][res][N], then d points [B][3][N], pre-filled with -4242 (what a
//                          guarded launch skips keeps it).  --guard and --limit: the range guard, decided per image;
//                          --amax a0,a1,..: each map's max |feature| (what the tensor-core program's G0 kernel would have
//                          left in the handle); --sms as for emu_fp32.
#define main emu_fp32_main
#include "emu_fp32.cpp"
#undef main

int main(int argc, char** argv) {
  EmuArgs a(argc, argv);
  if (!a.get("batch") || a.pos.size() < 3 || strcmp(a.pos[2], "grad") != 0) return emu_fp32_main(argc, argv);
  if (a.pos.size() > 4) { fprintf(stderr, "usage: emu_fp32_batch in.bin out.f32 grad [grad_out.f32] --batch B [--options]\n"); return 2; }
  const int B = (int)a.num("batch", 1);
  g_fake_sms = (int)a.num("sms", 3);
  EmuInput in = emu_read_input(a.pos[0], B, true);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in, a);
  EmuFeat ef = emu_make_feat(in, B);
  const int guard = emu_guard(a);
  if (const char* am = a.get("amax")) {
    for (int b = 0; b < B && *am; ++b) {
      char* e;
      const float amax = strtof(am, &e);
      memcpy(&ef.amax[b], &amax, 4);
      am = *e ? e + 1 : e;
    }
  }
  const std::vector<float> gout = emu_read_file(a.arg(0), (size_t)B * res * N);
  MpBatch bt;                       // (the [R|t] rows come from the device calibs)
  bt.B = B;
  bt.pt_stride = 3ll * N;
  bt.calibs = in.calibs.empty() ? nullptr : in.calibs.data();
  return emu_output(a, in.cal, nullptr, (size_t)B * (res + 3) * N, -4242.f, [&](const MpBatch*, float* out) {
    return mp_launch_query_grad(&m.mlp, &ef.feat, emu_rows_src(in), in.cal, gout.empty() ? nullptr : gout.data(), N, out, N,
                                out + (size_t)B * res * N, N, nullptr, guard, &bt);
  });
}
