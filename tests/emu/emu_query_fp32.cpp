// TEST INFRASTRUCTURE ONLY: monoport_b200/csrc/query_fp32.cu (the exact CUDA-core kernel: default path of the colour head
// and of every head shape the tensor-core programs do not cover) compiled unmodified on the CPU emulation layer.
//   emu_query_fp32 in.bin out.f32 [batch B]        (in.bin and out.f32 as for emu_query_tc, batch B included: one launch over
//   B images, what mp_query_points_batch sets up)
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_fp32.cu"

int main(int argc, char** argv) {
  const bool batched = argc == 5 && !strcmp(argv[3], "batch");
  if (argc != 3 && !batched) { fprintf(stderr, "usage: emu_query_fp32 in.bin out.f32 [batch B]\n"); return 2; }
  const int B = batched ? atoi(argv[4]) : 1;
  EmuInput in = emu_read_input(argv[1], B, batched);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in);
  EmuFeat ef = emu_make_feat(in, B);
  MpBatch bt;                     // (batched: the [R|t] rows come from the device calibs)
  bt.B = B;
  bt.pt_stride = 3ll * N;
  bt.out_stride = (long long)res * N;
  bt.calibs = in.calibs.empty() ? nullptr : in.calibs.data();
  std::vector<float> out((size_t)B * res * N + 1, -4242.f);
  MpOutDst dst;
  dst.out = out.data(); dst.ld = N; dst.scatter_vol = nullptr;
  const int rc = mp_launch_query_fp32(&m.mlp, &ef.feat, emu_rows_src(in), in.cal, dst, nullptr, MP_GUARD_NONE,
                                      batched ? &bt : nullptr);
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_fp32: %s\n", g_err); return 3; }
  if (out[(size_t)B * res * N] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  emu_write(argv[2], out.data(), (size_t)B * res * N);
  return 0;
}
