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

// the launcher (launch<P, Kernel>) expands this inside its template: P is the tile size it launches
#define MP_EMU_LAUNCH(grid, block, call)                                                                                 \
  (printf("launch P=%d\n", P), cuda_emu::launch(dim3((unsigned)(grid)), dim3((unsigned)(block)), [&] { call; }))
#include "emu_host.h"
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
  EmuInput in = emu_read_input(argv[1]);
  const int N = in.N, res = in.res;

  const char* s = argv[3];
  const bool skip = strncmp(s, "noskip:", 7) != 0;
  if (!skip) s += 7;
  std::vector<int> widths;
  for (char* e; *s && (int)widths.size() < MP_MAX_LAYERS; s = *e ? e + 1 : e) widths.push_back((int)strtol(s, &e, 10));
  if (widths.empty() || *s || widths.back() != res) { fprintf(stderr, "bad widths %s (res %d)\n", argv[3], res); return 2; }

  EmuMlp m = emu_make_mlp(in, widths, skip);
  EmuFeat ef = emu_make_feat(in);
  const MpPointSrc src = emu_rows_src(in);
  std::vector<float> out;
  int rc;
  if (surface) {
    const int R = atoi(argv[6]);
    const long long count = N;
    const EmuVerts v = emu_vertex_rows(in);
    out.assign((size_t)R * R * 3 + 1, 1.0f);
    out.back() = -4242.f;
    float bmin[3], bmax[3];
    emu_box_args(argv + 7, bmin, bmax);
    const MpSurfaceSrc surf = mp_surface_src(v.X.data(), v.Y.data(), v.Z.data(), &count, R, bmin, bmax, out.data());
    rc = mp_launch_surface_fp32(&m.mlp, &ef.feat, surf, N, in.cal, nullptr, MP_GUARD_NONE);
  } else if (!strcmp(mode, "grad")) {
    out.assign((size_t)(res + 3) * N + 1, -4242.f);    // value [res][N], gradient [3][N], then a sentinel
    rc = mp_launch_query_grad(&m.mlp, &ef.feat, src, in.cal, nullptr, N, out.data(), N, out.data() + (size_t)res * N, N, nullptr);
  } else {
    out.assign((size_t)res * N + 1, -4242.f);
    MpOutDst dst;
    dst.out = out.data(); dst.ld = N; dst.scatter_vol = nullptr;
    rc = mp_launch_query_fp32(&m.mlp, &ef.feat, src, in.cal, dst, nullptr, MP_GUARD_NONE);
  }
  if (rc != MP_OK) { fprintf(stderr, "launch refused: %s (%d)\n", g_err, rc); return 3; }
  if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  emu_write(argv[2], out.data(), out.size() - 1);
  return 0;
}
