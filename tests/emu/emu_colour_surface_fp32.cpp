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
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_fp32.cu"

int main(int argc, char** argv) {
  const bool surface = argc == 13 && !strcmp(argv[4], "surface");
  if (!surface && !(argc == 5 && !strcmp(argv[4], "rows"))) {
    fprintf(stderr, "usage: emu_colour_surface_fp32 in.bin out.f32 sms (surface R count bx0 by0 bz0 bx1 by1 bz1 | rows)\n");
    return 2;
  }
  g_fake_sms = atoi(argv[3]);
  EmuInput in = emu_read_input(argv[1]);
  const int N = in.N;
  EmuMlp m = emu_make_mlp(in);
  const int guard = getenv("EMU_GUARD") ? atoi(getenv("EMU_GUARD")) : MP_GUARD_NONE;
  EmuFeat ef = emu_make_feat(in);
  const float amax_f = getenv("EMU_AMAX") ? (float)atof(getenv("EMU_AMAX")) : 0.f;
  memcpy(&ef.amax[0], &amax_f, 4);
  std::vector<float> out;
  int rc;
  if (surface) {
    const int R = atoi(argv[5]);
    const long long count = atoll(argv[6]);
    const EmuVerts v = emu_vertex_rows(in);
    const float bg = getenv("EMU_CANVAS_BG") ? (float)atof(getenv("EMU_CANVAS_BG")) : 1.0f;
    out.assign((size_t)R * R * 3 + 1, bg);
    out.back() = -4242.f;
    float bmin[3], bmax[3];
    emu_box_args(argv + 7, bmin, bmax);
    const MpSurfaceSrc surf = mp_surface_src(v.X.data(), v.Y.data(), v.Z.data(), &count, R, bmin, bmax, out.data());
    rc = mp_launch_surface_fp32(&m.mlp, &ef.feat, surf, N, in.cal, nullptr, guard);
  } else {
    out.assign((size_t)in.res * N + 1, -4242.f);
    MpOutDst dst;
    dst.out = out.data(); dst.ld = N; dst.scatter_vol = nullptr;
    rc = mp_launch_query_fp32(&m.mlp, &ef.feat, emu_rows_src(in), in.cal, dst, nullptr, guard);
  }
  if (rc != MP_OK) { fprintf(stderr, "fp32 launch: %s (%d)\n", g_err, rc); return 3; }
  if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  emu_write(argv[2], out.data(), out.size() - 1);
  return 0;
}
