// TEST INFRASTRUCTURE ONLY: the surface render of monoport_b200/csrc/query_tc.cu (the colour head's tensor-core program
// writing the visible-surface colours into a canvas) compiled UNMODIFIED for the CPU (see emu_host.h).
//   emu_colour_surface_tc in.bin out.f32 sms R count bx0 by0 bz0 bx1 by1 bz1 [host]      (the box [b_min, b_max])
// in.bin as for emu_query_tc (one map); the N points are the capacity of the vertex buffers: rows X, Y (integers) and Z
// (index space).
//   default: mp_launch_surface_tc with the vertex count on the device (`count`, an int64 that may exceed N) and the range
//            guard of EMU_TC_GUARD (limit EMU_TC_LIMIT, default +inf) -- what mp_colorize_surface_async enqueues;
//   host   : mp_launch_colour_surface with `count` vertices counted on the host -- what mp_colorize_surface runs.
// out.f32: the [R,R,3] canvas, background EMU_CANVAS_BG (default 1).
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_tc.cu"

int mp_launch_query_fp32(const mp_mlp*, const mp_feat*, const MpPointSrc&, const MpCalib&, const MpOutDst&, cudaStream_t, int,
                         const MpBatch*) { return MP_E_UNSUPPORTED; }

int main(int argc, char** argv) {
  if (argc < 12) { fprintf(stderr, "usage: emu_colour_surface_tc in.bin out.f32 sms R count bx0 by0 bz0 bx1 by1 bz1 [host]\n"); return 2; }
  g_fake_sms = atoi(argv[3]);
  const int R = atoi(argv[4]);
  const long long count = atoll(argv[5]);
  float bmin[3], bmax[3];
  emu_box_args(argv + 6, bmin, bmax);
  const bool host = argc >= 13 && !strcmp(argv[12], "host");
  EmuInput in = emu_read_input(argv[1]);
  EmuMlp m = emu_make_mlp(in);
  mp_mlp& mlp = m.mlp;
  const int guard = getenv("EMU_TC_GUARD") ? atoi(getenv("EMU_TC_GUARD")) : MP_GUARD_NONE;
  tc::emu::set_smem(g_dyn_smem[0], sizeof(g_dyn_smem[0]), g_dyn_smem[1]);
  if (mp_tc_prepare(&mlp) != MP_OK || !mlp.tc_ok) { fprintf(stderr, "mp_tc_prepare: %s (tc_ok=%d)\n", g_err, mlp.tc_ok); return 3; }
  EmuFeat ef = emu_make_feat(in);
  const EmuVerts v = emu_vertex_rows(in);
  const float bg = getenv("EMU_CANVAS_BG") ? (float)atof(getenv("EMU_CANVAS_BG")) : 1.0f;
  std::vector<float> canvas((size_t)R * R * 3 + 1, bg);
  canvas[(size_t)R * R * 3] = -4242.f;
  int rc;
  if (host) {
    rc = mp_launch_colour_surface(&mlp, &ef.feat, v.X.data(), v.Y.data(), v.Z.data(), count, R, bmin, bmax, in.cal,
                                  canvas.data(), nullptr);
  } else {
    const MpSurfaceSrc surf = mp_surface_src(v.X.data(), v.Y.data(), v.Z.data(), &count, R, bmin, bmax, canvas.data());
    rc = mp_launch_surface_tc(&mlp, &ef.feat, surf, in.N, in.cal, nullptr, guard);
  }
  if (rc != MP_OK) { fprintf(stderr, "surface render: %s (%d)\n", g_err, rc); return 3; }
  if (canvas[(size_t)R * R * 3] != -4242.f) { fprintf(stderr, "wrote past the canvas\n"); return 3; }
  float a;
  memcpy(&a, &ef.amax[0], 4);
  printf("%.9g\n", a);                                   // the frame's max |feature| (the range guard's input)
  emu_write(argv[2], canvas.data(), (size_t)R * R * 3);
  mp_tc_release(&mlp);
  return 0;
}
