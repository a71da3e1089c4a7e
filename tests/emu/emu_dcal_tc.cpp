// TEST INFRASTRUCTURE ONLY: the programs of monoport_b200/csrc/query_tc.cu launched with the camera in device memory (a
// single-map MpBatch whose calibs point at a 12-float buffer; see dcal_emu.h), compiled UNMODIFIED for the CPU (see
// emu_host.h).
//   emu_dcal_tc in.bin out.f32 sms (nodes R res | grid R z0 nz | surface R count bx0 by0 bz0 bx1 by1 bz1 | jvp)
//   nodes  : the query over every third node of the res^3 level of an R^3 pyramid over [-1,1]^3 (index list, count on the
//            device), scattered into the res^3 volume = out
//   grid   : the query over planes [z0, z0+nz) of an R^3 grid over [-1,1]^3; out = the nz*R*R values
//   surface: the colour head's render of the N vertex rows of in.bin (capacity N, `count` on the device) over the box into an
//            [R,R,3] canvas of ones = out (what mp_colorize_surface_async enqueues)
//   jvp    : the forward-mode gradient program on the N points of in.bin; out = value [res][N], then dpoints [3][N]
// in.bin: the layout of emu_query_tc (one map).  EMU_DCAL (dcal_emu.h) selects the device camera; without it the launch
// takes the camera by value, so the two runs can be compared.
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_tc.cu"
#include "dcal_emu.h"

int mp_launch_query_fp32(const mp_mlp*, const mp_feat*, const MpPointSrc&, const MpCalib&, const MpOutDst&, cudaStream_t, int,
                         const MpBatch*) { return MP_E_UNSUPPORTED; }

int main(int argc, char** argv) {
  if (argc < 5) {
    fprintf(stderr, "usage: emu_dcal_tc in.bin out.f32 sms (nodes R res | grid R z0 nz | surface R count box[6] | jvp)\n");
    return 2;
  }
  g_fake_sms = atoi(argv[3]);
  const std::string mode = argv[4];
  EmuInput in = emu_read_input(argv[1]);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in);
  mp_mlp& mlp = m.mlp;
  tc::emu::set_smem(g_dyn_smem[0], sizeof(g_dyn_smem[0]), g_dyn_smem[1]);
  if (mp_tc_prepare(&mlp) != MP_OK || !mlp.tc_ok) { fprintf(stderr, "mp_tc_prepare: %s (tc_ok=%d)\n", g_err, mlp.tc_ok); return 3; }
  EmuFeat ef = emu_make_feat(in);
  float calib[12];
  memcpy(calib, in.cal.m, sizeof(calib));

  std::vector<int32_t> nodes;
  int32_t node_count = 0;
  MpPointSrc src = emu_rows_src(in);
  long long n_out = 0;
  if (mode == "nodes" && argc == 7) {
    const int lres = atoi(argv[6]);
    src = emu_node_src(atoi(argv[5]), lres, nodes, node_count);
    n_out = (long long)lres * lres * lres;
  } else if (mode == "grid" && argc == 8) {
    src = emu_grid_src(atoi(argv[5]), atoi(argv[6]), atoi(argv[7]));
    n_out = src.n;
  } else if (!(mode == "surface" && argc == 13) && !(mode == "jvp" && argc == 5)) {
    fprintf(stderr, "bad mode or argument count\n");
    return 2;
  }

  const int rc_all = emu_dcal_run(in.cal, calib, argv[2], [&](const MpBatch* bt, const char* path) {
    std::vector<float> out;
    int rc;
    if (mode == "surface") {
      const int R = atoi(argv[5]);
      const long long count = atoll(argv[6]);
      float bmin[3], bmax[3];
      emu_box_args(argv + 7, bmin, bmax);
      const EmuVerts v = emu_vertex_rows(in);
      out.assign((size_t)R * R * 3 + 1, 1.0f);
      out.back() = -4242.f;
      const MpSurfaceSrc surf = mp_surface_src(v.X.data(), v.Y.data(), v.Z.data(), &count, R, bmin, bmax, out.data());
      rc = mp_launch_surface_tc(&mlp, &ef.feat, surf, N, in.cal, nullptr, MP_GUARD_NONE, bt);
    } else if (mode == "jvp") {
      out.assign((size_t)(res + 3) * N + 1, -4242.f);
      rc = mp_launch_query_jvp_tc(&mlp, &ef.feat, src, in.cal, nullptr, N, out.data(), N, out.data() + (size_t)res * N, N,
                                  nullptr, MP_GUARD_NONE, bt);
    } else {
      out.assign((size_t)n_out + 1, -4242.f);
      MpOutDst dst;
      dst.out = out.data(); dst.ld = n_out; dst.scatter_vol = nullptr;
      if (mode == "nodes") { dst.out = nullptr; dst.ld = 0; dst.scatter_vol = out.data(); }
      rc = mp_launch_query_tc(&mlp, &ef.feat, src, in.cal, dst, nullptr, MP_GUARD_NONE, bt);
    }
    if (rc != MP_OK) { fprintf(stderr, "launch: %s (%d)\n", g_err, rc); return 3; }
    if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
    emu_write(path, out.data(), out.size() - 1);
    return 0;
  });
  mp_tc_release(&mlp);
  return rc_all;
}
