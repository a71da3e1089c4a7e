// TEST INFRASTRUCTURE ONLY: the kernels of monoport_b200/csrc/query_fp32.cu launched with the camera in device memory (a
// single-map MpBatch whose calibs point at a 12-float buffer; see dcal_emu.h), compiled unmodified on the CPU emulation
// layer.
//   emu_dcal_fp32 in.bin out.f32 sms (nodes R res | surface R count bx0 by0 bz0 bx1 by1 bz1 | grad)
//   nodes  : the exact query over every third node of the res^3 level of an R^3 pyramid over [-1,1]^3 (index list, count
//            on the device), scattered into the res^3 volume = out (what the octree engine's fused path launches)
//   surface: the exact surface render of the N vertex rows of in.bin (capacity N, `count` on the device) over the box into
//            an [R,R,3] canvas of ones = out
//   grad   : the gradient kernel on the N points of in.bin; out = value [res][N], then dpoints [3][N]
// in.bin as for emu_query_fp32.  EMU_DCAL (dcal_emu.h) selects the device camera; without it the launch takes the camera by
// value, so the two runs can be compared.
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_fp32.cu"
#include "dcal_emu.h"

int main(int argc, char** argv) {
  if (argc < 5) {
    fprintf(stderr, "usage: emu_dcal_fp32 in.bin out.f32 sms (nodes R res | surface R count box[6] | grad)\n");
    return 2;
  }
  g_fake_sms = atoi(argv[3]);
  const std::string mode = argv[4];
  if (!(mode == "nodes" && argc == 7) && !(mode == "surface" && argc == 13) && !(mode == "grad" && argc == 5)) {
    fprintf(stderr, "bad mode or argument count\n");
    return 2;
  }
  EmuInput in = emu_read_input(argv[1]);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in);
  EmuFeat ef = emu_make_feat(in);
  float calib[12];
  memcpy(calib, in.cal.m, sizeof(calib));

  return emu_dcal_run(in.cal, calib, argv[2], [&](const MpBatch* bt, const char* path) {
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
      rc = mp_launch_surface_fp32(&m.mlp, &ef.feat, surf, N, in.cal, nullptr, MP_GUARD_NONE, bt);
    } else if (mode == "grad") {
      out.assign((size_t)(res + 3) * N + 1, -4242.f);
      rc = mp_launch_query_grad(&m.mlp, &ef.feat, emu_rows_src(in), in.cal, nullptr, N, out.data(), N,
                                out.data() + (size_t)res * N, N, nullptr, MP_GUARD_NONE, bt);
    } else {
      const int lres = atoi(argv[6]);
      std::vector<int32_t> idx;
      int32_t node_count;
      const MpPointSrc src = emu_node_src(atoi(argv[5]), lres, idx, node_count);
      out.assign((size_t)lres * lres * lres + 1, -4242.f);
      MpOutDst dst;
      dst.out = nullptr; dst.ld = 0; dst.scatter_vol = out.data();
      rc = mp_launch_query_fp32(&m.mlp, &ef.feat, src, in.cal, dst, nullptr, MP_GUARD_NONE, bt);
    }
    if (rc != MP_OK) { fprintf(stderr, "launch: %s (%d)\n", g_err, rc); return 3; }
    if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
    emu_write(path, out.data(), out.size() - 1);
    return 0;
  });
}
