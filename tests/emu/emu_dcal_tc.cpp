// TEST INFRASTRUCTURE ONLY: the programs of monoport_b200/csrc/query_tc.cu launched with the camera in device memory (a
// single-map MpBatch whose calibs point at a 12-float buffer; see dcal_emu.h), compiled UNMODIFIED for the CPU against the
// execution-model emulation and the functional model of the wgmma layer.  The host-side stand-ins are emu_query_tc.cpp's,
// which it includes.
//   emu_dcal_tc in.bin out.f32 sms (nodes R res | grid R z0 nz | surface R count bx0 by0 bz0 bx1 by1 bz1 | jvp)
//   nodes  : the query over every third node of the res^3 level of an R^3 pyramid over [-1,1]^3 (index list, count on the
//            device), scattered into the res^3 volume = out
//   grid   : the query over planes [z0, z0+nz) of an R^3 grid over [-1,1]^3; out = the nz*R*R values
//   surface: the colour head's render of the N vertex rows of in.bin (capacity N, `count` on the device) over the box into an
//            [R,R,3] canvas of ones = out (what mp_colorize_surface_async enqueues)
//   jvp    : the forward-mode gradient program on the N points of in.bin; out = value [res][N], then dpoints [3][N]
// in.bin: the layout of emu_query_tc (one map).  EMU_DCAL (dcal_emu.h) selects the device camera; without it the launch
// takes the camera by value, so the two runs can be compared.
#define main emu_query_tc_main
#include "emu_query_tc.cpp"
#undef main
#include "dcal_emu.h"

int main(int argc, char** argv) {
  if (argc < 5) {
    fprintf(stderr, "usage: emu_dcal_tc in.bin out.f32 sms (nodes R res | grid R z0 nz | surface R count box[6] | jvp)\n");
    return 2;
  }
  g_fake_sms = atoi(argv[3]);
  const std::string mode = argv[4];
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  int32_t hd[8];
  float zs, calib[12];
  if (fread(hd, 4, 8, f) != 8 || fread(&zs, 4, 1, f) != 1 || fread(calib, 4, 12, f) != 12) { fprintf(stderr, "short header\n"); return 2; }
  const int C = hd[0], H = hd[1], W = hd[2], N = hd[3], has_calib = hd[4], persp = hd[5], res = hd[6], last_op = hd[7];
  auto rd = [&](size_t n) { std::vector<float> v(n); if (fread(v.data(), 4, n, f) != n) { fprintf(stderr, "short file\n"); exit(2); } return v; };
  std::vector<float> nchw = rd((size_t)C * H * W), pts = rd((size_t)3 * N);
  const int chans[6] = {C + 1, 1024, 512, 256, 128, res};
  mp_mlp mlp;
  memset(&mlp, 0, sizeof(mlp));
  mlp.n_layers = 5; mlp.skip = 1; mlp.last_op = last_op;
  mlp.gen = 1;
  mlp.tc_amax_limit = INFINITY;
  std::vector<std::vector<float>> Ws(5), Bs(5);
  for (int l = 0; l <= 5; ++l) mlp.channels[l] = chans[l];
  for (int l = 0; l < 5; ++l) {
    mlp.cin[l] = chans[l] + (l ? chans[0] : 0);
    mlp.cout[l] = chans[l + 1];
    Ws[l] = rd((size_t)mlp.cin[l] * mlp.cout[l]);
    Bs[l] = rd(mlp.cout[l]);
    mlp.w[l] = Ws[l].data();
    mlp.bias[l] = Bs[l].data();
  }
  fclose(f);
  tc::emu::set_smem(g_dyn_smem[0], sizeof(g_dyn_smem[0]), g_dyn_smem[1]);
  if (mp_tc_prepare(&mlp) != MP_OK || !mlp.tc_ok) { fprintf(stderr, "mp_tc_prepare: %s (tc_ok=%d)\n", g_err, mlp.tc_ok); return 3; }
  std::vector<float> nhwc((size_t)C * H * W);
  for (int c = 0; c < C; ++c)
    for (int p = 0; p < H * W; ++p) nhwc[(size_t)p * C + c] = nchw[(size_t)c * H * W + p];
  mp_feat feat;
  memset(&feat, 0, sizeof(feat));
  feat.B = 1; feat.C = C; feat.H = H; feat.W = W; feat.nhwc32 = nhwc.data(); feat.version = 1;
  unsigned amax = 0u;
  feat.amax = &amax;
  MpCalib cal;
  memset(&cal, 0, sizeof(cal));
  cal.has = has_calib;
  memcpy(cal.m, calib, sizeof(calib));
  cal.perspective = persp && has_calib;
  cal.z_scale = zs;

  std::vector<int32_t> nodes;
  int32_t node_count = 0;
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_ROWS;
  src.px = pts.data(); src.py = pts.data() + N; src.pz = pts.data() + 2 * (size_t)N;
  src.pstride = 1;
  src.n = N;
  long long n_out = 0;
  if (mode == "nodes" && argc == 7) {
    const int R = atoi(argv[5]), lres = atoi(argv[6]);
    for (int i = 0; i < lres * lres * lres; i += 3) nodes.push_back(i);
    node_count = (int32_t)nodes.size();
    nodes.resize(nodes.size() + 300, 0);            // capacity beyond the count: must not be evaluated
    memset(&src, 0, sizeof(src));
    src.kind = MP_SRC_NODES;
    fill_grid_geom(src, lres, (R - 1) / (lres - 1), R);
    src.nodes = nodes.data();
    src.count_dev = &node_count;
    src.n = (long long)nodes.size();
    n_out = (long long)lres * lres * lres;
  } else if (mode == "grid" && argc == 8) {
    const int R = atoi(argv[5]), z0 = atoi(argv[6]), nz = atoi(argv[7]);
    memset(&src, 0, sizeof(src));
    src.kind = MP_SRC_GRID;
    fill_grid_geom(src, R, 1, R);
    src.z0 = z0;
    src.lin0 = (long long)z0 * R * R;
    src.n = (long long)nz * R * R;
    n_out = src.n;
  } else if (!(mode == "surface" && argc == 13) && !(mode == "jvp" && argc == 5)) {
    fprintf(stderr, "bad mode or argument count\n");
    return 2;
  }

  const int rc_all = emu_dcal_run(cal, calib, argv[2], [&](const MpBatch* bt, const char* path) {
    std::vector<float> out;
    int rc;
    if (mode == "surface") {
      const int R = atoi(argv[5]);
      const long long count = atoll(argv[6]);
      float bmin[3], bmax[3];
      for (int a = 0; a < 3; ++a) { bmin[a] = strtof(argv[7 + a], nullptr); bmax[a] = strtof(argv[10 + a], nullptr); }
      std::vector<long long> X(N), Y(N);
      std::vector<float> Z(N);
      for (int i = 0; i < N; ++i) { X[i] = (long long)pts[i]; Y[i] = (long long)pts[(size_t)N + i]; Z[i] = pts[2 * (size_t)N + i]; }
      out.assign((size_t)R * R * 3 + 1, 1.0f);
      out.back() = -4242.f;
      const MpSurfaceSrc surf = mp_surface_src(X.data(), Y.data(), Z.data(), &count, R, bmin, bmax, out.data());
      rc = mp_launch_surface_tc(&mlp, &feat, surf, N, cal, nullptr, MP_GUARD_NONE, bt);
    } else if (mode == "jvp") {
      out.assign((size_t)(res + 3) * N + 1, -4242.f);
      rc = mp_launch_query_jvp_tc(&mlp, &feat, src, cal, nullptr, N, out.data(), N, out.data() + (size_t)res * N, N, nullptr,
                                  MP_GUARD_NONE, bt);
    } else {
      out.assign((size_t)n_out + 1, -4242.f);
      MpOutDst dst;
      dst.out = out.data(); dst.ld = n_out; dst.scatter_vol = nullptr;
      if (mode == "nodes") { dst.out = nullptr; dst.ld = 0; dst.scatter_vol = out.data(); }
      rc = mp_launch_query_tc(&mlp, &feat, src, cal, dst, nullptr, MP_GUARD_NONE, bt);
    }
    if (rc != MP_OK) { fprintf(stderr, "launch: %s (%d)\n", g_err, rc); return 3; }
    if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
    FILE* fo = fopen(path, "wb");
    fwrite(out.data(), 4, out.size() - 1, fo);
    fclose(fo);
    return 0;
  });
  mp_tc_release(&mlp);
  return rc_all;
}
