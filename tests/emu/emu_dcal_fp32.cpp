// TEST INFRASTRUCTURE ONLY: the kernels of monoport_b200/csrc/query_fp32.cu launched with the camera in device memory (a
// single-map MpBatch whose calibs point at a 12-float buffer; see dcal_emu.h), compiled unmodified on the CPU emulation
// layer.  The host-side stand-ins are emu_colour_surface_fp32.cpp's, which it includes.
//   emu_dcal_fp32 in.bin out.f32 sms (nodes R res | surface R count bx0 by0 bz0 bx1 by1 bz1 | grad)
//   nodes  : the exact query over every third node of the res^3 level of an R^3 pyramid over [-1,1]^3 (index list, count
//            on the device), scattered into the res^3 volume = out (what the octree engine's fused path launches)
//   surface: the exact surface render of the N vertex rows of in.bin (capacity N, `count` on the device) over the box into
//            an [R,R,3] canvas of ones = out
//   grad   : the gradient kernel on the N points of in.bin; out = value [res][N], then dpoints [3][N]
// in.bin as for emu_query_fp32.  EMU_DCAL (dcal_emu.h) selects the device camera; without it the launch takes the camera by
// value, so the two runs can be compared.
#define main emu_colour_surface_fp32_main
#include "emu_colour_surface_fp32.cpp"
#undef main
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
  mlp.tc_amax_limit = INFINITY;
  std::vector<std::vector<float>> Ws(5), Wt(5), Bs(5);
  for (int l = 0; l <= 5; ++l) mlp.channels[l] = chans[l];
  for (int l = 0; l < 5; ++l) {
    const int cin = chans[l] + (l ? chans[0] : 0), cout = chans[l + 1];
    mlp.cin[l] = cin; mlp.cout[l] = cout;
    Ws[l] = rd((size_t)cin * cout);
    Bs[l] = rd(cout);
    Wt[l].resize((size_t)cin * cout);                    // what transpose_w_kernel produces: [cin][cout]
    for (int o = 0; o < cout; ++o)
      for (int k = 0; k < cin; ++k) Wt[l][(size_t)k * cout + o] = Ws[l][(size_t)o * cin + k];
    mlp.w[l] = Ws[l].data(); mlp.wt[l] = Wt[l].data(); mlp.bias[l] = Bs[l].data();
  }
  fclose(f);
  std::vector<float> nhwc((size_t)C * H * W);
  for (int c = 0; c < C; ++c)
    for (int p = 0; p < H * W; ++p) nhwc[(size_t)p * C + c] = nchw[(size_t)c * H * W + p];
  mp_feat feat;
  memset(&feat, 0, sizeof(feat));
  feat.B = 1; feat.C = C; feat.H = H; feat.W = W; feat.nhwc32 = nhwc.data();
  unsigned amax = 0u;
  feat.amax = &amax;
  MpCalib cal;
  memset(&cal, 0, sizeof(cal));
  cal.has = has_calib;
  memcpy(cal.m, calib, sizeof(calib));
  cal.perspective = persp && has_calib;
  cal.z_scale = zs;

  return emu_dcal_run(cal, calib, argv[2], [&](const MpBatch* bt, const char* path) {
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
      rc = mp_launch_surface_fp32(&mlp, &feat, surf, N, cal, nullptr, MP_GUARD_NONE, bt);
    } else if (mode == "grad") {
      MpPointSrc src;
      memset(&src, 0, sizeof(src));
      src.kind = MP_SRC_ROWS;
      src.px = pts.data(); src.py = pts.data() + N; src.pz = pts.data() + 2 * (size_t)N;
      src.pstride = 1;
      src.n = N;
      out.assign((size_t)(res + 3) * N + 1, -4242.f);
      rc = mp_launch_query_grad(&mlp, &feat, src, cal, nullptr, N, out.data(), N, out.data() + (size_t)res * N, N, nullptr,
                                MP_GUARD_NONE, bt);
    } else {
      // every third node of the level, an index list longer than the device-side count (what octree.cu sets up)
      const int R = atoi(argv[5]), lres = atoi(argv[6]);
      std::vector<int32_t> idx;
      for (int i = 0; i < lres * lres * lres; i += 3) idx.push_back(i);
      const int32_t node_count = (int32_t)idx.size();
      idx.resize(idx.size() + 300, 0);
      MpPointSrc src;
      memset(&src, 0, sizeof(src));
      src.kind = MP_SRC_NODES;
      src.res = lres; src.node_stride = (R - 1) / (lres - 1); src.r_final = R;
      src.inv_r = 1.0f / (float)R;
      src.half_inv_r = (float)(1.0 / (2.0 * (double)R));
      for (int a = 0; a < 3; ++a) { src.bmin[a] = -1.f; src.bext[a] = 1.f - (-1.f); }
      src.nodes = idx.data();
      src.count_dev = &node_count;
      src.n = (long long)idx.size();
      out.assign((size_t)lres * lres * lres + 1, -4242.f);
      MpOutDst dst;
      dst.out = nullptr; dst.ld = 0; dst.scatter_vol = out.data();
      rc = mp_launch_query_fp32(&mlp, &feat, src, cal, dst, nullptr, MP_GUARD_NONE, bt);
    }
    if (rc != MP_OK) { fprintf(stderr, "launch: %s (%d)\n", g_err, rc); return 3; }
    if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
    FILE* fo = fopen(path, "wb");
    fwrite(out.data(), 4, out.size() - 1, fo);
    fclose(fo);
    return 0;
  });
}
