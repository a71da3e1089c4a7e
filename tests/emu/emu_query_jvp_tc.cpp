// TEST INFRASTRUCTURE ONLY: the forward-mode gradient program of monoport_b200/csrc/query_tc.cu (query_jvp_kernel, with
// the per-frame G0 kernel before it) compiled UNMODIFIED for the CPU against the execution-model emulation (cuda_emu.h) and
// the functional model of the wgmma / mbarrier / bulk-copy layer (tc_ptx_emu.h).  The host-side stand-ins are those of
// emu_query_tc.cpp, which it includes.
//   emu_query_jvp_tc in.bin out.f32 sms [grad_out.f32]
// in.bin: the layout of emu_query_tc (one map).  out.f32: value [res][N], then dpoints [3][N], pre-filled with -4242 (what a
// guarded launch skips, and the points at or beyond the device-side count, keep it).
// EMU_TC_LIMIT / EMU_TC_GUARD: the range guard as in emu_query_tc; EMU_COUNT=k: the point count on the device (n = N is
// then the capacity).
#define main emu_query_tc_main
#include "emu_query_tc.cpp"
#undef main

int main(int argc, char** argv) {
  if (argc < 4) { fprintf(stderr, "usage: emu_query_jvp_tc in.bin out.f32 sms [grad_out.f32]\n"); return 2; }
  g_fake_sms = atoi(argv[3]);
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  int32_t hd[8];
  float zs, calib[12];
  if (fread(hd, 4, 8, f) != 8 || fread(&zs, 4, 1, f) != 1 || fread(calib, 4, 12, f) != 12) { fprintf(stderr, "short header\n"); return 2; }
  const int C = hd[0], H = hd[1], W = hd[2], N = hd[3], has_calib = hd[4], persp = hd[5], res = hd[6], last_op = hd[7];
  auto rd = [&](FILE* in, size_t n) { std::vector<float> v(n); if (fread(v.data(), 4, n, in) != n) { fprintf(stderr, "short file\n"); exit(2); } return v; };
  std::vector<float> nchw = rd(f, (size_t)C * H * W), pts = rd(f, (size_t)3 * N);
  const int chans[6] = {C + 1, 1024, 512, 256, 128, res};
  mp_mlp mlp;
  memset(&mlp, 0, sizeof(mlp));
  mlp.n_layers = 5; mlp.skip = 1; mlp.last_op = last_op;
  mlp.gen = 1;
  mlp.tc_amax_limit = getenv("EMU_TC_LIMIT") ? (float)atof(getenv("EMU_TC_LIMIT")) : INFINITY;
  const int guard = getenv("EMU_TC_GUARD") ? atoi(getenv("EMU_TC_GUARD")) : MP_GUARD_NONE;
  std::vector<std::vector<float>> Ws(5), Bs(5);
  for (int l = 0; l <= 5; ++l) mlp.channels[l] = chans[l];
  for (int l = 0; l < 5; ++l) {
    mlp.cin[l] = chans[l] + (l ? chans[0] : 0);
    mlp.cout[l] = chans[l + 1];
    Ws[l] = rd(f, (size_t)mlp.cin[l] * mlp.cout[l]);
    Bs[l] = rd(f, mlp.cout[l]);
    mlp.w[l] = Ws[l].data();
    mlp.bias[l] = Bs[l].data();
  }
  fclose(f);
  std::vector<float> gout;
  if (argc >= 5) {
    FILE* g = fopen(argv[4], "rb");
    if (!g) { perror(argv[4]); return 2; }
    gout = rd(g, (size_t)res * N);
    fclose(g);
  }
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
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_ROWS;
  src.px = pts.data(); src.py = pts.data() + N; src.pz = pts.data() + 2 * (size_t)N;
  src.pstride = 1;
  src.n = N;
  int32_t count = 0;
  if (getenv("EMU_COUNT")) {
    count = atoi(getenv("EMU_COUNT"));
    src.count_dev = &count;
  }
  MpCalib cal;
  memset(&cal, 0, sizeof(cal));
  cal.has = has_calib;
  memcpy(cal.m, calib, sizeof(calib));
  cal.perspective = persp && has_calib;
  cal.z_scale = zs;
  std::vector<float> out((size_t)(res + 3) * N + 1, -4242.f);
  const int rc = mp_launch_query_jvp_tc(&mlp, &feat, src, cal, gout.empty() ? nullptr : gout.data(), N, out.data(), N,
                                        out.data() + (size_t)res * N, N, nullptr, guard);
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_jvp_tc: %s\n", g_err); return 3; }
  if (out[(size_t)(res + 3) * N] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  f = fopen(argv[2], "wb");
  fwrite(out.data(), 4, (size_t)(res + 3) * N, f);
  fclose(f);
  mp_tc_release(&mlp);
  return 0;
}
