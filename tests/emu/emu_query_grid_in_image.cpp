// TEST INFRASTRUCTURE ONLY: the in-image grid launch of monoport_b200/csrc/query_tc.cu (mp_launch_query_tc_grid: the ordered
// compaction of mp_scan.cuh, then the tensor-core program over the node list) compiled UNMODIFIED for the CPU (see emu_host.h).
//   emu_query_grid_in_image in.bin out.f32 sms R lin0 n [peers]
// out.f32: [2][n] -- the dense MP_SRC_GRID launch of nodes [lin0, lin0 + n), then the in-image launch of the same range into
// a buffer pre-filled with -4242 (every node must be written once: listed, or +0).  peers: the in-image launch writes through
// two peer volumes of R^3 nodes instead (the fused slab exchange), and the harness checks that nothing outside the range is
// touched.  Prints the number of nodes in the image, by the program's own predicate.
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_tc.cu"

int mp_launch_query_fp32(const mp_mlp*, const mp_feat*, const MpPointSrc&, const MpCalib&, const MpOutDst&, cudaStream_t, int,
                         const MpBatch*) { return MP_E_UNSUPPORTED; }

int main(int argc, char** argv) {
  if (argc < 7) { fprintf(stderr, "usage: emu_query_grid_in_image in.bin out.f32 sms R lin0 n [peers]\n"); return 2; }
  g_fake_sms = atoi(argv[3]);
  const int R = atoi(argv[4]);
  const long long lin0 = atoll(argv[5]), n = atoll(argv[6]);
  const bool peers = argc >= 8 && !strcmp(argv[7], "peers");
  EmuInput in = emu_read_input(argv[1]);
  EmuMlp m = emu_make_mlp(in);
  mp_mlp& mlp = m.mlp;
  tc::emu::set_smem(g_dyn_smem[0], sizeof(g_dyn_smem[0]), g_dyn_smem[1]);
  if (mp_tc_prepare(&mlp) != MP_OK || !mlp.tc_ok) { fprintf(stderr, "mp_tc_prepare: %s (tc_ok=%d)\n", g_err, mlp.tc_ok); return 3; }
  EmuFeat ef = emu_make_feat(in);
  std::vector<unsigned> nonfinite(1, 0u);
  ef.feat.nonfinite = nonfinite.data();
  MpPointSrc grid;
  memset(&grid, 0, sizeof(grid));
  grid.kind = MP_SRC_GRID;
  mp_fill_grid_geom(grid, R, 1, R, kUnitMin, kUnitMax);
  grid.lin0 = lin0;
  grid.n = n;
  std::vector<float> out(2 * (size_t)n + 1, -4242.f);
  MpOutDst dense;
  dense.out = out.data(); dense.ld = n; dense.scatter_vol = nullptr;
  if (mp_launch_query_tc(&mlp, &ef.feat, grid, in.cal, dense, nullptr, MP_GUARD_NONE) != MP_OK) {
    fprintf(stderr, "dense launch: %s\n", g_err);
    return 3;
  }
  MpOutDst dst;
  dst.out = out.data() + n; dst.ld = n; dst.scatter_vol = nullptr;
  std::vector<std::vector<float>> vols;
  if (peers) {
    vols.assign(2, std::vector<float>((size_t)R * R * R, -4242.f));
    dst.out = nullptr;
    for (int p = 0; p < 2; ++p) dst.peer[p] = vols[p].data();
    dst.n_peers = 2;
    dst.peer_off = lin0;
  }
  std::vector<uint8_t> scratch(mp_tc_grid_scratch_bytes(n), 0xAB);
  memset(scratch.data(), 0, 16);
  if (mp_launch_query_tc_grid(&mlp, &ef.feat, grid, in.cal, dst, scratch.data(), nullptr, MP_GUARD_NONE) != MP_OK) {
    fprintf(stderr, "in-image launch: %s\n", g_err);
    return 3;
  }
  if (out[2 * (size_t)n] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  if (peers) {
    for (int p = 0; p < 2; ++p)
      for (long long i = 0; i < (long long)R * R * R; ++i) {
        const bool inside = i >= lin0 && i < lin0 + n;
        if (!inside && vols[p][i] != -4242.f) { fprintf(stderr, "peer volume %d written outside the range at %lld\n", p, i); return 3; }
        if (inside && memcmp(&vols[p][i], &vols[0][i], 4) != 0) { fprintf(stderr, "peer volumes differ at %lld\n", i); return 3; }
      }
    memcpy(out.data() + n, vols[0].data() + lin0, (size_t)n * 4);
  }
  long long listed = 0;
  for (long long i = 0; i < n; ++i) {
    float x, y, z, u, v, w;
    mp_load_point(grid, MpBatch(), 0, i, x, y, z);
    listed += tc_project_in_image(in.cal, x, y, z, u, v, w) ? 1 : 0;
  }
  emu_write(argv[2], out.data(), 2 * (size_t)n);
  printf("%lld\n", listed);
  mp_tc_release(&mlp);
  return 0;
}
