// TEST INFRASTRUCTURE ONLY: the brick-ordered in-image list of monoport_b200/csrc/query_tc.cu (mp_launch_query_tc_grid)
// compiled UNMODIFIED for the CPU (see emu_host.h).
//   emu_query_grid_brick in.bin out.bin sms R lin0 n
// out.bin: int64 count, int64 size of the brick space; float [2][n]: the dense MP_SRC_GRID launch of nodes [lin0, lin0 + n),
// then the in-image launch of the same range into a buffer pre-filled with -4242; int32 list[count] (the scratch's list as
// the program read it); int32 visits[n]: how many indices of the brick space map to each node of the range; uint8 in[n]:
// the program's own in-image predicate per node, in ascending order.
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_tc.cu"

int mp_launch_query_fp32(const mp_mlp*, const mp_feat*, const MpPointSrc&, const MpCalib&, const MpOutDst&, cudaStream_t, int,
                         const MpBatch*) { return MP_E_UNSUPPORTED; }

int main(int argc, char** argv) {
  if (argc < 7) { fprintf(stderr, "usage: emu_query_grid_brick in.bin out.bin sms R lin0 n\n"); return 2; }
  g_fake_sms = atoi(argv[3]);
  const int R = atoi(argv[4]);
  const long long lin0 = atoll(argv[5]), n = atoll(argv[6]);
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
  std::vector<float> out(2 * (size_t)n, -4242.f);
  MpOutDst dense;
  dense.out = out.data(); dense.ld = n; dense.scatter_vol = nullptr;
  if (mp_launch_query_tc(&mlp, &ef.feat, grid, in.cal, dense, nullptr, MP_GUARD_NONE) != MP_OK) {
    fprintf(stderr, "dense launch: %s\n", g_err);
    return 3;
  }
  MpOutDst dst;
  dst.out = out.data() + n; dst.ld = n; dst.scatter_vol = nullptr;
  const size_t bytes = mp_tc_grid_scratch_bytes(n);
  std::vector<uint8_t> scratch(bytes + 64, 0xAB);       // 64 guard bytes past the scratch
  memset(scratch.data(), 0, 16);
  if (mp_launch_query_tc_grid(&mlp, &ef.feat, grid, in.cal, dst, scratch.data(), nullptr, MP_GUARD_NONE) != MP_OK) {
    fprintf(stderr, "in-image launch: %s\n", g_err);
    return 3;
  }
  for (size_t k = bytes; k < scratch.size(); ++k)
    if (scratch[k] != 0xAB) { fprintf(stderr, "wrote past the scratch\n"); return 3; }
  const int32_t* list = reinterpret_cast<const int32_t*>(scratch.data() + grid_list_offset(n));
  const long long count = list[-4];
  const BrickSpace bs = BrickSpace::of(R, lin0, n);
  std::vector<int32_t> visits((size_t)n, 0);
  for (long long j = 0; j < bs.size; ++j) {
    const long long i = bs.node(j);
    if (i >= 0) ++visits[(size_t)i];
  }
  std::vector<uint8_t> inside((size_t)n);
  for (long long i = 0; i < n; ++i) {
    float x, y, z, u, v, w;
    mp_load_point(grid, MpBatch(), 0, i, x, y, z);
    inside[(size_t)i] = tc_project_in_image(in.cal, x, y, z, u, v, w) ? 1 : 0;
  }
  FILE* f = fopen(argv[2], "wb");
  if (!f) { fprintf(stderr, "cannot write %s\n", argv[2]); return 3; }
  const long long head[2] = {count, bs.size};
  fwrite(head, 8, 2, f);
  fwrite(out.data(), 4, out.size(), f);
  fwrite(list, 4, (size_t)count, f);
  fwrite(visits.data(), 4, visits.size(), f);
  fwrite(inside.data(), 1, inside.size(), f);
  fclose(f);
  mp_tc_release(&mlp);
  return 0;
}
