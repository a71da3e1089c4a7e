// TEST INFRASTRUCTURE ONLY: monoport_b200/csrc/query_tc.cu -- host-side weight packing, launch logic, the per-frame G0
// GEMM kernel and the fused wgmma sample+MLP kernel -- compiled UNMODIFIED for the CPU (see emu_host.h).
//   emu_query_tc in.bin out.f32 program sms [grid R z0 nz | nodes R res | surface R | batch B]
// in.bin: see emu_host.h.  out.f32: [res][N].
// batch B: the batched launch (what mp_query_points_batch sets up: one launch over B images, the per-frame G0 kernel on a
//   texel-blocks x B grid, the range guard decided per tile).  in.bin then holds B feature maps, B point sets and, when
//   has_calib, B calibs; out.f32 is [B][res][N], pre-filled with -4242 (the tiles a guarded launch skips keep it).
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_tc.cu"

int mp_launch_query_fp32(const mp_mlp*, const mp_feat*, const MpPointSrc&, const MpCalib&, const MpOutDst&, cudaStream_t, int,
                         const MpBatch*) { return MP_E_UNSUPPORTED; }

int main(int argc, char** argv) {
  // optional point source (default: the rows of in.bin):  grid R z0 nz   |   nodes R res   |   surface R
  //   grid : node centres of planes [z0, z0+nz) of an R^3 grid over [-1,1]^3, generated in-kernel (mp_query_grid)
  //   nodes: every third node of the res^3 level of an R^3 pyramid, through an index list + a device-side count that
  //          is smaller than the list capacity, scattered into a res^3 volume (the octree engine's fused path)
  const char* src_kind = argc >= 6 ? argv[5] : "rows";
  if (argc < 5) { fprintf(stderr, "usage: emu_query_tc in.bin out.f32 program sms [grid R z0 nz | nodes R res | surface R | batch B]\n"); return 2; }
  const bool batched = !strcmp(src_kind, "batch");
  const int B = batched ? atoi(argv[6]) : 1;
  const int program = atoi(argv[3]);
  g_fake_sms = atoi(argv[4]);
  EmuInput in = emu_read_input(argv[1], B, batched);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in);
  mp_mlp& mlp = m.mlp;
  const int guard = getenv("EMU_TC_GUARD") ? atoi(getenv("EMU_TC_GUARD")) : MP_GUARD_NONE;   // (see mp_query_dispatch)
  tc::emu::set_smem(g_dyn_smem[0], sizeof(g_dyn_smem[0]), g_dyn_smem[1]);
  if (mp_tc_prepare(&mlp) != MP_OK || !mlp.tc_ok) { fprintf(stderr, "mp_tc_prepare: %s (tc_ok=%d)\n", g_err, mlp.tc_ok); return 3; }
  if (getenv("EMU_TC_DEBUG")) {
    const TcPack* pk = static_cast<const TcPack*>(mlp.tc);
    fprintf(stderr, "d_bias0[0..3] = %g %g %g %g   d_wz0[0..1] = %g %g  h_bias[0]=%g\n", __half2float(pk->d_bias0[0]), __half2float(pk->d_bias0[1]),
            __half2float(pk->d_bias0[2]), __half2float(pk->d_bias0[3]), __half2float(pk->d_wz0[0]), __half2float(pk->d_wz0[1]), pk->h_bias[0]);
  }
  EmuFeat ef = emu_make_feat(in, B);
  mp_feat& feat = ef.feat;
  MpPointSrc src = emu_rows_src(in);
  const MpCalib& cal = in.cal;
  long long n_out = N;
  std::vector<int32_t> nodes;
  int32_t node_count = 0;
  std::vector<float> scatter;
  if (!strcmp(src_kind, "grid")) {
    src = emu_grid_src(atoi(argv[6]), atoi(argv[7]), atoi(argv[8]));
    n_out = src.n;
  } else if (!strcmp(src_kind, "nodes")) {
    const int lres = atoi(argv[7]);
    src = emu_node_src(atoi(argv[6]), lres, nodes, node_count);
    n_out = (long long)lres * lres * lres;
    scatter.assign(n_out, -4242.f);
  }
  if (!strcmp(src_kind, "surface")) {
    // surface R: the first N "points" of in.bin are visible-surface vertices; the colour head renders them into an [R,R,3]
    // canvas of ones (mp_colorize_surface)
    const int R = atoi(argv[6]);
    const EmuVerts v = emu_vertex_rows(in);
    std::vector<float> canvas((size_t)R * R * 3 + 1, 1.0f);
    canvas[(size_t)R * R * 3] = -4242.f;
    const int rc = mp_launch_colour_surface(&mlp, &feat, v.X.data(), v.Y.data(), v.Z.data(), N, R, kUnitMin, kUnitMax, cal,
                                            canvas.data(), nullptr);
    if (rc != MP_OK) { fprintf(stderr, "mp_launch_colour_surface: %s\n", g_err); return 3; }
    if (canvas[(size_t)R * R * 3] != -4242.f) { fprintf(stderr, "wrote past the canvas\n"); return 3; }
    emu_write(argv[2], canvas.data(), (size_t)R * R * 3);
    mp_tc_release(&mlp);
    return 0;
  }
  MpBatch bt;                     // (batched: the [R|t] rows come from the device calibs)
  bt.B = B;
  bt.pt_stride = 3ll * N;
  bt.out_stride = (long long)res * N;
  bt.calibs = in.calibs.empty() ? nullptr : in.calibs.data();
  std::vector<float> out((size_t)B * res * n_out + 1, -4242.f);
  MpOutDst dst;
  dst.out = out.data(); dst.ld = n_out; dst.scatter_vol = nullptr;
  if (!scatter.empty()) { dst.out = nullptr; dst.ld = 0; dst.scatter_vol = scatter.data(); }
  // program 1xx: tensor-core program xx with the fused slab exchange -- three "peer volumes" (host buffers here)
  const int n_peers = program >= 100 ? 3 : 0, peer_off = 5;
  std::vector<std::vector<float>> peer(n_peers, std::vector<float>((size_t)n_out + 2 * peer_off, -4242.f));
  for (int p = 0; p < n_peers; ++p) dst.peer[p] = peer[p].data();
  dst.n_peers = n_peers;
  dst.peer_off = peer_off;
  if (program % 100 != 3 && program % 100 != 0) { fprintf(stderr, "unknown program %d (3 = the tensor-core program, 103 = with peer stores)\n", program); return 2; }
  // EMU_SHARD_WORLD=W: the query is evaluated as W launches, launch r taking the r-th window of the point list (what W
  // GPUs do with list sharding; here they share the output buffers, so together they must reproduce the unsharded result)
  const int shard_world = getenv("EMU_SHARD_WORLD") ? atoi(getenv("EMU_SHARD_WORLD")) : 1;
  int rc = MP_OK;
  for (int r = 0; r < shard_world && rc == MP_OK; ++r) {
    src.shard_rank = r;
    src.shard_world = shard_world;
    rc = mp_launch_query_tc(&mlp, &feat, src, cal, dst, nullptr, guard, batched ? &bt : nullptr);
  }
  if (getenv("EMU_TC_AMAX"))
    for (int b = 0; b < B; ++b) { float a; memcpy(&a, &ef.amax[b], 4); fprintf(stderr, "amax[%d] %.9g\n", b, a); }
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_tc: %s\n", g_err); return 3; }
  if (out[(size_t)B * res * n_out] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  if (!scatter.empty()) out.assign(scatter.begin(), scatter.end());       // report the scattered volume
  for (int p = 0; p < n_peers; ++p)
    for (long long i = 0; i < (long long)peer[p].size(); ++i) {
      float want = -4242.f;
      if (scatter.empty()) { if (i >= peer_off && i < peer_off + n_out) want = out[i - peer_off]; }
      else if (i >= peer_off && i < peer_off + node_count) want = scatter[nodes[i - peer_off]];     // peers receive the value LIST
      if (memcmp(&peer[p][i], &want, 4) != 0) { fprintf(stderr, "peer volume %d differs at %lld\n", p, i); return 3; }
    }
  emu_write(argv[2], out.data(), (size_t)B * res * n_out);
  if (const char* dump = getenv("EMU_TC_DUMP")) {       // per-texel products of the G0 kernel, for debugging the model
    if (feat.g0) {
      FILE* f = fopen(dump, "wb");
      fwrite(feat.g0, 2, (size_t)in.H * in.W * 1024, f);
      fwrite(feat.f16, 2, (size_t)in.H * in.W * in.C, f);
      fwrite(feat.s4tex, 4, (size_t)in.H * in.W, f);
      fclose(f);
    }
  }
  mp_tc_release(&mlp);
  return 0;
}
