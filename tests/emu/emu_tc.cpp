// TEST INFRASTRUCTURE ONLY: monoport_b200/csrc/query_tc.cu -- host-side weight packing, the launchers, the per-frame G0 GEMM
// kernel, the fused wgmma query program, its forward-mode gradient program, the surface render and the in-image grid
// compaction -- compiled UNMODIFIED for the CPU on the functional model of tc_ptx_emu.h.  The command line is emu_host.h's:
//   emu_tc in.bin out.f32 query [--batch B]     mp_launch_query_tc on the points of in.bin; out = [B][res][N].  --batch: one
//                                               launch over the B maps, point sets and calibs of a batched in.bin (the G0
//                                               kernel on a texel-blocks x B grid, the range guard decided per tile)
//   emu_tc in.bin out.f32 grid R z0 nz          the node centres of planes [z0, z0+nz) of an R^3 grid over [-1,1]^3,
//                                               generated in-kernel (mp_query_grid); out = the nz*R*R values
//   emu_tc in.bin out.f32 nodes R res           every third node of the res^3 level of an R^3 pyramid, through an index list
//                                               and a device-side count below the list's capacity, scattered into out = the
//                                               res^3 volume (the octree engine's fused path)
//     query, grid and nodes: --peers  the fused slab exchange: three "peer volumes" (host buffers here), checked to hold
//                                     the values at their offset and nothing else;
//                            --shard W  the query as W launches, launch r taking the r-th window of the point list (what
//                                     W GPUs do with list sharding: together they must give the unsharded result);
//                            --dump path  the G0 kernel's per-texel products (fp16 G0 [HW][1024], the fp16 map [HW][C],
//                                     fp32 S4 [HW]), for debugging the model
//   emu_tc in.bin out.f32 surface R [count bx0 by0 bz0 bx1 by1 bz1]
//                                               the colour head's render of the N vertex rows X, Y, Z of in.bin into an
//                                               [R,R,3] canvas of --canvas-bg (default 1): mp_launch_surface_tc with `count`
//                                               (default N, may exceed it) on the device, box default [-1,1]^3 -- what
//                                               mp_colorize_surface_async enqueues; --eager: mp_launch_colour_surface with
//                                               `count` counted on the host -- what mp_colorize_surface runs
//   emu_tc in.bin out.f32 jvp [grad_out.f32]    the forward-mode gradient program (grad_out [res][N], default ones); out =
//                                               the value [res][N], then d points [3][N].  --count k: the point count on the
//                                               device (N is then the capacity)
//   emu_tc in.bin out.f32 grid-in-image R lin0 n [--peers]
//                                               out = [2][n]: the dense MP_SRC_GRID launch of nodes [lin0, lin0 + n), then
//                                               mp_launch_query_tc_grid (the in-image list) of the same range; --peers: that
//                                               launch writes through two peer volumes of R^3 nodes, checked to be untouched
//                                               outside the range.  Prints the number of nodes in the image, by the
//                                               program's own predicate
//   emu_tc in.bin out.bin grid-brick R lin0 n   out.bin: int64 count, int64 size of the brick space; float [2][n] as
//                                               grid-in-image's; int32 list[count] (the scratch's list as the program read
//                                               it); int32 visits[n]: how many indices of the brick space map to each node
//                                               of the range; uint8 in[n]: the program's in-image predicate per node
// Outputs are pre-filled with -4242 (what a guarded launch skips, and the points at or beyond the device-side count, keep
// it).  --guard and --limit: the range guard of query, grid, nodes, jvp and the device-count surface render; --print-amax
// (query, grid, nodes, surface): the max |feature| of each map, which the G0 kernel leaves in the handle, on stdout.
// grid, nodes, jvp and the device-count surface render read --dcal (emu_output).
#include "emu_host.h"
#include "../../monoport_b200/csrc/query_tc.cu"

int mp_launch_query_fp32(const mp_mlp*, const mp_feat*, const MpPointSrc&, const MpCalib&, const MpOutDst&, cudaStream_t, int,
                         const MpBatch*) { return MP_E_UNSUPPORTED; }

static void print_amax(const EmuFeat& ef) {
  for (unsigned a : ef.amax) { float f; memcpy(&f, &a, 4); printf("%.9g\n", f); }
}

// the dense MP_SRC_GRID source of nodes [lin0, lin0 + n) of an R^3 grid over [-1,1]^3
static MpPointSrc grid_range(int R, long long lin0, long long n) {
  MpPointSrc grid;
  memset(&grid, 0, sizeof(grid));
  grid.kind = MP_SRC_GRID;
  mp_fill_grid_geom(grid, R, 1, R, kUnitMin, kUnitMax);
  grid.lin0 = lin0;
  grid.n = n;
  return grid;
}

// query, grid and nodes: one launch (W with --shard) of the tensor-core program
static int query(EmuArgs& a, const std::string& op, EmuInput& in, mp_mlp& mlp, EmuFeat& ef, int B, bool batched) {
  const int N = in.N, res = in.res;
  const int guard = emu_guard(a);
  const bool peers = a.get("peers"), amax = a.get("print-amax");
  const int shard_world = (int)a.num("shard", 1);
  const char* dump = a.get("dump");
  MpPointSrc src = emu_rows_src(in);
  std::vector<int32_t> nodes;
  int32_t node_count = 0;
  long long n_out = N;            // points per image (nodes: the volume)
  if (op == "grid") {
    src = emu_grid_src(atoi(a.arg(0)), atoi(a.arg(1)), atoi(a.arg(2)));
    n_out = src.n;
  } else if (op == "nodes") {
    const int lres = atoi(a.arg(1));
    src = emu_node_src(atoi(a.arg(0)), lres, nodes, node_count);
    n_out = (long long)lres * lres * lres;
  }
  MpBatch batch;                  // (batched: the [R|t] rows come from the device calibs)
  batch.B = B;
  batch.pt_stride = 3ll * N;
  batch.out_stride = (long long)res * N;
  batch.calibs = in.calibs.empty() ? nullptr : in.calibs.data();
  const int n_peers = peers ? 3 : 0, peer_off = 5;
  const size_t n_vals = op == "nodes" ? n_out : (size_t)B * res * n_out;
  return emu_output(a, in.cal, op == "query" ? nullptr : a.get("dcal"), n_vals, -4242.f, [&](const MpBatch* bt, float* out) {
    MpOutDst dst;
    dst.out = out; dst.ld = n_out; dst.scatter_vol = nullptr;
    if (op == "nodes") { dst.out = nullptr; dst.ld = 0; dst.scatter_vol = out; }
    std::vector<std::vector<float>> peer(n_peers, std::vector<float>((size_t)n_out + 2 * peer_off, -4242.f));
    for (int p = 0; p < n_peers; ++p) dst.peer[p] = peer[p].data();
    dst.n_peers = n_peers;
    dst.peer_off = peer_off;
    int rc = MP_OK;
    for (int r = 0; r < shard_world && rc == MP_OK; ++r) {
      src.shard_rank = r;
      src.shard_world = shard_world;
      rc = mp_launch_query_tc(&mlp, &ef.feat, src, in.cal, dst, nullptr, guard, batched ? &batch : bt);
    }
    if (amax) print_amax(ef);
    if (rc != MP_OK) return rc;
    for (int p = 0; p < n_peers; ++p)
      for (long long i = 0; i < (long long)peer[p].size(); ++i) {
        float want = -4242.f;
        if (op != "nodes") { if (i >= peer_off && i < peer_off + n_out) want = out[i - peer_off]; }
        else if (i >= peer_off && i < peer_off + node_count) want = out[nodes[i - peer_off]];     // peers receive the value LIST
        if (memcmp(&peer[p][i], &want, 4) != 0) { fprintf(stderr, "peer volume %d differs at %lld\n", p, i); exit(3); }
      }
    if (dump && ef.feat.g0) {
      FILE* f = fopen(dump, "wb");
      fwrite(ef.feat.g0, 2, (size_t)in.H * in.W * 1024, f);
      fwrite(ef.feat.f16, 2, (size_t)in.H * in.W * in.C, f);
      fwrite(ef.feat.s4tex, 4, (size_t)in.H * in.W, f);
      fclose(f);
    }
    return rc;
  });
}

// grid-in-image and grid-brick: the dense launch of a grid range into out[0, n), the in-image launch into out[n, 2n)
static int in_image(EmuArgs& a, const std::string& op, EmuInput& in, mp_mlp& mlp, EmuFeat& ef) {
  const int R = atoi(a.arg(0));
  const long long lin0 = atoll(a.arg(1)), n = atoll(a.arg(2));
  const bool peers = op == "grid-in-image" && a.get("peers");
  std::vector<unsigned> nonfinite(1, 0u);
  ef.feat.nonfinite = nonfinite.data();
  const MpPointSrc grid = grid_range(R, lin0, n);
  const size_t bytes = mp_tc_grid_scratch_bytes(n);
  std::vector<uint8_t> scratch(bytes + 64, 0xAB);       // 64 guard bytes past the scratch
  memset(scratch.data(), 0, 16);
  std::vector<float> out(2 * (size_t)n + 1, -4242.f);
  a.done();
  MpOutDst dense;
  dense.out = out.data(); dense.ld = n; dense.scatter_vol = nullptr;
  MpOutDst dst = dense;
  dst.out = out.data() + n;
  std::vector<std::vector<float>> vols;
  if (peers) {
    vols.assign(2, std::vector<float>((size_t)R * R * R, -4242.f));
    dst.out = nullptr;
    for (int p = 0; p < 2; ++p) dst.peer[p] = vols[p].data();
    dst.n_peers = 2;
    dst.peer_off = lin0;
  }
  int rc = mp_launch_query_tc(&mlp, &ef.feat, grid, in.cal, dense, nullptr, MP_GUARD_NONE);
  if (rc == MP_OK) rc = mp_launch_query_tc_grid(&mlp, &ef.feat, grid, in.cal, dst, scratch.data(), nullptr, MP_GUARD_NONE);
  if (rc != MP_OK) { fprintf(stderr, "launch refused: %s (%d)\n", g_err, rc); return 3; }
  if (out[2 * (size_t)n] != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  for (size_t k = bytes; k < scratch.size(); ++k)
    if (scratch[k] != 0xAB) { fprintf(stderr, "wrote past the scratch\n"); return 3; }
  if (peers) {
    for (int p = 0; p < 2; ++p)
      for (long long i = 0; i < (long long)R * R * R; ++i) {
        const bool inside = i >= lin0 && i < lin0 + n;
        if (!inside && vols[p][i] != -4242.f) { fprintf(stderr, "peer volume %d written outside the range at %lld\n", p, i); return 3; }
        if (inside && memcmp(&vols[p][i], &vols[0][i], 4) != 0) { fprintf(stderr, "peer volumes differ at %lld\n", i); return 3; }
      }
    memcpy(out.data() + n, vols[0].data() + lin0, (size_t)n * 4);
  }
  std::vector<uint8_t> inside((size_t)n);
  long long listed = 0;
  for (long long i = 0; i < n; ++i) {
    float x, y, z, u, v, w;
    mp_load_point(grid, MpBatch(), 0, i, x, y, z);
    inside[(size_t)i] = tc_project_in_image(in.cal, x, y, z, u, v, w) ? 1 : 0;
    listed += inside[(size_t)i];
  }
  if (op == "grid-in-image") {
    emu_write(a.pos[1], out.data(), 2 * (size_t)n);
    printf("%lld\n", listed);
    return 0;
  }
  const int32_t* list = reinterpret_cast<const int32_t*>(scratch.data() + grid_list_offset(n));
  const long long count = list[-4];
  const BrickSpace bs = BrickSpace::of(R, lin0, n);
  std::vector<int32_t> visits((size_t)n, 0);
  for (long long j = 0; j < bs.size; ++j) {
    const long long i = bs.node(j);
    if (i >= 0) ++visits[(size_t)i];
  }
  FILE* f = fopen(a.pos[1], "wb");
  if (!f) { fprintf(stderr, "cannot write %s\n", a.pos[1]); return 3; }
  const long long head[2] = {count, bs.size};
  fwrite(head, 8, 2, f);
  fwrite(out.data(), 4, 2 * (size_t)n, f);
  fwrite(list, 4, (size_t)count, f);
  fwrite(visits.data(), 4, visits.size(), f);
  fwrite(inside.data(), 1, inside.size(), f);
  fclose(f);
  return 0;
}

int main(int argc, char** argv) {
  EmuArgs a(argc, argv);
  const std::string op = a.op("emu_tc in.bin out.f32 (query | grid R z0 nz | nodes R res | surface R [count bx0 by0 bz0 "
                                    "bx1 by1 bz1] | jvp [grad_out.f32] | grid-in-image R lin0 n | grid-brick R lin0 n) "
                                    "[--options]");
  const size_t nargs = a.pos.size() - 3;
  if (!((op == "query" && nargs == 0) || (op == "grid" && nargs == 3) || (op == "nodes" && nargs == 2) ||
        (op == "surface" && (nargs == 1 || nargs == 8)) || (op == "jvp" && nargs <= 1) ||
        ((op == "grid-in-image" || op == "grid-brick") && nargs == 3))) {
    fprintf(stderr, "bad op or argument count: %s\n", op.c_str());
    return 2;
  }
  const bool batched = op == "query" && a.get("batch");
  const int B = op == "query" ? (int)a.num("batch", 1) : 1;
  g_fake_sms = (int)a.num("sms", 3);
  EmuInput in = emu_read_input(a.pos[0], B, batched);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in, a);
  mp_mlp& mlp = m.mlp;
  tc::emu::set_smem(g_dyn_smem[0], sizeof(g_dyn_smem[0]), g_dyn_smem[1]);
  if (mp_tc_prepare(&mlp) != MP_OK || !mlp.tc_ok) { fprintf(stderr, "mp_tc_prepare: %s (tc_ok=%d)\n", g_err, mlp.tc_ok); return 3; }
  EmuFeat ef = emu_make_feat(in, B);
  int rc;
  if (op == "query" || op == "grid" || op == "nodes") {
    rc = query(a, op, in, mlp, ef, B, batched);
  } else if (op == "grid-in-image" || op == "grid-brick") {
    rc = in_image(a, op, in, mlp, ef);
  } else if (op == "jvp") {
    const int guard = emu_guard(a);
    const std::vector<float> gout = emu_read_file(a.arg(0), (size_t)res * N);
    MpPointSrc src = emu_rows_src(in);
    int32_t count = 0;
    if (a.get("count")) {
      count = (int32_t)a.num("count", 0);
      src.count_dev = &count;
    }
    rc = emu_output(a, in.cal, a.get("dcal"), (size_t)(res + 3) * N, -4242.f, [&](const MpBatch* bt, float* out) {
      return mp_launch_query_jvp_tc(&mlp, &ef.feat, src, in.cal, gout.empty() ? nullptr : gout.data(), N, out, N,
                                    out + (size_t)res * N, N, nullptr, guard, bt);
    });
  } else {                                                   // surface
    const int R = atoi(a.arg(0));
    const long long count = nargs > 1 ? atoll(a.arg(1)) : N;
    float bmin[3] = {-1.f, -1.f, -1.f}, bmax[3] = {1.f, 1.f, 1.f};
    if (nargs > 1) emu_box_args(a, 2, bmin, bmax);
    const EmuVerts v = emu_vertex_rows(in);
    const bool eager = a.get("eager"), amax = a.get("print-amax");
    const int guard = eager ? MP_GUARD_NONE : emu_guard(a);
    const char* dcal = eager ? nullptr : a.get("dcal");
    rc = emu_output(a, in.cal, dcal, (size_t)R * R * 3, (float)a.num("canvas-bg", 1.0), [&](const MpBatch* bt, float* out) {
      const int r = eager ? mp_launch_colour_surface(&mlp, &ef.feat, v.X.data(), v.Y.data(), v.Z.data(), count, R, bmin, bmax,
                                                     in.cal, out, nullptr)
                          : mp_launch_surface_tc(&mlp, &ef.feat, mp_surface_src(v.X.data(), v.Y.data(), v.Z.data(), &count, R,
                                                                                bmin, bmax, out), N, in.cal, nullptr, guard, bt);
      if (amax) print_amax(ef);
      return r;
    });
  }
  mp_tc_release(&mlp);
  return rc;
}
