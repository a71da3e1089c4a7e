// TEST INFRASTRUCTURE ONLY: the exact kernels of monoport_b200/csrc/query_fp32.cu -- the query, the point gradient and the
// surface render, the programs of the colour head and of every head the tensor-core programs do not cover -- and the
// training backward of query_vjp.cu (query_vjp_kernel, wgrad_kernel, the radix sort, the gather and the layout step),
// compiled unmodified on the CPU emulation layer and driven by the library's launchers.  The command line is emu_host.h's:
//   emu_fp32 in.bin out.f32 query [--batch B]   mp_launch_query_fp32 on the points of in.bin; out = [B][res][N].  --batch:
//                                               one launch over the B maps, point sets and calibs of a batched in.bin
//   emu_fp32 in.bin out.f32 nodes R res         the query over every third node of the res^3 level of an R^3 pyramid over
//                                               [-1,1]^3 (index list, count on the device), scattered into out = the res^3
//                                               volume (the octree engine's fused path)
//   emu_fp32 in.bin out.f32 grad [grad_out.f32] mp_launch_query_grad (grad_out [res][N], default ones); out = the value
//                                               [res][N], then the point gradient [3][N].  --count k: the point count on
//                                               the device (N is then the capacity)
//   emu_fp32 in.bin out.f32 surface R count bx0 by0 bz0 bx1 by1 bz1
//                                               mp_launch_surface_fp32 over the box: the N "points" of in.bin are vertex
//                                               rows X, Y, Z (capacity N, `count` on the device); out = the [R,R,3] canvas,
//                                               background --canvas-bg (default 1)
//   emu_fp32 in.bin out.f32 vjp B grad_out.f32|- chunk_points [want]
//                                               mp_launch_query_vjp on a batched in.bin of B maps; grad_out [B][res][N] or
//                                               - for ones; chunk_points per weight-gradient chunk (0: one chunk); want the
//                                               requested outputs as letters f (features), p (points), w (weights and
//                                               biases), default fpw.  out = d features [B][C][H][W], d points [B][3][N],
//                                               d W_l [cout][cin] of every layer, d b_l of every layer (zeros where not
//                                               requested).  --vjp-flags F (default 0); --wmask / --bmask M: bit l set =
//                                               d W_l / d b_l requested, every other entry of the launcher's arrays null,
//                                               every d W / d b output pre-filled with -7 (default: all layers); --dump path
//                                               (MP_VJP_DETERMINISTIC, want f, one chunk): the ordered feature gradient's
//                                               scratch -- int64 {columns, C}, then fp32 dX rows [columns][C], fp32 tap
//                                               weights [columns][4], the sorted uint32 keys and their columns -- and
//                                               "radix passes <p>" on stdout
//   emu_fp32 limit res last_op                  prints mp_tc_default_feature_limit(res, last_op)
// Outputs other than vjp's are pre-filled with -4242 (what a guarded launch skips, and the points at or beyond the
// device-side count, keep it).  The range guard of query, grad and surface: --guard, --limit and --amax (the frame's
// max |feature|, which the tensor-core program's G0 kernel would have left in the handle).  nodes, grad and surface read
// --dcal (emu_output).  Every launch of the exact kernels prints "launch P=<tile size>" on stdout: the instantiation the
// launcher's shared-memory fit chose.

// the launcher (launch<P, Kernel>) expands this inside its template: P is the tile size it launches
#define MP_EMU_LAUNCH(grid, block, call)                                                                                 \
  (printf("launch P=%d\n", P), cuda_emu::launch(dim3((unsigned)(grid)), dim3((unsigned)(block)), [&] { call; }))
#include <algorithm>

#include "emu_host.h"
#include "../../monoport_b200/csrc/query_fp32.cu"
#undef MP_EMU_LAUNCH
#define MP_EMU_LAUNCH(grid, block, call) cuda_emu::launch(dim3((unsigned)(grid)), dim3((unsigned)(block)), [&] { call; })
#include "../../monoport_b200/csrc/query_vjp.cu"

static int vjp(EmuArgs& a, EmuInput& in, EmuMlp& m, EmuFeat& ef, int B) {
  const int N = in.N, L = m.mlp.n_layers;
  const char* want = a.arg(3) ? a.arg(3) : "fpw";
  const bool wf = strchr(want, 'f'), wpt = strchr(want, 'p'), ww = strchr(want, 'w');
  const long long chunk_points = atoll(a.arg(2));
  const std::vector<float> gout = emu_read_file(strcmp(a.arg(1), "-") ? a.arg(1) : nullptr, (size_t)B * in.res * N);
  const int flags = (int)a.num("vjp-flags", 0);
  const char* dump = a.get("dump");
  const char* wmask = a.get("wmask");
  const char* bmask = a.get("bmask");
  size_t n_w = 0, n_b = 0;
  for (int l = 0; l < L; ++l) { n_w += (size_t)m.mlp.cout[l] * m.mlp.cin[l]; n_b += m.mlp.cout[l]; }
  const size_t n_f = (size_t)B * in.C * in.H * in.W, n_p = (size_t)B * 3 * N;
  MpBatch bt;
  bt.B = B;
  bt.pt_stride = 3 * (long long)N;
  bt.calibs = in.calibs.empty() ? nullptr : in.calibs.data();
  return emu_output(a, in.cal, nullptr, n_f + n_p + n_w + n_b, 0.f, [&](const MpBatch*, float* dfeat) {
    float* dp = dfeat + n_f;
    std::vector<float*> dw(L), db(L);
    float* q = dp + n_p;
    for (int l = 0; l < L; ++l) { dw[l] = q; q += (size_t)m.mlp.cout[l] * m.mlp.cin[l]; }
    for (int l = 0; l < L; ++l) { db[l] = q; q += m.mlp.cout[l]; }
    if (wmask || bmask) {
      std::fill(dp + n_p, q, -7.f);
      const long wm = wmask ? atol(wmask) : -1, bm = bmask ? atol(bmask) : -1;
      for (int l = 0; l < L; ++l) {
        if (!((wm >> l) & 1)) dw[l] = nullptr;
        if (!((bm >> l) & 1)) db[l] = nullptr;
      }
    }
    const long long bytes = mp_vjp_scratch_bytes(&m.mlp, &ef.feat, B, N, chunk_points, wf, ww, flags);
    if (bytes < 0) return (int)bytes;
    std::vector<float> scratch((size_t)bytes / 4 + 1);
    const int rc = mp_launch_query_vjp(&m.mlp, &ef.feat, emu_rows_src(in), in.cal, bt, gout.empty() ? nullptr : gout.data(),
                                       wf ? dfeat : nullptr, wpt ? dp : nullptr, ww ? dw.data() : nullptr,
                                       ww ? db.data() : nullptr, bytes ? scratch.data() : nullptr, bytes, nullptr, flags);
    if (rc != MP_OK || !dump) return rc;
    if (!(flags & MP_VJP_DETERMINISTIC) || !wf || chunk_points > 0) { fprintf(stderr, "--dump: one ordered chunk only\n"); exit(2); }
    // the launcher's layout of a single chunk of every tile
    const int P = mp_query_vjp_tile(&m.mlp);
    const long long cols = (long long)B * ((N + P - 1) / P) * P, HW = (long long)in.H * in.W;
    const size_t rows = ww ? (size_t)row_layout(&m.mlp).total * P * sizeof(float) * (size_t)(cols / P) : 0;
    const char* area = reinterpret_cast<const char*>(scratch.data()) + round256((size_t)B * HW * in.C * sizeof(float)) + round256(rows);
    const OrderedLayout ol = ordered_layout(cols, in.C);
    const int passes = radix_passes((unsigned long long)B * HW), sorted = passes & 1;
    printf("radix passes %d\n", passes);
    FILE* f = fopen(dump, "wb");
    const long long hd[2] = {cols, in.C};
    fwrite(hd, 8, 2, f);
    fwrite(area + ol.dx, 4, (size_t)cols * in.C, f);
    fwrite(area + ol.wgt, 4, (size_t)cols * 4, f);
    fwrite(area + ol.key[sorted], 4, (size_t)cols, f);
    fwrite(area + ol.col[sorted], 4, (size_t)cols, f);
    fclose(f);
    return rc;
  });
}

int main(int argc, char** argv) {
  if (argc == 4 && !strcmp(argv[1], "limit")) {
    printf("%.9g\n", mp_tc_default_feature_limit(atoi(argv[2]), atoi(argv[3])));
    return 0;
  }
  EmuArgs a(argc, argv);
  const std::string op = a.op("emu_fp32 in.bin out.f32 (query | nodes R res | grad [grad_out.f32] | "
                                    "surface R count bx0 by0 bz0 bx1 by1 bz1 | vjp B grad_out.f32|- chunk_points [want]) "
                                    "[--options]\n       emu_fp32 limit res last_op");
  const size_t nargs = a.pos.size() - 3;
  if (!((op == "query" && nargs == 0) || (op == "nodes" && nargs == 2) || (op == "grad" && nargs <= 1) ||
        (op == "surface" && nargs == 8) || (op == "vjp" && (nargs == 3 || nargs == 4)))) {
    fprintf(stderr, "bad op or argument count: %s\n", op.c_str());
    return 2;
  }
  const bool batched = op == "vjp" || (op == "query" && a.get("batch"));
  const int B = op == "vjp" ? atoi(a.arg(0)) : op == "query" ? (int)a.num("batch", 1) : 1;
  g_fake_sms = (int)a.num("sms", 3);
  EmuInput in = emu_read_input(a.pos[0], B, batched);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in, a);
  EmuFeat ef = emu_make_feat(in, B);
  if (op == "vjp") return vjp(a, in, m, ef, B);
  if (op == "nodes") {
    const int lres = atoi(a.arg(1));
    std::vector<int32_t> idx;
    int32_t node_count;
    const MpPointSrc src = emu_node_src(atoi(a.arg(0)), lres, idx, node_count);
    return emu_output(a, in.cal, a.get("dcal"), (size_t)lres * lres * lres, -4242.f, [&](const MpBatch* bt, float* out) {
      MpOutDst dst;
      dst.out = nullptr; dst.ld = 0; dst.scatter_vol = out;
      return mp_launch_query_fp32(&m.mlp, &ef.feat, src, in.cal, dst, nullptr, MP_GUARD_NONE, bt);
    });
  }
  const int guard = emu_guard(a);
  if (a.get("amax")) {
    const float amax = (float)a.num("amax", 0);
    memcpy(&ef.amax[0], &amax, 4);
  }
  if (op == "query") {
    MpBatch bt;                   // (batched: the [R|t] rows come from the device calibs)
    bt.B = B;
    bt.pt_stride = 3ll * N;
    bt.out_stride = (long long)res * N;
    bt.calibs = in.calibs.empty() ? nullptr : in.calibs.data();
    return emu_output(a, in.cal, nullptr, (size_t)B * res * N, -4242.f, [&](const MpBatch*, float* out) {
      MpOutDst dst;
      dst.out = out; dst.ld = N; dst.scatter_vol = nullptr;
      return mp_launch_query_fp32(&m.mlp, &ef.feat, emu_rows_src(in), in.cal, dst, nullptr, guard, batched ? &bt : nullptr);
    });
  }
  if (op == "grad") {
    const std::vector<float> gout = emu_read_file(a.arg(0), (size_t)res * N);
    MpPointSrc src = emu_rows_src(in);
    int32_t count = 0;
    if (a.get("count")) {
      count = (int32_t)a.num("count", 0);
      src.count_dev = &count;
    }
    return emu_output(a, in.cal, a.get("dcal"), (size_t)(res + 3) * N, -4242.f, [&](const MpBatch* bt, float* out) {
      return mp_launch_query_grad(&m.mlp, &ef.feat, src, in.cal, gout.empty() ? nullptr : gout.data(), N, out, N,
                                  out + (size_t)res * N, N, nullptr, guard, bt);
    });
  }
  const int R = atoi(a.arg(0));                              // surface
  const long long count = atoll(a.arg(1));
  float bmin[3], bmax[3];
  emu_box_args(a, 2, bmin, bmax);
  const EmuVerts v = emu_vertex_rows(in);
  return emu_output(a, in.cal, a.get("dcal"), (size_t)R * R * 3, (float)a.num("canvas-bg", 1.0), [&](const MpBatch* bt, float* out) {
    const MpSurfaceSrc surf = mp_surface_src(v.X.data(), v.Y.data(), v.Z.data(), &count, R, bmin, bmax, out);
    return mp_launch_surface_fp32(&m.mlp, &ef.feat, surf, N, in.cal, nullptr, guard, bt);
  });
}
