// TEST INFRASTRUCTURE ONLY: the vector-Jacobian product of the exact query with the flags of mp_query_points_vjp_ex -- in
// particular MP_VJP_DETERMINISTIC, the ordered feature gradient -- query_vjp_kernel of monoport_b200/csrc/query_fp32.cu and
// the contraction, radix sort, gather and layout step of query_vjp.cu compiled unmodified on the CPU emulation layer, driven
// by mp_launch_query_vjp as the library drives it.  The arguments and the output are emu_query_vjp's:
//   emu_query_vjp_det in.bin out.f32 B widths grad_out.f32|- chunk_points [sms] [want]
// in.bin: a batched input of B maps / point sets / calibs (emu_host.h); widths: the head's widths after the first, comma
// separated; grad_out.f32: [B][Res][N] fp32, or - for ones; chunk_points: points per chunk (0: one chunk); want: the
// requested outputs as letters f (features), p (points), w (weights and biases), default fpw.  out.f32 = d features
// [B][C][H][W], d points [B][3][N], d W_l [cout][cin] for every layer, d b_l for every layer (zeros where not requested).
// EMU_VJP_FLAGS: the flags (default 0).  EMU_VJP_DUMP=path (with MP_VJP_DETERMINISTIC, want f and one chunk): the ordered
// feature gradient's scratch after the run -- int64 {columns, C}, then fp32 dX rows [columns][C] (zero for a column that
// contributes nothing), fp32 tap weights [columns][4], the sorted uint32 keys and their columns.
#include "emu_host.h"

extern "C" cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { memset(d, v, n); return cudaSuccess; }

#include "../../monoport_b200/csrc/query_fp32.cu"
#include "../../monoport_b200/csrc/query_vjp.cu"

int main(int argc, char** argv) {
  if (argc < 7 || argc > 9) {
    fprintf(stderr, "usage: emu_query_vjp_det in.bin out.f32 B widths grad_out.f32|- chunk_points [sms] [want]\n");
    return 2;
  }
  const int B = atoi(argv[3]);
  std::vector<int> widths;
  for (char* s = strtok(argv[4], ","); s; s = strtok(nullptr, ",")) widths.push_back(atoi(s));
  const long long chunk_points = atoll(argv[6]);
  if (argc >= 8) g_fake_sms = atoi(argv[7]);
  const char* want = argc >= 9 ? argv[8] : "fpw";
  const bool wf = strchr(want, 'f'), wpt = strchr(want, 'p'), ww = strchr(want, 'w');
  EmuInput in = emu_read_input(argv[1], B, true);
  const int N = in.N, res = in.res;
  EmuMlp m = emu_make_mlp(in, widths);
  EmuFeat ef = emu_make_feat(in, B);
  std::vector<float> gout;
  if (strcmp(argv[5], "-") != 0) {
    FILE* g = fopen(argv[5], "rb");
    if (!g) { perror(argv[5]); return 2; }
    gout = emu_read(g, (size_t)B * res * N);
    fclose(g);
  }
  const int L = m.mlp.n_layers;
  size_t n_w = 0, n_b = 0;
  for (int l = 0; l < L; ++l) { n_w += (size_t)m.mlp.cout[l] * m.mlp.cin[l]; n_b += m.mlp.cout[l]; }
  const size_t n_f = (size_t)B * in.C * in.H * in.W, n_p = (size_t)B * 3 * N;
  std::vector<float> out(n_f + n_p + n_w + n_b + 1, 0.f);
  out.back() = -4242.f;
  float* dfeat = out.data();
  float* dp = dfeat + n_f;
  std::vector<float*> dw(L), db(L);
  float* q = dp + n_p;
  for (int l = 0; l < L; ++l) { dw[l] = q; q += (size_t)m.mlp.cout[l] * m.mlp.cin[l]; }
  for (int l = 0; l < L; ++l) { db[l] = q; q += m.mlp.cout[l]; }

  MpPointSrc src = emu_rows_src(in);
  MpBatch bt;
  bt.B = B;
  bt.pt_stride = 3 * (long long)N;
  bt.calibs = in.calibs.empty() ? nullptr : in.calibs.data();
  const int flags = getenv("EMU_VJP_FLAGS") ? atoi(getenv("EMU_VJP_FLAGS")) : 0;
  const long long bytes = mp_vjp_scratch_bytes(&m.mlp, &ef.feat, B, N, chunk_points, wf, ww, flags);
  if (bytes < 0) { fprintf(stderr, "mp_vjp_scratch_bytes: %s\n", g_err); return 3; }
  std::vector<float> scratch((size_t)bytes / 4 + 1);
  const int rc = mp_launch_query_vjp(&m.mlp, &ef.feat, src, in.cal, bt, gout.empty() ? nullptr : gout.data(), wf ? dfeat : nullptr,
                                     wpt ? dp : nullptr, ww ? dw.data() : nullptr, ww ? db.data() : nullptr,
                                     bytes ? scratch.data() : nullptr, bytes, nullptr, flags);
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_vjp: %s\n", g_err); return 3; }
  if (const char* dump = getenv("EMU_VJP_DUMP")) {
    if (!(flags & MP_VJP_DETERMINISTIC) || !wf || chunk_points > 0) { fprintf(stderr, "EMU_VJP_DUMP: one ordered chunk only\n"); return 2; }
    // the launcher's layout of a single chunk of every tile
    const int P = mp_query_vjp_tile(&m.mlp);
    const long long cols = (long long)B * ((N + P - 1) / P) * P, HW = (long long)in.H * in.W;
    const size_t rows = ww ? (size_t)row_layout(&m.mlp).total * P * sizeof(float) * (size_t)(cols / P) : 0;
    const char* area = reinterpret_cast<const char*>(scratch.data()) + round256((size_t)B * HW * in.C * sizeof(float)) + round256(rows);
    const OrderedLayout ol = ordered_layout(cols, in.C);
    const int sorted = radix_passes((unsigned long long)B * HW) & 1;
    FILE* f = fopen(dump, "wb");
    const long long hd[2] = {cols, in.C};
    fwrite(hd, 8, 2, f);
    fwrite(area + ol.dx, 4, (size_t)cols * in.C, f);
    fwrite(area + ol.wgt, 4, (size_t)cols * 4, f);
    fwrite(area + ol.key[sorted], 4, (size_t)cols, f);
    fwrite(area + ol.col[sorted], 4, (size_t)cols, f);
    fclose(f);
  }
  if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  emu_write(argv[2], out.data(), out.size() - 1);
  return 0;
}
