// TEST INFRASTRUCTURE ONLY: the vector-Jacobian product of the exact query -- query_vjp_kernel of
// monoport_b200/csrc/query_fp32.cu and the contraction and layout step of query_vjp.cu -- compiled unmodified on the CPU
// emulation layer, driven by mp_launch_query_vjp as the library drives it.
//   emu_query_vjp in.bin out.f32 B widths grad_out.f32|- chunk_points [sms] [want]
// in.bin: a batched input of B maps / point sets / calibs (emu_host.h); widths: the head's widths after the first, comma
// separated; grad_out.f32: [B][Res][N] fp32, or - for ones; chunk_points: points per weight-gradient chunk (0: one chunk);
// want: the requested outputs as letters f (features), p (points), w (weights and biases), default fpw.  out.f32 = d features
// [B][C][H][W], d points [B][3][N], d W_l [cout][cin] for every layer, d b_l for every layer (zeros where not requested).
#include "emu_host.h"

extern "C" cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { memset(d, v, n); return cudaSuccess; }

#include "../../monoport_b200/csrc/query_fp32.cu"
#include "../../monoport_b200/csrc/query_vjp.cu"

int main(int argc, char** argv) {
  if (argc < 7 || argc > 9) {
    fprintf(stderr, "usage: emu_query_vjp in.bin out.f32 B widths grad_out.f32|- chunk_points [sms] [want]\n");
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
  const long long bytes = mp_vjp_scratch_bytes(&m.mlp, &ef.feat, B, N, chunk_points, wf, ww);
  if (bytes < 0) { fprintf(stderr, "mp_vjp_scratch_bytes: %s\n", g_err); return 3; }
  std::vector<float> scratch((size_t)bytes / 4 + 1);
  const int rc = mp_launch_query_vjp(&m.mlp, &ef.feat, src, in.cal, bt, gout.empty() ? nullptr : gout.data(), wf ? dfeat : nullptr,
                                     wpt ? dp : nullptr, ww ? dw.data() : nullptr, ww ? db.data() : nullptr,
                                     bytes ? scratch.data() : nullptr, bytes, nullptr);
  if (rc != MP_OK) { fprintf(stderr, "mp_launch_query_vjp: %s\n", g_err); return 3; }
  if (out.back() != -4242.f) { fprintf(stderr, "wrote past the output\n"); return 3; }
  emu_write(argv[2], out.data(), out.size() - 1);
  return 0;
}
