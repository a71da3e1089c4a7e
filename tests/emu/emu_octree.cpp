// TEST INFRASTRUCTURE ONLY: the coarse-to-fine engine's kernels (monoport_b200/csrc/octree_kernels.cuh + mp_scan.cuh) on
// the CPU emulation layer.  The launch sequence mirrors run_fused_levels / build_level_list / build_conflict_list of
// octree.cu; the occupancy query is a lookup into a dense final-resolution volume supplied by the test (every level's
// nodes are a subset of the final grid), so the oracle can be driven with exactly the same values.
//   emu_octree MODE balance dense.f32 out_vol.f32 out_idx.i32 n_levels r0 r1 ... [k0 k1 ...]     MODE = faster|lossless|topk
//   prints per level the number of evaluated nodes (their indices, in evaluation order, go to out_idx)
#include "cuda_emu.h"

#include "../../monoport_b200/csrc/octree_kernels.cuh"

#include <string>

using namespace octree_k;

static int grid_for(long long n, int threads = 256, int cap = 148 * 8) {
  long long b = (n + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}
static int radius_for(bool faster, int level) {
  if (!faster) return 1;
  return level == 1 ? 4 : (level == 2 ? 3 : 1);
}

struct Eng {
  int n_levels = 0, R = 0;
  std::vector<int> res, topk;
  float balance = 0.5f;
  bool faster = false, use_topk = false;
  long long cap = 0, V = 0;
  std::vector<float> vol[2], vals;
  std::vector<uint8_t> known[2], cand_t, conflict;
  std::vector<int32_t> idx;
  std::vector<unsigned long long> sums;
  unsigned long long total[2] = {0, 0};
  int32_t count = 0;
  int nonempty = 0;
  std::vector<long long> stats;
  SelectState sel;
  int cur = 0;
  const float* dense = nullptr;
  std::vector<std::vector<int32_t>> evaluated;     // per level, in evaluation order
};

template <class F, class E, class P>
static void scan_emit(F f, E em, long long n, Eng& e, P post) {
  const int nb = mpscan::num_blocks(n > 0 ? n : 1);
  cuda_emu::launch(dim3(nb), dim3(mpscan::kThreads),
                   [&] { mpscan::block_sums_kernel<F, P>(f, n > 0 ? n : 0, e.sums.data(), nb, e.total, post); });
  if (n > 0) cuda_emu::launch(dim3(nb), dim3(mpscan::kThreads), [&] { mpscan::emit_kernel<F, E>(f, em, n, e.sums.data()); });
}

static void build_level_list(Eng& e, int level) {
  const int res_c = e.res[level - 1], res_f = e.res[level];
  const long long nf = (long long)res_f * res_f * res_f;
  const int src = e.cur, dst = e.cur ^ 1;
  const bool last = level == e.n_levels - 1;
  const bool interp_only = e.use_topk || (e.faster && last);
  const dim3 grid((unsigned)(((long long)res_c * res_c + 255) / 256), (unsigned)res_c);
  const float* vc = e.vol[src].data();
  const uint8_t* kc = e.use_topk ? nullptr : e.known[src].data();
  float* vf = e.vol[dst].data();
  uint8_t* kf = (e.use_topk || (e.faster && last)) ? nullptr : e.known[dst].data();
  const int radius = radius_for(e.faster, level);
  uint8_t* ct = e.cand_t.data();
  const float bal = e.balance;
  if (interp_only) cuda_emu::launch(grid, dim3(256), [&] { upsample_kernel<0>(vc, kc, vf, kf, nullptr, res_c, res_f, radius, bal); });
  else if (radius <= 1) cuda_emu::launch(grid, dim3(256), [&] { upsample_kernel<3>(vc, kc, vf, kf, ct, res_c, res_f, radius, bal); });
  else if (radius <= 3) cuda_emu::launch(grid, dim3(256), [&] { upsample_kernel<5>(vc, kc, vf, kf, ct, res_c, res_f, radius, bal); });
  else cuda_emu::launch(grid, dim3(256), [&] { upsample_kernel<6>(vc, kc, vf, kf, ct, res_c, res_f, radius, bal); });
  e.cur = dst;
  if (e.use_topk) {
    long long k = e.topk[level] < 0 ? 0 : e.topk[level];
    if (k > nf) k = nf;
    if (k == 0) { e.count = 0; return; }
    SelectState* sp = &e.sel;
    cuda_emu::launch(dim3(1), dim3(256), [&] { select_init_kernel(sp, (uint32_t)k); });
    for (int pass = 0; pass < 4; ++pass) {
      cuda_emu::launch(dim3(grid_for(nf)), dim3(256), [&] { select_hist_kernel(vf, nf, bal, sp, pass); });
      cuda_emu::launch(dim3(1), dim3(256), [&] { select_pick_kernel(sp, pass); });
    }
    scan_emit(TopkF{vf, bal, sp}, TopkEmit{e.idx.data(), sp}, nf, e, mpscan::NoPost());
    topk_count_kernel(&e.count, &e.stats[level], &e.nonempty, (int32_t)k);   // a <<<1, 1>>> launch: one call
    return;
  }
  if (interp_only) { e.count = 0; return; }
  scan_emit(FlagF{ct}, EmitNodesT{e.idx.data(), res_f, e.cap}, nf, e, CountPost{&e.count, e.cap, &e.stats[level]});
}

static void build_conflict_list(Eng& e, int level) {
  const int res = e.res[level];
  const long long nf = (long long)res * res * res;
  const uint8_t* cf = e.conflict.data();
  const uint8_t* kn = e.known[e.cur].data();
  uint8_t* ct = e.cand_t.data();
  cuda_emu::launch(dim3(grid_for(nf)), dim3(256), [&] { conflict_neighbours_kernel(cf, kn, ct, res); });
  memset(e.conflict.data(), 0, nf);
  scan_emit(FlagF{ct}, EmitNodesT{e.idx.data(), res, e.cap}, nf, e, CountPost{&e.count, e.cap, &e.stats[level]});
}

// the fused sample+MLP kernel's role: value of node idx[i] of the level grid
static void query_nodes(Eng& e, int level, long long n, float* out_vals, float* scatter_vol) {
  const int res = e.res[level], stride = (e.R - 1) / (res - 1);
  for (long long i = 0; i < n; ++i) {
    const int lin = e.idx[i];
    const int z = lin / (res * res), r = lin - z * res * res, y = r / res, x = r - y * res;
    const float v = e.dense[((long long)z * stride * e.R + (long long)y * stride) * e.R + (long long)x * stride];
    if (out_vals) out_vals[i] = v;
    if (scatter_vol) scatter_vol[lin] = v;
    e.evaluated[level].push_back(lin);
  }
}

int main(int argc, char** argv) {
  if (argc < 8) { fprintf(stderr, "usage: see header\n"); return 2; }
  Eng e;
  const std::string mode = argv[1];
  e.faster = mode == "faster";
  e.use_topk = mode == "topk";
  e.balance = (float)atof(argv[2]);
  e.n_levels = atoi(argv[6]);
  for (int l = 0; l < e.n_levels; ++l) e.res.push_back(atoi(argv[7 + l]));
  if (e.use_topk) for (int l = 0; l < e.n_levels; ++l) e.topk.push_back(atoi(argv[7 + e.n_levels + l]));
  e.R = e.res.back();
  e.V = (long long)e.R * e.R * e.R;
  std::vector<float> dense(e.V);
  {
    FILE* f = fopen(argv[3], "rb");
    if (!f || fread(dense.data(), 4, e.V, f) != (size_t)e.V) { perror("dense"); return 2; }
    fclose(f);
  }
  e.dense = dense.data();
  // capacities as in mp_octree_create
  long long cap = (long long)e.res[0] * e.res[0] * e.res[0];
  if (e.use_topk) {
    for (int l = 1; l < e.n_levels; ++l) {
      const long long r3 = (long long)e.res[l] * e.res[l] * e.res[l];
      long long k = e.topk[l] < 0 ? 0 : e.topk[l];
      if (k > r3) k = r3;
      if (k > cap) cap = k;
    }
  } else {
    const int last_examined = (e.faster && e.n_levels > 1) ? e.n_levels - 2 : e.n_levels - 1;
    const long long r = e.res[last_examined];
    if (r * r * r > cap) cap = r * r * r;
  }
  e.cap = cap;
  for (int i = 0; i < 2; ++i) { e.vol[i].assign(e.V, -777.f); e.known[i].assign(e.V, 0xEE); }
  e.cand_t.assign(e.V, 0xEE);
  e.conflict.assign(e.V, 0);
  e.idx.assign(cap, -1);
  e.vals.assign(cap, -777.f);
  e.sums.assign(mpscan::num_blocks(e.V) + 1, 0);
  e.stats.assign(e.n_levels + 1, 0);
  e.evaluated.resize(e.n_levels);

  // ---- level 0: dense
  const int r0 = e.res[0];
  const long long n0 = (long long)r0 * r0 * r0;
  {
    int32_t* ip = e.idx.data();
    cuda_emu::launch(dim3(grid_for(n0)), dim3(256), [&] { iota_kernel(ip, (int)n0); });
    query_nodes(e, 0, n0, nullptr, e.vol[e.cur].data());
    uint8_t* kp = e.known[e.cur].data();
    cuda_emu::launch(dim3(grid_for(n0)), dim3(256), [&] { set_u8_kernel(kp, n0, 1); });
  }
  {
    const float* vp = e.vol[e.cur].data();
    const float bal = e.balance;
    int* ne = &e.nonempty;
    cuda_emu::launch(dim3(grid_for(n0)), dim3(256), [&] { any_gt_kernel(vp, n0, bal, ne); });
  }
  // like run_fused_levels, the levels run whatever level 0 found: an empty frame must produce empty node lists
  for (int level = 1; level < e.n_levels; ++level) {
    build_level_list(e, level);
    const bool last = level == e.n_levels - 1;
    if (!e.use_topk && e.faster && last) break;
    const bool lossless = !e.use_topk && !e.faster;
    for (;;) {
      long long n = e.count;
      if (e.use_topk) {
        const long long nf = (long long)e.res[level] * e.res[level] * e.res[level];
        const long long k = e.topk[level] > nf ? nf : e.topk[level];
        if (k <= 0) break;
        n = n < k ? n : k;
      }
      float* volp = e.vol[e.cur].data();
      query_nodes(e, level, n, lossless ? e.vals.data() : nullptr, lossless ? nullptr : volp);
      const int32_t* ip = e.idx.data();
      const float* vsrc = lossless ? e.vals.data() : volp;
      uint8_t* kn = e.use_topk ? nullptr : e.known[e.cur].data();
      uint8_t* cf = lossless ? e.conflict.data() : nullptr;
      const float bal = e.balance;
      const int32_t* cnt = &e.count;
      const long long nmax = e.use_topk ? n : e.cap;
      cuda_emu::launch(dim3(grid_for(e.cap > (1 << 20) ? (1 << 20) : e.cap)), dim3(256),
                       [&] { scatter_kernel(ip, cnt, nmax, vsrc, volp, kn, cf, bal, lossless); });
      if (!lossless) break;
      build_conflict_list(e, level);
      if (e.count == 0) break;
    }
  }
  if (e.total[1] != 0) { fprintf(stderr, "scan ticket not reset\n"); return 3; }
  // outputs
  printf("%d", e.nonempty);
  FILE* fi = fopen(argv[5], "wb");
  for (int l = 0; l < e.n_levels; ++l) {
    printf(" %zu", e.evaluated[l].size());
    if (!e.evaluated[l].empty()) fwrite(e.evaluated[l].data(), 4, e.evaluated[l].size(), fi);
  }
  fclose(fi);
  printf("\n");
  FILE* fv = fopen(argv[4], "wb");
  if (e.nonempty) fwrite(e.vol[e.cur].data(), 4, e.V, fv);
  fclose(fv);
  return 0;
}
