// TEST INFRASTRUCTURE ONLY: the lossless engine's device-driven conflict loop (mp_octree_run_fused_async) on the CPU
// emulation layer.  The kernels of monoport_b200/csrc/octree_kernels.cuh + octree_loop.cuh + mp_scan.cuh run unmodified;
// the launch sequence mirrors run_fused_levels / level_pass / device_conflict_loop of octree.cu: every level from 1 on runs
// the WHILE node's body (query, scatter with conflict detection, conflict list, loop_control_kernel) for as long as
// loop_control_kernel sets the node's condition.  The occupancy query is a lookup into a dense final-resolution volume
// supplied by the test, so the oracle can be driven with exactly the same values.
//   emu_octree_loop balance dense.f32 out_vol.f32 out_idx.i32 cap n_levels r0 r1 ...
//   cap: at most `cap` passes per level (0: the library's 8 x resolution).  Prints per level the number of evaluated
//   nodes (their indices, in evaluation order, go to out_idx), then on a second line the passes per level and the
//   truncated flag (level + 1, or 0).
#include "cuda_emu.h"

// the device runtime's call that sets a WHILE / IF node's condition: the harness reads back the last handle and value set
namespace emu_graph {
inline unsigned long long g_cond_handle = 0;
inline unsigned g_cond_value = 0;
}
inline void cudaGraphSetConditional(unsigned long long handle, unsigned value) {
  emu_graph::g_cond_handle = handle;
  emu_graph::g_cond_value = value;
}

#include "../../monoport_b200/csrc/octree_loop.cuh"

using namespace octree_k;

static int grid_for(long long n, int threads = 256, int cap = 148 * 8) {
  long long b = (n + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

struct Eng {
  int n_levels = 0, R = 0;
  std::vector<int> res;
  float balance = 0.5f;
  long long cap = 0, V = 0;
  std::vector<float> vol[2], vals;
  std::vector<uint8_t> known[2], cand_t, conflict;
  std::vector<int32_t> idx;
  std::vector<unsigned long long> sums;
  unsigned long long total[2] = {0, 0};
  int32_t count = 0;
  std::vector<long long> stats;
  std::vector<int32_t> loops;                      // passes per level, then the truncated flag (mp_octree::loops)
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

// build_level_list of the lossless engine: radius 1, every level examined
static void build_level_list(Eng& e, int level) {
  const int res_c = e.res[level - 1], res_f = e.res[level];
  const long long nf = (long long)res_f * res_f * res_f;
  const int src = e.cur, dst = e.cur ^ 1;
  const dim3 grid((unsigned)(((long long)res_c * res_c + 255) / 256), (unsigned)res_c);
  const float* vc = e.vol[src].data();
  const uint8_t* kc = e.known[src].data();
  float* vf = e.vol[dst].data();
  uint8_t* kf = e.known[dst].data();
  uint8_t* ct = e.cand_t.data();
  const float bal = e.balance;
  cuda_emu::launch(grid, dim3(256), [&] { upsample_kernel<3>(vc, kc, vf, kf, ct, res_c, res_f, 1, bal); });
  e.cur = dst;
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

// one execution of the WHILE node's body; returns the condition loop_control_kernel set
static bool loop_body(Eng& e, int level, int loop_cap) {
  query_nodes(e, level, e.count, e.vals.data(), nullptr);
  const int32_t* ip = e.idx.data();
  const float* vsrc = e.vals.data();
  float* volp = e.vol[e.cur].data();
  uint8_t* kn = e.known[e.cur].data();
  uint8_t* cf = e.conflict.data();
  const float bal = e.balance;
  const int32_t* cnt = &e.count;
  const long long nmax = e.cap;
  cuda_emu::launch(dim3(grid_for(e.cap > (1 << 20) ? (1 << 20) : e.cap)), dim3(256),
                   [&] { scatter_kernel(ip, cnt, nmax, vsrc, volp, kn, cf, bal, true); });
  build_conflict_list(e, level);
  int32_t* pp = &e.loops[level];
  int32_t* tp = &e.loops[e.n_levels];
  const int cap = loop_cap > 0 ? loop_cap : 8 * e.res[level];
  const unsigned long long cond = 100 + level;
  emu_graph::g_cond_handle = 0;
  // (one thread on the GPU; the CPU model launches whole warps, and the kernel acts in thread 0 only)
  cuda_emu::launch(dim3(1), dim3(32), [&] { loop_control_kernel(cnt, pp, tp, level, cap, cond); });
  if (emu_graph::g_cond_handle != cond) { fprintf(stderr, "condition not set\n"); exit(3); }
  return emu_graph::g_cond_value != 0;
}

int main(int argc, char** argv) {
  if (argc < 8) { fprintf(stderr, "usage: see header\n"); return 2; }
  Eng e;
  e.balance = (float)atof(argv[1]);
  const int loop_cap = atoi(argv[5]);
  e.n_levels = atoi(argv[6]);
  for (int l = 0; l < e.n_levels; ++l) e.res.push_back(atoi(argv[7 + l]));
  e.R = e.res.back();
  e.V = (long long)e.R * e.R * e.R;
  std::vector<float> dense(e.V);
  {
    FILE* f = fopen(argv[2], "rb");
    if (!f || fread(dense.data(), 4, e.V, f) != (size_t)e.V) { perror("dense"); return 2; }
    fclose(f);
  }
  e.dense = dense.data();
  // capacity as in mp_octree_create (lossless: the last level is examined)
  long long cap = (long long)e.res[0] * e.res[0] * e.res[0];
  if ((long long)e.R * e.R * e.R > cap) cap = (long long)e.R * e.R * e.R;
  e.cap = cap;
  for (int i = 0; i < 2; ++i) { e.vol[i].assign(e.V, -777.f); e.known[i].assign(e.V, 0xEE); }
  e.cand_t.assign(e.V, 0xEE);
  e.conflict.assign(e.V, 0);
  e.idx.assign(cap, -1);
  e.vals.assign(cap, -777.f);
  e.sums.assign(mpscan::num_blocks(e.V) + 1, 0);
  e.stats.assign(e.n_levels + 1, 0);
  e.loops.assign(e.n_levels + 1, 0);
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
  int nonempty = 0;
  {
    const float* vp = e.vol[e.cur].data();
    const float bal = e.balance;
    cuda_emu::launch(dim3(grid_for(n0)), dim3(256), [&] { any_gt_kernel(vp, n0, bal, &nonempty); });
  }
  // ---- levels 1..: the level list outside the loop, then the WHILE node (its condition defaults to 1: one pass at least)
  for (int level = 1; level < e.n_levels && nonempty; ++level) {
    build_level_list(e, level);
    while (loop_body(e, level, loop_cap)) {}
  }
  if (e.total[1] != 0) { fprintf(stderr, "scan ticket not reset\n"); return 3; }
  // outputs
  printf("%d", nonempty);
  FILE* fi = fopen(argv[4], "wb");
  for (int l = 0; l < e.n_levels; ++l) {
    printf(" %zu", e.evaluated[l].size());
    if (!e.evaluated[l].empty()) fwrite(e.evaluated[l].data(), 4, e.evaluated[l].size(), fi);
  }
  fclose(fi);
  printf("\n");
  for (int l = 0; l <= e.n_levels; ++l) printf(l ? " %d" : "%d", e.loops[l]);
  printf("\n");
  FILE* fv = fopen(argv[3], "wb");
  if (nonempty) fwrite(e.vol[e.cur].data(), 4, e.V, fv);
  fclose(fv);
  return 0;
}
