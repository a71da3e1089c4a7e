// TEST INFRASTRUCTURE ONLY: runs the device half of mp_mesh_refine_async (mcubes.cu) on the CPU emulation layer -- marching
// cubes (the enqueue-only sequence of mp_mcubes_run_async, or the eager count + mesh_emit_kernel), then mesh_edges_kernel,
// refine_init_kernel and `rounds` x refine_step_kernel, all from monoport_b200/csrc unmodified.  The query program between
// the rounds is replaced by a given value per vertex and round (sigma.f32: [rounds][count32] float32).  Every grid is forced
// to `blocks` CTAs.
//   emu_mesh_refine D H W iso v_cap blocks eager world R bmin0 bmin1 bmin2 bmax0 bmax1 bmax2 rounds vol.f32 sigma.f32 outdir
// eager = 1: mp_mcubes_count + mp_mcubes_emit's kernels (index-space vertices, every id written; v_cap is only the edge
// records' capacity) -- only the edge records are written then.
// Writes outdir/verts_mc.f32 (the emitted vertices, min(nV, v_cap) of them), outdir/edge_node.u32 and edge_axis.u8 (the
// records of ids < min(nV, v_cap)), outdir/rows.f32 (the query rows of every round, [rounds][3][count32]) and
// outdir/verts.f32 (the vertices after the refinement, count32 of them), and prints "nV nF count32".
// Exit code 3: a write outside the buffers (the guard words behind the records, the scratch arrays and the vertices).
#include "cuda_emu.h"

#include "../../monoport_b200/csrc/refine_kernels.cuh"

#include <string>

using namespace mcubes;

static std::vector<char> read_file(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) { perror(path); exit(2); }
  fseek(f, 0, SEEK_END);
  const long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  std::vector<char> b(n);
  if (n && fread(b.data(), 1, n, f) != (size_t)n) { perror("read"); exit(2); }
  fclose(f);
  return b;
}

static void write_file(const std::string& path, const void* p, size_t bytes) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) { perror(path.c_str()); exit(2); }
  if (bytes && fwrite(p, 1, bytes, f) != bytes) { perror("write"); exit(2); }
  fclose(f);
}

static void fail(const char* what) {
  fprintf(stderr, "%s\n", what);
  exit(3);
}

int main(int argc, char** argv) {
  if (argc != 20) {
    fprintf(stderr, "usage: emu_mesh_refine D H W iso v_cap blocks eager world R bmin0..2 bmax0..2 rounds vol.f32 sigma.f32 outdir\n");
    return 2;
  }
  const int D = atoi(argv[1]), H = atoi(argv[2]), W = atoi(argv[3]);
  const float iso = (float)atof(argv[4]);
  const long long v_cap = atoll(argv[5]);
  const unsigned blocks = (unsigned)atoi(argv[6]);
  const int eager = atoi(argv[7]), world = atoi(argv[8]);
  const float R = (float)atof(argv[9]);
  float bmin[3], bmax[3];
  for (int a = 0; a < 3; ++a) {
    bmin[a] = (float)atof(argv[10 + a]);
    bmax[a] = (float)atof(argv[13 + a]);
  }
  const int rounds = atoi(argv[16]);
  std::vector<char> raw = read_file(argv[17]);
  std::vector<char> sig_raw = read_file(argv[18]);
  const std::string outdir = argv[19];
  const long long n = (long long)D * H * W;
  if ((long long)raw.size() != n * 4) { fprintf(stderr, "volume size mismatch\n"); return 2; }
  const float* vol = reinterpret_cast<const float*>(raw.data());

  // the workspace (mp_mcubes_create)
  const long long n_words = (n + 31) >> 5;
  std::vector<uint32_t> bits(n_words + bits_pad_words(H, W), 0u);
  std::vector<WordInfo> info(n_words + 4);
  std::vector<unsigned long long> prefix(n_words + 4);
  std::vector<uint32_t> active(n_words + 4);
  const int nb = mpscan::num_blocks(n_words);
  std::vector<unsigned long long> sums(nb + 2, 0ull);
  uint32_t* n_active_dev = reinterpret_cast<uint32_t*>(sums.data() + nb + 1);
  unsigned long long total[2] = {0, 0};
  cuda_emu::launch(dim3(3), dim3(kBitsThreads), [&] { bits_kernel(vol, bits.data(), n, iso); });
  cuda_emu::launch(dim3((unsigned)((n_words + kClassifyWords - 1) / kClassifyWords)), dim3(kClassifyThreads),
                   [&] { classify_sums_kernel(bits.data(), info.data(), n, D, H, W, sums.data(), nb, total); });
  WordCountF f{info.data()};
  PrefixEmit em{prefix.data(), active.data(), n_active_dev};
  cuda_emu::launch(dim3(nb), dim3(mpscan::kThreads), [&] { mpscan::emit_kernel<WordCountF, PrefixEmit>(f, em, n_words, sums.data()); });
  const long long nv = (long long)(total[0] & 0xffffffffull), nf = (long long)(total[0] >> 32);

  constexpr int kGuard = 16;
  const long long kv = nv < v_cap ? nv : v_cap;
  int32_t count32 = (int32_t)kv;
  std::vector<float> verts;
  if (eager) {
    // mp_mcubes_emit: every vertex and face, index space, n_active from the host
    verts.assign((size_t)nv * 3 + kGuard, -12345.f);
    std::vector<int32_t> faces((size_t)nf * 3 + 1);
    const uint32_t n_act = *n_active_dev;
    const unsigned grid = (unsigned)((n_act + kEmitWarps - 1) / kEmitWarps);
    if (grid)
      cuda_emu::launch(dim3(grid), dim3(kEmitThreads), [&] {
        mesh_emit_kernel(vol, bits.data(), info.data(), prefix.data(), active.data(), n_act, verts.data(), faces.data(), D, H, W, n, iso);
      });
  } else {
    verts.assign((size_t)v_cap * 3 + kGuard, -12345.f);
    std::vector<int32_t> faces(1);
    long long counts[2];
    MeshOut out;
    memset(&out, 0, sizeof(out));
    out.verts = verts.data();
    out.faces = faces.data();
    out.v_cap = (uint32_t)v_cap;
    out.f_cap = 0;
    if (world) {
      out.world = 1;
      for (int a = 0; a < 3; ++a) {
        out.scale[a] = (bmax[a] - bmin[a]) / R;
        out.bmin[a] = bmin[a];
      }
    }
    cuda_emu::launch(dim3(blocks), dim3(kEmitThreads), [&] {
      mesh_emit_async_kernel(vol, bits.data(), info.data(), prefix.data(), active.data(), n_active_dev, total, out, counts, &count32,
                             D, H, W, n, iso);
    });
    if (count32 != (int32_t)kv) fail("count32 is not min(nV, v_cap)");
  }
  write_file(outdir + "/verts_mc.f32", verts.data(), (size_t)kv * 3 * sizeof(float));

  // the scratch of mp_mesh_refine_async, each array with guard words behind its capacity
  const size_t cap = (size_t)v_cap;
  std::vector<uint32_t> node(cap + kGuard, 0xA5A5A5A5u);
  std::vector<uint8_t> flags(cap + kGuard, 0xA5u);
  cuda_emu::launch(dim3(blocks), dim3(kEdgesThreads), [&] {
    mesh_edges_kernel(info.data(), prefix.data(), active.data(), n_active_dev, (uint32_t)v_cap, node.data(), flags.data());
  });
  for (int g = 0; g < kGuard; ++g)
    if (node[cap + g] != 0xA5A5A5A5u || flags[cap + g] != 0xA5u) fail("edge record written at or beyond v_cap");
  for (size_t v = (size_t)kv; v < cap; ++v)
    if (node[v] != 0xA5A5A5A5u || flags[v] != 0xA5u) fail("edge record written at or beyond nV");
  write_file(outdir + "/edge_node.u32", node.data(), (size_t)kv * sizeof(uint32_t));
  write_file(outdir + "/edge_axis.u8", flags.data(), (size_t)kv);
  printf("%lld %lld %d\n", nv, nf, count32);
  if (eager) return 0;

  std::vector<std::vector<float>> arrays(8, std::vector<float>(cap + kGuard, -777.f));
  std::vector<float> pts(3 * cap + kGuard, -777.f);
  mrefine::State s;
  s.pts = pts.data();
  s.sigma = arrays[0].data();
  s.ta = arrays[1].data(); s.fa = arrays[2].data(); s.tb = arrays[3].data(); s.fb = arrays[4].data();
  s.tbest = arrays[5].data(); s.fbest = arrays[6].data(); s.tcur = arrays[7].data();
  s.node = node.data();
  s.flags = flags.data();
  s.cap = (uint32_t)v_cap;
  mrefine::Geom g;
  g.H = H; g.W = W;
  g.iso = iso;
  for (int a = 0; a < 3; ++a) {
    g.scale[a] = (bmax[a] - bmin[a]) / R;
    g.bmin[a] = bmin[a];
  }
  if ((long long)sig_raw.size() != (long long)rounds * count32 * 4) { fprintf(stderr, "sigma size mismatch\n"); return 2; }
  const float* sig = reinterpret_cast<const float*>(sig_raw.data());
  std::vector<float> rows;
  if (rounds > 0) cuda_emu::launch(dim3(blocks), dim3(mrefine::kThreads), [&] { mrefine::refine_init_kernel(vol, &count32, s, g); });
  for (int r = 0; r < rounds; ++r) {
    for (int a = 0; a < 3; ++a) rows.insert(rows.end(), pts.begin() + a * cap, pts.begin() + a * cap + count32);
    for (int32_t v = 0; v < count32; ++v) s.sigma[v] = sig[(size_t)r * count32 + v];      // the query program's values
    cuda_emu::launch(dim3(blocks), dim3(mrefine::kThreads),
                     [&] { mrefine::refine_step_kernel(&count32, s, g, r == rounds - 1, verts.data()); });
  }
  for (int k = 0; k < 8; ++k)
    for (size_t v = cap; v < cap + kGuard; ++v)
      if (arrays[k][v] != -777.f) fail("scratch written beyond v_cap");
  for (size_t v = 3 * cap; v < 3 * cap + kGuard; ++v)
    if (pts[v] != -777.f) fail("query rows written beyond v_cap");
  for (size_t v = (size_t)count32; v < cap; ++v)
    if (pts[v] != -777.f || s.tcur[v] != -777.f) fail("scratch written at or beyond count32");
  for (size_t i = (size_t)count32 * 3; i < verts.size(); ++i)
    if (verts[i] != -12345.f) fail("a vertex at or beyond min(nV, v_cap) was written");
  write_file(outdir + "/rows.f32", rows.data(), rows.size() * sizeof(float));
  write_file(outdir + "/verts.f32", verts.data(), (size_t)count32 * 3 * sizeof(float));
  return 0;
}
