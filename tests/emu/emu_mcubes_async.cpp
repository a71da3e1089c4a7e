// TEST INFRASTRUCTURE ONLY: runs the enqueue-only marching-cubes sequence of mp_mcubes_run_async (mcubes.cu) on the CPU
// emulation layer -- bits_kernel, the zeroed chunk sums (n_active included), classify_sums_kernel, the scan's emit half and
// mesh_emit_async_kernel, all from monoport_b200/csrc/mcubes_kernels.cuh unmodified -- once per input volume, on ONE
// workspace and into the same output buffers, as a replayed graph does.  The emission grid is forced to `blocks` CTAs.
//   emu_mcubes_async D H W iso v_cap f_cap blocks world R bmin0 bmin1 bmin2 bmax0 bmax1 bmax2 outdir in0.f32 [in1.f32 ...]
// Run k writes outdir/verts<k>.f32 (min(nV, v_cap) vertices) and outdir/faces<k>.i32 (min(nF, f_cap) faces) and prints
// "nV nF count32".  Exit code 3: a write outside the buffers or the workspace, or a per-run word left set.
#include "cuda_emu.h"

#include "../../monoport_b200/csrc/mcubes_kernels.cuh"

#include <string>

using namespace mcubes;

static std::vector<char> read_file(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) { perror(path); exit(2); }
  fseek(f, 0, SEEK_END);
  const long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  std::vector<char> b(n);
  if (fread(b.data(), 1, n, f) != (size_t)n) { perror("read"); exit(2); }
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
  if (argc < 18) {
    fprintf(stderr, "usage: emu_mcubes_async D H W iso v_cap f_cap blocks world R bmin0..2 bmax0..2 outdir in0.f32 [...]\n");
    return 2;
  }
  const int D = atoi(argv[1]), H = atoi(argv[2]), W = atoi(argv[3]);
  const float iso = (float)atof(argv[4]);
  const long long v_cap = atoll(argv[5]), f_cap = atoll(argv[6]);
  const unsigned blocks = (unsigned)atoi(argv[7]);
  const int world = atoi(argv[8]);
  const float R = (float)atof(argv[9]);
  float bmin[3], bmax[3];
  for (int a = 0; a < 3; ++a) {
    bmin[a] = (float)atof(argv[10 + a]);
    bmax[a] = (float)atof(argv[13 + a]);
  }
  const std::string outdir = argv[16];
  const long long n = (long long)D * H * W;

  // workspace of mp_mcubes_create: the bit volume and its padding zeroed, the scan ticket zeroed, everything else left as
  // it comes (garbage here) -- the sequence must not depend on it.  Guard words behind every array.
  const long long n_words = (n + 31) >> 5;
  const long long pad = bits_pad_words(H, W);
  std::vector<uint32_t> bits(n_words + pad, 0u);
  std::vector<WordInfo> info(n_words + 4, WordInfo{0xEEEEEEEEu, 0xEEEEEEEEu, 0xEEEEEEEEu, 0xEEEEEEEEu});
  std::vector<unsigned long long> prefix(n_words + 4, 0xDEADBEEFDEADBEEFull);
  std::vector<uint32_t> active(n_words + 4, 0xABABABABu);
  const int nb = mpscan::num_blocks(n_words);
  std::vector<unsigned long long> sums(nb + 2, 0x5A5A5A5A5A5A5A5Aull);
  uint32_t* n_active_dev = reinterpret_cast<uint32_t*>(sums.data() + nb + 1);
  unsigned long long total[2] = {0, 0};

  // the caller's buffers (shared by all runs, like a graph's), with guard words behind both
  constexpr int kGuard = 16;
  std::vector<float> verts((size_t)v_cap * 3 + kGuard, -12345.f);
  std::vector<int32_t> faces((size_t)f_cap * 3 + kGuard, -7);
  long long counts[2] = {-1, -1};
  int32_t count32 = -1;

  MeshOut out;
  memset(&out, 0, sizeof(out));
  out.verts = verts.data();
  out.faces = faces.data();
  out.v_cap = (uint32_t)v_cap;
  out.f_cap = (uint32_t)f_cap;
  if (world) {
    out.world = 1;
    for (int a = 0; a < 3; ++a) {
      out.scale[a] = (bmax[a] - bmin[a]) / R;          // (mcubes.cu's host arithmetic)
      out.bmin[a] = bmin[a];
    }
  }

  for (int k = 0; 17 + k < argc; ++k) {
    std::vector<char> raw = read_file(argv[17 + k]);
    if ((long long)raw.size() != n * 4) { fprintf(stderr, "volume size mismatch\n"); return 2; }
    const float* vol = reinterpret_cast<const float*>(raw.data());
    {
      const long long warps_needed = (n_words + kBitsUnroll - 1) / kBitsUnroll;
      long long b = (warps_needed + kBitsThreads / 32 - 1) / (kBitsThreads / 32);
      if (b > 3) b = 3;
      cuda_emu::launch(dim3((unsigned)b), dim3(kBitsThreads), [&] { bits_kernel(vol, bits.data(), n, iso); });
    }
    std::fill(sums.begin(), sums.end(), 0ull);          // the cudaMemsetAsync of the sequence: chunk sums + n_active
    cuda_emu::launch(dim3((unsigned)((n_words + kClassifyWords - 1) / kClassifyWords)), dim3(kClassifyThreads),
                     [&] { classify_sums_kernel(bits.data(), info.data(), n, D, H, W, sums.data(), nb, total); });
    WordCountF f{info.data()};
    PrefixEmit em{prefix.data(), active.data(), n_active_dev};
    cuda_emu::launch(dim3(nb), dim3(mpscan::kThreads), [&] { mpscan::emit_kernel<WordCountF, PrefixEmit>(f, em, n_words, sums.data()); });
    if (total[1] != 0) fail("scan ticket not reset");
    cuda_emu::launch(dim3(blocks), dim3(kEmitThreads), [&] {
      mesh_emit_async_kernel(vol, bits.data(), info.data(), prefix.data(), active.data(), n_active_dev, total, out, counts,
                             &count32, D, H, W, n, iso);
    });
    for (long long w = n_words; w < n_words + pad; ++w)
      if (bits[w] != 0u) fail("wrote into the bit padding");
    for (long long w = n_words; w < n_words + 4; ++w)
      if (active[w] != 0xABABABABu || info[w].ex != 0xEEEEEEEEu || prefix[w] != 0xDEADBEEFDEADBEEFull)
        fail("wrote past the word arrays");
    for (int g = 0; g < kGuard; ++g)
      if (verts[(size_t)v_cap * 3 + g] != -12345.f || faces[(size_t)f_cap * 3 + g] != -7) fail("wrote past the output buffers");
    const long long nv = counts[0], nf = counts[1];
    if (nv != (long long)(total[0] & 0xffffffffull) || nf != (long long)(total[0] >> 32)) fail("counts differ from the scan total");
    const long long kv = nv < v_cap ? nv : v_cap, kf = nf < f_cap ? nf : f_cap;
    if (count32 != (int32_t)kv) fail("count32 is not min(nV, v_cap)");
    for (long long i = 0; i < kf * 3; ++i)
      if (faces[i] < 0 || faces[i] >= nv) fail("face index out of range");
    write_file(outdir + "/verts" + std::to_string(k) + ".f32", verts.data(), (size_t)kv * 3 * sizeof(float));
    write_file(outdir + "/faces" + std::to_string(k) + ".i32", faces.data(), (size_t)kf * 3 * sizeof(int32_t));
    printf("%lld %lld %d\n", nv, nf, count32);
  }
  return 0;
}
