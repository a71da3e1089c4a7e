// TEST INFRASTRUCTURE ONLY: runs the device half of mp_render_mesh_async (raster.cu) on the CPU emulation layer -- the key
// clear, raster_setup_kernel, raster_large_kernel and raster_resolve_kernel from monoport_b200/csrc/raster_kernels.cuh,
// unmodified.  The setup and large-face grids are forced to `setup_blocks` x views and `large_blocks` CTAs.
//   emu_raster v_cap f_cap views W H has_normals has_colours setup_blocks large_blocks in.bin outdir
// in.bin: counts int64[2], clear float32[4], mats float32[views][32], verts float32[v_cap][3], faces int32[f_cap][3], then
// normals and colours float32[v_cap][3] when present.
// Writes outdir/keys.u64 ([views][H][W] depth keys), outdir/normal.f32 and / or outdir/colour.f32 ([views][H][W][4]) and
// prints the length of the large-face list.  Exit code 3: a write outside the images or the list.
#include "cuda_emu.h"

#include <string>

// the device intrinsics the rasterizer uses beyond cuda_emu.h's (round-to-nearest-even is the host's default mode)
inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
inline int __float2int_rn(float a) { return (int)nearbyintf(a); }
inline long long __double2ll_rn(double a) { return llrint(a); }
inline float __double2float_rn(double a) { return (float)a; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dsub_rn(double a, double b) { return a - b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __ddiv_rn(double a, double b) { return a / b; }
inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  unsigned long long old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (old > v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}

#include "../../monoport_b200/csrc/raster_kernels.cuh"

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

template <class T>
static const T* take(const std::vector<char>& raw, size_t& off, size_t n) {
  const T* p = reinterpret_cast<const T*>(raw.data() + off);
  off += n * sizeof(T);
  if (off > raw.size()) { fprintf(stderr, "in.bin too short\n"); exit(2); }
  return p;
}

int main(int argc, char** argv) {
  if (argc != 12) {
    fprintf(stderr, "usage: emu_raster v_cap f_cap views W H has_normals has_colours setup_blocks large_blocks in.bin outdir\n");
    return 2;
  }
  const uint32_t v_cap = (uint32_t)atoll(argv[1]), f_cap = (uint32_t)atoll(argv[2]);
  const int views = atoi(argv[3]), W = atoi(argv[4]), H = atoi(argv[5]);
  const int has_n = atoi(argv[6]), has_c = atoi(argv[7]);
  const unsigned setup_blocks = (unsigned)atoi(argv[8]), large_blocks = (unsigned)atoi(argv[9]);
  const std::vector<char> raw = read_file(argv[10]);
  const std::string outdir = argv[11];
  size_t off = 0;
  mraster::Mesh m;
  m.counts = take<long long>(raw, off, 2);
  const float* clear = take<float>(raw, off, 4);
  const float* mats = take<float>(raw, off, (size_t)views * 32);
  m.verts = take<float>(raw, off, (size_t)v_cap * 3);
  m.faces = take<int32_t>(raw, off, (size_t)f_cap * 3);
  m.normals = has_n ? take<float>(raw, off, (size_t)v_cap * 3) : nullptr;
  m.colours = has_c ? take<float>(raw, off, (size_t)v_cap * 3) : nullptr;
  m.v_cap = v_cap;
  m.f_cap = f_cap;
  if (off != raw.size()) { fprintf(stderr, "in.bin size mismatch\n"); return 2; }

  constexpr int kGuard = 16;
  const size_t npx = (size_t)W * H * views;
  std::vector<unsigned long long> keys(npx, mraster::kClearKey);        // the memset node
  std::vector<uint2> list((size_t)views * f_cap + kGuard, uint2{0xA5A5A5A5u, 0xA5A5A5A5u});
  uint32_t list_len = 0;
  mraster::Target t;
  t.mats = mats;
  t.views = views;
  t.W = W;
  t.H = H;
  t.keys = keys.data();
  t.list = list.data();
  t.list_len = &list_len;
  std::vector<float> normal(has_n ? npx * 4 + kGuard : 0, -777.f), colour(has_c ? npx * 4 + kGuard : 0, -777.f);
  mraster::Shade s;
  s.normal = has_n ? normal.data() : nullptr;
  s.colour = has_c ? colour.data() : nullptr;
  for (int k = 0; k < 4; ++k) s.clear[k] = clear[k];
  if (f_cap > 0) {
    cuda_emu::launch(dim3(setup_blocks, views), dim3(mraster::kSetupThreads), [&] { mraster::raster_setup_kernel(m, t); });
    cuda_emu::launch(dim3(large_blocks), dim3(mraster::kLargeThreads), [&] { mraster::raster_large_kernel(m, t); });
  }
  cuda_emu::launch(dim3((unsigned)((W * H + mraster::kResolveThreads - 1) / mraster::kResolveThreads), views),
                   dim3(mraster::kResolveThreads), [&] { mraster::raster_resolve_kernel(m, t, s); });
  for (size_t k = (size_t)views * f_cap; k < list.size(); ++k)
    if (list[k].x != 0xA5A5A5A5u || list[k].y != 0xA5A5A5A5u) { fprintf(stderr, "list written beyond its capacity\n"); return 3; }
  for (int g = 0; g < kGuard; ++g)
    if ((has_n && normal[npx * 4 + g] != -777.f) || (has_c && colour[npx * 4 + g] != -777.f)) {
      fprintf(stderr, "image written beyond its end\n");
      return 3;
    }
  write_file(outdir + "/keys.u64", keys.data(), npx * 8);
  if (has_n) write_file(outdir + "/normal.f32", normal.data(), npx * 16);
  if (has_c) write_file(outdir + "/colour.f32", colour.data(), npx * 16);
  printf("%u\n", list_len);
  return 0;
}
