// TEST INFRASTRUCTURE ONLY: the normal-image kernel (monoport_b200/csrc/surface_kernels.cuh) on the CPU emulation layer,
// launched like mp_render_normals_async in surface.cu.
//   emu_render_normals R cap count blocks in.bin out.f32
// in.bin: X [cap] int64, Y [cap] int64, norm [cap*3] float32.  out.f32: the [R,R,3] canvas, background 1.
#include "cuda_emu.h"

#include "../../monoport_b200/csrc/surface_kernels.cuh"

using namespace surface_k;

int main(int argc, char** argv) {
  if (argc != 7) { fprintf(stderr, "usage: emu_render_normals R cap count blocks in.bin out.f32\n"); return 2; }
  const int R = atoi(argv[1]);
  const long long cap = atoll(argv[2]), count = atoll(argv[3]);
  const int blocks = atoi(argv[4]);
  std::vector<long long> X(cap), Y(cap);
  std::vector<float> N(3 * cap);
  FILE* f = fopen(argv[5], "rb");
  if (!f || fread(X.data(), 8, cap, f) != (size_t)cap || fread(Y.data(), 8, cap, f) != (size_t)cap ||
      fread(N.data(), 4, 3 * cap, f) != (size_t)(3 * cap)) { fprintf(stderr, "short input\n"); return 2; }
  fclose(f);
  std::vector<float> canvas((size_t)R * R * 3 + 1, 1.0f);
  canvas[(size_t)R * R * 3] = -4242.f;
  const long long* xp = X.data();
  const long long* yp = Y.data();
  const float* np_ = N.data();
  const long long* cp = &count;
  float* out = canvas.data();
  cuda_emu::launch(dim3((unsigned)blocks), dim3(kNormThreads), [&] { render_normals_kernel(xp, yp, np_, cp, cap, R, out); });
  if (canvas[(size_t)R * R * 3] != -4242.f) { fprintf(stderr, "wrote past the canvas\n"); return 3; }
  f = fopen(argv[6], "wb");
  fwrite(canvas.data(), 4, (size_t)R * R * 3, f);
  fclose(f);
  return 0;
}
