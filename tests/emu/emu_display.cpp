// TEST INFRASTRUCTURE ONLY: the display-image kernel (monoport_b200/csrc/surface_kernels.cuh) on the CPU emulation layer,
// launched like mp_display_async in surface.cu, on `blocks` CTAs (grid-stride).
//   emu_display R S blocks images in.bin out.bin
// images: "both", "norm" or "tex".  in.bin: the present [R,R,3] float32 canvases, normal image first.
// out.bin: the present [S,S,3] float32 images, normal image first, then the [S,S] uint8 mask.
#include "cuda_emu.h"

#include "../../monoport_b200/csrc/surface_kernels.cuh"

using namespace surface_k;

int main(int argc, char** argv) {
  if (argc != 7) { fprintf(stderr, "usage: emu_display R S blocks both|norm|tex in.bin out.bin\n"); return 2; }
  const int R = atoi(argv[1]), S = atoi(argv[2]), blocks = atoi(argv[3]);
  const bool has_norm = strcmp(argv[4], "tex") != 0, has_tex = strcmp(argv[4], "norm") != 0;
  const size_t in_n = (size_t)R * R * 3, px = (size_t)S * S;
  std::vector<float> norm(has_norm ? in_n : 0), tex(has_tex ? in_n : 0);
  FILE* f = fopen(argv[5], "rb");
  if (!f || fread(norm.data(), 4, norm.size(), f) != norm.size() || fread(tex.data(), 4, tex.size(), f) != tex.size()) {
    fprintf(stderr, "short input\n");
    return 2;
  }
  fclose(f);
  // every output is followed by a guard value: a write past its end fails the run
  std::vector<float> norm_out(3 * px + 1, -4242.f), tex_out(3 * px + 1, -4242.f);
  std::vector<uint8_t> mask(px + 1, 77);
  const float* np_ = has_norm ? norm.data() : nullptr;
  const float* tp = has_tex ? tex.data() : nullptr;
  float* no = has_norm ? norm_out.data() : nullptr;
  float* to = has_tex ? tex_out.data() : nullptr;
  uint8_t* mp = mask.data();
  cuda_emu::launch(dim3((unsigned)blocks), dim3(kDispThreads), [&] { display_kernel(np_, tp, R, S, no, to, mp); });
  if (norm_out[3 * px] != -4242.f || tex_out[3 * px] != -4242.f || mask[px] != 77) {
    fprintf(stderr, "wrote past an output\n");
    return 3;
  }
  f = fopen(argv[6], "wb");
  if (has_norm) fwrite(norm_out.data(), 4, 3 * px, f);
  if (has_tex) fwrite(tex_out.data(), 4, 3 * px, f);
  fwrite(mask.data(), 1, px, f);
  fclose(f);
  return 0;
}
