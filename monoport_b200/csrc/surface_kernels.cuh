// Device code of the visible-surface extraction (see surface.cu).  Free of host API calls and CUDA runtime types so that
// tests/emu can run these kernels unmodified on the CPU emulation layer.
#pragma once
#include <stdint.h>
#include "mp_scan.cuh"

namespace surface_k {


// A[x,y,k] of RTL/recon.py:53-55 expressed on the raw [z,y,x] volume for the four directions.
//   front: A[x,y,k] = vol[R-1-k, y, x]          back : A[x,y,k] = vol[k, y, x]
//   left : A[x,y,k] = vol[x, y, R-1-k]          right: A[x,y,k] = vol[R-1-x, y, R-1-k]   (see derivation in DESIGN.md)
__device__ __forceinline__ long long a_index(int dir, int R, int x, int y, int k) {
  switch (dir) {
    case 0: return ((long long)(R - 1 - k) * R + y) * R + x;
    case 1: return ((long long)k * R + y) * R + x;
    case 2: return ((long long)x * R + y) * R + (R - 1 - k);
    default: return ((long long)(R - 1 - x) * R + y) * R + (R - 1 - k);
  }
}

// A[x,y,k] = vol[base + k * stride]: the column walk of a_index as an affine index
__device__ __forceinline__ void column_walk(int dir, int R, int x, int y, long long& base, long long& stride) {
  base = a_index(dir, R, x, y, 0);
  stride = a_index(dir, R, x, y, 1) - base;
}

// 32 columns x 8 depth slices per block: every thread walks ONE slice of its column (R/8 nodes, in batches of independent
// loads), the block keeps the first slice with a hit.  One thread per whole column made an empty column a chain of R/16
// dependent memory round trips (17 at R = 257: 24 us); here it is ceil(R/8/17) = 2.  For front/back the 32 lanes of a warp
// walk 32 consecutive x (coalesced); for left/right k is the contiguous axis and a thread reads 17 consecutive floats.
constexpr int kHitCols = 32, kHitSlices = 8, kHitBatch = 17;
__global__ void __launch_bounds__(kHitCols * kHitSlices)
first_hit_kernel(const float* __restrict__ vol, int R, int dir, int32_t* __restrict__ first_t) {
  __shared__ int s_hit[kHitSlices][kHitCols];
  const int n = R * R;
  const int cx = threadIdx.x % kHitCols, sl = threadIdx.x / kHitCols;
  const int len = (R + kHitSlices - 1) / kHitSlices;
  for (int c0 = blockIdx.x * kHitCols; c0 < n; c0 += gridDim.x * kHitCols) {     // (block-uniform trip count)
    const int c = c0 + cx;
    int hit = -1;
    if (c < n) {
      const int x = c % R, y = c / R;
      long long base, stride;
      column_walk(dir, R, x, y, base, stride);
      const int k_end = min(R, (sl + 1) * len);
      for (int k0 = sl * len; k0 < k_end && hit < 0; k0 += kHitBatch) {
        float v[kHitBatch];
#pragma unroll
        for (int j = 0; j < kHitBatch; ++j) v[j] = (k0 + j < k_end) ? __ldg(vol + base + (long long)(k0 + j) * stride) : 0.f;
#pragma unroll
        for (int j = kHitBatch - 1; j >= 0; --j)
          if (v[j] > 0.5f) hit = k0 + j;
      }
    }
    s_hit[sl][cx] = hit;
    __syncthreads();
    if (sl == 0 && c < n) {
      int h = -1;
#pragma unroll
      for (int q = kHitSlices - 1; q >= 0; --q)
        if (s_hit[q][cx] >= 0) h = s_hit[q][cx];
      first_t[(c % R) * R + c / R] = h;    // transposed: scan order is x-major
    }
    __syncthreads();
  }
}

struct HitF {
  const int32_t* first_t;
  static constexpr bool kVec8 = false;
  __device__ unsigned long long operator()(long long i) const { return first_t[i] >= 0 ? 1ull : 0ull; }
};

struct HitEmit {
  const float* vol; const int32_t* first_t; int R; int dir;
  long long* X; long long* Y; float* Z; float* N;
  __device__ void operator()(long long i, unsigned long long v, unsigned long long pos) const {
    if (!v) return;
    const int x = (int)(i / R), y = (int)(i % R), k = first_t[i];
    const int k2 = max(k - 2, 0), y2 = max(y - 2, 0), x2 = max(x - 2, 0);      // RTL/recon.py:63-68
    const float v1 = vol[a_index(dir, R, x, y, k)];
    const float v2 = vol[a_index(dir, R, x, y, k2)];
    const float v3 = vol[a_index(dir, R, x, y2, k)];
    const float v4 = vol[a_index(dir, R, x2, y, k)];
    // :77  Z = k2*(0.5-v1)/(v2-v1) + k*(v2-0.5)/(v2-v1), evaluated left to right with separate roundings
    const float d = __fsub_rn(v2, v1);
    float z = __fadd_rn(__fdiv_rn(__fmul_rn((float)k2, __fsub_rn(0.5f, v1)), d),
                        __fdiv_rn(__fmul_rn((float)k, __fsub_rn(v2, 0.5f)), d));
    if (z == z) z = fminf(fmaxf(z, 0.f), (float)R);                              // :78 (NaN stays NaN like torch.clamp)
    const float nx = __fsub_rn(v4, v1), ny = __fsub_rn(v3, v1), nz = __fsub_rn(v2, v1);
    // torch.norm(p=2): sqrt(sum of squares) -- accumulate in the same x,y,z order
    const float nn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
    X[pos] = x; Y[pos] = y; Z[pos] = z;
    N[3 * pos + 0] = __fdiv_rn(nx, nn); N[3 * pos + 1] = __fdiv_rn(ny, nn); N[3 * pos + 2] = __fdiv_rn(nz, nn);
  }
};

// The normal image of the demo (RTL/main.py:212-228): canvas[X[i], Y[i], :] = clamp((norm[i] + 1) / 2, 0, 1) for the
// min(*count, cap) vertices of forward_vertices.  The bits are torch's: one rounding for the sum, the halving is exact, and
// the clamp lets NaN through (the normals of a column whose finite differences vanish are NaN) -- no fminf / fmaxf.
constexpr int kNormThreads = 256;
__global__ void __launch_bounds__(kNormThreads)
render_normals_kernel(const long long* __restrict__ X, const long long* __restrict__ Y, const float* __restrict__ norm,
                      const long long* __restrict__ count, long long cap, int R, float* __restrict__ canvas) {
  long long n = *count;
  if (n > cap) n = cap;
  const long long step = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += step) {
    float* px = canvas + ((size_t)X[i] * R + (size_t)Y[i]) * 3;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      float v = __fmul_rn(__fadd_rn(norm[3 * i + a], 1.f), 0.5f);
      v = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
      px[a] = v;
    }
  }
}

// The display images of the demo (visulization, RTL/main.py:252-281) for one S x S output: each [R,R,3] canvas C (either
// may be NULL, not both) becomes C * 255 rotated by torch.rot90(k=1, dims [0,1]) and resized by nearest F.interpolate,
// i.e. out[y][x] = C[nx][R-1-ny] * 255 with upsample_nearest2d's index n = min((int)floorf(dst * (R / S)), R - 1) (its
// S == R and S == 2R special cases select the same texels).  mask[y][x] = 0 iff the three values of the reference image
// (the texture image if present, else the normal image) all equal 255 after the multiply -- a NaN value is foreground.
// One thread per output pixel when launched with ceil(S^2 / kDispThreads) blocks (grid-stride for smaller grids).
constexpr int kDispThreads = 256;
__global__ void __launch_bounds__(kDispThreads)
display_kernel(const float* __restrict__ norm, const float* __restrict__ tex, int R, int S, float* __restrict__ norm_out,
               float* __restrict__ tex_out, uint8_t* __restrict__ mask) {
  const float scale = (float)R / (float)S;
  const long long n = (long long)S * S;
  const long long step = (long long)gridDim.x * blockDim.x;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += step) {
    const int y = (int)(p / S), x = (int)(p % S);
    const int ny = min((int)floorf(__fmul_rn((float)y, scale)), R - 1);
    const int nx = min((int)floorf(__fmul_rn((float)x, scale)), R - 1);
    const size_t src = ((size_t)nx * R + (size_t)(R - 1 - ny)) * 3;
    float nv[3] = {0.f, 0.f, 0.f}, tv[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (norm) norm_out[3 * p + c] = nv[c] = __fmul_rn(norm[src + c], 255.0f);
      if (tex) tex_out[3 * p + c] = tv[c] = __fmul_rn(tex[src + c], 255.0f);
    }
    const bool from_tex = tex != nullptr;             // the mask's reference image
    bool bg = true;
#pragma unroll
    for (int c = 0; c < 3; ++c) bg = bg && (from_tex ? tv[c] : nv[c]) == 255.0f;
    mask[p] = bg ? 0 : 1;
  }
}

}  // namespace surface_k
