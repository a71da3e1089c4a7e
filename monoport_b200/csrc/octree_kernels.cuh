// Device code of the coarse-to-fine occupancy engine (see octree.cu for the pipeline and the host side).  Free of host
// API calls and CUDA runtime types so that tests/emu can run these kernels unmodified on the CPU emulation layer.
#pragma once
#include <stdint.h>
#include "mp_scan.cuh"

namespace octree_k {


__device__ __forceinline__ float up_axis(float a, float b, bool odd) {
  // align_corners=True 2x: even fine index -> coarse node; odd -> 0.5*a + 0.5*b (exact products, one rounding)
  return odd ? __fadd_rn(__fmul_rn(0.5f, a), __fmul_rn(0.5f, b)) : a;
}

// candidates_t may be null (top-k engine / last "faster" level): then only the interpolation runs (W = 0).
// One thread = one COARSE cell (k,j,i) -> its 2x2x2 fine nodes (2k+a, 2j+b, 2i+c): the eight corner loads are shared by
// the eight interpolations (same operations per output as the per-node form, so bit-identical), and the eight box
// tests share one pass over the union of their boxes -- per axis the box of parity 0 is [l0,h0], of parity 1 [l1,h1]
// with l0<=l1<=h0<=h1, so the union is [l0,h1] (at most W = radius + 2 wide); a box is "mixed" iff OR != AND of its
// occupancy bits, and OR/AND separate per axis.  A z slice of the union (W x W values) is loaded unconditionally
// (clamped addresses, masked afterwards) before any of it is used: the loads of a slice overlap, which matters on the
// small levels where a handful of threads per SM walk a cold L1 (a load-test-branch chain costs ~30 us there).
// Launch: grid (ceil(res_c^2 / 256), res_c).
template <int W>
__global__ void __launch_bounds__(256)
upsample_kernel(const float* __restrict__ vc, const uint8_t* __restrict__ known_c, float* __restrict__ vf,
                uint8_t* __restrict__ known_f, uint8_t* __restrict__ candidates_t, int res_c, int res_f, int radius,
                float balance) {
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= res_c * res_c) return;
  const int i = blockIdx.y;
  const int j = p / res_c, k = p - j * res_c;
  const int ex = (k + 1 < res_c) ? 1 : 0, ey = (j + 1 < res_c) ? 1 : 0, ez = (i + 1 < res_c) ? 1 : 0;   // odd nodes exist
  float c[2][2][2];
#pragma unroll
  for (int zi = 0; zi < 2; ++zi)
#pragma unroll
    for (int yj = 0; yj < 2; ++yj) {
      const float* row = vc + ((long long)(i + zi * ez) * res_c + (j + yj * ey)) * res_c + k;
      c[zi][yj][0] = __ldg(row);
      c[zi][yj][1] = __ldg(row + ex);
    }
  const long long plane_f = (long long)res_f * res_f;
  const bool cell_known = known_c == nullptr || known_c[((long long)i * res_c + j) * res_c + k];
#pragma unroll
  for (int cz = 0; cz < 2; ++cz)
#pragma unroll
    for (int by = 0; by < 2; ++by)
#pragma unroll
      for (int ax = 0; ax < 2; ++ax) {
        if ((cz && !ez) || (by && !ey) || (ax && !ex)) continue;
        const float c00 = up_axis(c[0][0][0], c[0][0][1], ax), c01 = up_axis(c[0][1][0], c[0][1][1], ax);
        const float c10 = up_axis(c[1][0][0], c[1][0][1], ax), c11 = up_axis(c[1][1][0], c[1][1][1], ax);
        const float v = up_axis(up_axis(c00, c01, by), up_axis(c10, c11, by), cz);
        const long long o = (long long)(2 * i + cz) * plane_f + (long long)(2 * j + by) * res_f + (2 * k + ax);
        vf[o] = v;
        if (known_f) known_f[o] = (!(cz | by | ax) && cell_known) ? 1 : 0;
      }
  if constexpr (W > 0) {
    int lx[2], hx[2], ly[2], hy[2], lz[2], hz[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int fx = 2 * k + q, fy = 2 * j + q, fz = 2 * i + q;
      lx[q] = max(fx - radius, 0) >> 1; hx[q] = (min(fx + radius, res_f - 1) + 1) >> 1;
      ly[q] = max(fy - radius, 0) >> 1; hy[q] = (min(fy + radius, res_f - 1) + 1) >> 1;
      lz[q] = max(fz - radius, 0) >> 1; hz[q] = (min(fz + radius, res_f - 1) + 1) >> 1;
    }
    // bit (4*cz + 2*by + ax) of orm / andm: OR / AND of the occupancy bits over that node's box
    unsigned orm = 0u, andm = 0xFFu;
    for (int zz = lz[0]; zz <= hz[1]; ++zz) {
      const unsigned zin = ((zz <= hz[0]) ? 1u : 0u) | ((zz >= lz[1]) ? 2u : 0u);
      float v[W][W];
#pragma unroll
      for (int yi = 0; yi < W; ++yi) {
        const float* row = vc + ((long long)zz * res_c + min(ly[0] + yi, res_c - 1)) * res_c;
#pragma unroll
        for (int xi = 0; xi < W; ++xi) v[yi][xi] = __ldg(row + min(lx[0] + xi, res_c - 1));
      }
#pragma unroll
      for (int yi = 0; yi < W; ++yi) {
        const int yy = ly[0] + yi;
        // rows beyond the union take part in no box: yin = 0
        const unsigned yin = (yy <= hy[1]) ? (((yy <= hy[0]) ? 1u : 0u) | ((yy >= ly[1]) ? 2u : 0u)) : 0u;
        unsigned o0 = 0u, a0 = 1u, o1 = 0u, a1 = 1u;
#pragma unroll
        for (int xi = 0; xi < W; ++xi) {
          const int xx = lx[0] + xi;
          const unsigned bit = (v[yi][xi] > balance) ? 1u : 0u;
          if (xx <= hx[0]) { o0 |= bit; a0 &= bit; }
          if (xx >= lx[1] && xx <= hx[1]) { o1 |= bit; a1 &= bit; }
        }
        const unsigned orow = o0 | (o1 << 1), arow = a0 | (a1 << 1);   // per x parity
#pragma unroll
        for (int cz = 0; cz < 2; ++cz)
#pragma unroll
          for (int by = 0; by < 2; ++by)
            if (((zin >> cz) & 1u) && ((yin >> by) & 1u)) {
              const int sh = 4 * cz + 2 * by;
              orm |= orow << sh;
              andm &= ~(0x3u << sh) | (arow << sh);
            }
      }
    }
    const unsigned mixed = orm & ~andm;
#pragma unroll
    for (int cz = 0; cz < 2; ++cz)
#pragma unroll
      for (int by = 0; by < 2; ++by)
#pragma unroll
        for (int ax = 0; ax < 2; ++ax) {
          if ((cz && !ez) || (by && !ey) || (ax && !ex)) continue;
          const bool known = !(cz | by | ax) && cell_known;
          const bool cand = !known && ((mixed >> (4 * cz + 2 * by + ax)) & 1u);
          candidates_t[((long long)(2 * k + ax) * res_f + (2 * j + by)) * res_f + (2 * i + cz)] = cand ? 1 : 0;
        }
  }
}

// functors for the ordered compaction -------------------------------------------------------------
struct FlagF {
  const uint8_t* flags;       // cudaMalloc'ed (8-byte aligned) 0/1 flags
  static constexpr bool kVec8 = true;
  __device__ unsigned long long operator()(long long i) const { return flags[i]; }
  __device__ void load8(long long i, unsigned long long (&v)[8]) const {
    uint32_t b[8];
    mpscan::load_bytes8(flags, i, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = b[j];
  }
};
struct EmitNodesT {      // i indexes the transposed [x][y][z] flag volume
  int32_t* idx;
  int res;
  long long cap;
  __device__ void operator()(long long i, unsigned long long v, unsigned long long pos) const {
    if (v && (long long)pos < cap) {
      const int z = (int)(i % res), y = (int)((i / res) % res), x = (int)(i / ((long long)res * res));
      idx[pos] = (z * res + y) * res + x;
    }
  }
};

// scan hook: clamp the number of candidates to the list capacity and publish it as the device-side point count
struct CountPost {
  int32_t* count; long long cap; long long* stat;
  __device__ void operator()(unsigned long long t) const {
    if ((long long)t > cap) t = (unsigned long long)cap;
    *count = (int32_t)t;
    if (stat) *stat += (long long)t;
  }
};

__global__ void iota_kernel(int32_t* idx, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) idx[i] = i;
}

// a scalar parameter -> device memory (instead of a host-to-device copy from a stack variable: graph-capturable)
__global__ void set_i64_kernel(long long* p, long long v) { *p = v; }

__global__ void set_u8_kernel(uint8_t* p, long long n, uint8_t v) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

__global__ void any_gt_kernel(const float* __restrict__ v, long long n, float thr, int* flag) {
  bool any = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    any |= v[i] > thr;
  if (__syncthreads_or(any) && threadIdx.x == 0) atomicOr(flag, 1);
}

// scatter values of the evaluated nodes; mark them known; (lossless) flag sign conflicts with the interpolation
__global__ void scatter_kernel(const int32_t* __restrict__ idx, const int32_t* count_dev, long long n_max,
                               const float* __restrict__ vals, float* __restrict__ vol, uint8_t* __restrict__ known,
                               uint8_t* __restrict__ conflict, float balance, bool write_vals) {
  long long n = n_max;
  if (count_dev) { const long long c = *count_dev; n = c < n ? c : n; }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int node = idx[i];
    const float nv = vals[i];
    if (conflict) {
      const float ov = vol[node];
      conflict[node] = ((ov - balance) * (nv - balance) < 0.f) ? 1 : 0;
    }
    if (write_vals) vol[node] = nv;
    if (known) known[node] = 1;
  }
}

// candidates = unknown nodes with a conflict in their 27-neighbourhood (transposed output); clears nothing
__global__ void conflict_neighbours_kernel(const uint8_t* __restrict__ conflict, const uint8_t* __restrict__ known,
                                           uint8_t* __restrict__ candidates_t, int res) {
  const long long n = (long long)res * res * res;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % res), y = (int)((i / res) % res), z = (int)(i / ((long long)res * res));
    bool cand = false;
    if (!known[i]) {
      for (int dz = -1; dz <= 1 && !cand; ++dz)
        for (int dy = -1; dy <= 1 && !cand; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            const int xx = x + dx, yy = y + dy, zz = z + dz;
            if (xx < 0 || yy < 0 || zz < 0 || xx >= res || yy >= res || zz >= res) continue;
            if (conflict[((long long)zz * res + yy) * res + xx]) { cand = true; break; }
          }
    }
    candidates_t[((long long)x * res + y) * res + z] = cand ? 1 : 0;
  }
}

// ---- device-driven conflict loop (lossless engine, body of a CUDA-graph WHILE node) ---------------------------------
// After one pass of a level (evaluate the list, scatter with conflict detection, build the next conflict list): count the
// pass, and run another while the new list is non-empty.  A level that reaches `cap` passes with nodes still listed stops
// and is reported in *truncated (level + 1).  Every continuing pass makes at least one unknown node known, so the loop ends
// by itself; the cap only bounds how long a defect could keep the GPU busy.
__device__ __forceinline__ unsigned conflict_loop_continue(const int32_t* count, int32_t* passes, int32_t* truncated,
                                                           int level, int cap) {
  const int32_t p = *passes + 1;
  *passes = p;
  if (*count <= 0) return 0u;
  if (p >= cap) { *truncated = level + 1; return 0u; }
  return 1u;
}
// (the kernel that hands this decision to the WHILE node is loop_control_kernel in octree_loop.cuh)

// ---- top-k (Seg3dTopk): radix select of the k smallest |v - balance| with index tie-break ------------
__device__ __forceinline__ uint32_t topk_key(float v, float balance) { return __float_as_uint(fabsf(v - balance)); }

struct SelectState {          // device-resident
  uint32_t prefix;            // known high bits of the k-th key
  uint32_t remaining;         // rank still to locate inside the prefix bucket (1-based)
  uint32_t hist[256];
  uint32_t threshold;         // final k-th smallest key
  uint32_t need_equal;        // how many keys == threshold to take (lowest indices first)
};

__global__ void select_init_kernel(SelectState* s, uint32_t k) {
  if (threadIdx.x < 256) s->hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) { s->prefix = 0; s->remaining = k; s->threshold = 0; s->need_equal = 0; }
}

__global__ void select_hist_kernel(const float* __restrict__ v, long long n, float balance, SelectState* s, int pass) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int shift = 24 - 8 * pass;
  const uint32_t mask_hi = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
  const uint32_t prefix = s->prefix;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t key = topk_key(v[i], balance);
    if ((key & mask_hi) == prefix) atomicAdd(&h[(key >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&s->hist[threadIdx.x], h[threadIdx.x]);
}

__global__ void select_pick_kernel(SelectState* s, int pass) {
  if (threadIdx.x == 0) {
    const int shift = 24 - 8 * pass;
    uint32_t rem = s->remaining, b = 0;
    for (; b < 256; ++b) {
      const uint32_t c = s->hist[b];
      if (rem <= c) break;
      rem -= c;
    }
    if (b > 255) b = 255;
    s->prefix |= (b << shift);
    s->remaining = rem;
    if (pass == 3) { s->threshold = s->prefix; s->need_equal = rem; }
  }
  __syncthreads();
  if (threadIdx.x < 256) s->hist[threadIdx.x] = 0;
}

// A top-k level's node count: k after a non-empty level 0, else 0 (the generic run stops there and evaluates nothing
// more); decided on the device so that a captured frame needs no host read.  Also the level's evaluated-node stat.
__global__ void topk_count_kernel(int32_t* count, long long* stat, const int* nonempty, int32_t k) {
  const int32_t n = *nonempty ? k : 0;
  *count = n;
  if (stat) *stat = n;
}

struct TopkF {   // low 32 bits: key < T ; high 32 bits: key == T
  const float* v; float balance; const SelectState* s;
  static constexpr bool kVec8 = false;
  __device__ unsigned long long operator()(long long i) const {
    const uint32_t key = topk_key(v[i], balance), t = s->threshold;
    return key < t ? 1ull : (key == t ? (1ull << 32) : 0ull);
  }
};
struct TopkEmit {
  int32_t* idx; const SelectState* s;
  __device__ void operator()(long long i, unsigned long long val, unsigned long long pre) const {
    if (!val) return;
    const uint32_t less_before = (uint32_t)pre, eq_before = (uint32_t)(pre >> 32), need = s->need_equal;
    if (val >> 32) { if (eq_before >= need) return; }
    idx[less_before + min(eq_before, need)] = (int32_t)i;
  }
};

}  // namespace octree_k
