// Device code of F3 marching cubes (see mcubes.cu for the pipeline).  Kept free of host API calls and of CUDA runtime
// types so that tests/emu can run these kernels unmodified on the CPU emulation layer of the build container.
//
// Everything after the first pass works on a BIT VOLUME: one occupancy bit (value > iso) per node in linear node order,
// word w = nodes 32w .. 32w+31 (a word may straddle rows).  At 257^3 that is 2.1 MB instead of 68 MB, so the volume is
// read from HBM exactly once (bits_kernel, streaming); neighbour lookups become funnel shifts of L1/L2-resident words, and
// the ~95 % of words whose eight shifted copies agree (no surface inside) cost a dozen loads and seven XORs.
#pragma once
#include <stdint.h>
#include "mp_scan.cuh"
#include "mc_table.inc"

namespace mcubes {

constexpr int kBitsThreads = 256;
constexpr int kBitsUnroll = 8;      // words (= 128 B lines of the volume) a warp has in flight per iteration

// zero words the bit volume carries behind the last node so that neighbour reads (+1, +W, +H*W and their sums) of the
// last words never leave the allocation
__host__ __device__ inline long long bits_pad_words(int H, int W) { return ((long long)H * W + W + 1) / 32 + 3; }

// ---- pass 1: volume -> bits.  HBM-bound: 4 B read per node, 1 bit written.
__global__ void __launch_bounds__(kBitsThreads)
bits_kernel(const float* __restrict__ vol, uint32_t* __restrict__ bits, long long n, float iso) {
  const long long n_words = (n + 31) >> 5;
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * (kBitsThreads / 32) + (threadIdx.x >> 5);
  const long long n_warps = (long long)gridDim.x * (kBitsThreads / 32);
  for (long long w0 = warp0 * kBitsUnroll; w0 < n_words; w0 += n_warps * kBitsUnroll) {     // (warp-uniform trip count)
    float v[kBitsUnroll];
#pragma unroll
    for (int j = 0; j < kBitsUnroll; ++j) {
      const long long i = (w0 + j) * 32 + lane;
      v[j] = i < n ? __ldg(vol + i) : iso;                  // (iso > iso is false: nodes past the end read as outside)
    }
#pragma unroll
    for (int j = 0; j < kBitsUnroll; ++j) {
      const uint32_t m = __ballot_sync(0xffffffffu, v[j] > iso);
      if (lane == j && w0 + j < n_words) bits[w0 + j] = m;  // lanes 0..7 store eight consecutive words: one 32 B segment
    }
  }
}

// bits of nodes 32w + s .. 32w + s + 31
__device__ __forceinline__ uint32_t shifted_word(const uint32_t* __restrict__ bits, long long w, long long s) {
  const long long i = 32 * w + s;
  const long long q = i >> 5;
  return __funnelshift_r(__ldg(bits + q), __ldg(bits + q + 1), (uint32_t)(i & 31));
}

// the eight corner bit-vectors of the cells whose corner 0 is a node of word w: index c = dx | dy << 1 | dz << 2
__device__ __forceinline__ void corner_words(const uint32_t* __restrict__ bits, long long w, int H, int W, uint32_t (&v)[8]) {
  const long long sy = W, sz = (long long)H * W;
  v[0] = __ldg(bits + w);
  v[1] = shifted_word(bits, w, 1);
  v[2] = shifted_word(bits, w, sy);
  v[3] = shifted_word(bits, w, sy + 1);
  v[4] = shifted_word(bits, w, sz);
  v[5] = shifted_word(bits, w, sz + 1);
  v[6] = shifted_word(bits, w, sz + sy);
  v[7] = shifted_word(bits, w, sz + sy + 1);
}

__device__ __forceinline__ int case_of(const uint32_t (&v)[8], int b) {
  int k = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) k |= (int)((v[c] >> b) & 1u) << c;
  return k;
}

// per word: x / y / z edge masks (bit b: node 32w+b owns an active +x / +y / +z edge) and the triangle count of its cells
struct WordInfo {
  uint32_t ex, ey, ez, nt;
};

// ---- pass 2 (runs inside the scan's first pass): edge masks + triangle count of one word.  Uniform words (all eight
// shifted copies equal) leave at once.
// `ntri`: the 256 triangle counts (byte 15 of the table rows), staged in shared memory by the caller
__device__ __forceinline__ WordInfo classify_word(const uint32_t* __restrict__ bits, long long w, long long n, int D, int H, int W,
                                                  const uint8_t* ntri) {
  uint32_t v[8];
  corner_words(bits, w, H, W, v);
  uint32_t mixed = 0;
#pragma unroll
  for (int c = 1; c < 8; ++c) mixed |= v[0] ^ v[c];
  WordInfo wi{0u, 0u, 0u, 0u};
  if (mixed) {
    // which nodes of the word have a +x / +y / +z neighbour (a word may straddle rows and planes)
    uint32_t xi = 0, yi = 0, zi = 0;
    const long long i0 = 32 * w;
    const uint32_t i0u = (uint32_t)i0;                              // (the volume has fewer than 2^31 nodes)
    const uint32_t t = i0u / (uint32_t)W;
    int x = (int)(i0u - t * (uint32_t)W);
    int z = (int)(t / (uint32_t)H), y = (int)(t - (uint32_t)z * (uint32_t)H);
    for (int b = 0; b < 32 && i0 + b < n; ++b) {
      if (x + 1 < W) xi |= 1u << b;
      if (y + 1 < H) yi |= 1u << b;
      if (z + 1 < D) zi |= 1u << b;
      if (++x == W) { x = 0; if (++y == H) { y = 0; ++z; } }
    }
    wi.ex = (v[0] ^ v[1]) & xi;
    wi.ey = (v[0] ^ v[2]) & yi;
    wi.ez = (v[0] ^ v[4]) & zi;
    uint32_t cm = mixed & xi & yi & zi;
    while (cm) {
      const int b = __ffs((int)cm) - 1;
      cm &= cm - 1;
      wi.nt += (uint32_t)ntri[case_of(v, b)];
    }
  }
  return wi;
}

__device__ __forceinline__ unsigned long long word_counts(const uint4 q) {
  return (unsigned long long)(__popc(q.x) + __popc(q.y) + __popc(q.z)) | ((unsigned long long)q.w << 32);
}

// The scan's first pass, specialised: one thread per word classifies it (coalesced), stores its info, and the CTA reduces the
// (vertex, triangle) counts.  A CTA covers a QUARTER of a 2048-word chunk of mp_scan (256 threads x 2 words) and adds its total
// into the chunk's slot: the words with a surface cluster in a few z ranges, and with whole chunks per CTA (1024 threads) the
// few CTAs that got them set the kernel's time (19.4 us; the classification as its own 256-thread kernel + a sums pass took
// 11.0 + 6.6).  The last CTA turns the chunk totals into offsets (mpscan::finish_block_sums).  sums[] must be zero on entry.
// A functor inside the generic block_sums_kernel was slower still (23.6 us: one thread classified eight consecutive words).
constexpr int kClassifyThreads = 256;
constexpr int kClassifyWords = 2 * kClassifyThreads;                  // words per CTA
constexpr int kClassifySplit = mpscan::kChunk / kClassifyWords;       // CTAs per chunk of the ordered scan
static_assert(mpscan::kChunk % kClassifyWords == 0, "a CTA must not straddle two chunks of the ordered scan");
__global__ void __launch_bounds__(kClassifyThreads)
classify_sums_kernel(const uint32_t* __restrict__ bits, WordInfo* __restrict__ info, long long n, int D, int H, int W,
                     unsigned long long* __restrict__ sums, int nb, unsigned long long* __restrict__ total) {
  // the triangle counts of the 256 cases: a word with a surface inside looks up one per mixed cell, back to back
  __shared__ uint8_t s_ntri[256];
  if (threadIdx.x < 256) s_ntri[threadIdx.x] = g_mc_tri[threadIdx.x][15];
  __syncthreads();
  const long long n_words = (n + 31) >> 5;
  unsigned long long s = 0;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const long long w = (long long)blockIdx.x * kClassifyWords + j * kClassifyThreads + threadIdx.x;
    if (w < n_words) {
      const WordInfo wi = classify_word(bits, w, n, D, H, W, s_ntri);
      const uint4 q = make_uint4(wi.ex, wi.ey, wi.ez, wi.nt);
      *reinterpret_cast<uint4*>(info + w) = q;
      s += word_counts(q);
    }
  }
  // CTA total: warp shuffles, then one warp over the warp totals
  __shared__ unsigned long long s_warp[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) s_warp[warp] = s;
  __syncthreads();
  if (warp == 0) {
    unsigned long long t = lane < kClassifyThreads / 32 ? s_warp[lane] : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) s_warp[0] = t;
  }
  __syncthreads();
  mpscan::finish_block_sums<kClassifyThreads>(s_warp[0], sums, nb, total, mpscan::NoPost(), (int)(blockIdx.x / kClassifySplit),
                                              (int)gridDim.x, true);
}

// functor of the scan's SECOND pass (and of everything after it): the stored info
struct WordCountF {    // low 32: vertices owned by the word's nodes, high 32: triangles of its cells
  const WordInfo* info;
  static constexpr bool kVec8 = false;
  __device__ unsigned long long operator()(long long w) const {
    // (plain load, not __ldg: the first pass of the same scan wrote it)
    return word_counts(*reinterpret_cast<const uint4*>(info + w));
  }
};

// exclusive (vertex, triangle) prefix of every word; words with a surface inside are also appended to the ACTIVE LIST the
// emission walks (one warp per entry).  The list's order is whatever the atomics give -- it does not matter: every word
// carries its own output offsets, so the mesh is the same for any order.
struct PrefixEmit {
  unsigned long long* prefix;
  uint32_t* active;            // [n_words] word indices
  uint32_t* n_active;          // zeroed before the scan
  __device__ void operator()(long long w, unsigned long long v, unsigned long long pre) const {
    prefix[w] = pre;
    if (v) active[atomicAdd(n_active, 1u)] = (uint32_t)w;
  }
};

// id of the vertex on the +`axis` edge owned by node i (the edge must be active)
__device__ __forceinline__ int32_t vertex_id(const WordInfo* __restrict__ info, const unsigned long long* __restrict__ prefix,
                                             uint32_t i, int axis) {
  const uint32_t w = i >> 5;
  const int b = (int)(i & 31u);
  const uint4 q = __ldg(reinterpret_cast<const uint4*>(info + w));
  const uint32_t below = (1u << b) - 1u;
  uint32_t id = (uint32_t)__ldg(prefix + w) + __popc(q.x & below) + __popc(q.y & below) + __popc(q.z & below);
  if (axis >= 1) id += (q.x >> b) & 1u;
  if (axis == 2) id += (q.y >> b) & 1u;
  return (int32_t)id;
}

// The vertex arithmetic of the emission, shared with mesh_edges_kernel and the refinement (refine_kernels.cuh), which must
// reproduce the emitted vertices bit for bit.
// (x, y, z) of node i (32-bit: mp_mcubes_create bounds the volume below 2^31 nodes)
__device__ __forceinline__ void node_xyz(uint32_t i, uint32_t plane, int W, uint32_t& x, uint32_t& y, uint32_t& z) {
  z = i / plane;
  const uint32_t r = i - z * plane;
  y = r / (uint32_t)W;
  x = r - y * (uint32_t)W;
}

// id of the first vertex owned by node `lane` of a word: the word's prefix + the owned edges of the nodes below it
__device__ __forceinline__ uint32_t word_vertex_base(unsigned long long pre, uint32_t ex, uint32_t ey, uint32_t ez, int lane) {
  const uint32_t below = (1u << lane) - 1u;
  return (uint32_t)pre + __popc(ex & below) + __popc(ey & below) + __popc(ez & below);
}

// the owned edges of node `lane` of a word: bit a = its +a edge is active
__device__ __forceinline__ uint32_t lane_edge_code(uint32_t ex, uint32_t ey, uint32_t ez, int lane) {
  return ((ex >> lane) & 1u) | (((ey >> lane) & 1u) << 1) | (((ez >> lane) & 1u) << 2);
}

// the linear interpolation of marching cubes: the parameter of iso between va (t = 0) and vb (t = 1)
__device__ __forceinline__ float edge_t0(float va, float vb, float iso) { return __fdiv_rn(__fsub_rn(iso, va), __fsub_rn(vb, va)); }

// index-space point at parameter t on the +axis edge of node (x, y, z)
__device__ __forceinline__ void edge_point(uint32_t x, uint32_t y, uint32_t z, int axis, float t, float (&p)[3]) {
  p[0] = (float)x; p[1] = (float)y; p[2] = (float)z;
  p[axis] = __fadd_rn(p[axis], t);
}

// index space -> reconstruction()'s world point (p + 0.5) * scale + b_min, with torch's three fp32 roundings (intrinsics, so
// that no FMA contraction fuses them)
__device__ __forceinline__ void world_point(const float (&scale)[3], const float (&bmin)[3], float (&p)[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) p[a] = __fadd_rn(__fmul_rn(__fadd_rn(p[a], 0.5f), scale[a]), bmin[a]);
}

// ---- pass 4: emission, two phases per round of a CTA.
// (a) one warp per word with a surface inside (the active list), one lane per node: up to three vertices (vertex id = rank of
//     (node, axis) in node order), and the cell's triangles are QUEUED in shared memory -- (corner-0 node, triangle index,
//     its three edge numbers); triangle index = the word's prefix + a warp scan, i.e. face order = (cell linear index, table
//     order).
// (b) the whole CTA walks the queue densely, one thread per face corner: edge -> owning node -> vertex id (the owning
//     word's prefix + popcounts) -> faces.
// Only about one cell in ten of an active word has triangles: resolving the corners in phase (a) made every warp run the
// 15-corner loop for its few cells (27-63 us at 257^3); walking 32 consecutive words per warp instead of a list left most
// warps empty and a few with a dozen dependent chains.  Node indices are 32-bit (mp_mcubes_create bounds the volume).
constexpr int kEmitThreads = 256;
constexpr int kEmitWarps = kEmitThreads / 32;
constexpr int kEmitQueue = kEmitWarps * 32 * MC_MAX_TRI;

// Where the emission writes, for the enqueue-only run (mesh_emit_async_kernel): vertex ids >= v_cap and face indices >=
// f_cap are not written, and with `world` set a vertex v is stored as (v + 0.5) * scale + b_min -- reconstruction()'s
// node-centre mapping, with torch's three fp32 roundings (intrinsics, so that no FMA contraction fuses them).
struct MeshOut {
  float* verts;
  int32_t* faces;
  uint32_t v_cap, f_cap;
  int world;
  float scale[3], bmin[3];
};

// The emission of one grid (the algorithm above), shared by the eager kernel (kCapped = false: every id is written, index
// space, n_active from the host) and the enqueue-only one (kCapped = true: MeshOut's capacities and world mapping, n_active
// read from the device).  `n_active` must be the same for every thread of the grid (it sets the uniform round count).
template <bool kCapped>
__device__ __forceinline__ void mesh_emit_body(const float* __restrict__ vol, const uint32_t* __restrict__ bits,
                                               const WordInfo* __restrict__ info, const unsigned long long* __restrict__ prefix,
                                               const uint32_t* __restrict__ active, uint32_t n_active, const MeshOut& out,
                                               int D, int H, int W, long long n, float iso) {
  float* __restrict__ verts = out.verts;
  int32_t* __restrict__ faces = out.faces;
  __shared__ uint32_t q_node[kEmitQueue], q_tri[kEmitQueue], q_edges[kEmitQueue];
  __shared__ uint32_t q_count;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t plane = (uint32_t)H * (uint32_t)W;
  const uint32_t per_round = gridDim.x * kEmitWarps;
  const uint32_t rounds = (n_active + per_round - 1) / per_round;                 // (uniform over the grid)
  for (uint32_t round = 0; round < rounds; ++round) {
    if (threadIdx.x == 0) q_count = 0;
    __syncthreads();
    const uint32_t e = (round * gridDim.x + blockIdx.x) * kEmitWarps + warp;
    if (e < n_active) {                                                           // (warp-uniform)
      const uint32_t w = __ldg(active + e);
      const uint4 wi = __ldg(reinterpret_cast<const uint4*>(info + w));
      const uint32_t ex = wi.x, ey = wi.y, ez = wi.z, nt = wi.w;
      const unsigned long long pre = __ldg(prefix + w);
      const uint32_t i = 32u * w + (uint32_t)lane;                                // this lane's node
      uint32_t x, y, z;
      node_xyz(i, plane, W, x, y, z);
      // ---- vertices on the owned edges
      const uint32_t code = lane_edge_code(ex, ey, ez, lane);
      if (code) {
        uint32_t vi = word_vertex_base(pre, ex, ey, ez, lane);
        const float va = __ldg(vol + i);
#pragma unroll
        for (int axis = 0; axis < 3; ++axis) {
          if (!((code >> axis) & 1u)) continue;
          const uint32_t step = axis == 0 ? 1u : (axis == 1 ? (uint32_t)W : plane);
          const float vb = __ldg(vol + i + step);
          float p[3];
          edge_point(x, y, z, axis, edge_t0(va, vb, iso), p);
          if (!kCapped || vi < out.v_cap) {
            if (kCapped && out.world) world_point(out.scale, out.bmin, p);
            float* o = verts + 3ull * vi;
            o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
          }
          ++vi;
        }
      }
      // ---- triangles of the cell whose corner 0 is this node: queue them
      if (nt) {                                                                   // (warp-uniform)
        uint32_t v[8];
        corner_words(bits, w, H, W, v);
        const bool cell = (long long)i < n && x + 1 < (uint32_t)W && y + 1 < (uint32_t)H && z + 1 < (uint32_t)D;
        const int k = cell ? case_of(v, lane) : 0;
        // one 16-byte load: bytes 0..14 = edge numbers of the cell's triangles, byte 15 = their number
        const uint4 row = __ldg(reinterpret_cast<const uint4*>(&g_mc_tri[k][0]));
        const uint32_t rw[4] = {row.x, row.y, row.z, row.w};
        const uint32_t mytri = row.w >> 24;
        const uint32_t incl = (uint32_t)mpscan::warp_incl_scan((unsigned long long)mytri, lane);
        const uint32_t warp_total = __shfl_sync(0xffffffffu, incl, 31);
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&q_count, warp_total);
        base = __shfl_sync(0xffffffffu, base, 0);
        const uint32_t slot = base + incl - mytri, tri0 = (uint32_t)(pre >> 32) + incl - mytri;
#pragma unroll
        for (int t = 0; t < MC_MAX_TRI; ++t)
          if ((uint32_t)t < mytri) {
            uint32_t ed3 = 0;
#pragma unroll
            for (int c = 0; c < 3; ++c) ed3 |= ((rw[(3 * t + c) >> 2] >> (8 * ((3 * t + c) & 3))) & 0xFFu) << (8 * c);
            q_node[slot + t] = i;
            q_tri[slot + t] = tri0 + (uint32_t)t;
            q_edges[slot + t] = ed3;
          }
      }
    }
    __syncthreads();
    // ---- phase (b): one thread per face corner of the queued triangles
    const uint32_t corners = 3u * q_count;
    for (uint32_t idx = threadIdx.x; idx < corners; idx += kEmitThreads) {
      const uint32_t tq = idx / 3u, c = idx - 3u * tq;
      const int ed = (int)((q_edges[tq] >> (8 * c)) & 0xFFu);
      // edge -> owning node + axis.  edges 0-3 along x at (y,z) offsets, 4-7 along y at (x,z), 8-11 along z at (x,y)
      const int axis = ed >> 2, q = ed & 3;
      uint32_t ox = 0, oy = 0, oz = 0;
      if (axis == 0) { oy = q & 1; oz = q >> 1; }
      else if (axis == 1) { ox = q & 1; oz = q >> 1; }
      else { ox = q & 1; oy = q >> 1; }
      const uint32_t node = q_node[tq] + (oz * (uint32_t)H + oy) * (uint32_t)W + ox;
      if (!kCapped || q_tri[tq] < out.f_cap) faces[3ull * q_tri[tq] + c] = vertex_id(info, prefix, node, axis);
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kEmitThreads)
mesh_emit_kernel(const float* __restrict__ vol, const uint32_t* __restrict__ bits, const WordInfo* __restrict__ info,
                 const unsigned long long* __restrict__ prefix, const uint32_t* __restrict__ active, uint32_t n_active,
                 float* __restrict__ verts, int32_t* __restrict__ faces, int D, int H, int W, long long n, float iso) {
  MeshOut out;
  out.verts = verts;
  out.faces = faces;
  mesh_emit_body<false>(vol, bits, info, prefix, active, n_active, out, D, H, W, n, iso);
}

// ---- pass 4 without the host (mp_mcubes_run_async): the grid is fixed when the launch is recorded, every thread reads the
// active-list length the scan left on the device, and the rounds cover it.  Block 0 also publishes the totals of the packed
// scan total (low 32 bits vertices, high 32 faces): counts[0..1] = (nv, nf), the true ones even when they exceed the
// capacities, and count32 = min(nv, v_cap), the point count of the queries at the vertices.
__global__ void __launch_bounds__(kEmitThreads)
mesh_emit_async_kernel(const float* __restrict__ vol, const uint32_t* __restrict__ bits, const WordInfo* __restrict__ info,
                       const unsigned long long* __restrict__ prefix, const uint32_t* __restrict__ active,
                       const uint32_t* __restrict__ n_active_dev, const unsigned long long* __restrict__ total, MeshOut out,
                       long long* __restrict__ counts, int32_t* __restrict__ count32, int D, int H, int W, long long n,
                       float iso) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const unsigned long long tot = *total;
    const uint32_t nv = (uint32_t)(tot & 0xffffffffull), nf = (uint32_t)(tot >> 32);
    counts[0] = (long long)nv;
    counts[1] = (long long)nf;
    *count32 = (int32_t)(nv < out.v_cap ? nv : out.v_cap);
  }
  mesh_emit_body<true>(vol, bits, info, prefix, active, *n_active_dev, out, D, H, W, n, iso);
}

// ---- edge records of the vertices (mp_mesh_refine_async): vertex v -> (owning node, axis), for every id < v_cap.  The walk
// of pass 4: a warp per listed word, a lane per node, the id from the word's prefix + popcounts.  It reads the active-list
// length on the device, so it follows both mp_mcubes_run_async and the eager count + emit.  A persistent grid of any size.
constexpr int kEdgesThreads = 256;
__global__ void __launch_bounds__(kEdgesThreads)
mesh_edges_kernel(const WordInfo* __restrict__ info, const unsigned long long* __restrict__ prefix, const uint32_t* __restrict__ active,
                  const uint32_t* __restrict__ n_active_dev, uint32_t v_cap, uint32_t* __restrict__ edge_node,
                  uint8_t* __restrict__ edge_axis) {
  const uint32_t n_active = *n_active_dev;
  const int lane = threadIdx.x & 31;
  const uint32_t n_warps = gridDim.x * (kEdgesThreads / 32);
  for (uint32_t e = blockIdx.x * (kEdgesThreads / 32) + (threadIdx.x >> 5); e < n_active; e += n_warps) {
    const uint32_t w = __ldg(active + e);
    const uint4 wi = __ldg(reinterpret_cast<const uint4*>(info + w));
    const uint32_t code = lane_edge_code(wi.x, wi.y, wi.z, lane);
    if (!code) continue;
    uint32_t vi = word_vertex_base(__ldg(prefix + w), wi.x, wi.y, wi.z, lane);
    const uint32_t i = 32u * w + (uint32_t)lane;
#pragma unroll
    for (int axis = 0; axis < 3; ++axis) {
      if (!((code >> axis) & 1u)) continue;
      if (vi < v_cap) {
        edge_node[vi] = i;
        edge_axis[vi] = (uint8_t)axis;
      }
      ++vi;
    }
  }
}

}  // namespace mcubes
