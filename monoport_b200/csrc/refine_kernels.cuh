// Device code of the mesh refinement (mp_mesh_refine_async in mcubes.cu; the algorithm: DESIGN.md §F3.1).  Every vertex of a
// marching-cubes mesh lies on a grid edge whose two end nodes bracket the iso level; K rounds of regula falsi with the
// Illinois modification, each evaluating the network at one candidate per vertex through the query program, move it
// toward the network's own root on that edge, and the candidate with the smallest |sigma - iso| is written back.
// Kept free of host API calls and of CUDA runtime types so that tests/emu can run these kernels unmodified on the CPU
// emulation layer.  Every float operation is an __f*_rn intrinsic (or a compare / select), so no FMA contraction changes
// the bits and tests/mesh_refine_ref.py restates them exactly in float32 torch ops.
#pragma once
#include <stdint.h>
#include "mcubes_kernels.cuh"

namespace mrefine {

constexpr int kThreads = 256;

// flag byte of a vertex: bits 0-1 the edge's axis, bits 2-3 the bracket end kept by the last update (0 none, 1 the t = 0
// side "a", 2 the t = 1 side "b"), bit 4 set once a round hit f == 0 exactly (the candidate stops moving)
constexpr uint8_t kAxisMask = 3u, kKeptShift = 2, kKeptMask = 3u << kKeptShift, kDone = 16u;
constexpr uint8_t kKeptA = 1u, kKeptB = 2u;

// The scratch of a refinement, structure of arrays over the capacity v_cap (mp_mesh_refine_scratch_bytes):
//   pts   [3][cap]  the candidates' world points, the rows the query program reads
//   sigma [cap]     the query's values there
//   ta, fa, tb, fb  the bracket: parameter and f = value - iso at its t = 0 side (a) and its t = 1 side (b)
//   tbest, fbest    the candidate with the smallest |f| so far
//   tcur            the candidate evaluated by the current round
//   node, flags     the edge record (owning node, axis) and the flag byte above
struct State {
  float* pts;
  float* sigma;
  float *ta, *fa, *tb, *fb, *tbest, *fbest, *tcur;
  uint32_t* node;
  uint8_t* flags;
  uint32_t cap;
};

// the grid of the volume marching cubes read, its iso level, and reconstruction()'s world mapping
struct Geom {
  int H, W;
  float iso;
  float scale[3], bmin[3];
};

// the number of vertices to refine: the emission's count32, clamped to the capacity
__device__ __forceinline__ uint32_t vertex_count(const int32_t* __restrict__ count32, uint32_t cap) {
  const int32_t c = *count32;
  return c <= 0 ? 0u : ((uint32_t)c < cap ? (uint32_t)c : cap);
}

// the world point at parameter t on vertex v's edge, as the emission makes it (mcubes::edge_point + world_point)
__device__ __forceinline__ void edge_world_point(const Geom& g, uint32_t node, int axis, float t, float (&p)[3]) {
  uint32_t x, y, z;
  mcubes::node_xyz(node, (uint32_t)g.H * (uint32_t)g.W, g.W, x, y, z);
  mcubes::edge_point(x, y, z, axis, t, p);
  mcubes::world_point(g.scale, g.bmin, p);
}

__device__ __forceinline__ void store_rows(const State& s, uint32_t v, const float (&p)[3]) {
  s.pts[v] = p[0];
  s.pts[s.cap + v] = p[1];
  s.pts[2ull * s.cap + v] = p[2];
}

// round 0's set-up: the bracket (0, va - iso), (1, vb - iso) from the volume marching cubes read, the candidate t0 = the
// emitted vertex's parameter, and its world point in the query rows.  (s.node / s.flags hold mesh_edges_kernel's records.)
__global__ void __launch_bounds__(kThreads)
refine_init_kernel(const float* __restrict__ vol, const int32_t* __restrict__ count32, State s, Geom g) {
  const uint32_t n = vertex_count(count32, s.cap);
  const uint32_t step = gridDim.x * kThreads;
  for (uint32_t v = blockIdx.x * kThreads + threadIdx.x; v < n; v += step) {
    const uint32_t i = s.node[v];
    const int axis = (int)(s.flags[v] & kAxisMask);
    const uint32_t off = axis == 0 ? 1u : (axis == 1 ? (uint32_t)g.W : (uint32_t)g.H * (uint32_t)g.W);
    const float va = __ldg(vol + i), vb = __ldg(vol + i + off);
    const float t0 = mcubes::edge_t0(va, vb, g.iso);
    s.ta[v] = 0.f;
    s.fa[v] = __fsub_rn(va, g.iso);
    s.tb[v] = 1.f;
    s.fb[v] = __fsub_rn(vb, g.iso);
    s.tbest[v] = t0;
    s.fbest[v] = INFINITY;                  // (round 0's candidate always becomes the best, unless its value is NaN)
    s.tcur[v] = t0;
    s.flags[v] = (uint8_t)axis;
    float p[3];
    edge_world_point(g, i, axis, t0, p);
    store_rows(s, v, p);
  }
}

// One round's update from the query's values at the candidates: keep the best candidate, replace the bracket end on f's side
// (halving the retained end's f when the same end is retained twice in a row), and put the next candidate -- the secant
// root of the bracket, clamped into it, bisection when the secant is undefined -- in the query rows.  `last`: instead,
// write the best candidate's world point into verts [cap][3].
__global__ void __launch_bounds__(kThreads)
refine_step_kernel(const int32_t* __restrict__ count32, State s, Geom g, int last, float* __restrict__ verts) {
  const uint32_t n = vertex_count(count32, s.cap);
  const uint32_t step = gridDim.x * kThreads;
  for (uint32_t v = blockIdx.x * kThreads + threadIdx.x; v < n; v += step) {
    const float t = s.tcur[v];
    const float f = __fsub_rn(s.sigma[v], g.iso);
    uint8_t flags = s.flags[v];
    const int axis = (int)(flags & kAxisMask);
    float tbest = s.tbest[v];
    if (fabsf(f) < fabsf(s.fbest[v])) {     // (strict: the earlier candidate wins a tie)
      tbest = t;
      s.tbest[v] = t;
      s.fbest[v] = f;
    }
    float p[3];
    if (last) {
      edge_world_point(g, s.node[v], axis, tbest, p);
      float* o = verts + 3ull * v;
      o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
      continue;
    }
    float tn = t;                            // a root was hit (now or before): the candidate stays
    if (f == 0.f) flags |= kDone;
    if (!(flags & kDone)) {
      float ta = s.ta[v], fa = s.fa[v], tb = s.tb[v], fb = s.fb[v];
      const bool side_a = (f > 0.f) == (fa > 0.f);
      const uint8_t kept = side_a ? kKeptB : kKeptA;
      if (side_a) { ta = t; fa = f; } else { tb = t; fb = f; }
      if (((flags & kKeptMask) >> kKeptShift) == kept) {       // Illinois: the same end retained twice in a row
        if (kept == kKeptA) fa = __fmul_rn(fa, 0.5f);
        else fb = __fmul_rn(fb, 0.5f);
      }
      flags = (uint8_t)((flags & ~kKeptMask) | (kept << kKeptShift));
      const float d = __fsub_rn(fb, fa);
      tn = __fsub_rn(ta, __fmul_rn(__fdiv_rn(fa, d), __fsub_rn(tb, ta)));
      if (d == 0.f || tn != tn) tn = __fmul_rn(__fadd_rn(ta, tb), 0.5f);
      const float lo = ta < tb ? ta : tb, hi = ta < tb ? tb : ta;
      tn = tn < lo ? lo : (tn > hi ? hi : tn);
      s.ta[v] = ta; s.fa[v] = fa; s.tb[v] = tb; s.fb[v] = fb;
    }
    s.flags[v] = flags;
    s.tcur[v] = tn;
    edge_world_point(g, s.node[v], axis, tn, p);
    store_rows(s, v, p);
  }
}

}  // namespace mrefine
