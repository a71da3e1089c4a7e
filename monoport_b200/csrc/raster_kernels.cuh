// Device code of the mesh renderer (mp_render_mesh_async in raster.cu; the rules: DESIGN.md §F3.2).  A deterministic
// restatement of what the reference's NormalRender / ColorRender GL programs draw: the vertex transform PerspMat * ModelMat,
// window coordinates snapped to 1/256 pixel, coverage on integer edge functions with a top-left rule, GL_LESS on a 24-bit
// depth in draw order (a 64-bit atomicMin of (depth << 32 | face id)), then one resolve pass that shades the winning face
// of every pixel with perspective-correct barycentrics.
// Kept free of host API calls and of CUDA runtime types so that tests/emu can run these kernels unmodified on the CPU
// emulation layer.  Every float operation is an __f*_rn / __d*_rn intrinsic (or a compare / select), so no FMA contraction
// changes the bits and tests/raster_ref.py restates them exactly in numpy.
#pragma once
#include <stdint.h>

namespace mraster {

constexpr int kSetupThreads = 256;
constexpr int kLargeThreads = 256;
constexpr int kResolveThreads = 256;
constexpr int kMaxSize = 8192;            // width and height limit: the snapped guard band stays below 2^22 in 1/256 px
constexpr int kMaxViews = 65535;          // the grids' y dimension
constexpr float kGuard = 2.f;             // |x/w|, |y/w| <= kGuard: the guard band, in normalised device coordinates
constexpr float kMinW = 1.0e-5f;          // the clip plane w >= kMinW that keeps clipped vertices in front of the eye
constexpr int kSmallPixels = 16;          // faces whose pixel box holds at most this many pixels are drawn by the setup thread
constexpr int kMaxPoly = 9;               // a triangle clipped by six planes
constexpr int kMaxPieces = kMaxPoly - 2;
constexpr unsigned long long kClearKey = ~0ull;
constexpr double kDepthScale = 16777215.0;   // 2^24 - 1: a DEPTH24 buffer

// the mesh: mp_mcubes_run_async's buffers and counts (or any indexed mesh with its counts on the device)
struct Mesh {
  const float* verts;           // [v_cap][3]
  const int32_t* faces;         // [f_cap][3]
  const long long* counts;      // (nV, nF)
  const float* normals;         // [v_cap][3] or null
  const float* colours;         // [v_cap][3] or null
  uint32_t v_cap, f_cap;
};

// the views and the raster state (scratch of mp_render_mesh_scratch_bytes)
struct Target {
  const float* mats;            // [views][32]: ModelMat then PerspMat, each row-major 4x4
  int views, W, H;
  unsigned long long* keys;     // [views][H][W], row j counted from the bottom; cleared to kClearKey
  uint2* list;                  // (view, face) of the faces the large-face kernel draws
  uint32_t* list_len;           // cleared to 0
};

// what the resolve writes: [views][H][W][4] images (null when absent) and the clear colour
struct Shade {
  float* normal;
  float* colour;
  float clear[4];
};

// a piece ready for coverage: snapped window vertices (1/256 px, counter-clockwise) and its pixel box in the viewport
struct Tri {
  int32_t x[3], y[3];
  int32_t bx0, by0, bx1, by1;
};

// (nV, nF): the counts on the device, capped at the capacities
__device__ __forceinline__ void mesh_counts(const Mesh& m, uint32_t& nv, uint32_t& nf) {
  const long long a = m.counts[0], b = m.counts[1];
  nv = a <= 0 ? 0u : (a < (long long)m.v_cap ? (uint32_t)a : m.v_cap);
  nf = b <= 0 ? 0u : (b < (long long)m.f_cap ? (uint32_t)b : m.f_cap);
}

// face f's vertex ids; false when one lies outside [0, nv)
__device__ __forceinline__ bool load_face(const Mesh& m, uint32_t f, uint32_t nv, int32_t (&idx)[3]) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    idx[k] = m.faces[3ull * f + k];
    ok = ok && idx[k] >= 0 && (uint32_t)idx[k] < nv;
  }
  return ok;
}

// e = ModelMat [p, 1] and clip = PerspMat e, row by row ((m0 x + m1 y) + m2 z) + m3 (with + m3 e3 for PerspMat)
__device__ __forceinline__ void transform(const float* __restrict__ mat, const float* __restrict__ p, float (&c)[4]) {
  float e[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    e[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(mat[4 * i], p[0]), __fmul_rn(mat[4 * i + 1], p[1])), __fmul_rn(mat[4 * i + 2], p[2])),
                     mat[4 * i + 3]);
  const float* P = mat + 16;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    c[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[4 * i], e[0]), __fmul_rn(P[4 * i + 1], e[1])), __fmul_rn(P[4 * i + 2], e[2])),
                     __fmul_rn(P[4 * i + 3], e[3]));
}

__device__ __forceinline__ void face_clip(const Mesh& m, const float* __restrict__ mat, const int32_t (&idx)[3], float (&c)[3][4]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) transform(mat, m.verts + 3ull * (uint32_t)idx[k], c[k]);
}

// the window coordinate (ndc + 1) * size / 2 of one axis, snapped to 1/256 px (round to nearest even)
__device__ __forceinline__ int32_t snap(float ndc, int size) {
  const float win = __fmul_rn(__fadd_rn(ndc, 1.f), __fmul_rn((float)size, 0.5f));
  return __float2int_rn(__fmul_rn(win, 256.f));
}

// the direct path: every w > 0 and every vertex inside the guard band -> the snapped vertices
__device__ __forceinline__ bool direct(const float (&c)[3][4], int W, int H, int32_t (&x)[3], int32_t (&y)[3]) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float nx = __fdiv_rn(c[k][0], c[k][3]), ny = __fdiv_rn(c[k][1], c[k][3]);
    ok = ok && c[k][3] > 0.f && nx >= -kGuard && nx <= kGuard && ny >= -kGuard && ny <= kGuard;
    x[k] = ok ? snap(nx, W) : 0;
    y[k] = ok ? snap(ny, H) : 0;
  }
  return ok;
}

__device__ __forceinline__ bool finite_face(const float (&c)[3][4]) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int q = 0; q < 4; ++q) ok = ok && c[k][q] - c[k][q] == 0.f;
  return ok;
}

// floor(a / 256) and ceil(a / 256) of a snapped coordinate
__device__ __forceinline__ int32_t floor256(int32_t a) { return a >> 8; }
__device__ __forceinline__ int32_t ceil256(int32_t a) { return -((-a) >> 8); }

// the winding normalised to counter-clockwise and the pixel box (centres (i + 1/2, j + 1/2)) clamped to the viewport;
// false for a zero-area piece or an empty box
__device__ __forceinline__ bool tri_setup(const int32_t (&x)[3], const int32_t (&y)[3], int W, int H, Tri& t) {
  const long long area = (long long)(x[1] - x[0]) * (y[2] - y[0]) - (long long)(y[1] - y[0]) * (x[2] - x[0]);
  if (area == 0) return false;
  const bool ccw = area > 0;
  t.x[0] = x[0]; t.y[0] = y[0];
  t.x[1] = ccw ? x[1] : x[2]; t.y[1] = ccw ? y[1] : y[2];
  t.x[2] = ccw ? x[2] : x[1]; t.y[2] = ccw ? y[2] : y[1];
  const int32_t xmin = min(min(x[0], x[1]), x[2]), xmax = max(max(x[0], x[1]), x[2]);
  const int32_t ymin = min(min(y[0], y[1]), y[2]), ymax = max(max(y[0], y[1]), y[2]);
  t.bx0 = max(ceil256(xmin - 128), 0);
  t.bx1 = min(floor256(xmax - 128), W - 1);
  t.by0 = max(ceil256(ymin - 128), 0);
  t.by1 = min(floor256(ymax - 128), H - 1);
  return t.bx0 <= t.bx1 && t.by0 <= t.by1;
}

// pixel (i, j) is covered: every edge function > 0, or = 0 on a top or left edge (counter-clockwise, y up: an edge going
// down, or a horizontal edge going left)
__device__ __forceinline__ bool covered(const Tri& t, int i, int j) {
  const long long px = 256ll * i + 128, py = 256ll * j + 128;
  bool in = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int a = k == 2 ? 0 : k + 1, b = k == 0 ? 2 : (k == 1 ? 0 : 1);
    const long long dx = (long long)t.x[b] - t.x[a], dy = (long long)t.y[b] - t.y[a];
    const long long e = dx * (py - t.y[a]) - dy * (px - t.x[a]);
    in = in && (e > 0 || (e == 0 && (dy < 0 || (dy == 0 && dx < 0))));
  }
  return in;
}

// perspective-correct barycentrics of pixel centre (i, j) with respect to the face's clip coordinates, in the 2D-homogeneous
// form: b_k proportional to (v_{k+1} x v_{k+2}) . (px, py, 1) with v = (x, y, w), px = (2i + 1) / W - 1, in float64
__device__ __forceinline__ void barycentrics(const float (&c)[3][4], int i, int j, int W, int H, double (&b)[3]) {
  const double px = __dsub_rn(__ddiv_rn((double)(2 * i + 1), (double)W), 1.0);
  const double py = __dsub_rn(__ddiv_rn((double)(2 * j + 1), (double)H), 1.0);
  double e[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int u = k == 2 ? 0 : k + 1, v = k == 0 ? 2 : (k == 1 ? 0 : 1);
    const double ux = c[u][0], uy = c[u][1], uw = c[u][3], vx = c[v][0], vy = c[v][1], vw = c[v][3];
    const double cx = __dsub_rn(__dmul_rn(uy, vw), __dmul_rn(uw, vy));
    const double cy = __dsub_rn(__dmul_rn(uw, vx), __dmul_rn(ux, vw));
    const double cw = __dsub_rn(__dmul_rn(ux, vy), __dmul_rn(uy, vx));
    e[k] = __dadd_rn(__dadd_rn(__dmul_rn(cx, px), __dmul_rn(cy, py)), cw);
  }
  const double s = __dadd_rn(__dadd_rn(e[0], e[1]), e[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) b[k] = __ddiv_rn(e[k], s);
}

// ((b0 a0 + b1 a1) + b2 a2) in float64
__device__ __forceinline__ double lerp3(const double (&b)[3], double a0, double a1, double a2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(b[0], a0), __dmul_rn(b[1], a1)), __dmul_rn(b[2], a2));
}

// THE coverage-and-depth function of both raster paths: a covered pixel whose window depth lies in [0, 1] takes part in the
// depth test with key (round(z_w (2^24 - 1)) << 32) | face
__device__ __forceinline__ void fragment(const Tri& t, const float (&c)[3][4], uint32_t face, int i, int j, int W, int H,
                                         unsigned long long* __restrict__ keys) {
  if (!covered(t, i, j)) return;
  double b[3];
  barycentrics(c, i, j, W, H, b);
  const double z = lerp3(b, c[0][2], c[1][2], c[2][2]), w = lerp3(b, c[0][3], c[1][3], c[2][3]);
  const double zw = __dmul_rn(__dadd_rn(__ddiv_rn(z, w), 1.0), 0.5);
  if (!(zw >= 0.0 && zw <= 1.0)) return;
  const unsigned long long d = (unsigned long long)__double2ll_rn(__dmul_rn(zw, kDepthScale));
  atomicMin(keys + (size_t)j * W + i, (d << 32) | face);
}

// signed distance of clip-space point v to clip plane p: z >= -w, w >= kMinW, then the guard band x >= -2w, x <= 2w,
// y >= -2w, y <= 2w
__device__ __forceinline__ float plane_dist(const float* v, int p) {
  switch (p) {
    case 0: return __fadd_rn(v[2], v[3]);
    case 1: return __fsub_rn(v[3], kMinW);
    case 2: return __fadd_rn(__fmul_rn(kGuard, v[3]), v[0]);
    case 3: return __fsub_rn(__fmul_rn(kGuard, v[3]), v[0]);
    case 4: return __fadd_rn(__fmul_rn(kGuard, v[3]), v[1]);
    default: return __fsub_rn(__fmul_rn(kGuard, v[3]), v[1]);
  }
}

// The face's pieces into t[] (returns how many; one thread): the face itself on the direct path, else the triangle clipped in
// clip space against the six planes above (Sutherland-Hodgman; an edge's crossing is always computed from its inside end) and
// fan-triangulated from its first vertex.  poly: 2 x kMaxPoly x 4 floats of working memory.
__device__ __forceinline__ int face_pieces(const float (&c)[3][4], int W, int H, float (*poly)[kMaxPoly][4], Tri* t) {
  int32_t x[3], y[3];
  if (direct(c, W, H, x, y)) return tri_setup(x, y, W, H, t[0]) ? 1 : 0;
  int n = 3;
  for (int k = 0; k < 3; ++k)
    for (int q = 0; q < 4; ++q) poly[0][k][q] = c[k][q];
  for (int p = 0; p < 6; ++p) {
    const float (*in)[4] = poly[p & 1];
    float (*out)[4] = poly[(p & 1) ^ 1];
    int m = 0;
    for (int k = 0; k < n; ++k) {
      const float* a = in[k];
      const float* b = in[k + 1 == n ? 0 : k + 1];
      const float da = plane_dist(a, p), db = plane_dist(b, p);
      const bool ia = da >= 0.f, ib = db >= 0.f;
      if (ia)
        for (int q = 0; q < 4; ++q) out[m][q] = a[q];
      if (ia) ++m;
      if (ia != ib) {
        const float* s = ia ? a : b;
        const float* e = ia ? b : a;
        const float ds = ia ? da : db, de = ia ? db : da;
        const float u = __fdiv_rn(ds, __fsub_rn(ds, de));
        for (int q = 0; q < 4; ++q) out[m][q] = __fadd_rn(s[q], __fmul_rn(u, __fsub_rn(e[q], s[q])));
        ++m;
      }
    }
    n = m;
  }
  const float (*v)[4] = poly[0];        // (six planes: the result is back in poly[0])
  int np = 0;
  for (int k = 1; k + 1 < n; ++k) {
    const int id[3] = {0, k, k + 1};
    for (int r = 0; r < 3; ++r) {
      x[r] = snap(__fdiv_rn(v[id[r]][0], v[id[r]][3]), W);
      y[r] = snap(__fdiv_rn(v[id[r]][1], v[id[r]][3]), H);
    }
    if (tri_setup(x, y, W, H, t[np])) ++np;
  }
  return np;
}

// One thread per (view, face), grid-stride over the face count read on the device: transform, classify and snap the face; a
// direct face with a small pixel box is drawn here, every other face goes on the list of the large-face kernel.
__global__ void __launch_bounds__(kSetupThreads)
raster_setup_kernel(Mesh m, Target t) {
  uint32_t nv, nf;
  mesh_counts(m, nv, nf);
  const uint32_t view = blockIdx.y;
  const float* mat = t.mats + 32ull * view;
  unsigned long long* keys = t.keys + (size_t)view * t.H * t.W;
  const uint32_t step = gridDim.x * kSetupThreads;
  for (uint32_t f = blockIdx.x * kSetupThreads + threadIdx.x; f < nf; f += step) {
    int32_t idx[3];
    if (!load_face(m, f, nv, idx)) continue;
    float c[3][4];
    face_clip(m, mat, idx, c);
    if (!finite_face(c)) continue;
    int32_t x[3], y[3];
    Tri tri;
    bool large = !direct(c, t.W, t.H, x, y);
    if (!large) {
      if (!tri_setup(x, y, t.W, t.H, tri)) continue;
      large = (tri.bx1 - tri.bx0 + 1) * (tri.by1 - tri.by0 + 1) > kSmallPixels;
    }
    if (large) {
      const uint32_t k = atomicAdd(t.list_len, 1u);
      t.list[k] = make_uint2(view, f);
      continue;
    }
    for (int j = tri.by0; j <= tri.by1; ++j)
      for (int i = tri.bx0; i <= tri.bx1; ++i) fragment(tri, c, f, i, j, t.W, t.H, keys);
  }
}

// A persistent grid over the list (its length read on the device), one CTA per listed face: one thread makes the pieces,
// then the CTA tiles each piece's pixel box.
__global__ void __launch_bounds__(kLargeThreads)
raster_large_kernel(Mesh m, Target t) {
  __shared__ float s_c[3][4];
  __shared__ float s_poly[2][kMaxPoly][4];
  __shared__ Tri s_tri[kMaxPieces];
  __shared__ int s_n;
  uint32_t nv, nf;
  mesh_counts(m, nv, nf);
  const uint32_t n = *t.list_len;
  for (uint32_t k = blockIdx.x; k < n; k += gridDim.x) {
    const uint2 e = t.list[k];
    if (threadIdx.x == 0) {
      int32_t idx[3];
      load_face(m, e.y, nv, idx);                  // (listed faces passed this test in the setup kernel)
      float c[3][4];
      face_clip(m, t.mats + 32ull * e.x, idx, c);
      for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 4; ++q) s_c[r][q] = c[r][q];
      s_n = face_pieces(c, t.W, t.H, s_poly, s_tri);
    }
    __syncthreads();
    unsigned long long* keys = t.keys + (size_t)e.x * t.H * t.W;
    const int np = s_n;
    for (int p = 0; p < np; ++p) {
      const Tri& tri = s_tri[p];
      const int bw = tri.bx1 - tri.bx0 + 1, bh = tri.by1 - tri.by0 + 1;
      for (int q = threadIdx.x; q < bw * bh; q += kLargeThreads) fragment(tri, s_c, e.y, tri.bx0 + q % bw, tri.by0 + q / bw, t.W, t.H, keys);
    }
    __syncthreads();
  }
}

// n_cam = (ModelMat [n, 0]).xyz, rows ((m0 nx + m1 ny) + m2 nz)
__device__ __forceinline__ void cam_normal(const float* __restrict__ mat, const float* __restrict__ n, float (&o)[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
    o[i] = __fadd_rn(__fadd_rn(__fmul_rn(mat[4 * i], n[0]), __fmul_rn(mat[4 * i + 1], n[1])), __fmul_rn(mat[4 * i + 2], n[2]));
}

// One thread per pixel per view: the clear colour, or the winning face's attributes at the pixel centre -- the normal program's
// (n / sqrt(n.n) + 1) / 2 of the interpolated camera-space normal, the colour program's interpolated colour, alpha 1.  Output
// row r is window row H - 1 - r (get_color()'s orientation).
__global__ void __launch_bounds__(kResolveThreads)
raster_resolve_kernel(Mesh m, Target t, Shade s) {
  const uint32_t npx = (uint32_t)t.W * (uint32_t)t.H;
  const uint32_t q = blockIdx.x * kResolveThreads + threadIdx.x;
  if (q >= npx) return;
  const uint32_t view = blockIdx.y;
  const int i = (int)(q % (uint32_t)t.W), r = (int)(q / (uint32_t)t.W), j = t.H - 1 - r;
  const unsigned long long key = t.keys[(size_t)view * npx + (size_t)j * t.W + i];
  const size_t o = ((size_t)view * npx + q) * 4;
  if (key == kClearKey) {
    for (int k = 0; k < 4; ++k) {
      if (s.normal) s.normal[o + k] = s.clear[k];
      if (s.colour) s.colour[o + k] = s.clear[k];
    }
    return;
  }
  const uint32_t f = (uint32_t)(key & 0xffffffffull);
  const float* mat = t.mats + 32ull * view;
  int32_t idx[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) idx[k] = m.faces[3ull * f + k];
  float c[3][4];
  face_clip(m, mat, idx, c);
  double b[3];
  barycentrics(c, i, j, t.W, t.H, b);
  if (s.normal) {
    float n[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) cam_normal(mat, m.normals + 3ull * (uint32_t)idx[k], n[k]);
    float v[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) v[a] = __double2float_rn(lerp3(b, n[0][a], n[1][a], n[2][a]));
    const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])));
#pragma unroll
    for (int a = 0; a < 3; ++a) s.normal[o + a] = __fmul_rn(__fadd_rn(__fdiv_rn(v[a], len), 1.f), 0.5f);
    s.normal[o + 3] = 1.f;
  }
  if (s.colour) {
    const float* c0 = m.colours + 3ull * (uint32_t)idx[0];
    const float* c1 = m.colours + 3ull * (uint32_t)idx[1];
    const float* c2 = m.colours + 3ull * (uint32_t)idx[2];
#pragma unroll
    for (int a = 0; a < 3; ++a) s.colour[o + a] = __double2float_rn(lerp3(b, c0[a], c1[a], c2[a]));
    s.colour[o + 3] = 1.f;
  }
}

}  // namespace mraster
