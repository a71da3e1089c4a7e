// Shared internals of libmonoport_b200 (sm_90a only).  Not part of the ABI.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdarg.h>
#include <vector>

#include "../../include/monoport_b200.h"

// dynamic shared memory of a kernel (tests/emu runs the kernels on the CPU, where it is a buffer the harness hands out --
// one per CTA of a cluster)
#ifdef MP_CUDA_EMU
void* mp_emu_dyn_smem();
#define MP_DYN_SMEM(type, name) type* const name = static_cast<type*>(mp_emu_dyn_smem())
#define MP_DYN_SMEM_ALIGNED(type, name, bytes) type* const name = static_cast<type*>(mp_emu_dyn_smem())
#else
#define MP_DYN_SMEM(type, name) extern __shared__ type name[]
#define MP_DYN_SMEM_ALIGNED(type, name, bytes) extern __shared__ __align__(bytes) type name[]
#endif

// NVTX ranges around the entry points of the hot path (F1 query, F2 octree, F3 marching cubes / visible surface): header-only
// NVTX3, a no-op unless a profiler (nsys / ncu --nvtx) is attached
#ifndef MP_CUDA_EMU
#include <nvtx3/nvToolsExt.h>
struct MpRange {
  explicit MpRange(const char* name) { nvtxRangePushA(name); }
  ~MpRange() { nvtxRangePop(); }
};
#else
struct MpRange {
  explicit MpRange(const char*) {}
};
#endif

#define MP_LEAKY_SLOPE 0.01f   // F.leaky_relu default (heads/SurfaceClassifier.py:58)
#define MP_MAX_LAYERS 8

void mp_set_error(const char* fmt, ...);
void mp_ensure_pool();

#define MP_CUDA(call)                                                                        \
  do {                                                                                       \
    cudaError_t e_ = (call);                                                                 \
    if (e_ != cudaSuccess) {                                                                 \
      mp_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return MP_E_CUDA;                                                                      \
    }                                                                                        \
  } while (0)

#define MP_REQUIRE(cond, ...)      \
  do {                             \
    if (!(cond)) {                 \
      mp_set_error(__VA_ARGS__);   \
      return MP_E_INVALID;         \
    }                              \
  } while (0)

// entry points that evaluate one map refuse a batch handle instead of silently evaluating its image 0
#define MP_REQUIRE_SINGLE_MAP(feat, what)                                                                          \
  MP_REQUIRE((feat)->B == 1, "%s takes a single-map feature handle, this one holds %d maps (batched queries: "      \
             "mp_query_points_batch)", what, (feat)->B)

// ---------------------------------------------------------------------------------------------
// handles
// ---------------------------------------------------------------------------------------------
struct mp_mlp {
  int n_layers;
  int channels[MP_MAX_LAYERS + 1];   // filter_channels
  int cin[MP_MAX_LAYERS];            // per-layer total input width (hidden + skip)
  int cout[MP_MAX_LAYERS];
  int skip;                          // !no_residual
  int last_op;
  // fp32 path: per layer W^T as [cin][cout] (k-major rows, cout contiguous) + bias
  float* wt[MP_MAX_LAYERS];
  float* bias[MP_MAX_LAYERS];
  // original [cout][cin] fp32 (row-major) kept for the fp32 last layer of the tensor-core path
  float* w[MP_MAX_LAYERS];
  // tensor-core path (query_tc.cu): packed fp16 weight tiles + fp32 side vectors; null when unsupported
  void* tc;
  int tc_ok;
  int device;
  unsigned long long gen;            // unique per mp_mlp_create (process-wide counter, never 0): keys per-feature caches
  // validated range of the tensor-core program: frames whose largest |feature| exceeds this limit are evaluated by the
  // exact fp32 kernel instead (decided on the DEVICE, per launch; see mp_query_dispatch).  +inf disables the guard.
  float tc_amax_limit;
};

// Default tc_amax_limit of a head with `res` outputs and last op `last_op` (DESIGN.md §5, "Feature limit per last op").  The
// tensor-core programs run the geometry widths (res 1) and the colour widths (res 3) with any last op; the error of the
// logit reaches the output times the last op's slope (Sigmoid 1/4, Tanh and none 1), so the validated range depends on
// both.  The geometry head's Sigmoid (12) and the colour head's Tanh (8) are the shipped limits; the others were measured on
// the CPU model of the wgmma program to keep the geometry head's Sigmoid margin under the 1e-4 bar.
inline float mp_tc_default_feature_limit(int res, int last_op) {
  if (last_op == MP_LAST_SIGMOID) return 12.0f;
  if (res == 3) return last_op == MP_LAST_TANH ? 8.0f : 4.0f;
  return 3.0f;                                       // the geometry widths with Tanh or no last op
}

struct mp_feat {
  int C, H, W;
  int B;            // maps held (mp_feat_create: 1; mp_feat_create_batch: B).  Every per-texel array below is B
                    // consecutive per-image blocks, image b's at offset b * (its per-image size); amax has B entries.
  float* nhwc32;    // [H][W][C] fp32 (one bilinear tap = one contiguous C*4-byte vector): the CURRENT map -- the handle's own
                    // repacked copy (nhwc_own) or, after mp_feat_bind_nhwc, the caller's channel-last tensor itself
  float* nhwc_own;
  float* staging;   // [C][H][W] device staging for host uploads
  int device;
  // layer-0 pre-activation per texel, G0 = W0[:, :C] . F  ([H*W][g0_n] fp16), built lazily by the tensor-core path
  // (bilinear sampling is linear, so sampling G0 equals applying W0 to the sampled features); valid for
  // (g0_owner == generation id of the head handle, g0_version == version).  The owner is the head's generation id, not
  // its address: a head rebuilt after a weight change may be handed the freed handle's address again.
  __half* g0;
  __half* f16;      // [H*W][C] fp16 copy of the map (X operand taps of the v3 program), same validity as g0
  float* s4tex;     // [H*W][n_out] fp32: last layer's feature part applied per texel (sampled in fp32 by the v3 program)
  int g0_n;
  unsigned long long g0_owner;
  unsigned long long g0_version;
  unsigned long long version;   // bumped by every mp_feat_upload
  // max |feature| of the current frame as float bits (non-negative floats order like unsigned integers): zeroed by every
  // upload, raised by the staging pass of the per-frame G0 kernels; read by the range guard of the query kernels
  unsigned* amax;
  // [B] after amax (the same allocation, zeroed with it): nonzero when the current map holds a NaN or an infinity (raised by
  // the same staging pass); the in-image grid launch then lists every node
  unsigned* nonfinite;
};

// ---------------------------------------------------------------------------------------------
// where the points of a query come from
// ---------------------------------------------------------------------------------------------
enum { MP_SRC_ROWS = 0, MP_SRC_GRID = 1, MP_SRC_NODES = 2 };

struct MpPointSrc {
  int kind;
  // MP_SRC_ROWS: three rows x[n], y[n], z[n]
  const float* px;
  const float* py;
  const float* pz;
  long long pstride;          // element stride between consecutive points
  // MP_SRC_NODES: linear node indices of a res^3 level grid; count may live on the device
  const int32_t* nodes;
  const int32_t* count_dev;   // nullable; when set, n is only an upper bound
  // MP_SRC_GRID / MP_SRC_NODES geometry
  int res;          // nodes per axis of the (level) grid
  int node_stride;  // index-space stride of a node (final-resolution units)
  int r_final;      // final resolution (divisor of the world mapping)
  int z0;           // (host-side bookkeeping only: first plane of a MP_SRC_GRID slab; the kernels use lin0)
  long long lin0;   // MP_SRC_GRID: linear index (z slowest) of the node point 0 stands for -- a z slab starts at z0*res*res,
                    // a balanced shard anywhere (contiguous z-major ranges need not end on plane boundaries)
  // list sharding (multi-GPU): of the n points (after the device-side count) this launch evaluates only the window
  // [rank * per, rank * per + per) with per = ceil(n / world) rounded up to a multiple of 128; 0/1 = everything
  int shard_rank, shard_world;
  float inv_r, half_inv_r;    // 1/r_final, 1/(2 r_final) rounded to fp32
  float bmin[3], bext[3];     // b_min, (b_max - b_min)
  long long n;
};

struct MpCalib {
  float m[12];        // rows 0..2 of [R|t]
  int has;            // 0 => calibs=None (points already in image space)
  int perspective;
  float z_scale;
};

// The images of a query launch: B images of n points each, evaluated by one launch whose tiles never straddle two images
// (tile t belongs to image t / tiles_per_image).  Image b reads its points at px/py/pz + b * pt_stride, its calibration
// (rows 0..2 of [R|t], when MpCalib::has) from calibs[12 b ..] in device memory (null: MpCalib::m), its map's per-texel
// arrays at the per-image offsets of mp_feat, and writes its outputs at out + b * out_stride.  The default is a
// single-map launch.  B == 1 with calibs set is a single-map launch whose camera is read from device memory when the kernel
// runs (a captured frame whose camera changes between replays): every point source and output of a single-map launch, the
// projection and z_scale still from MpCalib (has = 1).
struct MpBatch {
  int B = 1;
  long long pt_stride = 0;
  long long out_stride = 0;
  const float* calibs = nullptr;   // [B][12] device
};

// Direct rendering of the visible surface (RTL/main.py:212-249), shared by both query programs: point i is the vertex
// (X[i], Y[i], R - Z[i]) of forward_vertices mapped to world space by mat_color (RTL/main.py:201-210: diag((b_max-b_min)/R),
// translation b_min), and its colour pred * 0.5 + 0.5 (:244) is scattered to canvas[X[i], Y[i], :] (:247-248) -- no
// intermediate point / prediction tensors.  X == nullptr: the ordinary point sources and the [R,N] output.
struct MpSurfaceSrc {
  const long long* X;
  const long long* Y;
  const float* Z;
  const long long* count;       // nullable: the vertex count on the device (mp_forward_vertices_async's count_dev); the
                                // launch's n is then the capacity, and vertices at or beyond min(*count, n) are not touched
  float scale[3], bmin[3];      // (b_max - b_min) / R and b_min, fp32 like torch's
  float R;
  float* canvas;                // [R, R, 3]
  int canvas_R;
};

inline MpSurfaceSrc mp_surface_src(const long long* X, const long long* Y, const float* Z, const long long* count, int R,
                                   const float* b_min3, const float* b_max3, float* canvas) {
  MpSurfaceSrc s;
  memset(&s, 0, sizeof(s));
  s.X = X; s.Y = Y; s.Z = Z; s.count = count;
  for (int a = 0; a < 3; ++a) {
    s.scale[a] = (b_max3[a] - b_min3[a]) / (float)R;          // mat[a,a] = length / resolution  (RTL/main.py:207)
    s.bmin[a] = b_min3[a];
  }
  s.R = (float)R;
  s.canvas = canvas;
  s.canvas_R = R;
  return s;
}

// world position of vertex i: the two fp32 roundings of torch's `verts * scale + b_min` (RTL/main.py:231-237)
__device__ __forceinline__ void mp_surface_point(const MpSurfaceSrc& s, long long i, float& x, float& y, float& z) {
  const float vx = (float)__ldg(s.X + i), vy = (float)__ldg(s.Y + i), vz = __fsub_rn(s.R, __ldg(s.Z + i));
  x = __fadd_rn(__fmul_rn(vx, s.scale[0]), s.bmin[0]);
  y = __fadd_rn(__fmul_rn(vy, s.scale[1]), s.bmin[1]);
  z = __fadd_rn(__fmul_rn(vz, s.scale[2]), s.bmin[2]);
}

// the canvas pixel of vertex i takes channel r of its value v as v * 0.5 + 0.5 (RTL/main.py:244-248)
__device__ __forceinline__ void mp_surface_store(const MpSurfaceSrc& s, long long i, int r, float v) {
  float* px = s.canvas + ((size_t)__ldg(s.X + i) * s.canvas_R + (size_t)__ldg(s.Y + i)) * 3;
  px[r] = __fadd_rn(__fmul_rn(v, 0.5f), 0.5f);
}

// where results go
#define MP_MAX_PEERS 8
struct MpOutDst {
  float* out;          // MP_SRC_ROWS/GRID: [Res][ld]; value of point i, channel c at out[c*ld + i]
  long long ld;
  float* scatter_vol;  // if non-null: channel 0 is ALSO scattered to scatter_vol[nodes[i]]
  // fused slab exchange of the z-sharded grid query (mp_query_grid_peers): channel 0 of point i is ALSO stored at
  // peer[p][peer_off + i] for p < n_peers -- peer-memory pointers (NVLink P2P) to the full volumes of every rank, the
  // own one included -- so the volume is assembled on every GPU while the tiles are computed, without a collective.
  float* peer[MP_MAX_PEERS] = {};
  long long peer_off = 0;
  int n_peers = 0;
  // MP_SRC_NODES over the full volumes (the in-image list of a grid query): if set, the peer stores of point i go to
  // peer[p][nodes[i]] instead of peer[p][peer_off + i].  (An int in the struct's tail padding: the exact kernel keeps a
  // copy of dst on its stack.)
  int peer_by_node = 0;
};

// ---------------------------------------------------------------------------------------------
// device helpers shared by the fp32 and tensor-core kernels
// ---------------------------------------------------------------------------------------------
// point i of image b (batched launches: MP_SRC_ROWS only)
__device__ __forceinline__ void mp_load_point(const MpPointSrc& s, const MpBatch& bt, int b, long long i, float& x, float& y,
                                              float& z) {
  if (s.kind == MP_SRC_ROWS) {
    const long long o = (long long)b * bt.pt_stride + i * s.pstride;
    x = __ldg(s.px + o);
    y = __ldg(s.py + o);
    z = __ldg(s.pz + o);
    return;
  }
  int ix, iy, iz;
  if (s.kind == MP_SRC_GRID) {
    const long long plane = (long long)s.res * s.res;
    const long long li = i + s.lin0;
    iz = (int)(li / plane);
    const int r = (int)(li % plane);
    iy = r / s.res;
    ix = r - iy * s.res;
  } else {
    const int lin = __ldg(s.nodes + i);
    const int plane = s.res * s.res;
    iz = lin / plane;
    const int r = lin - iz * plane;
    iy = r / s.res;
    ix = r - iy * s.res;
  }
  // world = (c / R + 1/(2R)) * (b_max-b_min) + b_min, each op rounded separately (no FMA contraction)
  // so that the result is bit-identical to the engine's torch expression (oracle/spec.py:level_points)
  const float cx = (float)(ix * s.node_stride), cy = (float)(iy * s.node_stride), cz = (float)(iz * s.node_stride);
  const float R = (float)s.r_final;
  x = __fadd_rn(__fmul_rn(__fadd_rn(__fdiv_rn(cx, R), s.half_inv_r), s.bext[0]), s.bmin[0]);
  y = __fadd_rn(__fmul_rn(__fadd_rn(__fdiv_rn(cy, R), s.half_inv_r), s.bext[1]), s.bmin[1]);
  z = __fadd_rn(__fmul_rn(__fadd_rn(__fdiv_rn(cz, R), s.half_inv_r), s.bext[2]), s.bmin[2]);
}

// Image of tile t.  Divisions stay 32-bit (a 64-bit one is a call, whose saved registers would spill in the tensor-core
// program): mp_query_points_batch keeps a batched launch under 2^31 tiles, and a single-map launch, which has no such
// bound, maps every tile to image 0 without dividing.
__device__ __forceinline__ int mp_tile_image(const MpBatch& bt, long long t, long long tiles_per_image) {
  return bt.B == 1 ? 0 : (int)((unsigned)t / (unsigned)tiles_per_image);
}

// Tile t of image b is skipped by the range guard, and so is the rest of image b: the tile from which the launch's
// grid-stride loop goes on to this CTA's first tile of image b + 1 (for the last image, one from which it ends).
__device__ __forceinline__ long long mp_skip_image(const MpBatch& bt, long long t, int b, long long tiles_per_image) {
  const long long end = (long long)(b + 1) * tiles_per_image;
  if (b == bt.B - 1) return end - 1;
  return t + (long long)((unsigned)(end - 1 - t) / gridDim.x) * gridDim.x;
}

// image b's calibration (the same projection and depth scale, its own [R|t] rows)
__device__ __forceinline__ MpCalib mp_image_calib(const MpCalib& c, const MpBatch& bt, int b) {
  if (!bt.calibs) return c;
  MpCalib r = c;
#pragma unroll
  for (int k = 0; k < 12; ++k) r.m[k] = __ldg(bt.calibs + 12 * (long long)b + k);
  return r;
}

// the window [i0, i1) of a query's n points that this launch evaluates (see MpPointSrc::shard_rank)
__device__ __forceinline__ void mp_shard_window(const MpPointSrc& s, long long n, long long& i0, long long& i1) {
  i0 = 0; i1 = n;
  if (s.shard_world > 1) {
    long long per = (n + s.shard_world - 1) / s.shard_world;
    per = (per + 127) / 128 * 128;
    i0 = per * s.shard_rank;
    i1 = i0 + per;
    if (i0 > n) i0 = n;
    if (i1 > n) i1 = n;
  }
}

// geometry.py:19-34 / :37-55.  The roundings of every row m0 x + m1 y + m2 z + m3 are written out, so the result does not
// depend on which product the compiler would leave unfused: the fp32 kernels round m1 y first, the tensor-core program
// (X_FIRST) m0 x -- the results each program has always given.
template <bool X_FIRST = false>
__device__ __forceinline__ void mp_project(const MpCalib& c, float x, float y, float z, float& u, float& v, float& w) {
  if (!c.has) {
    u = x; v = y; w = z;
    return;
  }
  auto row = [&](const float* m) {
    const float p = X_FIRST ? fmaf(m[1], y, __fmul_rn(m[0], x)) : fmaf(m[0], x, __fmul_rn(m[1], y));
    return __fadd_rn(fmaf(m[2], z, p), m[3]);
  };
  u = row(c.m);
  v = row(c.m + 4);
  w = row(c.m + 8);
  if (c.perspective) {
    u = u / w;
    v = v / w;
  }
}

// Bilinear tap set of grid_sample(align_corners=True, padding zeros)  (geometry.py:15)
struct MpTaps {
  int off[4];     // texel index y*W+x of nw, ne, sw, se (clamped; weight is 0 when the tap is outside)
  float wgt[4];
};

__device__ __forceinline__ MpTaps mp_taps(float u, float v, int H, int W) {
  MpTaps t;
  const float ix = ((u + 1.f) / 2.f) * (float)(W - 1);
  const float iy = ((v + 1.f) / 2.f) * (float)(H - 1);
  const float x0 = floorf(ix), y0 = floorf(iy);
  const float x1 = x0 + 1.f, y1 = y0 + 1.f;
  float w_nw = (x1 - ix) * (y1 - iy);
  float w_ne = (ix - x0) * (y1 - iy);
  float w_sw = (x1 - ix) * (iy - y0);
  float w_se = (ix - x0) * (iy - y0);
  const bool x0ok = (x0 >= 0.f) && (x0 <= (float)(W - 1));
  const bool x1ok = (x1 >= 0.f) && (x1 <= (float)(W - 1));
  const bool y0ok = (y0 >= 0.f) && (y0 <= (float)(H - 1));
  const bool y1ok = (y1 >= 0.f) && (y1 <= (float)(H - 1));
  const int xi0 = min(max((int)x0, 0), W - 1), xi1 = min(max((int)x1, 0), W - 1);
  const int yi0 = min(max((int)y0, 0), H - 1), yi1 = min(max((int)y1, 0), H - 1);
  t.off[0] = yi0 * W + xi0; t.wgt[0] = (x0ok && y0ok) ? w_nw : 0.f;
  t.off[1] = yi0 * W + xi1; t.wgt[1] = (x1ok && y0ok) ? w_ne : 0.f;
  t.off[2] = yi1 * W + xi0; t.wgt[2] = (x0ok && y1ok) ? w_sw : 0.f;
  t.off[3] = yi1 * W + xi1; t.wgt[3] = (x1ok && y1ok) ? w_se : 0.f;
  return t;
}

__device__ __forceinline__ float mp_last_op(float v, int last_op) {
  if (last_op == MP_LAST_SIGMOID) return 1.f / (1.f + expf(-v));
  if (last_op == MP_LAST_TANH) return tanhf(v);
  return v;
}

// atomicAdd on a float (the VJP kernel's feature-gradient scatter).  The CPU model of tests/emu runs the threads of a CTA
// concurrently and models only the integer atomics: there it is a compare-and-swap loop on the float's bits.
__device__ __forceinline__ float mp_atomic_add(float* p, float v) {
#ifndef MP_CUDA_EMU
  return atomicAdd(p, v);
#else
  unsigned* u = reinterpret_cast<unsigned*>(p);
  unsigned old = __atomic_load_n(u, __ATOMIC_SEQ_CST), upd;
  float f;
  do {
    memcpy(&f, &old, 4);
    const float sum = f + v;
    memcpy(&upd, &sum, 4);
  } while (!__atomic_compare_exchange_n(u, &old, upd, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST));
  return f;
#endif
}

__device__ __forceinline__ float mp_lrelu(float v) { return v > 0.f ? v : v * MP_LEAKY_SLOPE; }

// host-side launchers implemented in the kernel files
// `guard`: the launch is conditional on the frame's feature range (feat->amax vs mlp->tc_amax_limit), evaluated on the device:
//   MP_GUARD_NONE always run, MP_GUARD_IN_RANGE run when max|feature| <= limit, MP_GUARD_OUT_OF_RANGE run when it is above.
// `bt` (batched launches; nullptr = one map): the launch covers bt->B images of src.n points.  The guard is decided per tile
// from the maximum of the tile's own image (feat->amax[b]).  A bt with B == 1 only moves the camera to device memory
// (MpBatch::calibs); the gradient and surface launchers take such a bt too.
enum { MP_GUARD_NONE = 0, MP_GUARD_IN_RANGE = 1, MP_GUARD_OUT_OF_RANGE = 2 };
int mp_launch_query_fp32(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal,
                         const MpOutDst& dst, cudaStream_t st, int guard = MP_GUARD_NONE, const MpBatch* bt = nullptr);
int mp_launch_query_tc(const mp_mlp* mlp, mp_feat* feat, const MpPointSrc& src, const MpCalib& cal,
                       const MpOutDst& dst, cudaStream_t st, int guard = MP_GUARD_NONE, const MpBatch* bt = nullptr);
// The tensor-core program over the nodes of an MP_SRC_GRID range that project into the image, for a head whose last op is
// Sigmoid (there a node outside the image has the value 0 * act = +0 exactly).  An ordered compaction lists those nodes in
// 4x4x4-brick order and stores +0 for the others into dst (out[i] and / or peer[p][peer_off + i]); the program then runs
// over the list with a device-side count.  One map, calib by value, R^3 < 2^31; the output is the dense launch's bit for
// bit.  `guard` as above.  scratch: mp_tc_grid_scratch_bytes(grid.n) bytes of device memory (a bound for every R) whose
// first 16 are zero (they are left at zero).
size_t mp_tc_grid_scratch_bytes(long long n);
int mp_launch_query_tc_grid(const mp_mlp* mlp, mp_feat* feat, const MpPointSrc& grid, const MpCalib& cal, const MpOutDst& dst,
                            void* scratch, cudaStream_t st, int guard);
// gradient of the fp32 query with respect to the points (query_fp32.cu): value -> out[r*ld_out+i] (out may be null; written
// by a query_fp32_kernel launch, so it is that kernel's value bit for bit),
// d(sum_r grad_out[r*ld_grad+i] * value_r)/d point_i -> dpoints[a*ld_dp+i] (grad_out null = ones): one launch of the VJP
// kernel below, for d points only; MP_SRC_ROWS.  bt: the images, as many as the handle's maps (nullptr: one map); image b's
// rows follow image b-1's, at grad_out + b*Res*ld_grad, out + b*Res*ld_out and dpoints + b*3*ld_dp (bt->out_stride is
// not read).  src.count_dev (when set) is the point count on the device; `guard` as for the query launchers.
int mp_launch_query_grad(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal,
                         const float* grad_out, long long ld_grad, float* out, long long ld_out, float* dpoints,
                         long long ld_dp, cudaStream_t st, int guard = MP_GUARD_NONE, const MpBatch* bt = nullptr);
// the same outputs, for the same images and layout, from the tensor-core program's forward-mode derivative (query_tc.cu:
// query_jvp_kernel), whose value is the tensor-core query's bit for bit; the shipped heads, MP_SRC_ROWS, maps of at most
// 65536 texels
int mp_launch_query_jvp_tc(const mp_mlp* mlp, mp_feat* feat, const MpPointSrc& src, const MpCalib& cal, const float* grad_out,
                           long long ld_grad, float* out, long long ld_out, float* dpoints, long long ld_dp, cudaStream_t st,
                           int guard, const MpBatch* bt = nullptr);
// The vector-Jacobian product of the exact query (query_fp32.cu: query_vjp_kernel; query_vjp.cu drives it).  The caller of
// mp_launch_query_vjp_tiles fills the outputs, the row tables and the chunk; the launcher fills w, mask_off and mask_words.
struct MpVjpParams {
  const float* w[MP_MAX_LAYERS];   // [cout][cin] row-major
  int mask_off[MP_MAX_LAYERS];     // words (of P points) before hidden layer l's sign mask
  int mask_words;
  const float* grad_out;           // image b, channel r, point i at grad_out[b * gout_stride + r * ld_grad + i]; null = ones
  long long ld_grad, gout_stride;
  float* dp;                       // null, or d points: image b, coordinate a, point i at dp[b * dp_stride + a * ld_dp + i]
  long long ld_dp, dp_stride;
  float* dfeat;                    // null, or [B][H][W][C] fp32, accumulated with atomicAdd
  // the ordered feature gradient (query_vjp.cu): when dx_rows is set, dfeat is not touched and column j of the chunk gets
  // dX[:C] at dx_rows[j * C ..] (in-image points only), its four tap weights at dx_wgt[4 j ..] and its cell key at dx_key[j]:
  // b * H * W + (the nw tap's texel) for an in-image point, B * H * W for a point at or beyond n or outside the image
  float* dx_rows;
  float* dx_wgt;
  unsigned* dx_key;
  float* rows;                     // null, or the saved rows [act rows ; delta rows][ld_rows] of the chunk's points
  long long ld_rows;
  int act_row[MP_MAX_LAYERS];      // row of hidden layer l's activations (the input X: rows 0 .. c0-1)
  int delta_row[MP_MAX_LAYERS];    // row of layer l's δ
  long long tile0, tile1;          // the chunk: tiles [tile0, tile1) of the B * ceil(n / P) tiles of the batch
};
// P of the VJP kernel for this head on the current device (a positive tile size), or an MP_E_* code
int mp_query_vjp_tile(const mp_mlp* mlp);
// one launch of query_vjp_kernel over the chunk of `outs` (src: MP_SRC_ROWS, n points per image -- src.count_dev, when set,
// the count on the device of a single-map launch; bt: the batch); `guard` as for the query launchers
int mp_launch_query_vjp_tiles(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal,
                              const MpBatch& bt, const MpVjpParams& outs, cudaStream_t st, int guard = MP_GUARD_NONE);
// the whole VJP (query_vjp.cu): outputs zeroed, then chunk by chunk the kernel and the weight-gradient contraction (and, with
// MP_VJP_DETERMINISTIC in flags, the ordered feature gradient's sort and gather), then the feature gradient's layout step.
// dweights / dbiases: n_layers device pointers each, or null; scratch as sized by mp_vjp_scratch_bytes for the same requests
// and flags.
long long mp_vjp_scratch_bytes(const mp_mlp* mlp, const mp_feat* feat, int B, long long n, long long chunk_points, bool dfeat,
                               bool dweights, int flags = 0);
int mp_launch_query_vjp(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal, const MpBatch& bt,
                        const float* grad_out, float* dfeat_nchw, float* dpoints, float* const* dweights, float* const* dbiases,
                        void* scratch, long long scratch_bytes, cudaStream_t st, int flags = 0);
// device-side predicate shared by the kernels: true = the tiles of this image (amax = its entry) must do nothing.  In the
// tensor-core program the weight producer and the consumers both take it, per tile, from the same word.
__device__ __forceinline__ bool mp_guard_skips(const unsigned* amax, float limit, int guard) {
  if (guard == MP_GUARD_NONE || amax == nullptr) return false;
  const bool above = __uint_as_float(*amax) > limit;
  return guard == MP_GUARD_IN_RANGE ? above : !above;
}
// colour head only: vertices (X, Y, R - Z) of the visible surface -> world -> colour -> canvas[X, Y, :]   (query_tc.cu)
// The eager entry point: the vertex count n on the host, the feature range checked on the host (MP_E_RANGE above the limit).
int mp_launch_colour_surface(const mp_mlp* mlp, mp_feat* feat, const long long* X, const long long* Y, const float* Z, long long n,
                             int R, const float* b_min3, const float* b_max3, const MpCalib& cal, float* canvas, cudaStream_t st);
// The same render by either program, enqueue-only: n = the capacity (surf.count, when set, the count on the device) and the
// range guard decided on the device (`guard` as above).  _tc: the colour head's tensor-core program (query_tc.cu); _fp32: the
// exact kernel (query_fp32.cu), any head with 3 outputs.
int mp_launch_surface_tc(const mp_mlp* mlp, mp_feat* feat, const MpSurfaceSrc& surf, long long n, const MpCalib& cal,
                         cudaStream_t st, int guard, const MpBatch* bt = nullptr);
int mp_launch_surface_fp32(const mp_mlp* mlp, const mp_feat* feat, const MpSurfaceSrc& surf, long long n, const MpCalib& cal,
                           cudaStream_t st, int guard, const MpBatch* bt = nullptr);
// the single-map MpBatch whose camera is the 12 floats at calib_dev (device memory); nullptr: the camera in MpCalib
inline MpBatch mp_device_calib(const float* calib_dev) {
  MpBatch b;
  b.calibs = calib_dev;
  return b;
}
int mp_tc_prepare(mp_mlp* mlp);     // builds mlp->tc; sets tc_ok
void mp_tc_release(mp_mlp* mlp);

// generic query dispatch (mode handling) used by the API and the octree engine
int mp_query_dispatch(mp_mlp* mlp, mp_feat* feat, const MpPointSrc& src, const MpCalib& cal, const MpOutDst& dst,
                      int mode, cudaStream_t st, const MpBatch* bt = nullptr);

// Host helpers of the launches (header-only, so that the CPU model of tests/emu runs these very lines)
inline void mp_fill_calib(MpCalib& c, const float* calib12, int projection, float z_scale) {
  memset(&c, 0, sizeof(c));
  c.has = calib12 != nullptr;
  if (calib12) memcpy(c.m, calib12, 12 * sizeof(float));
  c.perspective = (projection == MP_PROJ_PERSPECTIVE) && c.has;
  c.z_scale = z_scale;
}

// The camera of a single-map call: calib12 (host memory, or none) in the kernel parameters, or -- calib_dev set, the _dcal
// entry points -- 12 floats in device memory that the kernels read when they run.  Returns the batch to launch with
// (nullptr: the by-value camera).
inline const MpBatch* mp_single_calib(MpCalib& cal, MpBatch& bt, const float* calib12, const float* calib_dev, int projection,
                                      float z_scale) {
  if (!calib_dev) {
    mp_fill_calib(cal, calib12, projection, z_scale);
    return nullptr;
  }
  mp_fill_calib(cal, nullptr, projection, z_scale);
  cal.has = 1;
  cal.perspective = projection == MP_PROJ_PERSPECTIVE;
  bt = mp_device_calib(calib_dev);
  return &bt;
}

inline void mp_fill_grid_geom(MpPointSrc& s, int res, int node_stride, int r_final, const float* bmin, const float* bmax) {
  s.res = res;
  s.node_stride = node_stride;
  s.r_final = r_final;
  s.inv_r = 1.0f / (float)r_final;
  s.half_inv_r = (float)(1.0 / (2.0 * (double)r_final));
  for (int a = 0; a < 3; ++a) {
    s.bmin[a] = bmin[a];
    s.bext[a] = bmax[a] - bmin[a];   // fp32 subtraction, like torch's (b_max - b_min)
  }
}
