// F1 (fp32 flavour): fused  project -> in-image mask -> bilinear gather -> z-concat -> skip-MLP -> last_op -> mask
// on CUDA cores, fp32 end to end.  Replaces MonoPortNet.query (monoport/lib/modeling/MonoPortNet.py:48-91):
//   orthogonal()/perspective() geometry.py:19-55, index() geometry.py:4-16, DepthNormalizer.py:32,
//   SurfaceClassifier.forward heads/SurfaceClassifier.py:39-71.
// This is the exact (|err| ~1e-6) path and the one every head shape can use; the tensor-core kernel
// (query_tc.cu) is the fast path for the shipped heads.
//
// One CTA owns a tile of P points and walks all layers with the activations resident in shared memory:
//   sX  [C0 ][P]   sampled features + z (the skip input, read by every layer)
//   sA/sB [.][P]   ping/pong hidden activations
// Layout [k][P]: for a fixed input channel k the P point values are contiguous, so a thread that owns
// output channels reads them as broadcast float4s.  Weights are pre-transposed to [k][cout] so a warp's
// weight loads are coalesced; they stream from L2 (4.7 MB total, L2 resident).
#include "mp_common.cuh"

namespace {

constexpr int kThreads = 256;

struct Fp32Params {
  int n_layers;
  int c0;                       // input width (C + 1)
  int C, H, W;
  int cin[MP_MAX_LAYERS], cout[MP_MAX_LAYERS], hid[MP_MAX_LAYERS];   // hid = hidden part of cin
  const float* wt[MP_MAX_LAYERS];
  const float* bias[MP_MAX_LAYERS];
  const float* w_last;          // [cout_last][cin_last] row-major
  int last_op;
  int h_ping, h_pong;
  const float* feat;            // NHWC fp32
  const unsigned* amax;         // range guard (see mp_guard_skips)
  float amax_limit;
  int guard;
};

// acc[j][p] += w_j * act[p]
template <int P, int NCO>
__device__ __forceinline__ void fma_rows(float (&acc)[NCO][P], const float* __restrict__ act, const float (&w)[NCO]) {
#pragma unroll
  for (int q = 0; q < P / 4; ++q) {
    const float4 a = *reinterpret_cast<const float4*>(act + 4 * q);
#pragma unroll
    for (int j = 0; j < NCO; ++j) {
      acc[j][4 * q + 0] = fmaf(w[j], a.x, acc[j][4 * q + 0]);
      acc[j][4 * q + 1] = fmaf(w[j], a.y, acc[j][4 * q + 1]);
      acc[j][4 * q + 2] = fmaf(w[j], a.z, acc[j][4 * q + 2]);
      acc[j][4 * q + 3] = fmaf(w[j], a.w, acc[j][4 * q + 3]);
    }
  }
}

// One hidden layer: out[co][p] = lrelu(b[co] + sum_k Wt[k][co] * in[k][p]),  in = [hidden rows ; skip rows]
// MASK (the VJP kernel): also store the sign of every pre-activation, bit co % 32 of sMask[(co / 32) * P + p]
template <int P, int NCO, bool MASK = false>
__device__ void dense_layer(const float* __restrict__ wt, const float* __restrict__ bias, int cin_hidden, int cin_skip,
                            int cout, const float* sHidden, const float* sSkip, float* sOut, unsigned* sMask = nullptr) {
  const int tid = threadIdx.x;
  for (int base = 0; base < cout; base += kThreads * NCO) {
    int co[NCO];
    bool ok[NCO];
#pragma unroll
    for (int j = 0; j < NCO; ++j) {
      co[j] = base + j * kThreads + tid;
      ok[j] = co[j] < cout;
      if (!ok[j]) co[j] = cout - 1;
    }
    float acc[NCO][P];
#pragma unroll
    for (int j = 0; j < NCO; ++j) {
      const float b = __ldg(bias + co[j]);
#pragma unroll
      for (int p = 0; p < P; ++p) acc[j][p] = b;
    }
    // hidden part then skip part -- the reference concatenates [hidden, input] (SurfaceClassifier.py:55)
    for (int part = 0; part < 2; ++part) {
      const int nk = part == 0 ? cin_hidden : cin_skip;
      const float* act = part == 0 ? sHidden : sSkip;
      const float* wrow = wt + (size_t)(part == 0 ? 0 : cin_hidden) * cout;
      int k = 0;
      for (; k + 4 <= nk; k += 4) {
        float w[4][NCO];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
          for (int j = 0; j < NCO; ++j) w[kk][j] = __ldg(wrow + (size_t)(k + kk) * cout + co[j]);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) fma_rows<P, NCO>(acc, act + (size_t)(k + kk) * P, w[kk]);
      }
      for (; k < nk; ++k) {
        float w[NCO];
#pragma unroll
        for (int j = 0; j < NCO; ++j) w[j] = __ldg(wrow + (size_t)k * cout + co[j]);
        fma_rows<P, NCO>(acc, act + (size_t)k * P, w);
      }
    }
    if constexpr (MASK) {
      // lane l of a warp owns channel 32 w + l (kThreads is a multiple of 32), so one ballot per point is one mask word;
      // lane p stores point p's word.  (Bits of clamped channels >= cout are never read.)
      const int lane = tid & 31;
#pragma unroll
      for (int j = 0; j < NCO; ++j) {
        const int word = (base + j * kThreads + (tid & ~31)) >> 5;
        unsigned mine = 0u;
#pragma unroll
        for (int p = 0; p < P; ++p) {
          const unsigned bits = __ballot_sync(0xffffffffu, acc[j][p] > 0.f);
          if (lane == p) mine = bits;
        }
        if (lane < P && word * 32 < cout) sMask[(size_t)word * P + lane] = mine;
      }
    }
#pragma unroll
    for (int j = 0; j < NCO; ++j) {
      if (!ok[j]) continue;
      float* o = sOut + (size_t)co[j] * P;
#pragma unroll
      for (int q = 0; q < P / 4; ++q) {
        float4 v;
        v.x = mp_lrelu(acc[j][4 * q + 0]);
        v.y = mp_lrelu(acc[j][4 * q + 1]);
        v.z = mp_lrelu(acc[j][4 * q + 2]);
        v.w = mp_lrelu(acc[j][4 * q + 3]);
        *reinterpret_cast<float4*>(o + 4 * q) = v;
      }
    }
  }
}

// ---- the steps of a tile, shared by query_fp32_kernel and the forward half of query_vjp_kernel --------------------------
// 1. projection, mask, taps of image b's points; 2. bilinear gather from its map `feat`: sX = [sampled features ;
// z * z_scale], sMeta[p] = in_img.  SURF: the points are the vertices of *surf (one map) instead of src's.
template <int P, bool SURF = false>
__device__ __forceinline__ void tile_sample(const Fp32Params& prm, const MpPointSrc& src, const MpCalib& cal, const MpBatch& bt,
                                            int b, const float* feat, long long p0, long long n, float* sX, float* sMeta,
                                            int (&sOff)[4][P], float (&sWgt)[4][P], const MpSurfaceSrc* surf = nullptr) {
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  if (tid < P) {
    const long long i = p0 + tid;
    float u = 0.f, v = 0.f, w = 0.f;
    bool valid = i < n;
    if (valid) {
      float x, y, z;
      if constexpr (SURF) mp_surface_point(*surf, i, x, y, z);
      else mp_load_point(src, bt, b, i, x, y, z);
      mp_project(mp_image_calib(cal, bt, b), x, y, z, u, v, w);
    }
    const bool in_img = valid && (u >= -1.f) && (u <= 1.f) && (v >= -1.f) && (v <= 1.f);   // MonoPortNet.py:74
    MpTaps t = mp_taps(valid ? u : 0.f, valid ? v : 0.f, prm.H, prm.W);
    // NaN coordinates (perspective with w==0): in_img is false; keep taps finite
    if (!(u == u) || !(v == v)) {
#pragma unroll
      for (int a = 0; a < 4; ++a) { t.off[a] = 0; t.wgt[a] = 0.f; }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) { sOff[a][tid] = t.off[a]; sWgt[a][tid] = t.wgt[a]; }
    sMeta[0 * P + tid] = in_img ? 1.f : 0.f;
    sX[(size_t)prm.C * P + tid] = w * cal.z_scale;                                          // DepthNormalizer.py:32
  }
  __syncthreads();
  // warp per point, lanes over channels (NHWC => contiguous)
  for (int p = warp; p < P; p += kThreads / 32) {
    const float* f0 = feat + (size_t)sOff[0][p] * prm.C;
    const float* f1 = feat + (size_t)sOff[1][p] * prm.C;
    const float* f2 = feat + (size_t)sOff[2][p] * prm.C;
    const float* f3 = feat + (size_t)sOff[3][p] * prm.C;
    const float w0 = sWgt[0][p], w1 = sWgt[1][p], w2 = sWgt[2][p], w3 = sWgt[3][p];
    for (int c = lane; c < prm.C; c += 32) {
      // same accumulation order as grid_sample: nw, ne, sw, se (the first sum rounded as written: ne's product first)
      float v = fmaf(__ldg(f0 + c), w0, __fmul_rn(__ldg(f1 + c), w1));
      v += __ldg(f2 + c) * w2;
      v += __ldg(f3 + c) * w3;
      sX[(size_t)c * P + p] = v;
    }
  }
  __syncthreads();
}

// what tile_hidden hands every finished hidden layer (l, its [cout][P] activations): nothing, except in the VJP kernel
struct NoLayerSink {
  __device__ __forceinline__ void operator()(int, const float*) const {}
};

// 3. hidden layers, ping-ponging between sA and sB (layer l writes sA for even l, sB for odd l); returns the last hidden
// layer's activations.  MASK: layer l also stores its pre-activation signs at sMask + mask_off[l].  `sink` sees each layer's
// activations after the barrier that ends it, before the next-but-one layer overwrites them.
template <int P, bool MASK, class Sink = NoLayerSink>
__device__ __forceinline__ const float* tile_hidden(const Fp32Params& prm, const float* sX, float* sA, float* sB,
                                                    unsigned* sMask = nullptr, const int* mask_off = nullptr,
                                                    const Sink& sink = Sink()) {
  const float* sIn = sX;
  float* sOut = sA;
  for (int l = 0; l < prm.n_layers - 1; ++l) {
    const int hid = prm.hid[l];
    const int skipw = prm.cin[l] - hid;
    unsigned* m = MASK ? sMask + mask_off[l] : nullptr;
    if (l == 0) {
      dense_layer<P, 2, MASK>(prm.wt[l], prm.bias[l], 0, prm.cin[l], prm.cout[l], sX, sX, sOut, m);
    } else if (prm.cout[l] > kThreads) {
      dense_layer<P, 2, MASK>(prm.wt[l], prm.bias[l], hid, skipw, prm.cout[l], sIn, sX, sOut, m);
    } else {
      dense_layer<P, 1, MASK>(prm.wt[l], prm.bias[l], hid, skipw, prm.cout[l], sIn, sX, sOut, m);
    }
    __syncthreads();
    sink(l, sOut);
    sIn = sOut;
    sOut = (sOut == sA) ? sB : sA;
  }
  return sIn;
}

// 4. last layer, one warp per (point p, out channel r): the logit without its bias, on every lane
template <int P>
__device__ __forceinline__ float last_layer_dot(const Fp32Params& prm, const float* sX, const float* sIn, int p, int r, int lane) {
  const int l = prm.n_layers - 1;
  const int hid = prm.n_layers == 1 ? 0 : prm.hid[l];
  const int cin = prm.cin[l];
  const float* wrow = prm.w_last + (size_t)r * cin;
  float acc = 0.f;
  for (int k = lane; k < cin; k += 32) {
    const float a = (prm.n_layers == 1) ? sX[(size_t)k * P + p]
                    : (k < hid ? sIn[(size_t)k * P + p] : sX[(size_t)(k - hid) * P + p]);
    acc = fmaf(__ldg(wrow + k), a, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// bt.B images of src.n points (more than one: MP_SRC_ROWS); tile t is tile t % n_tiles of image t / n_tiles, which samples
// its own map and calibration and writes its own outputs; the range guard is decided per tile from that image's maximum.
// SURF (a separate instantiation, so the query instantiations keep their code): the exact twin of the tensor-core program's
// surface render -- src.n vertices of surf (one map; surf.count, when set, the count on the device), their colours into
// surf.canvas.
template <int P, bool SURF>
__global__ void __launch_bounds__(kThreads, 1)
query_fp32_kernel(Fp32Params prm, MpPointSrc src, MpCalib cal, MpOutDst dst, MpBatch bt, MpSurfaceSrc surf) {
  MP_DYN_SMEM_ALIGNED(float, smem, 16);
  float* sX = smem;                                  // [c0][P]
  float* sA = sX + (size_t)prm.c0 * P;               // [h_ping][P]
  float* sB = sA + (size_t)prm.h_ping * P;           // [h_pong][P]
  float* sMeta = sB + (size_t)prm.h_pong * P;        // [8][P]: in_img, u, v, z_feat, (4 spare)
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;

  long long n = src.n;
  if (src.count_dev) {
    const long long c = *src.count_dev;
    n = c < n ? c : n;
  }
  if constexpr (SURF) {
    if (surf.count) {
      const long long c = *surf.count;
      n = c < n ? c : n;
    }
  }
  long long win0, win1;
  mp_shard_window(src, n, win0, win1);
  n = win1;                                          // points >= n are padding; the first evaluated one is win0
  const long long n_tiles = (win1 - win0 + P - 1) / P;          // (per image)
  const long long all_tiles = n_tiles * bt.B;

  for (long long at = blockIdx.x; at < all_tiles; at += gridDim.x) {
    const int b = mp_tile_image(bt, at, n_tiles);
    if (mp_guard_skips(prm.amax + b, prm.amax_limit, prm.guard)) {      // (uniform over the CTA)
      at = mp_skip_image(bt, at, b, n_tiles);
      continue;
    }
    const long long p0 = win0 + (at - (long long)b * n_tiles) * P;
    __shared__ int sOff[4][P];
    __shared__ float sWgt[4][P];
    tile_sample<P, SURF>(prm, src, cal, bt, b, prm.feat + (size_t)b * prm.H * prm.W * prm.C, p0, n, sX, sMeta, sOff, sWgt, &surf);
    const float* sIn = tile_hidden<P, false>(prm, sX, sA, sB);
    const int l = prm.n_layers - 1;
    float* out = dst.out + b * bt.out_stride;
    for (int job = warp; job < P * prm.cout[l]; job += kThreads / 32) {
      const int p = job % P, r = job / P;
      const float acc = last_layer_dot<P>(prm, sX, sIn, p, r, lane);
      if (lane == 0) {
        const long long i = p0 + p;
        if (i < n) {
          float v = mp_last_op(acc + __ldg(prm.bias[l] + r), prm.last_op);
          v = sMeta[p] * v;                                                              // MonoPortNet.py:89
          if constexpr (SURF) {
            mp_surface_store(surf, i, r, v);                                             // RTL/main.py:244-248
            continue;
          }
          if (out) out[(long long)r * dst.ld + i] = v;
          if (dst.scatter_vol && r == 0) dst.scatter_vol[__ldg(src.nodes + i)] = v;
          if (r == 0)
            for (int pp = 0; pp < dst.n_peers; ++pp) dst.peer[pp][dst.peer_off + i] = v;      // peer-memory stores (NVLink)
        }
      }
    }
    __syncthreads();
  }
}

// ---- F1'' and F1'''': the reverse pass of the query (the point gradient, and the vector-Jacobian product for training) ---
// Forward half = the fp32 kernel's tile steps (tile_sample / tile_hidden / last_layer_dot above), which also record the sign
// of every hidden pre-activation as bit masks (1920 bits per point for the shipped heads).  Reverse half, per tile:
//   g      = grad_out * last_op'(value) * in_img                                    -> sG    [Res][P]
//   δ_l    = (W_{l+1}[:, :hid]^T δ_{l+1}) * lrelu'(pre_l)   (δ_l in layer l's ping/pong block)
//   dX     = W_0^T δ_0 + sum_{l>=1} W_l[:, hid:]^T δ_l         (accumulated in sX, which the forward half no longer needs)
//   d(u,v) = sum_c dX_c * dX_c/d(u,v)   (grid_sample's backward: the tap differences), dw = z_scale * dX_C
//   dp     = J^T d(u,v,w),  J = d(u,v,w)/dp of the projection
// The transposed products read the row-major [cout][cin] weight copy: the thread that owns input channel k reads w[co][k].

// out[k][p] = sum_co W[co][k] * delta[co][p] for the cin input channels k of a layer; rows k < hid are the previous layer's
// δ (times lrelu' from its mask), rows k >= hid go to dX[k - hid] (assigned when `first`, accumulated otherwise)
template <int P, int NCO>
__device__ void transposed_layer(const float* __restrict__ w, int cin, int cout, int hid, const float* sDelta, float* sHid,
                                 const unsigned* sMask, float* sDX, bool first) {
  const int tid = threadIdx.x;
  for (int base = 0; base < cin; base += kThreads * NCO) {
    int k[NCO];
    bool ok[NCO];
#pragma unroll
    for (int j = 0; j < NCO; ++j) {
      k[j] = base + j * kThreads + tid;
      ok[j] = k[j] < cin;
      if (!ok[j]) k[j] = cin - 1;
    }
    float acc[NCO][P];
#pragma unroll
    for (int j = 0; j < NCO; ++j)
#pragma unroll
      for (int p = 0; p < P; ++p) acc[j][p] = 0.f;
    int co = 0;
    for (; co + 4 <= cout; co += 4) {
      float wv[4][NCO];
#pragma unroll
      for (int cc = 0; cc < 4; ++cc)
#pragma unroll
        for (int j = 0; j < NCO; ++j) wv[cc][j] = __ldg(w + (size_t)(co + cc) * cin + k[j]);
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) fma_rows<P, NCO>(acc, sDelta + (size_t)(co + cc) * P, wv[cc]);
    }
    for (; co < cout; ++co) {
      float wv[NCO];
#pragma unroll
      for (int j = 0; j < NCO; ++j) wv[j] = __ldg(w + (size_t)co * cin + k[j]);
      fma_rows<P, NCO>(acc, sDelta + (size_t)co * P, wv);
    }
#pragma unroll
    for (int j = 0; j < NCO; ++j) {
      if (!ok[j]) continue;
      if (k[j] < hid) {
        const unsigned* m = sMask + (size_t)(k[j] >> 5) * P;
        const unsigned bit = 1u << (k[j] & 31);
        float* o = sHid + (size_t)k[j] * P;
#pragma unroll
        for (int p = 0; p < P; ++p) o[p] = (m[p] & bit) ? acc[j][p] : acc[j][p] * MP_LEAKY_SLOPE;   // torch: lrelu'(0) = slope
      } else {
        float* o = sDX + (size_t)(k[j] - hid) * P;
#pragma unroll
        for (int p = 0; p < P; ++p) o[p] = first ? acc[j][p] : o[p] + acc[j][p];
      }
    }
  }
}

// the input gradient dX (in sX) of the tile's points of image b -> d(u,v,w) -> d point, written at dp[a * ld_dp + i]: warp
// per point, lanes over channels
template <int P>
__device__ __forceinline__ void tile_point_grad(const Fp32Params& prm, const MpPointSrc& src, const MpCalib& cal, const MpBatch& bt,
                                                int b, const float* feat, long long p0, long long n, const float* sX,
                                                const float* sMeta, const int (&sOff)[4][P], float* dp_img, long long ld_dp) {
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  for (int p = warp; p < P; p += kThreads / 32) {
    const long long i = p0 + p;
    if (i >= n) continue;
    float* dp = dp_img + i;
    if (sMeta[p] == 0.f) {                             // outside the image: exactly 0
      if (lane < 3) dp[lane * ld_dp] = 0.f;
      continue;
    }
    // the projection and its Jacobian below: one MpCalib, the camera tile_sample projected with
    const MpCalib c = mp_image_calib(cal, bt, b);
    float x, y, z, u, v, w;
    mp_load_point(src, bt, b, i, x, y, z);
    mp_project(c, x, y, z, u, v, w);
    // the tap cell of mp_taps; a tap outside the map is zero padding and contributes nothing
    const float ix = ((u + 1.f) / 2.f) * (float)(prm.W - 1);
    const float iy = ((v + 1.f) / 2.f) * (float)(prm.H - 1);
    const float x0 = floorf(ix), y0 = floorf(iy);
    const float fx = ix - x0, fy = iy - y0;
    const float x1 = x0 + 1.f, y1 = y0 + 1.f;
    const bool x0ok = (x0 >= 0.f) && (x0 <= (float)(prm.W - 1));
    const bool x1ok = (x1 >= 0.f) && (x1 <= (float)(prm.W - 1));
    const bool y0ok = (y0 >= 0.f) && (y0 <= (float)(prm.H - 1));
    const bool y1ok = (y1 >= 0.f) && (y1 <= (float)(prm.H - 1));
    const bool ok_nw = x0ok && y0ok, ok_ne = x1ok && y0ok, ok_sw = x0ok && y1ok, ok_se = x1ok && y1ok;
    const float* f0 = feat + (size_t)sOff[0][p] * prm.C;
    const float* f1 = feat + (size_t)sOff[1][p] * prm.C;
    const float* f2 = feat + (size_t)sOff[2][p] * prm.C;
    const float* f3 = feat + (size_t)sOff[3][p] * prm.C;
    float du = 0.f, dv = 0.f;
    for (int c = lane; c < prm.C; c += 32) {
      const float fnw = ok_nw ? __ldg(f0 + c) : 0.f, fne = ok_ne ? __ldg(f1 + c) : 0.f;
      const float fsw = ok_sw ? __ldg(f2 + c) : 0.f, fse = ok_se ? __ldg(f3 + c) : 0.f;
      const float dx = sX[(size_t)c * P + p];
      du = fmaf(dx, (1.f - fy) * (fne - fnw) + fy * (fse - fsw), du);
      dv = fmaf(dx, (1.f - fx) * (fsw - fnw) + fx * (fse - fne), dv);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      du += __shfl_xor_sync(0xffffffffu, du, o);
      dv += __shfl_xor_sync(0xffffffffu, dv, o);
    }
    if (lane == 0) {
      du *= 0.5f * (float)(prm.W - 1);
      dv *= 0.5f * (float)(prm.H - 1);
      const float dw = c.z_scale * sX[(size_t)prm.C * P + p];
      float g[3];
      if (!c.has) {
        g[0] = du; g[1] = dv; g[2] = dw;
      } else if (!c.perspective) {                     // J = R
#pragma unroll
        for (int a = 0; a < 3; ++a) g[a] = c.m[a] * du + c.m[4 + a] * dv + c.m[8 + a] * dw;
      } else {                                         // J rows: (R0 - u R2) / w, (R1 - v R2) / w, R2
        const float su = du / w, sv = dv / w;
        const float s2 = dw - su * u - sv * v;
#pragma unroll
        for (int a = 0; a < 3; ++a) g[a] = c.m[a] * su + c.m[4 + a] * sv + c.m[8 + a] * s2;
      }
#pragma unroll
      for (int a = 0; a < 3; ++a) dp[a * ld_dp] = g[a];
    }
  }
}

// query_vjp_kernel runs these steps over the B * ceil(n / P) tiles of a batch (tile t of image t / ceil(n / P), as
// query_fp32_kernel maps them), for the tiles [vp.tile0, vp.tile1) of one chunk.  n is src.n, or the count on the device
// when src.count_dev is set (single-map launches: the tile bound follows the count); the range guard skips an image as in
// query_fp32_kernel.  Besides d points it can
//   - save the rows the weight gradient contracts: the input X and every hidden activation in the forward half, every δ_l
//     (the last layer's g included) in the reverse half -- column (t - tile0) * P + p of vp.rows (query_vjp.cu sums them);
//   - scatter dX[:C] of each in-image point onto its four taps with grid_sample's weights (atomicAdd into [B][H][W][C]), or,
//     with vp.dx_rows set, record dX[:C], the tap weights and the cell key of each column for query_vjp.cu's ordered gather.
// It writes no values.
template <int P>
__device__ __forceinline__ void save_rows(float* dst, long long ld, const float* src, int rows) {
  for (int e = threadIdx.x; e < rows * P; e += kThreads) {
    const int r = e / P, p = e % P;
    dst[(long long)r * ld + p] = src[(size_t)r * P + p];
  }
}

template <int P>
struct SaveActivations {
  float* rows;                 // this tile's first column, or null
  long long ld;
  const int* act_row;
  const int* cout;
  __device__ __forceinline__ void operator()(int l, const float* sOut) const {
    if (rows) save_rows<P>(rows + (long long)act_row[l] * ld, ld, sOut, cout[l]);
  }
};

template <int P>
__global__ void __launch_bounds__(kThreads, 1)
query_vjp_kernel(Fp32Params prm, MpVjpParams vp, MpPointSrc src, MpCalib cal, MpBatch bt) {
  MP_DYN_SMEM_ALIGNED(float, smem, 16);
  float* sX = smem;                                  // [c0][P]: sampled input, then dX
  float* sA = sX + (size_t)prm.c0 * P;               // [h_ping][P]: activations of even layers, then their δ
  float* sB = sA + (size_t)prm.h_ping * P;           // [h_pong][P]: odd layers
  float* sMeta = sB + (size_t)prm.h_pong * P;        // [8][P]: in_img
  unsigned* sMask = reinterpret_cast<unsigned*>(sMeta + 8 * P);          // [mask_words][P]
  float* sG = reinterpret_cast<float*>(sMask + (size_t)vp.mask_words * P);   // [Res][P]
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int L = prm.n_layers;
  const int res = prm.cout[L - 1];
  long long n = src.n;
  if (src.count_dev) {                               // (the point count on the device: src.n is then the capacity)
    const long long c = *src.count_dev;
    n = c < n ? c : n;
  }
  const long long n_tiles = (n + P - 1) / P;         // (per image)
  const long long tile1 = vp.tile1 < n_tiles * bt.B ? vp.tile1 : n_tiles * bt.B;
  const bool need_dx = vp.dp || vp.dfeat;            // (else the reverse pass stops at δ_0)

  for (long long at = vp.tile0 + blockIdx.x; at < tile1; at += gridDim.x) {
    const int b = mp_tile_image(bt, at, n_tiles);
    if (mp_guard_skips(prm.amax + b, prm.amax_limit, prm.guard)) {      // (uniform over the CTA)
      at = mp_skip_image(bt, at, b, n_tiles);
      continue;
    }
    const long long p0 = (at - (long long)b * n_tiles) * P;
    const float* feat = prm.feat + (size_t)b * prm.H * prm.W * prm.C;
    float* rows = vp.rows ? vp.rows + (at - vp.tile0) * P : nullptr;
    // ---- forward half ----------------------------------------------------------------------------
    __shared__ int sOff[4][P];
    __shared__ float sWgt[4][P];
    tile_sample<P>(prm, src, cal, bt, b, feat, p0, n, sX, sMeta, sOff, sWgt);
    if (rows) save_rows<P>(rows, vp.ld_rows, sX, prm.c0);
    const float* sIn = tile_hidden<P, true>(prm, sX, sA, sB, sMask, vp.mask_off,
                                            SaveActivations<P>{rows, vp.ld_rows, vp.act_row, prm.cout});
    for (int job = warp; job < P * res; job += kThreads / 32) {
      const int p = job % P, r = job / P;
      const float acc = last_layer_dot<P>(prm, sX, sIn, p, r, lane);
      if (lane == 0) {
        const long long i = p0 + p;
        float g = 0.f;
        if (i < n) {
          const float y = mp_last_op(acc + __ldg(prm.bias[L - 1] + r), prm.last_op);
          const float d = prm.last_op == MP_LAST_SIGMOID ? y * (1.f - y) : (prm.last_op == MP_LAST_TANH ? 1.f - y * y : 1.f);
          g = (vp.grad_out ? __ldg(vp.grad_out + b * vp.gout_stride + (long long)r * vp.ld_grad + i) : 1.f) * d;
          if (sMeta[p] == 0.f) g = 0.f;                  // in_img multiplies the output (and y may be NaN/inf there)
        }
        sG[r * P + p] = g;
      }
    }
    __syncthreads();
    if (rows) save_rows<P>(rows + (long long)vp.delta_row[L - 1] * vp.ld_rows, vp.ld_rows, sG, res);
    // ---- reverse half: last layer down to layer 0 (layer 0 only for dX) ----------------------------
    const float* sDelta = sG;
    for (int l = L - 1; l >= (need_dx ? 0 : 1); --l) {
      const int hid = l == 0 ? 0 : prm.hid[l];
      float* sHid = l == 0 ? nullptr : (((l - 1) & 1) ? sB : sA);
      const unsigned* m = l == 0 ? nullptr : sMask + vp.mask_off[l - 1];
      if (prm.cin[l] > kThreads)
        transposed_layer<P, 2>(vp.w[l], prm.cin[l], prm.cout[l], hid, sDelta, sHid, m, sX, l == L - 1);
      else
        transposed_layer<P, 1>(vp.w[l], prm.cin[l], prm.cout[l], hid, sDelta, sHid, m, sX, l == L - 1);
      __syncthreads();
      if (rows && l > 0) save_rows<P>(rows + (long long)vp.delta_row[l - 1] * vp.ld_rows, vp.ld_rows, sHid, prm.cout[l - 1]);
      sDelta = sHid;
    }
    // ---- dX -> d points, and dX[:C] -> the four taps of the feature map -----------------------------
    if (vp.dp) tile_point_grad<P>(prm, src, cal, bt, b, feat, p0, n, sX, sMeta, sOff, vp.dp + b * vp.dp_stride, vp.ld_dp);
    if (vp.dx_rows) {
      // the ordered path: the chunk's columns for the sort and gather of query_vjp.cu, no atomics
      const long long HW = (long long)prm.H * prm.W;
      for (int p = warp; p < P; p += kThreads / 32) {
        const long long col = (at - vp.tile0) * P + p;
        const bool in = p0 + p < n && sMeta[p] != 0.f;
        if (in) {
          float* d = vp.dx_rows + col * prm.C;
          for (int c = lane; c < prm.C; c += 32) d[c] = sX[(size_t)c * P + p];
        }
        if (lane < 4) vp.dx_wgt[col * 4 + lane] = sWgt[lane][p];
        if (lane == 0) vp.dx_key[col] = (unsigned)(in ? b * HW + sOff[0][p] : bt.B * HW);
      }
    } else if (vp.dfeat) {
      float* df = vp.dfeat + (size_t)b * prm.H * prm.W * prm.C;
      for (int p = warp; p < P; p += kThreads / 32) {
        if (p0 + p >= n || sMeta[p] == 0.f) continue;          // outside the image: nothing, anywhere
        for (int a = 0; a < 4; ++a) {
          const float wa = sWgt[a][p];
          if (wa == 0.f) continue;                             // (a tap off the map has weight 0)
          float* t = df + (size_t)sOff[a][p] * prm.C;
          for (int c = lane; c < prm.C; c += 32) mp_atomic_add(t + c, wa * sX[(size_t)c * P + p]);
        }
      }
    }
    __syncthreads();
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------------
struct DeviceLimits {
  int sms, max_smem;            // SM count, shared-memory opt-in limit per block
};

// The shared memory of a head's tiles: the widest even and odd hidden layers (the ping / pong blocks sA / sB) and, for the
// reverse pass, the sign-mask words per point of the hidden layers (mask_off[l]: the words before hidden layer l's).
struct HeadLayout {
  int c0, ping, pong, res;
  int mask_words, mask_off[MP_MAX_LAYERS];
  // bytes of a P-point tile: sX, sA, sB and sMeta [8][P]; the reverse pass adds sMask and sG [res][P]
  size_t tile_bytes(int P, bool reverse) const {
    return (size_t)(c0 + ping + pong + 8 + (reverse ? mask_words + res : 0)) * P * sizeof(float);
  }
  // the largest tile of 32, 16 or 8 points that fits beside the 2 KB kept for the kernels' static shared memory; 0: none
  int fit_tile(bool reverse, int max_smem) const {
    for (int P = 32; P >= 8; P /= 2)
      if (tile_bytes(P, reverse) + 2048 <= (size_t)max_smem) return P;
    return 0;
  }
};

HeadLayout head_layout(const mp_mlp* mlp) {
  HeadLayout h;
  memset(&h, 0, sizeof(h));
  h.c0 = mlp->channels[0];
  h.res = mlp->cout[mlp->n_layers - 1];
  for (int l = 0; l + 1 < mlp->n_layers; ++l) {
    int& width = l % 2 == 0 ? h.ping : h.pong;
    width = width > mlp->cout[l] ? width : mlp->cout[l];
    h.mask_off[l] = h.mask_words;
    h.mask_words += (mlp->cout[l] + 31) / 32;
  }
  return h;
}

// the current device's limits, read once per device and thread
int device_limits(DeviceLimits& dev) {
  static thread_local DeviceLimits cached[64] = {};
  int d = 0;
  MP_CUDA(cudaGetDevice(&d));
  if (d >= 0 && d < 64 && cached[d].sms) {
    dev = cached[d];
    return MP_OK;
  }
  MP_CUDA(cudaDeviceGetAttribute(&dev.sms, cudaDevAttrMultiProcessorCount, d));
  MP_CUDA(cudaDeviceGetAttribute(&dev.max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, d));
  if (d >= 0 && d < 64) cached[d] = dev;
  return MP_OK;
}

// Fp32Params of a head and a map, with the range guard `guard` on the map's maxima; the head's layout; the device's limits
int fill_params(const mp_mlp* mlp, const mp_feat* feat, int guard, Fp32Params& prm, HeadLayout& h, DeviceLimits& dev) {
  memset(&prm, 0, sizeof(prm));
  prm.n_layers = mlp->n_layers;
  prm.c0 = mlp->channels[0];
  prm.C = feat->C; prm.H = feat->H; prm.W = feat->W;
  if (prm.c0 != feat->C + 1) {
    mp_set_error("head expects %d input channels but the feature map has %d (+1 depth)", prm.c0, feat->C);
    return MP_E_INVALID;
  }
  for (int l = 0; l < mlp->n_layers; ++l) {
    prm.cin[l] = mlp->cin[l];
    prm.cout[l] = mlp->cout[l];
    prm.hid[l] = (l == 0) ? 0 : mlp->channels[l];
    prm.wt[l] = mlp->wt[l];
    prm.bias[l] = mlp->bias[l];
    if (l > 0 && !mlp->skip) {
      mp_set_error("no_residual heads are not supported");
      return MP_E_UNSUPPORTED;
    }
  }
  prm.w_last = mlp->w[mlp->n_layers - 1];
  prm.last_op = mlp->last_op;
  h = head_layout(mlp);
  prm.h_ping = h.ping; prm.h_pong = h.pong;
  prm.feat = feat->nhwc32;
  prm.amax = feat->amax; prm.amax_limit = mlp->tc_amax_limit; prm.guard = guard;
  return device_limits(dev);
}

// One launch of Kernel, an exact kernel whose tiles are P points, on min(tiles, SMs) CTAs (at least one) with `smem` bytes
// of dynamic shared memory.  The opt-in is a property of the kernel instantiation, shared by every thread, and heads of
// different widths launch the same instantiation with different sizes: it is always set to the same bound -- the device's
// maximum less the 2 KB HeadLayout::fit_tile keeps free for the kernel's static shared memory -- so no thread lowers it
// under another thread's launch.  (Sticky per device, and recorded per instantiation: Kernel is a template argument, so each
// one has its own `opted`.  Raising it again for every launch costs a driver call per query.)
template <int P, auto Kernel, class... Args>
int launch(long long tiles, size_t smem, const DeviceLimits& dev, cudaStream_t st, const Args&... args) {
  static thread_local bool opted[64] = {};
  int d = 0;
  MP_CUDA(cudaGetDevice(&d));
  if (d < 0 || d >= 64 || !opted[d]) {
    MP_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dev.max_smem - 2048));
    if (d >= 0 && d < 64) opted[d] = true;
  }
  const int grid = (int)(tiles < (long long)dev.sms ? (tiles > 0 ? tiles : 1) : dev.sms);
#ifndef MP_CUDA_EMU
  Kernel<<<grid, kThreads, smem, st>>>(args...);
#else
  // tests/emu: CPU model of the execution model
  MP_EMU_LAUNCH(grid, kThreads, Kernel(args...));
#endif
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

// query_fp32_kernel over bt.B images of src.n points
template <bool SURF>
int launch_query(const Fp32Params& prm, const HeadLayout& h, const DeviceLimits& dev, const MpPointSrc& src, const MpCalib& cal,
                 const MpOutDst& dst, const MpBatch& bt, const MpSurfaceSrc& surf, cudaStream_t st) {
  const int P = h.fit_tile(false, dev.max_smem);
  if (!P) {
    mp_set_error("head too wide for the fp32 kernel's shared-memory tiling");
    return MP_E_UNSUPPORTED;
  }
  const long long tiles = bt.B * ((src.n + P - 1) / P);
  const size_t smem = h.tile_bytes(P, false);
  if (P == 32) return launch<32, query_fp32_kernel<32, SURF>>(tiles, smem, dev, st, prm, src, cal, dst, bt, surf);
  if (P == 16) return launch<16, query_fp32_kernel<16, SURF>>(tiles, smem, dev, st, prm, src, cal, dst, bt, surf);
  return launch<8, query_fp32_kernel<8, SURF>>(tiles, smem, dev, st, prm, src, cal, dst, bt, surf);
}

// the VJP kernel's tile for this head on the current device, or an MP_E_* code (`what` names the kernel in the refusal)
int reverse_tile(const mp_mlp* mlp, const char* what) {
  DeviceLimits dev;
  const int rc = device_limits(dev);
  if (rc != MP_OK) return rc;
  const int P = head_layout(mlp).fit_tile(true, dev.max_smem);
  if (!P) {
    mp_set_error("head too wide for the %s's shared-memory tiling", what);
    return MP_E_UNSUPPORTED;
  }
  return P;
}

}  // namespace

int mp_launch_query_fp32(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal,
                         const MpOutDst& dst, cudaStream_t st, int guard, const MpBatch* bt) {
  if (src.n <= 0) return MP_OK;
  Fp32Params prm;
  HeadLayout h;
  DeviceLimits dev;
  const int rc = fill_params(mlp, feat, guard, prm, h, dev);
  if (rc != MP_OK) return rc;
  if (bt && bt->B > 1 && (src.kind != MP_SRC_ROWS || dst.scatter_vol || dst.n_peers > 0 || !dst.out)) {
    mp_set_error("batched launches take point rows and write [R,N] outputs");
    return MP_E_UNSUPPORTED;
  }
  return launch_query<false>(prm, h, dev, src, cal, dst, bt ? *bt : MpBatch(), MpSurfaceSrc(), st);
}

int mp_launch_surface_fp32(const mp_mlp* mlp, const mp_feat* feat, const MpSurfaceSrc& surf, long long n, const MpCalib& cal,
                           cudaStream_t st, int guard, const MpBatch* bt) {
  if (n <= 0) return MP_OK;
  if (mlp->cout[mlp->n_layers - 1] != 3) {
    mp_set_error("surface colourisation needs a head with 3 outputs (got %d)", mlp->cout[mlp->n_layers - 1]);
    return MP_E_INVALID;
  }
  if (bt && bt->B != 1) {
    mp_set_error("the surface render takes one map");
    return MP_E_UNSUPPORTED;
  }
  Fp32Params prm;
  HeadLayout h;
  DeviceLimits dev;
  const int rc = fill_params(mlp, feat, guard, prm, h, dev);
  if (rc != MP_OK) return rc;
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_ROWS;
  src.n = n;
  MpOutDst dst;
  dst.out = nullptr; dst.ld = 0; dst.scatter_vol = nullptr;
  // (one map, its camera in device memory when bt->calibs is set)
  return launch_query<true>(prm, h, dev, src, cal, dst, bt ? *bt : MpBatch(), surf, st);
}

int mp_launch_query_grad(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal,
                         const float* grad_out, long long ld_grad, float* out, long long ld_out, float* dpoints,
                         long long ld_dp, cudaStream_t st, int guard, const MpBatch* bt) {
  if (src.n <= 0) return MP_OK;
  if (src.kind != MP_SRC_ROWS || (bt && bt->B != 1)) {
    mp_set_error("the gradient kernel takes point rows of one map");
    return MP_E_UNSUPPORTED;
  }
  if (out) {                                      // the value: query_fp32_kernel's own, bit for bit
    MpOutDst dst;
    dst.out = out; dst.ld = ld_out; dst.scatter_vol = nullptr;
    const int rq = mp_launch_query_fp32(mlp, feat, src, cal, dst, st, guard, bt);
    if (rq != MP_OK) return rq;
  }
  const int P = reverse_tile(mlp, "gradient kernel");
  if (P < 0) return P;
  MpVjpParams vp;                                 // d points of every tile of the map; no rows, no feature gradient
  memset(&vp, 0, sizeof(vp));
  vp.grad_out = grad_out; vp.ld_grad = ld_grad;
  vp.dp = dpoints; vp.ld_dp = ld_dp;
  vp.tile1 = (src.n + P - 1) / P;
  return mp_launch_query_vjp_tiles(mlp, feat, src, cal, bt ? *bt : MpBatch(), vp, st, guard);
}

int mp_query_vjp_tile(const mp_mlp* mlp) { return reverse_tile(mlp, "VJP kernel"); }

int mp_launch_query_vjp_tiles(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal,
                              const MpBatch& bt, const MpVjpParams& outs, cudaStream_t st, int guard) {
  Fp32Params prm;
  HeadLayout h;
  DeviceLimits dev;
  const int rc = fill_params(mlp, feat, guard, prm, h, dev);
  if (rc != MP_OK) return rc;
  const int P = mp_query_vjp_tile(mlp);
  if (P < 0) return P;
  MpVjpParams vp = outs;
  for (int l = 0; l < mlp->n_layers; ++l) {
    vp.w[l] = mlp->w[l];
    vp.mask_off[l] = h.mask_off[l] * P;           // (in words of a P-point tile)
  }
  vp.mask_words = h.mask_words;
  const long long tiles = vp.tile1 - vp.tile0;
  const size_t smem = h.tile_bytes(P, true);
  if (P == 32) return launch<32, query_vjp_kernel<32>>(tiles, smem, dev, st, prm, vp, src, cal, bt);
  if (P == 16) return launch<16, query_vjp_kernel<16>>(tiles, smem, dev, st, prm, vp, src, cal, bt);
  return launch<8, query_vjp_kernel<8>>(tiles, smem, dev, st, prm, vp, src, cal, bt);
}
