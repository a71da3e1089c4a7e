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

template <int P>
struct Fp32Smem {
  // sizes in floats
  static __host__ __device__ size_t bytes(int c0, int h_ping, int h_pong) {
    return (size_t)(c0 + h_ping + h_pong) * P * sizeof(float) + (size_t)P * 8 * sizeof(float);
  }
};

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
template <int P, int NCO>
__device__ void dense_layer(const float* __restrict__ wt, const float* __restrict__ bias, int cin_hidden, int cin_skip,
                            int cout, const float* sHidden, const float* sSkip, float* sOut) {
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

// BATCH: bt.B images of src.n points (MP_SRC_ROWS); tile t is tile t % n_tiles of image t / n_tiles, which samples its own
// map and calibration and writes its own outputs; the range guard is decided per tile from that image's maximum.
template <int P, bool BATCH = false>
__global__ void __launch_bounds__(kThreads, 1)
query_fp32_kernel(Fp32Params prm, MpPointSrc src, MpCalib cal, MpOutDst dst, MpBatch bt) {
  MP_DYN_SMEM_ALIGNED(float, smem, 16);
  float* sX = smem;                                  // [c0][P]
  float* sA = sX + (size_t)prm.c0 * P;               // [h_ping][P]
  float* sB = sA + (size_t)prm.h_ping * P;           // [h_pong][P]
  float* sMeta = sB + (size_t)prm.h_pong * P;        // [8][P]: in_img, u, v, z_feat, (4 spare)
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  if constexpr (!BATCH) {
    if (mp_guard_skips(prm.amax, prm.amax_limit, prm.guard)) return;      // (uniform over the grid)
  }

  long long n = src.n;
  if (src.count_dev) {
    const long long c = *src.count_dev;
    n = c < n ? c : n;
  }
  long long win0, win1;
  mp_shard_window(src, n, win0, win1);
  n = win1;                                          // points >= n are padding; the first evaluated one is win0
  const long long n_tiles = (win1 - win0 + P - 1) / P;          // (per image)
  const long long all_tiles = BATCH ? n_tiles * bt.B : n_tiles;

  for (long long at = blockIdx.x; at < all_tiles; at += gridDim.x) {
    const int b = BATCH ? mp_tile_image(at, n_tiles) : 0;
    if (BATCH && mp_guard_skips(prm.amax + b, prm.amax_limit, prm.guard)) continue;      // (uniform over the CTA)
    const long long tile = BATCH ? at - (long long)b * n_tiles : at;
    const float* feat = BATCH ? prm.feat + (size_t)b * prm.H * prm.W * prm.C : prm.feat;
    float* out = BATCH ? dst.out + b * bt.out_stride : dst.out;
    const long long p0 = win0 + tile * P;
    // ---- 1. projection, mask, taps ------------------------------------------------------------
    __shared__ int sOff[4][P];
    __shared__ float sWgt[4][P];
    if (tid < P) {
      const long long i = p0 + tid;
      float u = 0.f, v = 0.f, w = 0.f;
      bool valid = i < n;
      if (valid) {
        float x, y, z;
        if constexpr (BATCH) {
          mp_load_image_point(src, bt, b, i, x, y, z);
          mp_project(mp_image_calib(cal, bt, b), x, y, z, u, v, w);
        } else {
          mp_load_point(src, i, x, y, z);
          mp_project(cal, x, y, z, u, v, w);
        }
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
    // ---- 2. bilinear gather: warp per point, lanes over channels (NHWC => contiguous) ---------
    for (int p = warp; p < P; p += kThreads / 32) {
      const float* f0 = feat + (size_t)sOff[0][p] * prm.C;
      const float* f1 = feat + (size_t)sOff[1][p] * prm.C;
      const float* f2 = feat + (size_t)sOff[2][p] * prm.C;
      const float* f3 = feat + (size_t)sOff[3][p] * prm.C;
      const float w0 = sWgt[0][p], w1 = sWgt[1][p], w2 = sWgt[2][p], w3 = sWgt[3][p];
      for (int c = lane; c < prm.C; c += 32) {
        // same accumulation order as grid_sample: nw, ne, sw, se
        float v = __ldg(f0 + c) * w0;
        v += __ldg(f1 + c) * w1;
        v += __ldg(f2 + c) * w2;
        v += __ldg(f3 + c) * w3;
        sX[(size_t)c * P + p] = v;
      }
    }
    __syncthreads();
    // ---- 3. hidden layers ---------------------------------------------------------------------
    const float* sIn = sX;
    float* sOut = sA;
    for (int l = 0; l < prm.n_layers - 1; ++l) {
      const int hid = prm.hid[l];
      const int skipw = prm.cin[l] - hid;
      if (l == 0) {
        dense_layer<P, 2>(prm.wt[l], prm.bias[l], 0, prm.cin[l], prm.cout[l], sX, sX, sOut);
      } else if (prm.cout[l] > kThreads) {
        dense_layer<P, 2>(prm.wt[l], prm.bias[l], hid, skipw, prm.cout[l], sIn, sX, sOut);
      } else {
        dense_layer<P, 1>(prm.wt[l], prm.bias[l], hid, skipw, prm.cout[l], sIn, sX, sOut);
      }
      __syncthreads();
      sIn = sOut;
      sOut = (sOut == sA) ? sB : sA;
    }
    // ---- 4. last layer: one warp per (point, out channel) dot product -------------------------
    {
      const int l = prm.n_layers - 1;
      const int res = prm.cout[l];
      const int hid = prm.n_layers == 1 ? 0 : prm.hid[l];
      const int cin = prm.cin[l];
      for (int job = warp; job < P * res; job += kThreads / 32) {
        const int p = job % P, r = job / P;
        const float* wrow = prm.w_last + (size_t)r * cin;
        float acc = 0.f;
        for (int k = lane; k < cin; k += 32) {
          const float a = (prm.n_layers == 1) ? sX[(size_t)k * P + p]
                          : (k < hid ? sIn[(size_t)k * P + p] : sX[(size_t)(k - hid) * P + p]);
          acc = fmaf(__ldg(wrow + k), a, acc);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) {
          const long long i = p0 + p;
          if (i < n) {
            float v = mp_last_op(acc + __ldg(prm.bias[l] + r), prm.last_op);
            v = sMeta[p] * v;                                                              // MonoPortNet.py:89
            if (out) out[(long long)r * dst.ld + i] = v;
            if (dst.scatter_vol && r == 0) dst.scatter_vol[__ldg(src.nodes + i)] = v;
            if (r == 0)
              for (int pp = 0; pp < dst.n_peers; ++pp) dst.peer[pp][dst.peer_off + i] = v;      // peer-memory stores (NVLink)
          }
        }
      }
    }
    __syncthreads();
  }
}

template <int P>
int launch(const Fp32Params& prm, const MpPointSrc& src, const MpCalib& cal, const MpOutDst& dst, cudaStream_t st,
           int sm_count, int max_smem, const MpBatch* bt) {
  const size_t smem = Fp32Smem<P>::bytes(prm.c0, prm.h_ping, prm.h_pong);
  // The opt-in is a property of the kernel, shared by every thread, and heads of different widths launch the same
  // instantiation with different sizes: it is always set to the same bound -- the device's maximum less the 2 KB the size
  // selection below keeps free for the kernel's static shared memory -- so no thread lowers it under another thread's
  // launch.  (Sticky per device: raising it again for every launch costs a driver call per query.)
  const int opt_in = max_smem - 2048;
  static thread_local bool opted[2][64] = {};
  const int variant = bt ? 1 : 0;
  int dev_ = 0;
  MP_CUDA(cudaGetDevice(&dev_));
  if (dev_ < 0 || dev_ >= 64 || !opted[variant][dev_]) {
    if (bt) MP_CUDA(cudaFuncSetAttribute(query_fp32_kernel<P, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, opt_in));
    else MP_CUDA(cudaFuncSetAttribute(query_fp32_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, opt_in));
    if (dev_ >= 0 && dev_ < 64) opted[variant][dev_] = true;
  }
  long long tiles = (bt ? bt->B : 1) * ((src.n + P - 1) / P);
  int grid = (int)(tiles < (long long)sm_count ? (tiles > 0 ? tiles : 1) : sm_count);
  MpBatch b1;
  memset(&b1, 0, sizeof(b1));
  const MpBatch& bb = bt ? *bt : b1;
#ifndef MP_CUDA_EMU
  if (bt) query_fp32_kernel<P, true><<<grid, kThreads, smem, st>>>(prm, src, cal, dst, bb);
  else query_fp32_kernel<P><<<grid, kThreads, smem, st>>>(prm, src, cal, dst, bb);
#else
  // tests/emu: CPU model of the execution model
  if (bt) MP_EMU_LAUNCH(grid, kThreads, (query_fp32_kernel<P, true>(prm, src, cal, dst, bb)));
  else MP_EMU_LAUNCH(grid, kThreads, query_fp32_kernel<P>(prm, src, cal, dst, bb));
#endif
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

}  // namespace

int mp_launch_query_fp32(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal,
                         const MpOutDst& dst, cudaStream_t st, int guard, const MpBatch* bt) {
  if (src.n <= 0) return MP_OK;
  Fp32Params prm;
  memset(&prm, 0, sizeof(prm));
  prm.n_layers = mlp->n_layers;
  prm.c0 = mlp->channels[0];
  prm.C = feat->C; prm.H = feat->H; prm.W = feat->W;
  if (prm.c0 != feat->C + 1) {
    mp_set_error("head expects %d input channels but the feature map has %d (+1 depth)", prm.c0, feat->C);
    return MP_E_INVALID;
  }
  int ping = 0, pong = 0;
  for (int l = 0; l < mlp->n_layers; ++l) {
    prm.cin[l] = mlp->cin[l];
    prm.cout[l] = mlp->cout[l];
    prm.hid[l] = (l == 0) ? 0 : mlp->channels[l];
    prm.wt[l] = mlp->wt[l];
    prm.bias[l] = mlp->bias[l];
    if (l < mlp->n_layers - 1) {
      if (l % 2 == 0) ping = ping > mlp->cout[l] ? ping : mlp->cout[l];
      else pong = pong > mlp->cout[l] ? pong : mlp->cout[l];
    }
    if (l > 0 && !mlp->skip) {
      mp_set_error("no_residual heads are not supported");
      return MP_E_UNSUPPORTED;
    }
  }
  prm.w_last = mlp->w[mlp->n_layers - 1];
  prm.last_op = mlp->last_op;
  prm.h_ping = ping; prm.h_pong = pong;
  prm.feat = feat->nhwc32;
  prm.amax = feat->amax; prm.amax_limit = mlp->tc_amax_limit; prm.guard = guard;
  int dev = 0, sms = 148, max_smem = 0;
  MP_CUDA(cudaGetDevice(&dev));
  {
    static thread_local int c_sms[64] = {}, c_smem[64] = {};
    if (dev >= 0 && dev < 64 && c_sms[dev]) { sms = c_sms[dev]; max_smem = c_smem[dev]; }
    else {
      MP_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
      MP_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
      if (dev >= 0 && dev < 64) { c_sms[dev] = sms; c_smem[dev] = max_smem; }
    }
  }
  if (bt && (src.kind != MP_SRC_ROWS || dst.scatter_vol || dst.n_peers > 0 || !dst.out)) {
    mp_set_error("batched launches take point rows and write [R,N] outputs");
    return MP_E_UNSUPPORTED;
  }
  if (Fp32Smem<32>::bytes(prm.c0, ping, pong) + 2048 <= (size_t)max_smem) return launch<32>(prm, src, cal, dst, st, sms, max_smem, bt);
  if (Fp32Smem<16>::bytes(prm.c0, ping, pong) + 2048 <= (size_t)max_smem) return launch<16>(prm, src, cal, dst, st, sms, max_smem, bt);
  if (Fp32Smem<8>::bytes(prm.c0, ping, pong) + 2048 <= (size_t)max_smem) return launch<8>(prm, src, cal, dst, st, sms, max_smem, bt);
  mp_set_error("head too wide for the fp32 kernel's shared-memory tiling");
  return MP_E_UNSUPPORTED;
}
