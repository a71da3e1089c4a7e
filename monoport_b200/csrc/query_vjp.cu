// F1'''' (host side and the contraction): the vector-Jacobian product of the exact query for training -- d features, d points
// and the head's d weights / d biases of sum(grad_out * query(...)), the backward of MonoPortNet.py:63-91 in train mode.
//
// Per chunk of points, query_vjp_kernel (query_fp32.cu) writes the rows the weight gradient needs to a scratch buffer, and
// wgrad_kernel below contracts them over the chunk's points:
//   dW_l[co][k] += sum_n δ_l[co][n] * in_l[k][n],   db_l[co] += sum_n δ_l[co][n]
// with in_l = [h_{l-1} ; X] (torch.cat([y, feature], 1), SurfaceClassifier.py:55) and in_0 = X.  Scratch rows, each one
// column per point of the chunk (column (t - tile0) * P + p):
//   rows [0, c0)                   X: the sampled features and the depth feature
//   act_row[l] .. + cout_l         h_l, the post-activation of hidden layer l
//   delta_row[l] .. + cout_l       δ_l = d sum / d (pre-activation of layer l); for the last layer, g
// Determinism: every element of dW / db is owned by one thread of wgrad_kernel, which sums the chunk's points in column
// order; chunks follow one another on the stream in point order.  For one scratch size (one chunk size) the weight, bias and
// point gradients are the same bits from run to run.  The feature gradient is accumulated with atomicAdd, like torch's
// grid_sample backward, and its roundings depend on the order in which the points' taps land.
#include "mp_common.cuh"

namespace {

constexpr int kGemmTile = 64;      // dW tile: 64 output channels x 64 input channels (the bias as input channel cin)
constexpr int kGemmCols = 32;      // points per shared-memory stage

struct WgradParams {
  int n_layers;
  int cin[MP_MAX_LAYERS], cout[MP_MAX_LAYERS], hid[MP_MAX_LAYERS];
  int in_row[MP_MAX_LAYERS];       // row of h_{l-1} (l >= 1)
  int delta_row[MP_MAX_LAYERS];
  int k_tiles[MP_MAX_LAYERS];      // 64-wide tiles over cin + 1 (0: the layer is not wanted)
  int first_tile[MP_MAX_LAYERS + 1];
  float* dw[MP_MAX_LAYERS];        // [cout][cin] or null
  float* db[MP_MAX_LAYERS];        // [cout] or null
  const float* rows;
  long long ld;
  int cols;                        // points of this chunk
};

// One CTA per 64 x 64 tile of one layer's [dW | db]; thread (ty, tx) owns output channels co0 + ty + 16 i and input channels
// k0 + tx + 16 j (i, j < 4), accumulated over the chunk's points in order.
__global__ void __launch_bounds__(256) wgrad_kernel(WgradParams wp) {
  __shared__ float sD[kGemmCols][kGemmTile + 1];
  __shared__ float sI[kGemmCols][kGemmTile + 1];
  int l = 0;
  while (l + 1 < wp.n_layers && (int)blockIdx.x >= wp.first_tile[l + 1]) ++l;
  const int t = (int)blockIdx.x - wp.first_tile[l];
  const int co0 = (t / wp.k_tiles[l]) * kGemmTile, k0 = (t % wp.k_tiles[l]) * kGemmTile;
  const int cin = wp.cin[l], cout = wp.cout[l], hid = l == 0 ? 0 : wp.hid[l];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int c0 = 0; c0 < wp.cols; c0 += kGemmCols) {
    // row r of both tiles, 32 consecutive points: coalesced loads, conflict-free transposed stores
    for (int e = tid; e < kGemmTile * kGemmCols; e += 256) {
      const int r = e / kGemmCols, c = e % kGemmCols, col = c0 + c;
      float d = 0.f, x = 0.f;
      if (col < wp.cols) {
        const int co = co0 + r;
        if (co < cout) d = __ldg(wp.rows + (long long)(wp.delta_row[l] + co) * wp.ld + col);
        const int k = k0 + r;
        if (k < cin) {
          const int row = k < hid ? wp.in_row[l] + k : k - hid;
          x = __ldg(wp.rows + (long long)row * wp.ld + col);
        } else if (k == cin) {
          x = 1.f;                                     // the bias column
        }
      }
      sD[c][r] = d;
      sI[c][r] = x;
    }
    __syncthreads();
#pragma unroll 4
    for (int c = 0; c < kGemmCols; ++c) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = sD[c][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = sI[c][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + ty + 16 * i;
    if (co >= cout) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tx + 16 * j;
      if (k < cin) {
        if (wp.dw[l]) wp.dw[l][(long long)co * cin + k] += acc[i][j];
      } else if (k == cin && wp.db[l]) {
        wp.db[l][co] += acc[i][j];
      }
    }
  }
}

// [B][HW][C] -> [B][C][HW], 32 x 32 tiles through shared memory; block = 256 threads as 8 rows of 32
__global__ void __launch_bounds__(256) nhwc_to_nchw_kernel(const float* in, float* out, int C, long long HW, int p_tiles,
                                                           int c_tiles) {
  __shared__ float t[32][33];
  const int per_image = p_tiles * c_tiles;
  const int b = (int)blockIdx.x / per_image, r = (int)blockIdx.x % per_image;
  const long long p0 = (long long)(r / c_tiles) * 32;
  const int c0 = (r % c_tiles) * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  in += (size_t)b * HW * C;
  out += (size_t)b * HW * C;
  for (int j = ty; j < 32; j += 8) {
    const long long p = p0 + j;
    const int c = c0 + tx;
    if (p < HW && c < C) t[j][tx] = in[p * C + c];
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    const long long p = p0 + tx;
    if (p < HW && c < C) out[(long long)c * HW + p] = t[tx][j];
  }
}

// the scratch rows of a head: act_row / delta_row (see the top of this file) and their total
struct RowLayout {
  int act_row[MP_MAX_LAYERS];
  int delta_row[MP_MAX_LAYERS];
  int total;
};

RowLayout row_layout(const mp_mlp* mlp) {
  RowLayout r;
  memset(&r, 0, sizeof(r));
  int row = mlp->channels[0];
  for (int l = 0; l + 1 < mlp->n_layers; ++l) { r.act_row[l] = row; row += mlp->cout[l]; }
  for (int l = 0; l < mlp->n_layers; ++l) { r.delta_row[l] = row; row += mlp->cout[l]; }
  r.total = row;
  return r;
}

size_t round256(size_t b) { return (b + 255) / 256 * 256; }

}  // namespace

long long mp_vjp_scratch_bytes(const mp_mlp* mlp, const mp_feat* feat, int B, long long n, long long chunk_points, bool dfeat,
                               bool dweights) {
  const int P = mp_query_vjp_tile(mlp);
  if (P < 0) return P;
  size_t bytes = dfeat ? round256((size_t)B * feat->H * feat->W * feat->C * sizeof(float)) : 0;
  if (dweights) {
    const long long tiles = (long long)B * ((n + P - 1) / P);
    long long chunk = chunk_points > 0 ? (chunk_points + P - 1) / P : tiles;
    chunk = chunk < tiles ? chunk : tiles;
    bytes += (size_t)row_layout(mlp).total * P * sizeof(float) * (size_t)chunk;
  }
  return (long long)bytes;
}

int mp_launch_query_vjp(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal, const MpBatch& bt,
                        const float* grad_out, float* dfeat_nchw, float* dpoints, float* const* dweights, float* const* dbiases,
                        void* scratch, long long scratch_bytes, cudaStream_t st) {
  const int L = mlp->n_layers;
  bool want_w = false;
  for (int l = 0; l < L; ++l) want_w |= (dweights && dweights[l]) || (dbiases && dbiases[l]);
  if (!want_w && !dfeat_nchw && !dpoints) return MP_OK;
  const int P = mp_query_vjp_tile(mlp);
  if (P < 0) return P;
  const long long n = src.n;
  const long long tiles = (long long)bt.B * ((n + P - 1) / P);
  const long long HW = (long long)feat->H * feat->W;
  const size_t dfeat_elems = dfeat_nchw ? (size_t)bt.B * HW * feat->C : 0;
  const size_t dfeat_bytes = round256(dfeat_elems * sizeof(float));
  const RowLayout rl = row_layout(mlp);
  MP_REQUIRE(scratch || (!dfeat_nchw && !want_w), "the feature and weight gradients need a scratch buffer");
  MP_REQUIRE(scratch_bytes >= (long long)dfeat_bytes, "scratch of %lld bytes is smaller than the feature gradient's %lld",
             scratch_bytes, (long long)dfeat_bytes);
  long long chunk = tiles;
  if (want_w) {
    chunk = (scratch_bytes - (long long)dfeat_bytes) / ((long long)rl.total * P * (long long)sizeof(float));
    MP_REQUIRE(chunk >= 1, "scratch of %lld bytes holds no chunk (%lld bytes per %d points; see mp_query_points_vjp_scratch_bytes)",
               scratch_bytes, (long long)rl.total * P * (long long)sizeof(float), P);
    chunk = chunk < tiles ? chunk : tiles;
  }

  MpVjpParams vp;
  memset(&vp, 0, sizeof(vp));
  const int res = mlp->cout[L - 1];
  vp.grad_out = grad_out; vp.ld_grad = n; vp.gout_stride = (long long)res * n;
  vp.dp = dpoints; vp.ld_dp = n; vp.dp_stride = 3 * n;
  float* nhwc = dfeat_nchw ? static_cast<float*>(scratch) : nullptr;
  vp.dfeat = nhwc;
  vp.rows = want_w ? reinterpret_cast<float*>(static_cast<char*>(scratch) + dfeat_bytes) : nullptr;
  vp.ld_rows = chunk * P;
  memcpy(vp.act_row, rl.act_row, sizeof(vp.act_row));
  memcpy(vp.delta_row, rl.delta_row, sizeof(vp.delta_row));

  // outputs: the feature gradient accumulates into the zeroed NHWC buffer, the weight gradients chunk by chunk
  if (nhwc) MP_CUDA(cudaMemsetAsync(nhwc, 0, dfeat_elems * sizeof(float), st));
  WgradParams wp;
  memset(&wp, 0, sizeof(wp));
  int grid_w = 0;
  if (want_w) {
    wp.n_layers = L;
    for (int l = 0; l < L; ++l) {
      wp.cin[l] = mlp->cin[l]; wp.cout[l] = mlp->cout[l];
      wp.hid[l] = l == 0 ? 0 : mlp->channels[l];
      wp.in_row[l] = l == 0 ? 0 : rl.act_row[l - 1];
      wp.delta_row[l] = rl.delta_row[l];
      wp.dw[l] = dweights ? dweights[l] : nullptr;
      wp.db[l] = dbiases ? dbiases[l] : nullptr;
      const bool on = wp.dw[l] || wp.db[l];
      wp.k_tiles[l] = on ? (mlp->cin[l] + 1 + kGemmTile - 1) / kGemmTile : 0;
      wp.first_tile[l] = grid_w;
      grid_w += on ? wp.k_tiles[l] * ((mlp->cout[l] + kGemmTile - 1) / kGemmTile) : 0;
      if (wp.dw[l]) MP_CUDA(cudaMemsetAsync(wp.dw[l], 0, (size_t)mlp->cout[l] * mlp->cin[l] * sizeof(float), st));
      if (wp.db[l]) MP_CUDA(cudaMemsetAsync(wp.db[l], 0, (size_t)mlp->cout[l] * sizeof(float), st));
    }
    for (int l = L; l <= MP_MAX_LAYERS; ++l) wp.first_tile[l] = grid_w;
    wp.rows = vp.rows;
    wp.ld = vp.ld_rows;
  }

  for (long long t0 = 0; t0 < tiles; t0 += chunk) {
    vp.tile0 = t0;
    vp.tile1 = t0 + chunk < tiles ? t0 + chunk : tiles;
    const int rc = mp_launch_query_vjp_tiles(mlp, feat, src, cal, bt, vp, st);
    if (rc != MP_OK) return rc;
    if (want_w && grid_w > 0) {
      wp.cols = (int)((vp.tile1 - vp.tile0) * P);
#ifndef MP_CUDA_EMU
      wgrad_kernel<<<grid_w, 256, 0, st>>>(wp);
#else
      MP_EMU_LAUNCH(grid_w, 256, wgrad_kernel(wp));
#endif
      MP_CUDA(cudaGetLastError());
    }
  }
  if (dfeat_nchw) {
    const int p_tiles = (int)((HW + 31) / 32), c_tiles = (feat->C + 31) / 32;
    const int grid = bt.B * p_tiles * c_tiles;
#ifndef MP_CUDA_EMU
    nhwc_to_nchw_kernel<<<grid, 256, 0, st>>>(nhwc, dfeat_nchw, feat->C, HW, p_tiles, c_tiles);
#else
    MP_EMU_LAUNCH(grid, 256, nhwc_to_nchw_kernel(nhwc, dfeat_nchw, feat->C, HW, p_tiles, c_tiles));
#endif
    MP_CUDA(cudaGetLastError());
  }
  return MP_OK;
}
