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
// grid_sample backward, and its roundings depend on the order in which the points' taps land -- unless it is requested
// ordered (MP_VJP_DETERMINISTIC, below): then it is the same bits too, for one chunk size.
#include "mp_common.cuh"
#include "mp_scan.cuh"

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

// ---- the ordered feature gradient (MP_VJP_DETERMINISTIC) ------------------------------------------------------------------
// Per chunk, query_vjp_kernel records column j (one point) as dX[:C], its four tap weights and its cell key: b * H * W plus the
// texel of its nw tap (always on the map for an in-image point), or B * H * W for a point that contributes nothing.  Then:
//  1. A stable LSD radix sort of the chunk's columns by key, 8 bits per pass: radix_count_kernel counts the digits of each
//     block of 2048 columns (shared-memory integer atomics, which only count), the ordered scan of mp_scan.cuh turns the
//     digit-major [256][blocks] counts into offsets, and radix_scatter_kernel places each block's columns in column order
//     (ranks from warp ballots).  So within a cell the columns stay in ascending order, whatever the keys.
//  2. dfeat_gather_kernel: the thread of texel (b, y, x) and channel c owns that element of the [B][H][W][C] buffer.  It
//     sums, over the cells (y-1, x-1), (y-1, x), (y, x-1), (y, x) in that order -- whose points have the texel as their se,
//     sw, ne and nw tap -- and within a cell over its columns j in ascending order, with w the weight of that tap:
//         if (w != 0) s = fmaf(w, dX_j[c], s)            (s = +0 at the start; a tap of weight 0 is off the map)
//     and adds s to the buffer when some term was taken.  Chunks follow one another on the stream in point order.
// The feature gradient is then a function of the chunk size alone: not of the SM count, the schedule or the other requests.
constexpr int kRadixBits = 8;
constexpr int kRadixBins = 1 << kRadixBits;
constexpr int kRadixThreads = 256;
constexpr int kRadixItems = 8;
constexpr int kRadixBlock = kRadixThreads * kRadixItems;   // columns per CTA
static_assert(kRadixBins == kRadixThreads, "thread t owns digit t");

// counts[d * nb + block] = the columns of the block whose digit (key >> shift) & 255 is d
__global__ void __launch_bounds__(kRadixThreads) radix_count_kernel(const unsigned* __restrict__ keys, int n, int shift,
                                                                    unsigned* __restrict__ counts, int nb) {
  __shared__ unsigned hist[kRadixBins];
  hist[threadIdx.x] = 0u;
  __syncthreads();
  for (int r = 0; r < kRadixItems; ++r) {
    const int i = (int)blockIdx.x * kRadixBlock + r * kRadixThreads + (int)threadIdx.x;
    if (i < n) atomicAdd(&hist[(keys[i] >> shift) & (kRadixBins - 1)], 1u);
  }
  __syncthreads();
  counts[threadIdx.x * nb + blockIdx.x] = hist[threadIdx.x];
}

// the ordered scan over the digit-major counts
struct DigitCounts {
  static constexpr bool kVec8 = false;
  const unsigned* counts;
  __device__ unsigned long long operator()(long long i) const { return counts[i]; }
};
struct DigitOffsets {
  unsigned* offsets;
  __device__ void operator()(long long i, unsigned long long, unsigned long long prefix) const { offsets[i] = (unsigned)prefix; }
};

// One pass: the block's columns, 256 at a time in column order, go to offsets[d * nb + block] plus their rank among the
// block's earlier columns of digit d.  vals null: the values are the column indices.
__global__ void __launch_bounds__(kRadixThreads) radix_scatter_kernel(const unsigned* __restrict__ keys,
                                                                      const unsigned* __restrict__ vals, int n, int shift,
                                                                      const unsigned* __restrict__ offsets, int nb,
                                                                      unsigned* __restrict__ keys_out,
                                                                      unsigned* __restrict__ vals_out) {
  constexpr int kWarps = kRadixThreads / 32;
  __shared__ unsigned base[kRadixBins];              // digit t: where the block's next column of that digit goes
  __shared__ unsigned wcount[kWarps][kRadixBins];    // per warp: its columns of each digit, then where they start
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  base[tid] = offsets[tid * nb + blockIdx.x];
  for (int r = 0; r < kRadixItems; ++r) {
#pragma unroll
    for (int w = 0; w < kWarps; ++w) wcount[w][tid] = 0u;
    __syncthreads();
    const int i = (int)blockIdx.x * kRadixBlock + r * kRadixThreads + tid;
    const bool valid = i < n;
    const unsigned key = valid ? keys[i] : 0u;
    const unsigned d = (key >> shift) & (kRadixBins - 1);
    // the lanes holding the same digit, then this lane's rank among them
    unsigned peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
    for (int bit = 0; bit < kRadixBits; ++bit) {
      const unsigned set = __ballot_sync(0xffffffffu, (d >> bit) & 1u);
      peers &= ((d >> bit) & 1u) ? set : ~set;
    }
    const unsigned rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) wcount[warp][d] = __popc(peers);
    __syncthreads();
    unsigned run = base[tid];
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const unsigned c = wcount[w][tid];
      wcount[w][tid] = run;
      run += c;
    }
    base[tid] = run;
    __syncthreads();
    if (valid) {
      const unsigned dst = wcount[warp][d] + rank;
      keys_out[dst] = key;
      vals_out[dst] = vals ? vals[i] : (unsigned)i;
    }
    __syncthreads();
  }
}

struct GatherParams {
  const float* dx;             // [cols][C]
  const float* wgt;            // [cols][4]: nw, ne, sw, se
  const unsigned* keys;        // the sorted keys
  const unsigned* cols;        // the columns in that order
  int n;                       // columns of the chunk
  float* nhwc;                 // [B][H][W][C]
  int C, H, W;
  long long texels;            // B * H * W
};

// the first of the n sorted keys that is >= k
__device__ __forceinline__ int lower_bound_key(const unsigned* keys, int n, unsigned k) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < k) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// one warp per texel, lanes over channels (the order at the top of this section)
__global__ void __launch_bounds__(256) dfeat_gather_kernel(GatherParams gp) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long t = (long long)blockIdx.x * 8 + warp;
  if (t >= gp.texels) return;
  const long long r = t % ((long long)gp.H * gp.W);
  const bool up = r >= gp.W, left = r % gp.W != 0;
  int lo[4], hi[4];
  bool any = false;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const bool ok = a == 0 ? up && left : (a == 1 ? up : (a == 2 ? left : true));
    const long long cell = t - (a < 2 ? gp.W : 0) - (a % 2 == 0 ? 1 : 0);
    lo[a] = hi[a] = 0;
    if (ok) {
      lo[a] = lower_bound_key(gp.keys, gp.n, (unsigned)cell);
      hi[a] = lower_bound_key(gp.keys, gp.n, (unsigned)cell + 1u);
    }
    any |= lo[a] < hi[a];
  }
  if (!any) return;
  float* out = gp.nhwc + t * gp.C;
  for (int c = lane; c < gp.C; c += 32) {
    float s = 0.f;
    bool took = false;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int tap = 3 - a;                         // se, sw, ne, nw
      for (int j = lo[a]; j < hi[a]; ++j) {
        const unsigned col = __ldg(gp.cols + j);
        const float w = __ldg(gp.wgt + (size_t)col * 4 + tap);
        if (w == 0.f) continue;
        s = fmaf(w, __ldg(gp.dx + (size_t)col * gp.C + c), s);
        took = true;
      }
    }
    if (took) out[c] += s;
  }
}

size_t round256(size_t b) { return (b + 255) / 256 * 256; }

// The ordered path's part of the scratch for a chunk of `cols` columns (byte offsets from its start): the scan's words first
// (total[2], whose ticket total[1] must be zero before the first scan, then the chunk sums), the recorded columns, the two
// key / column buffers of the sort and the digit counts and offsets.
struct OrderedLayout {
  size_t scan, dx, wgt, key[2], col[2], counts, offsets, bytes;
  int blocks;                  // radix blocks of the chunk
};

OrderedLayout ordered_layout(long long cols, int C) {
  OrderedLayout o;
  size_t at = 0;
  auto take = [&at](size_t b) {
    const size_t p = at;
    at += round256(b);
    return p;
  };
  o.blocks = (int)((cols + kRadixBlock - 1) / kRadixBlock);
  const long long digits = (long long)kRadixBins * o.blocks;
  o.scan = take(8 * (size_t)(2 + mpscan::num_blocks(digits)));
  o.dx = take((size_t)cols * C * sizeof(float));
  o.wgt = take((size_t)cols * 4 * sizeof(float));
  for (int k = 0; k < 2; ++k) o.key[k] = take((size_t)cols * sizeof(unsigned));
  for (int k = 0; k < 2; ++k) o.col[k] = take((size_t)cols * sizeof(unsigned));
  o.counts = take((size_t)digits * sizeof(unsigned));
  o.offsets = take((size_t)digits * sizeof(unsigned));
  o.bytes = at;
  return o;
}

// radix passes for keys up to max_key; the sorted keys and columns end in buffer (passes & 1)
int radix_passes(unsigned long long max_key) {
  int p = 1;
  while (p < 4 && (max_key >> (kRadixBits * p)) != 0) ++p;
  return p;
}

// the sort of one chunk's n columns (keys in buffer 0)
int sort_columns(char* area, const OrderedLayout& o, int n, int passes, cudaStream_t st) {
  unsigned* keys[2] = {reinterpret_cast<unsigned*>(area + o.key[0]), reinterpret_cast<unsigned*>(area + o.key[1])};
  unsigned* cols[2] = {reinterpret_cast<unsigned*>(area + o.col[0]), reinterpret_cast<unsigned*>(area + o.col[1])};
  unsigned* counts = reinterpret_cast<unsigned*>(area + o.counts);
  unsigned* offsets = reinterpret_cast<unsigned*>(area + o.offsets);
  unsigned long long* total = reinterpret_cast<unsigned long long*>(area + o.scan);
  const int nb = (n + kRadixBlock - 1) / kRadixBlock;
  const long long digits = (long long)kRadixBins * nb;
  const DigitCounts f{counts};
  const DigitOffsets em{offsets};
  for (int p = 0; p < passes; ++p) {
    const int in = p & 1, out = in ^ 1, shift = kRadixBits * p;
    const unsigned* vals = p == 0 ? nullptr : cols[in];
#ifndef MP_CUDA_EMU
    radix_count_kernel<<<nb, kRadixThreads, 0, st>>>(keys[in], n, shift, counts, nb);
    MP_CUDA(mpscan::scan_emit(f, em, digits, total + 2, total, st));
    radix_scatter_kernel<<<nb, kRadixThreads, 0, st>>>(keys[in], vals, n, shift, offsets, nb, keys[out], cols[out]);
#else
    const int sb = mpscan::num_blocks(digits);
    MP_EMU_LAUNCH(nb, kRadixThreads, radix_count_kernel(keys[in], n, shift, counts, nb));
    MP_EMU_LAUNCH(sb, mpscan::kThreads, (mpscan::block_sums_kernel<DigitCounts, mpscan::NoPost>(f, digits, total + 2, sb, total,
                                                                                              mpscan::NoPost())));
    MP_EMU_LAUNCH(sb, mpscan::kThreads, (mpscan::emit_kernel<DigitCounts, DigitOffsets>(f, em, digits, total + 2)));
    MP_EMU_LAUNCH(nb, kRadixThreads, radix_scatter_kernel(keys[in], vals, n, shift, offsets, nb, keys[out], cols[out]));
#endif
    MP_CUDA(cudaGetLastError());
  }
  return MP_OK;
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

// the scratch of one chunk of `chunk` tiles after the NHWC buffer: the saved rows, then the ordered path's part
size_t chunk_bytes(const RowLayout& rl, int P, int C, bool want_w, bool ordered, long long chunk) {
  const size_t rows = want_w ? (size_t)rl.total * P * sizeof(float) * (size_t)chunk : 0;
  return ordered ? round256(rows) + ordered_layout(chunk * P, C).bytes : rows;
}

// the chunk of a request, in tiles: chunk_points rounded up to tiles (<= 0: every tile), at most every tile
long long chunk_tiles(long long chunk_points, int P, long long tiles) {
  const long long chunk = chunk_points > 0 ? (chunk_points + P - 1) / P : tiles;
  return chunk < tiles ? chunk : tiles;
}

}  // namespace

long long mp_vjp_scratch_bytes(const mp_mlp* mlp, const mp_feat* feat, int B, long long n, long long chunk_points, bool dfeat,
                               bool dweights, int flags) {
  const int P = mp_query_vjp_tile(mlp);
  if (P < 0) return P;
  const bool ordered = dfeat && (flags & MP_VJP_DETERMINISTIC);
  size_t bytes = dfeat ? round256((size_t)B * feat->H * feat->W * feat->C * sizeof(float)) : 0;
  if (dweights || ordered) {
    const long long tiles = (long long)B * ((n + P - 1) / P);
    bytes += chunk_bytes(row_layout(mlp), P, feat->C, dweights, ordered, chunk_tiles(chunk_points, P, tiles));
  }
  return (long long)bytes;
}

int mp_launch_query_vjp(const mp_mlp* mlp, const mp_feat* feat, const MpPointSrc& src, const MpCalib& cal, const MpBatch& bt,
                        const float* grad_out, float* dfeat_nchw, float* dpoints, float* const* dweights, float* const* dbiases,
                        void* scratch, long long scratch_bytes, cudaStream_t st, int flags) {
  const int L = mlp->n_layers;
  bool want_w = false;
  for (int l = 0; l < L; ++l) want_w |= (dweights && dweights[l]) || (dbiases && dbiases[l]);
  if (!want_w && !dfeat_nchw && !dpoints) return MP_OK;
  MP_REQUIRE((flags & ~MP_VJP_DETERMINISTIC) == 0, "unknown VJP flags %d", flags);
  const int P = mp_query_vjp_tile(mlp);
  if (P < 0) return P;
  const long long n = src.n;
  const long long tiles = (long long)bt.B * ((n + P - 1) / P);
  const bool ordered = dfeat_nchw && (flags & MP_VJP_DETERMINISTIC) && tiles > 0;
  const long long HW = (long long)feat->H * feat->W;
  const size_t dfeat_elems = dfeat_nchw ? (size_t)bt.B * HW * feat->C : 0;
  const size_t dfeat_bytes = round256(dfeat_elems * sizeof(float));
  const RowLayout rl = row_layout(mlp);
  MP_REQUIRE(scratch || (!dfeat_nchw && !want_w), "the feature and weight gradients need a scratch buffer");
  MP_REQUIRE(scratch_bytes >= (long long)dfeat_bytes, "scratch of %lld bytes is smaller than the feature gradient's %lld",
             scratch_bytes, (long long)dfeat_bytes);
  long long chunk = tiles;
  if (ordered) {
    // the largest chunk whose scratch fits: the chunk mp_vjp_scratch_bytes sized for the same requests
    MP_REQUIRE((unsigned long long)bt.B * HW < 0xFFFFFFFFull, "%d maps of %lld texels: too many cells for the ordered feature gradient",
               bt.B, HW);
    const long long room = scratch_bytes - (long long)dfeat_bytes;
    MP_REQUIRE((long long)chunk_bytes(rl, P, feat->C, want_w, true, 1) <= room,
               "scratch of %lld bytes holds no chunk (see mp_query_points_vjp_scratch_bytes_ex)", scratch_bytes);
    long long lo = 1, hi = tiles;
    while (lo < hi) {
      const long long mid = lo + (hi - lo + 1) / 2;
      if ((long long)chunk_bytes(rl, P, feat->C, want_w, true, mid) <= room) lo = mid;
      else hi = mid - 1;
    }
    chunk = lo;
    MP_REQUIRE(chunk * P < (1ll << 31), "a chunk of %lld points is too large for the ordered feature gradient", chunk * P);
  } else if (want_w) {
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
  char* area = nullptr;                             // the ordered path's part of the scratch
  OrderedLayout ol;
  memset(&ol, 0, sizeof(ol));
  const int passes = radix_passes((unsigned long long)bt.B * HW);
  if (ordered) {
    area = static_cast<char*>(scratch) + dfeat_bytes + round256(want_w ? (size_t)rl.total * P * sizeof(float) * chunk : 0);
    ol = ordered_layout(chunk * P, feat->C);
    vp.dx_rows = reinterpret_cast<float*>(area + ol.dx);
    vp.dx_wgt = reinterpret_cast<float*>(area + ol.wgt);
    vp.dx_key = reinterpret_cast<unsigned*>(area + ol.key[0]);
    MP_CUDA(cudaMemsetAsync(area + ol.scan, 0, 16, st));   // the scan's ticket (the scans leave it at zero)
  }

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
    if (ordered) {
      const int cols = (int)((vp.tile1 - vp.tile0) * P);
      const int rs = sort_columns(area, ol, cols, passes, st);
      if (rs != MP_OK) return rs;
      GatherParams gp;
      gp.dx = vp.dx_rows; gp.wgt = vp.dx_wgt;
      gp.keys = reinterpret_cast<const unsigned*>(area + ol.key[passes & 1]);
      gp.cols = reinterpret_cast<const unsigned*>(area + ol.col[passes & 1]);
      gp.n = cols;
      gp.nhwc = nhwc;
      gp.C = feat->C; gp.H = feat->H; gp.W = feat->W;
      gp.texels = (long long)bt.B * HW;
      const long long grid = (gp.texels + 7) / 8;
#ifndef MP_CUDA_EMU
      dfeat_gather_kernel<<<(unsigned)grid, 256, 0, st>>>(gp);
#else
      MP_EMU_LAUNCH(grid, 256, dfeat_gather_kernel(gp));
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
