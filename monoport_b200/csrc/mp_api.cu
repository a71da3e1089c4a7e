// C-ABI entry points: error channel, handles (head weights, feature volume), query dispatch.
// See include/monoport_b200.h for the contract of every function and the reference interface it replaces.
#include "mp_common.cuh"
#include <mutex>
#include <stdlib.h>
#include <atomic>
#include <math.h>

static thread_local char g_err[512] = "";

void mp_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* mp_last_error(void) { return g_err; }

// cudaMallocAsync scratch: keep freed blocks in the pool (the default release threshold of 0 hands memory back to
// the driver at every synchronisation, which costs milliseconds per frame).
void mp_ensure_pool() {
  static thread_local int done_for = -1;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev == done_for) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    unsigned long long thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  done_for = dev;
}
extern "C" int mp_version(void) { return 100; }

extern "C" int mp_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  MP_CUDA(cudaGetDevice(&dev));
  if (sm_count) MP_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
  if (cc_major) MP_CUDA(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev));
  if (cc_minor) MP_CUDA(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
  return MP_OK;
}

// ---------------------------------------------------------------------------------------------
// head weights
// ---------------------------------------------------------------------------------------------
__global__ void transpose_w_kernel(const float* __restrict__ w, float* __restrict__ wt, int cout, int cin) {
  // w [cout][cin] -> wt [cin][cout]
  __shared__ float tile[32][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = by + j, c = bx + threadIdx.x;
    tile[j][threadIdx.x] = (r < cout && c < cin) ? w[(size_t)r * cin + c] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = bx + j, c = by + threadIdx.x;   // r: cin index, c: cout index
    if (r < cin && c < cout) wt[(size_t)r * cout + c] = tile[threadIdx.x][j];
  }
}

extern "C" int mp_mlp_destroy(mp_mlp_t* h) {
  if (!h) return MP_OK;
  mp_tc_release(h);
  for (int l = 0; l < MP_MAX_LAYERS; ++l) {
    if (h->wt[l]) cudaFree(h->wt[l]);
    if (h->w[l]) cudaFree(h->w[l]);
    if (h->bias[l]) cudaFree(h->bias[l]);
  }
  delete h;
  return MP_OK;
}

extern "C" int mp_mlp_create(int n_layers, const int* channels, const float* const* weights,
                             const float* const* biases, int skip, int last_op, int on_device, mp_mlp_t** out) {
  MP_REQUIRE(out != nullptr, "out is NULL");
  *out = nullptr;
  MP_REQUIRE(n_layers >= 1 && n_layers <= MP_MAX_LAYERS, "n_layers=%d out of range [1,%d]", n_layers, MP_MAX_LAYERS);
  MP_REQUIRE(channels && weights && biases, "NULL channels/weights/biases");
  MP_REQUIRE(last_op >= MP_LAST_NONE && last_op <= MP_LAST_TANH, "bad last_op %d", last_op);
  for (int l = 0; l <= n_layers; ++l) MP_REQUIRE(channels[l] >= 1 && channels[l] <= 8192, "channels[%d]=%d", l, channels[l]);
  mp_mlp* h = new mp_mlp();
  memset(h, 0, sizeof(*h));
  h->n_layers = n_layers;
  h->skip = skip ? 1 : 0;
  h->last_op = last_op;
  static std::atomic<unsigned long long> next_gen{1};
  h->gen = next_gen.fetch_add(1);
  {
    // validated feature range of the tensor-core programs, per output count and last op (DESIGN.md, precision)
    const char* v = getenv("MONOPORT_B200_TC_FEATURE_LIMIT");
    h->tc_amax_limit = v ? (float)atof(v) : mp_tc_default_feature_limit(channels[n_layers], last_op);
  }
  cudaGetDevice(&h->device);
  for (int l = 0; l <= n_layers; ++l) h->channels[l] = channels[l];
  const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  for (int l = 0; l < n_layers; ++l) {
    h->cin[l] = channels[l] + ((l > 0 && skip) ? channels[0] : 0);
    h->cout[l] = channels[l + 1];
    const size_t nw = (size_t)h->cin[l] * h->cout[l];
    cudaError_t e = cudaMalloc(&h->w[l], nw * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&h->wt[l], nw * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&h->bias[l], h->cout[l] * sizeof(float));
    if (e == cudaSuccess) e = cudaMemcpy(h->w[l], weights[l], nw * sizeof(float), kind);
    if (e == cudaSuccess) e = cudaMemcpy(h->bias[l], biases[l], h->cout[l] * sizeof(float), kind);
    if (e != cudaSuccess) {
      mp_set_error("mp_mlp_create: layer %d upload failed: %s", l, cudaGetErrorString(e));
      mp_mlp_destroy(h);
      return MP_E_CUDA;
    }
    dim3 grid((h->cin[l] + 31) / 32, (h->cout[l] + 31) / 32), block(32, 8);
    transpose_w_kernel<<<grid, block>>>(h->w[l], h->wt[l], h->cout[l], h->cin[l]);
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    mp_set_error("mp_mlp_create: %s", cudaGetErrorString(e));
    mp_mlp_destroy(h);
    return MP_E_CUDA;
  }
  int rc = mp_tc_prepare(h);   // sets tc_ok (0 when the head shape is not handled by the tensor-core kernel)
  if (rc != MP_OK) {
    mp_mlp_destroy(h);
    return rc;
  }
  *out = h;
  return MP_OK;
}

extern "C" int mp_mlp_tc_supported(const mp_mlp_t* h) { return h ? h->tc_ok : 0; }

extern "C" int mp_mlp_set_tc_feature_limit(mp_mlp_t* h, float limit) {
  MP_REQUIRE(h, "NULL handle");
  MP_REQUIRE(limit > 0.f, "the limit must be positive (+inf disables the guard)");
  h->tc_amax_limit = limit;
  return MP_OK;
}

// ---------------------------------------------------------------------------------------------
// feature volume: NCHW fp32 -> NHWC fp32 (channel-last: one bilinear tap = one contiguous vector)
// ---------------------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ o32, int C, int HW) {
  // tile transpose [C][HW] -> [HW][C]
  __shared__ float tile[32][33];
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, p = p0 + threadIdx.x;
    tile[j][threadIdx.x] = (c < C && p < HW) ? in[(size_t)c * HW + p] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int p = p0 + j, c = c0 + threadIdx.x;
    if (p < HW && c < C) {
      o32[(size_t)p * C + c] = tile[threadIdx.x][j];
    }
  }
}

extern "C" int mp_feat_destroy(mp_feat_t* h) {
  if (!h) return MP_OK;
  if (h->nhwc_own) cudaFree(h->nhwc_own);
  if (h->staging) cudaFree(h->staging);
  if (h->g0) cudaFree(h->g0);
  if (h->f16) cudaFree(h->f16);
  if (h->s4tex) cudaFree(h->s4tex);
  if (h->amax) cudaFree(h->amax);
  delete h;
  return MP_OK;
}

extern "C" int mp_feat_create_batch(int B, int C, int H, int W, mp_feat_t** out) {
  MP_REQUIRE(out != nullptr, "out is NULL");
  *out = nullptr;
  MP_REQUIRE(C >= 1 && H >= 1 && W >= 1 && (long long)C * H * W < (1ll << 31), "bad feature shape %dx%dx%d", C, H, W);
  MP_REQUIRE(B >= 1 && (long long)B * C * H * W < (1ll << 40), "bad batch size %d for %dx%dx%d maps", B, C, H, W);
  mp_feat* h = new mp_feat();
  memset(h, 0, sizeof(*h));
  h->B = B; h->C = C; h->H = H; h->W = W;
  cudaGetDevice(&h->device);
  const size_t n = (size_t)B * C * H * W;
  cudaError_t e = cudaMalloc(&h->nhwc_own, n * sizeof(float));
  h->nhwc32 = h->nhwc_own;
  if (e == cudaSuccess) e = cudaMalloc(&h->staging, n * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->amax, 2 * B * sizeof(unsigned));
  if (e == cudaSuccess) e = cudaMemset(h->amax, 0, 2 * B * sizeof(unsigned));
  if (e == cudaSuccess) h->nonfinite = h->amax + B;
  if (e != cudaSuccess) {
    mp_set_error("mp_feat_create: %s", cudaGetErrorString(e));
    mp_feat_destroy(h);
    return MP_E_NOMEM;
  }
  *out = h;
  return MP_OK;
}

extern "C" int mp_feat_create(int C, int H, int W, mp_feat_t** out) { return mp_feat_create_batch(1, C, H, W, out); }

extern "C" int mp_feat_upload(mp_feat_t* h, const float* nchw, int on_device, void* stream) {
  MP_REQUIRE(h && nchw, "NULL handle or data");
  MpRange nvtx("monoport_b200: feature upload (channel-last repack)");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t per_map = (size_t)h->C * h->H * h->W;
  const float* src = nchw;
  if (!on_device) {
    MP_CUDA(cudaMemcpyAsync(h->staging, nchw, h->B * per_map * sizeof(float), cudaMemcpyHostToDevice, st));
    src = h->staging;
  }
  const int HW = h->H * h->W;
  dim3 grid((HW + 31) / 32, (h->C + 31) / 32), block(32, 8);
  h->nhwc32 = h->nhwc_own;
  for (int b = 0; b < h->B; ++b) nchw_to_nhwc_kernel<<<grid, block, 0, st>>>(src + b * per_map, h->nhwc32 + b * per_map, h->C, HW);
  MP_CUDA(cudaGetLastError());
  MP_CUDA(cudaMemsetAsync(h->amax, 0, 2 * h->B * sizeof(unsigned), st));
  h->version += 1;
  return MP_OK;
}

// The map is already channel-last on the device (a torch.channels_last tensor: what a channels_last encoder emits,
// SURVEY.md §8f-3): one device-to-device copy instead of the transposing kernel.
extern "C" int mp_feat_upload_nhwc(mp_feat_t* h, const float* nhwc_dev, void* stream) {
  MP_REQUIRE(h && nhwc_dev, "NULL handle or data");
  const size_t n = (size_t)h->B * h->C * h->H * h->W;
  h->nhwc32 = h->nhwc_own;
  MP_CUDA(cudaMemcpyAsync(h->nhwc32, nhwc_dev, n * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  MP_CUDA(cudaMemsetAsync(h->amax, 0, 2 * h->B * sizeof(unsigned), (cudaStream_t)stream));
  h->version += 1;
  return MP_OK;
}

// Zero-copy hand-off (SURVEY.md 8f-3): the kernels read the caller's channel-last map in place -- no repack, no copy.  The
// memory must stay valid and unchanged until the queries of this frame have completed (the binding keeps the tensor alive).
extern "C" int mp_feat_bind_nhwc(mp_feat_t* h, const float* nhwc_dev, void* stream) {
  MP_REQUIRE(h && nhwc_dev, "NULL handle or data");
  MP_REQUIRE((reinterpret_cast<uintptr_t>(nhwc_dev) & 15) == 0, "the channel-last map must be 16-byte aligned");
  h->nhwc32 = const_cast<float*>(nhwc_dev);
  MP_CUDA(cudaMemsetAsync(h->amax, 0, 2 * h->B * sizeof(unsigned), (cudaStream_t)stream));
  h->version += 1;
  return MP_OK;
}

// ---------------------------------------------------------------------------------------------
// query
// ---------------------------------------------------------------------------------------------
int mp_query_dispatch(mp_mlp* mlp, mp_feat* feat, const MpPointSrc& src, const MpCalib& cal, const MpOutDst& dst,
                      int mode, cudaStream_t st, const MpBatch* bt) {
  MpRange nvtx("monoport_b200: F1 fused sample+MLP query");
  // (bt: a batched launch; the guard below is then decided per tile, from the maximum of the tile's image)
  // the tensor-core program covers maps of at most 65536 texels (16-bit texel indices in registers)
  const bool tc_can = mlp->tc_ok && (long long)feat->H * feat->W <= 65536;
  if (mode == MP_MODE_AUTO) mode = tc_can ? MP_MODE_TC : MP_MODE_FP32;
  if (mode == MP_MODE_TC || mode == MP_MODE_TC_V3) {
    if (!mlp->tc_ok) {
      mp_set_error("MP_MODE_TC requested but the tensor-core kernel does not support this head/device");
      return MP_E_UNSUPPORTED;
    }
    // Range guard: the tensor-core program is validated (<= 1e-4 on what query() returns) for frames whose largest
    // |feature| stays under the head's limit.  The decision is taken on the device, per launch, from the frame's own
    // maximum (no host synchronisation, graph-capturable): the tensor-core launch runs when the frame is in range, the
    // exact fp32 launch when it is not; the other one returns at once.
    const bool guarded = isfinite(mlp->tc_amax_limit);
    int rc = mp_launch_query_tc(mlp, feat, src, cal, dst, st, guarded ? MP_GUARD_IN_RANGE : MP_GUARD_NONE, bt);
    if (rc != MP_OK || !guarded) return rc;
    return mp_launch_query_fp32(mlp, feat, src, cal, dst, st, MP_GUARD_OUT_OF_RANGE, bt);
  }
  if (mode != MP_MODE_FP32) {
    mp_set_error("bad mode %d (3 was the removed MP_MODE_TC_V2)", mode);
    return MP_E_INVALID;
  }
  return mp_launch_query_fp32(mlp, feat, src, cal, dst, st, MP_GUARD_NONE, bt);
}

// mp_query_points and mp_query_points_batch: B images of n points.  calibs_dev == nullptr: the single-map call, whose calib
// (calib12, host memory, or none) travels in the kernel parameters; otherwise B calibs in device memory and a batched launch.
static int query_points(mp_mlp_t* mlp, mp_feat_t* feat, int B, const float* points_dev, int64_t n, int64_t batch_stride,
                        int64_t row_stride, int64_t point_stride, const float* calib12, const float* calibs_dev, int projection,
                        float z_scale, float* out_dev, int64_t out_batch_stride, int64_t ld_out, int mode, void* stream,
                        bool batched, const int32_t* count_dev = nullptr, const float* calib_dev = nullptr) {
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE(n >= 0 && row_stride >= 1 && point_stride >= 1 && ld_out >= n, "bad sizes n=%lld strides=%lld,%lld ld_out=%lld",
             (long long)n, (long long)row_stride, (long long)point_stride, (long long)ld_out);
  if (batched) {
    MP_REQUIRE(B == feat->B, "batch size %d does not match the feature handle's %d maps", B, feat->B);
    MP_REQUIRE(B == 1 || (batch_stride >= 1 && out_batch_stride >= 1), "bad batch strides %lld, %lld", (long long)batch_stride,
               (long long)out_batch_stride);
    // (the kernels find a tile's image with a 32-bit division: at most 2^31 tiles of 8 points per launch)
    MP_REQUIRE((long long)B * ((n + 7) / 8) < (1ll << 31), "batch too large: %d x %lld points", B, (long long)n);
  } else {
    MP_REQUIRE_SINGLE_MAP(feat, "mp_query_points");
  }
  if (n == 0) return MP_OK;
  MP_REQUIRE(points_dev && out_dev, "NULL points/out");
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_ROWS;
  src.px = points_dev; src.py = points_dev + row_stride; src.pz = points_dev + 2 * row_stride;
  src.pstride = point_stride;
  src.n = n;
  src.count_dev = count_dev;
  MpCalib cal;
  MpBatch one;
  const MpBatch* single = mp_single_calib(cal, one, calib12, calib_dev, projection, z_scale);
  MpOutDst dst;
  dst.out = out_dev; dst.ld = ld_out; dst.scatter_vol = nullptr;
  if (!batched) return mp_query_dispatch(mlp, feat, src, cal, dst, mode, (cudaStream_t)stream, single);
  MpBatch bt;
  bt.B = B;
  bt.pt_stride = batch_stride;
  bt.out_stride = out_batch_stride;
  bt.calibs = calibs_dev;
  cal.has = calibs_dev != nullptr;
  cal.perspective = projection == MP_PROJ_PERSPECTIVE && cal.has;
  return mp_query_dispatch(mlp, feat, src, cal, dst, mode, (cudaStream_t)stream, &bt);
}

extern "C" int mp_query_points(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                               int64_t point_stride, const float* calib12, int projection, float z_scale,
                               float* out_dev, int64_t ld_out, int mode, void* stream) {
  return query_points(mlp, feat, 1, points_dev, n, 0, row_stride, point_stride, calib12, nullptr, projection, z_scale, out_dev, 0,
                      ld_out, mode, stream, false);
}

extern "C" int mp_query_points_count(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                                     int64_t point_stride, const float* calib12, int projection, float z_scale, float* out_dev,
                                     int64_t ld_out, const int32_t* count_dev, int mode, void* stream) {
  return query_points(mlp, feat, 1, points_dev, n, 0, row_stride, point_stride, calib12, nullptr, projection, z_scale, out_dev, 0,
                      ld_out, mode, stream, false, count_dev);
}

extern "C" int mp_query_points_count_dcal(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                                          int64_t point_stride, const float* calib_dev, int projection, float z_scale, float* out_dev,
                                          int64_t ld_out, const int32_t* count_dev, int mode, void* stream) {
  MP_REQUIRE(calib_dev, "NULL calib_dev");
  return query_points(mlp, feat, 1, points_dev, n, 0, row_stride, point_stride, nullptr, nullptr, projection, z_scale, out_dev, 0,
                      ld_out, mode, stream, false, count_dev, calib_dev);
}

extern "C" int mp_query_points_batch(mp_mlp_t* mlp, mp_feat_t* feat, int B, const float* points_dev, int64_t n,
                                     int64_t batch_stride, int64_t row_stride, int64_t point_stride, const float* calibs_dev,
                                     int projection, float z_scale, float* out_dev, int64_t out_batch_stride, int64_t ld_out,
                                     int mode, void* stream) {
  return query_points(mlp, feat, B, points_dev, n, batch_stride, row_stride, point_stride, nullptr, calibs_dev, projection, z_scale,
                      out_dev, out_batch_stride, ld_out, mode, stream, true);
}

// mp_query_points_grad and mp_query_points_grad_mode
static int query_points_grad(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                             int64_t point_stride, const float* calib12, int projection, float z_scale, const float* grad_out_dev,
                             int64_t ld_grad, float* out_dev, int64_t ld_out, float* dpoints_dev, int64_t ld_dpoints,
                             const int32_t* count_dev, int mode, void* stream, const char* what,
                             const float* calib_dev = nullptr) {
  MpRange nvtx("monoport_b200: F1'' query gradient");
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE_SINGLE_MAP(feat, what);
  MP_REQUIRE(n >= 0 && row_stride >= 1 && point_stride >= 1 && ld_dpoints >= n && (!out_dev || ld_out >= n) &&
                 (!grad_out_dev || ld_grad >= n),
             "bad sizes n=%lld strides=%lld,%lld ld_grad=%lld ld_out=%lld ld_dpoints=%lld", (long long)n, (long long)row_stride,
             (long long)point_stride, (long long)ld_grad, (long long)ld_out, (long long)ld_dpoints);
  if (n == 0) return MP_OK;
  MP_REQUIRE(points_dev && dpoints_dev, "NULL points/dpoints");
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_ROWS;
  src.px = points_dev; src.py = points_dev + row_stride; src.pz = points_dev + 2 * row_stride;
  src.pstride = point_stride;
  src.n = n;
  src.count_dev = count_dev;
  MpCalib cal;
  MpBatch one;
  const MpBatch* single = mp_single_calib(cal, one, calib12, calib_dev, projection, z_scale);
  cudaStream_t st = (cudaStream_t)stream;
  // the rule of mp_query_dispatch: the tensor-core program covers maps of at most 65536 texels, and a frame above the head's
  // feature limit is taken by the exact kernel, decided on the device
  const bool tc_can = mlp->tc_ok && (long long)feat->H * feat->W <= 65536;
  if (mode == MP_MODE_AUTO) mode = tc_can ? MP_MODE_TC : MP_MODE_FP32;
  if (mode == MP_MODE_TC || mode == MP_MODE_TC_V3) {
    if (!mlp->tc_ok) {
      mp_set_error("MP_MODE_TC requested but the tensor-core kernel does not support this head/device");
      return MP_E_UNSUPPORTED;
    }
    const bool guarded = isfinite(mlp->tc_amax_limit);
    int rc = mp_launch_query_jvp_tc(mlp, feat, src, cal, grad_out_dev, ld_grad, out_dev, ld_out, dpoints_dev, ld_dpoints, st,
                                    guarded ? MP_GUARD_IN_RANGE : MP_GUARD_NONE, single);
    if (rc != MP_OK || !guarded) return rc;
    return mp_launch_query_grad(mlp, feat, src, cal, grad_out_dev, ld_grad, out_dev, ld_out, dpoints_dev, ld_dpoints, st,
                                MP_GUARD_OUT_OF_RANGE, single);
  }
  MP_REQUIRE(mode == MP_MODE_FP32, "bad mode %d", mode);
  return mp_launch_query_grad(mlp, feat, src, cal, grad_out_dev, ld_grad, out_dev, ld_out, dpoints_dev, ld_dpoints, st, MP_GUARD_NONE,
                              single);
}

extern "C" int mp_query_points_grad(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                                    int64_t point_stride, const float* calib12, int projection, float z_scale,
                                    const float* grad_out_dev, int64_t ld_grad, float* out_dev, int64_t ld_out,
                                    float* dpoints_dev, int64_t ld_dpoints, void* stream) {
  return query_points_grad(mlp, feat, points_dev, n, row_stride, point_stride, calib12, projection, z_scale, grad_out_dev, ld_grad,
                           out_dev, ld_out, dpoints_dev, ld_dpoints, nullptr, MP_MODE_FP32, stream, "mp_query_points_grad");
}

extern "C" int mp_query_points_grad_mode(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                                         int64_t point_stride, const float* calib12, int projection, float z_scale,
                                         const float* grad_out_dev, int64_t ld_grad, float* out_dev, int64_t ld_out,
                                         float* dpoints_dev, int64_t ld_dpoints, const int32_t* count_dev, int mode, void* stream) {
  return query_points_grad(mlp, feat, points_dev, n, row_stride, point_stride, calib12, projection, z_scale, grad_out_dev, ld_grad,
                           out_dev, ld_out, dpoints_dev, ld_dpoints, count_dev, mode, stream, "mp_query_points_grad_mode");
}

// ---------------------------------------------------------------------------------------------
// the vector-Jacobian product of the exact query, for training (query_vjp.cu)
// ---------------------------------------------------------------------------------------------
extern "C" int64_t mp_query_points_vjp_scratch_bytes_ex(mp_mlp_t* mlp, mp_feat_t* feat, int B, int64_t n, int64_t chunk_points,
                                                        int want_dfeat, int want_dweights, int flags) {
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE(B == feat->B && n >= 0, "bad batch %d (the handle holds %d maps) or n=%lld", B, feat->B, (long long)n);
  MP_REQUIRE((flags & ~MP_VJP_DETERMINISTIC) == 0, "unknown VJP flags %d", flags);
  return mp_vjp_scratch_bytes(mlp, feat, B, n, chunk_points, want_dfeat != 0, want_dweights != 0, flags);
}

extern "C" int64_t mp_query_points_vjp_scratch_bytes(mp_mlp_t* mlp, mp_feat_t* feat, int B, int64_t n, int64_t chunk_points,
                                                     int want_dfeat, int want_dweights) {
  return mp_query_points_vjp_scratch_bytes_ex(mlp, feat, B, n, chunk_points, want_dfeat, want_dweights, 0);
}

extern "C" int mp_query_points_vjp_ex(mp_mlp_t* mlp, mp_feat_t* feat, int B, const float* points_dev, int64_t n,
                                      int64_t batch_stride, int64_t row_stride, int64_t point_stride, const float* calibs_dev,
                                      int projection, float z_scale, const float* grad_out_dev, float* dfeat_dev,
                                      float* dpoints_dev, float* const* dweights_dev, float* const* dbiases_dev, void* scratch_dev,
                                      int64_t scratch_bytes, int flags, void* stream) {
  MpRange nvtx("monoport_b200: F1'''' query VJP");
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE(B == feat->B, "batch size %d does not match the feature handle's %d maps", B, feat->B);
  MP_REQUIRE(n >= 0 && row_stride >= 1 && point_stride >= 1 && (B == 1 || batch_stride >= 1) && scratch_bytes >= 0,
             "bad sizes n=%lld strides=%lld,%lld,%lld scratch=%lld", (long long)n, (long long)batch_stride, (long long)row_stride,
             (long long)point_stride, (long long)scratch_bytes);
  // (the kernel finds a tile's image with a 32-bit division: at most 2^31 tiles of 8 points per launch)
  MP_REQUIRE((long long)B * ((n + 7) / 8) < (1ll << 31), "batch too large: %d x %lld points", B, (long long)n);
  MP_REQUIRE(n == 0 || points_dev, "NULL points");
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_ROWS;
  src.px = points_dev; src.py = points_dev + row_stride; src.pz = points_dev + 2 * row_stride;
  src.pstride = point_stride;
  src.n = n;
  MpCalib cal;
  mp_fill_calib(cal, nullptr, projection, z_scale);
  cal.has = calibs_dev != nullptr;
  cal.perspective = projection == MP_PROJ_PERSPECTIVE && cal.has;
  MpBatch bt;
  bt.B = B;
  bt.pt_stride = batch_stride;
  bt.calibs = calibs_dev;
  return mp_launch_query_vjp(mlp, feat, src, cal, bt, grad_out_dev, dfeat_dev, dpoints_dev, dweights_dev, dbiases_dev, scratch_dev,
                             scratch_bytes, (cudaStream_t)stream, flags);
}

extern "C" int mp_query_points_vjp(mp_mlp_t* mlp, mp_feat_t* feat, int B, const float* points_dev, int64_t n,
                                   int64_t batch_stride, int64_t row_stride, int64_t point_stride, const float* calibs_dev,
                                   int projection, float z_scale, const float* grad_out_dev, float* dfeat_dev, float* dpoints_dev,
                                   float* const* dweights_dev, float* const* dbiases_dev, void* scratch_dev,
                                   int64_t scratch_bytes, void* stream) {
  return mp_query_points_vjp_ex(mlp, feat, B, points_dev, n, batch_stride, row_stride, point_stride, calibs_dev, projection,
                                z_scale, grad_out_dev, dfeat_dev, dpoints_dev, dweights_dev, dbiases_dev, scratch_dev, scratch_bytes,
                                0, stream);
}

// ---------------------------------------------------------------------------------------------
// analytic normals of the visible surface, enqueue-only (mp_surface_normals_async)
// ---------------------------------------------------------------------------------------------
// step 1: vertex i -> its world point (mp_surface_point's two roundings) in rows [3][cap]; the count, clamped to the
// capacity, as the int32 point count of the gradient launches
__global__ void normals_points_kernel(MpSurfaceSrc s, long long cap, float* __restrict__ pts, int32_t* __restrict__ count32) {
  long long n = *s.count;
  n = n < 0 ? 0 : (n > cap ? cap : n);
  if (blockIdx.x == 0 && threadIdx.x == 0) *count32 = (int32_t)n;
  const long long step = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += step) {
    float x, y, z;
    mp_surface_point(s, i, x, y, z);
    pts[i] = x;
    pts[cap + i] = y;
    pts[2 * cap + i] = z;
  }
}

// step 3: the world gradient g [3][cap] -> -(g_x a_x, g_y a_y, g_z a_z) normalised into norm [cap][3], zero where g vanishes
__global__ void normals_finish_kernel(const float* __restrict__ g, const long long* __restrict__ count, long long cap, float ax,
                                      float ay, float az, float* __restrict__ norm) {
  long long n = *count;
  n = n < 0 ? 0 : (n > cap ? cap : n);
  const long long step = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += step) {
    const float v[3] = {-(g[i] * ax), -(g[cap + i] * ay), -(g[2 * cap + i] * az)};
    const float len = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
#pragma unroll
    for (int a = 0; a < 3; ++a) norm[3 * i + a] = len > 0.f ? v[a] / len : 0.f;
  }
}

static int surface_normals_async(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev, const float* z_dev,
                                 const int64_t* count_dev, int64_t capacity, int R, const float* b_min3, const float* b_max3,
                                 const float* calib12, const float* calib_dev, int projection, float z_scale, int mode,
                                 float* scratch_dev, float* norm_dev, void* stream) {
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE_SINGLE_MAP(feat, "mp_surface_normals_async");
  MP_REQUIRE(mlp->cout[mlp->n_layers - 1] == 1, "surface normals need a head with one output (got %d)", mlp->cout[mlp->n_layers - 1]);
  MP_REQUIRE(capacity >= 0 && R >= 1 && capacity <= (int64_t)R * R, "bad sizes capacity=%lld R=%d", (long long)capacity, R);
  MP_REQUIRE(x_dev && y_dev && z_dev && count_dev && b_min3 && b_max3 && scratch_dev && norm_dev, "NULL argument");
  if (capacity == 0) return MP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const MpSurfaceSrc surf = mp_surface_src(reinterpret_cast<const long long*>(x_dev), reinterpret_cast<const long long*>(y_dev), z_dev,
                                           reinterpret_cast<const long long*>(count_dev), R, b_min3, b_max3, nullptr);
  float* pts = scratch_dev;
  float* grad = scratch_dev + 3 * capacity;
  int32_t* count32 = reinterpret_cast<int32_t*>(scratch_dev + 6 * capacity);
  const long long blocks = (capacity + 255) / 256;
  const int grid = (int)(blocks < 1024 ? blocks : 1024);
  normals_points_kernel<<<grid, 256, 0, st>>>(surf, capacity, pts, count32);
  MP_CUDA(cudaGetLastError());
  const int rc = query_points_grad(mlp, feat, pts, capacity, capacity, 1, calib12, projection, z_scale, nullptr, 0, nullptr, 0, grad,
                                   capacity, count32, mode, stream, "mp_surface_normals_async", calib_dev);
  if (rc != MP_OK) return rc;
  // forward_vertices' frame: its (X, Y, Z) index axes are the world axes scaled by R / (b_max - b_min), Z reversed
  float a[3];
  for (int k = 0; k < 3; ++k) a[k] = (b_max3[k] - b_min3[k]) / (float)R;
  normals_finish_kernel<<<grid, 256, 0, st>>>(grad, reinterpret_cast<const long long*>(count_dev), capacity, a[0], a[1], -a[2], norm_dev);
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

extern "C" int mp_surface_normals_async(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev,
                                        const float* z_dev, const int64_t* count_dev, int64_t capacity, int R,
                                        const float* b_min3, const float* b_max3, const float* calib12, int projection,
                                        float z_scale, int mode, float* scratch_dev, float* norm_dev, void* stream) {
  return surface_normals_async(mlp, feat, x_dev, y_dev, z_dev, count_dev, capacity, R, b_min3, b_max3, calib12, nullptr, projection,
                               z_scale, mode, scratch_dev, norm_dev, stream);
}

extern "C" int mp_surface_normals_async_dcal(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev,
                                             const float* z_dev, const int64_t* count_dev, int64_t capacity, int R,
                                             const float* b_min3, const float* b_max3, const float* calib_dev, int projection,
                                             float z_scale, int mode, float* scratch_dev, float* norm_dev, void* stream) {
  MP_REQUIRE(calib_dev, "NULL calib_dev");
  return surface_normals_async(mlp, feat, x_dev, y_dev, z_dev, count_dev, capacity, R, b_min3, b_max3, nullptr, calib_dev, projection,
                               z_scale, mode, scratch_dev, norm_dev, stream);
}

// Analytic normals at the vertices of a mesh (mp_mcubes_run_async's world-space [cap][3] vertices), enqueue-only: the
// gradient launches of mp_surface_normals_async read the vertex rows in place (row stride 1, point stride 3) with the int32
// count of the emission, and normals_finish_kernel takes unit axes: -g / |g|, zero where g vanishes.
static int mesh_normals_async(mp_mlp_t* mlp, mp_feat_t* feat, const float* verts_dev, const int64_t* counts_dev,
                              const int32_t* count32_dev, int64_t capacity, const float* calib12, const float* calib_dev,
                              int projection, float z_scale, int mode, float* scratch_dev, float* norm_dev, void* stream) {
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE_SINGLE_MAP(feat, "mp_mesh_normals_async");
  MP_REQUIRE(mlp->cout[mlp->n_layers - 1] == 1, "mesh normals need a head with one output (got %d)", mlp->cout[mlp->n_layers - 1]);
  MP_REQUIRE(capacity >= 0, "bad capacity %lld", (long long)capacity);
  MP_REQUIRE(verts_dev && counts_dev && count32_dev && scratch_dev && norm_dev, "NULL argument");
  if (capacity == 0) return MP_OK;
  float* grad = scratch_dev;
  const int rc = query_points_grad(mlp, feat, verts_dev, capacity, 1, 3, calib12, projection, z_scale, nullptr, 0, nullptr, 0, grad,
                                   capacity, count32_dev, mode, stream, "mp_mesh_normals_async", calib_dev);
  if (rc != MP_OK) return rc;
  const long long blocks = (capacity + 255) / 256;
  const int grid = (int)(blocks < 1024 ? blocks : 1024);
  normals_finish_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(grad, reinterpret_cast<const long long*>(counts_dev), capacity,
                                                                1.f, 1.f, 1.f, norm_dev);
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

extern "C" int mp_mesh_normals_async(mp_mlp_t* mlp, mp_feat_t* feat, const float* verts_dev, const int64_t* counts_dev,
                                     const int32_t* count32_dev, int64_t capacity, const float* calib12, int projection,
                                     float z_scale, int mode, float* scratch_dev, float* norm_dev, void* stream) {
  return mesh_normals_async(mlp, feat, verts_dev, counts_dev, count32_dev, capacity, calib12, nullptr, projection, z_scale, mode,
                            scratch_dev, norm_dev, stream);
}

extern "C" int mp_mesh_normals_async_dcal(mp_mlp_t* mlp, mp_feat_t* feat, const float* verts_dev, const int64_t* counts_dev,
                                          const int32_t* count32_dev, int64_t capacity, const float* calib_dev, int projection,
                                          float z_scale, int mode, float* scratch_dev, float* norm_dev, void* stream) {
  MP_REQUIRE(calib_dev, "NULL calib_dev");
  return mesh_normals_async(mlp, feat, verts_dev, counts_dev, count32_dev, capacity, nullptr, calib_dev, projection, z_scale, mode,
                            scratch_dev, norm_dev, stream);
}

extern "C" int mp_query_points_host(mp_mlp_t* mlp, mp_feat_t* feat, const float* feat_nchw_host, const float* points_host,
                                    int64_t n, const float* calib12, int projection, float z_scale, float* out_host,
                                    int mode, void* stream) {
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE_SINGLE_MAP(feat, "mp_query_points_host");
  MP_REQUIRE(n >= 0, "bad n");
  cudaStream_t st = (cudaStream_t)stream;
  if (feat_nchw_host) {
    int rc = mp_feat_upload(feat, feat_nchw_host, 0, stream);
    if (rc != MP_OK) return rc;
  }
  if (n == 0) {
    MP_CUDA(cudaStreamSynchronize(st));
    return MP_OK;
  }
  MP_REQUIRE(points_host && out_host, "NULL points/out");
  const int res = mlp->cout[mlp->n_layers - 1];
  float* d_pts = nullptr;
  float* d_out = nullptr;
  mp_ensure_pool();
  MP_CUDA(cudaMallocAsync(&d_pts, (size_t)3 * n * sizeof(float), st));
  MP_CUDA(cudaMallocAsync(&d_out, (size_t)res * n * sizeof(float), st));
  MP_CUDA(cudaMemcpyAsync(d_pts, points_host, (size_t)3 * n * sizeof(float), cudaMemcpyHostToDevice, st));
  int rc = mp_query_points(mlp, feat, d_pts, n, n, 1, calib12, projection, z_scale, d_out, n, mode, stream);
  if (rc == MP_OK) {
    cudaError_t e = cudaMemcpyAsync(out_host, d_out, (size_t)res * n * sizeof(float), cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) { mp_set_error("D2H failed: %s", cudaGetErrorString(e)); rc = MP_E_CUDA; }
  }
  cudaFreeAsync(d_pts, st);
  cudaFreeAsync(d_out, st);
  cudaError_t e = cudaStreamSynchronize(st);
  if (rc == MP_OK && e != cudaSuccess) { mp_set_error("sync failed: %s", cudaGetErrorString(e)); rc = MP_E_CUDA; }
  return rc;
}

// One implementation behind the four grid entry points: nodes [lin0, lin0 + n) of the R^3 grid in z-major linear order
// (a z slab is the range [z0*R*R, (z0+nz)*R*R)), values to out_dev[0..n) and / or to every peer volume at offset lin0.
static int query_grid_range(mp_mlp_t* mlp, mp_feat_t* feat, int R, long long lin0, long long n, const float* b_min3,
                            const float* b_max3, const float* calib12, int projection, float z_scale, float* out_dev,
                            float* const* peer_vols, int n_peers, int mode, void* stream) {
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE_SINGLE_MAP(feat, "the grid query");
  MP_REQUIRE(R >= 1 && lin0 >= 0 && n >= 0 && lin0 + n <= (long long)R * R * R, "bad range R=%d lin0=%lld n=%lld", R, lin0, n);
  MP_REQUIRE(b_min3 && b_max3, "NULL bounds");
  MP_REQUIRE(mlp->cout[mlp->n_layers - 1] == 1, "grid queries need a single-channel head");
  MP_REQUIRE(n_peers >= 0 && n_peers <= MP_MAX_PEERS && (n_peers == 0 || peer_vols), "n_peers=%d out of range [0,%d]", n_peers, MP_MAX_PEERS);
  for (int p = 0; p < n_peers; ++p) MP_REQUIRE(peer_vols[p] != nullptr, "peer volume %d is NULL", p);
  if (n == 0) return MP_OK;
  MP_REQUIRE(out_dev || n_peers > 0, "NULL out");
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_GRID;
  mp_fill_grid_geom(src, R, 1, R, b_min3, b_max3);
  src.lin0 = lin0;
  src.n = n;
  MpCalib cal;
  mp_fill_calib(cal, calib12, projection, z_scale);
  MpOutDst dst;
  dst.out = out_dev; dst.ld = n; dst.scatter_vol = nullptr;
  for (int p = 0; p < n_peers; ++p) dst.peer[p] = peer_vols[p];
  dst.n_peers = n_peers;
  dst.peer_off = lin0;        // the range's position inside every full [R,R,R] volume
  // (the value of a node never depends on the range it is evaluated in, so a sharded volume is bit-identical to the
  // single-GPU volume for every rank count)
  // With a Sigmoid head on the tensor-core route a node outside the image has the value 0 * act = +0, so the program runs
  // over the list of in-image nodes only (DESIGN.md §F1).  Other heads carry act's sign in that zero, and node indices
  // are int32: those keep the dense launch.
  const bool tc_route = mlp->tc_ok && (long long)feat->H * feat->W <= 65536 &&
                        (mode == MP_MODE_AUTO || mode == MP_MODE_TC || mode == MP_MODE_TC_V3);
  if (!tc_route || mlp->last_op != MP_LAST_SIGMOID || (long long)R * R * R >= (1ll << 31))
    return mp_query_dispatch(mlp, feat, src, cal, dst, mode, (cudaStream_t)stream);
  MpRange nvtx("monoport_b200: F1 fused sample+MLP query, in-image nodes");
  // mp_query_dispatch's two guarded launches: the compaction's zero stores come first, the list launch skips an
  // out-of-range frame on the device, and the exact launch then overwrites every node of the range
  const cudaStream_t st = (cudaStream_t)stream;
  void* scratch = nullptr;
  mp_ensure_pool();
  MP_CUDA(cudaMallocAsync(&scratch, mp_tc_grid_scratch_bytes(n), st));
  const bool guarded = isfinite(mlp->tc_amax_limit);
  cudaError_t e = cudaMemsetAsync(scratch, 0, 16, st);
  int rc = e == cudaSuccess ? mp_launch_query_tc_grid(mlp, feat, src, cal, dst, scratch, st, guarded ? MP_GUARD_IN_RANGE : MP_GUARD_NONE)
                            : MP_E_CUDA;
  if (e != cudaSuccess) mp_set_error("scratch of the grid query: %s", cudaGetErrorString(e));
  if (rc == MP_OK && guarded) rc = mp_launch_query_fp32(mlp, feat, src, cal, dst, st, MP_GUARD_OUT_OF_RANGE);
  cudaFreeAsync(scratch, st);
  return rc;
}

extern "C" int mp_query_grid(mp_mlp_t* mlp, mp_feat_t* feat, int R, int z0, int nz, const float* b_min3, const float* b_max3,
                             const float* calib12, int projection, float z_scale, float* out_dev, int mode, void* stream) {
  MP_REQUIRE(R >= 1 && z0 >= 0 && nz >= 0 && z0 + nz <= R, "bad slab R=%d z0=%d nz=%d", R, z0, nz);
  return query_grid_range(mlp, feat, R, (long long)z0 * R * R, (long long)nz * R * R, b_min3, b_max3, calib12, projection, z_scale,
                          out_dev, nullptr, 0, mode, stream);
}

extern "C" int mp_query_grid_range(mp_mlp_t* mlp, mp_feat_t* feat, int R, int64_t lin0, int64_t n, const float* b_min3,
                                   const float* b_max3, const float* calib12, int projection, float z_scale, float* out_dev,
                                   int mode, void* stream) {
  return query_grid_range(mlp, feat, R, lin0, n, b_min3, b_max3, calib12, projection, z_scale, out_dev, nullptr, 0, mode, stream);
}

// ---------------------------------------------------------------------------------------------
// fused slab exchange (multi-GPU sharding of the grid without a data collective)
// ---------------------------------------------------------------------------------------------
extern "C" int mp_query_grid_peers(mp_mlp_t* mlp, mp_feat_t* feat, int R, int z0, int nz, const float* b_min3,
                                   const float* b_max3, const float* calib12, int projection, float z_scale,
                                   float* const* peer_vols, int n_peers, int mode, void* stream) {
  MP_REQUIRE(R >= 1 && z0 >= 0 && nz >= 0 && z0 + nz <= R, "bad slab R=%d z0=%d nz=%d", R, z0, nz);
  MP_REQUIRE(peer_vols && n_peers >= 1, "n_peers=%d out of range [1,%d]", n_peers, MP_MAX_PEERS);
  return query_grid_range(mlp, feat, R, (long long)z0 * R * R, (long long)nz * R * R, b_min3, b_max3, calib12, projection, z_scale,
                          nullptr, peer_vols, n_peers, mode, stream);
}

extern "C" int mp_query_grid_range_peers(mp_mlp_t* mlp, mp_feat_t* feat, int R, int64_t lin0, int64_t n, const float* b_min3,
                                         const float* b_max3, const float* calib12, int projection, float z_scale,
                                         float* const* peer_vols, int n_peers, int mode, void* stream) {
  MP_REQUIRE(peer_vols && n_peers >= 1, "n_peers=%d out of range [1,%d]", n_peers, MP_MAX_PEERS);
  return query_grid_range(mlp, feat, R, lin0, n, b_min3, b_max3, calib12, projection, z_scale, nullptr, peer_vols, n_peers, mode, stream);
}

// ---------------------------------------------------------------------------------------------
// direct rendering of the visible surface with the colour head, one launch (RTL/main.py:212-249)
// ---------------------------------------------------------------------------------------------
extern "C" int mp_colorize_surface(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev, const float* z_dev,
                                   int64_t n, int R, const float* b_min3, const float* b_max3, const float* calib12, int projection,
                                   float z_scale, float* canvas_dev, void* stream) {
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE_SINGLE_MAP(feat, "mp_colorize_surface");
  MP_REQUIRE(n >= 0 && R >= 1, "bad sizes n=%lld R=%d", (long long)n, R);
  if (n == 0) return MP_OK;
  MP_REQUIRE(x_dev && y_dev && z_dev && canvas_dev && b_min3 && b_max3, "NULL argument");
  MpCalib cal;
  mp_fill_calib(cal, calib12, projection, z_scale);
  return mp_launch_colour_surface(mlp, feat, reinterpret_cast<const long long*>(x_dev), reinterpret_cast<const long long*>(y_dev), z_dev,
                                  n, R, b_min3, b_max3, cal, canvas_dev, (cudaStream_t)stream);
}

// The same render, enqueue-only (graph-capturable): the vertex count stays on the device and the range guard is decided
// there, exactly as mp_query_dispatch decides it for a query -- the tensor-core launch renders a frame inside the head's
// range, its exact fp32 twin one outside it, and the other launch returns at once.
static int colorize_surface_async(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev, const float* z_dev,
                                  const int64_t* count_dev, int64_t capacity, int R, const float* b_min3, const float* b_max3,
                                  const float* calib12, const float* calib_dev, int projection, float z_scale, int mode,
                                  float* canvas_dev, void* stream) {
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE_SINGLE_MAP(feat, "mp_colorize_surface_async");
  MP_REQUIRE(mlp->cout[mlp->n_layers - 1] == 3, "surface colourisation needs a head with 3 outputs (got %d)",
             mlp->cout[mlp->n_layers - 1]);
  MP_REQUIRE(capacity >= 0 && R >= 1 && capacity <= (int64_t)R * R, "bad sizes capacity=%lld R=%d", (long long)capacity, R);
  MP_REQUIRE(x_dev && y_dev && z_dev && count_dev && canvas_dev && b_min3 && b_max3, "NULL argument");
  if (capacity == 0) return MP_OK;
  MpRange nvtx("monoport_b200: F1 fused surface colourisation");
  MpCalib cal;
  MpBatch one;
  const MpBatch* single = mp_single_calib(cal, one, calib12, calib_dev, projection, z_scale);
  const MpSurfaceSrc surf = mp_surface_src(reinterpret_cast<const long long*>(x_dev), reinterpret_cast<const long long*>(y_dev), z_dev,
                                           reinterpret_cast<const long long*>(count_dev), R, b_min3, b_max3, canvas_dev);
  cudaStream_t st = (cudaStream_t)stream;
  const bool tc_can = mlp->tc_ok && (long long)feat->H * feat->W <= 65536;
  if (mode == MP_MODE_AUTO) mode = tc_can ? MP_MODE_TC : MP_MODE_FP32;
  if (mode == MP_MODE_TC || mode == MP_MODE_TC_V3) {
    if (!mlp->tc_ok) {
      mp_set_error("MP_MODE_TC requested but the tensor-core kernel does not support this head/device");
      return MP_E_UNSUPPORTED;
    }
    const bool guarded = isfinite(mlp->tc_amax_limit);
    int rc = mp_launch_surface_tc(mlp, feat, surf, capacity, cal, st, guarded ? MP_GUARD_IN_RANGE : MP_GUARD_NONE, single);
    if (rc != MP_OK || !guarded) return rc;
    return mp_launch_surface_fp32(mlp, feat, surf, capacity, cal, st, MP_GUARD_OUT_OF_RANGE, single);
  }
  MP_REQUIRE(mode == MP_MODE_FP32, "bad mode %d", mode);
  return mp_launch_surface_fp32(mlp, feat, surf, capacity, cal, st, MP_GUARD_NONE, single);
}

extern "C" int mp_colorize_surface_async(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev,
                                         const float* z_dev, const int64_t* count_dev, int64_t capacity, int R, const float* b_min3,
                                         const float* b_max3, const float* calib12, int projection, float z_scale, int mode,
                                         float* canvas_dev, void* stream) {
  return colorize_surface_async(mlp, feat, x_dev, y_dev, z_dev, count_dev, capacity, R, b_min3, b_max3, calib12, nullptr, projection,
                                z_scale, mode, canvas_dev, stream);
}

extern "C" int mp_colorize_surface_async_dcal(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev,
                                              const float* z_dev, const int64_t* count_dev, int64_t capacity, int R,
                                              const float* b_min3, const float* b_max3, const float* calib_dev, int projection,
                                              float z_scale, int mode, float* canvas_dev, void* stream) {
  MP_REQUIRE(calib_dev, "NULL calib_dev");
  return colorize_surface_async(mlp, feat, x_dev, y_dev, z_dev, count_dev, capacity, R, b_min3, b_max3, nullptr, calib_dev,
                                projection, z_scale, mode, canvas_dev, stream);
}

// Volumes that other processes of the node write into: plain cudaMalloc blocks (exportable; the caching allocators of
// frameworks hand out sub-blocks, which legacy IPC handles cannot describe) + their 64-byte IPC handle.
extern "C" int mp_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64) {
  MP_REQUIRE(dev_ptr && handle64 && bytes > 0, "bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  *dev_ptr = nullptr;
  MP_CUDA(cudaMalloc(dev_ptr, bytes));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, *dev_ptr);
  if (e != cudaSuccess) {
    cudaFree(*dev_ptr);
    *dev_ptr = nullptr;
    mp_set_error("cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    return MP_E_CUDA;
  }
  memcpy(handle64, &h, 64);
  return MP_OK;
}

extern "C" int mp_ipc_open(const unsigned char* handle64, void** dev_ptr) {
  MP_REQUIRE(dev_ptr && handle64, "bad argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  *dev_ptr = nullptr;
  MP_CUDA(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return MP_OK;
}

extern "C" int mp_ipc_close(void* dev_ptr) {
  if (dev_ptr) MP_CUDA(cudaIpcCloseMemHandle(dev_ptr));
  return MP_OK;
}

extern "C" int mp_ipc_free(void* dev_ptr) {
  if (dev_ptr) MP_CUDA(cudaFree(dev_ptr));
  return MP_OK;
}

extern "C" int mp_query_grid_host(mp_mlp_t* mlp, mp_feat_t* feat, const float* feat_nchw_host, int R, int z0, int nz,
                                  const float* b_min3, const float* b_max3, const float* calib12, int projection,
                                  float z_scale, float* out_host, int mode, void* stream) {
  MP_REQUIRE(mlp && feat, "NULL handle");
  MP_REQUIRE_SINGLE_MAP(feat, "mp_query_grid_host");
  MP_REQUIRE(R >= 1 && z0 >= 0 && nz >= 0 && z0 + nz <= R, "bad slab R=%d z0=%d nz=%d", R, z0, nz);
  cudaStream_t st = (cudaStream_t)stream;
  if (feat_nchw_host) {
    int rc = mp_feat_upload(feat, feat_nchw_host, 0, stream);
    if (rc != MP_OK) return rc;
  }
  if (nz == 0) {
    MP_CUDA(cudaStreamSynchronize(st));
    return MP_OK;
  }
  MP_REQUIRE(out_host, "NULL out");
  const size_t bytes = (size_t)nz * R * R * sizeof(float);
  float* d_out = nullptr;
  mp_ensure_pool();
  MP_CUDA(cudaMallocAsync(&d_out, bytes, st));
  // Large slabs go out in a few z-chunks: the read-back of chunk k (copy stream, gated by an event) overlaps the evaluation of
  // chunk k+1, so only the last chunk's copy is exposed (257^3: 68 MB = 1.2 ms of a 35 ms call otherwise).
  const long long plane = (long long)R * R;
  const int n_chunks = (plane * nz >= (4ll << 20) && nz >= 8) ? 4 : 1;
  // one copy stream per device (shared by concurrent callers: it only orders copies); the events are per call
  cudaStream_t copy_st = nullptr;
  cudaEvent_t ev_done[4] = {nullptr, nullptr, nullptr, nullptr}, ev_copied = nullptr;
  int rc = MP_OK;
  if (n_chunks > 1) {
    static std::mutex mu;
    static cudaStream_t per_device[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess && dev >= 0 && dev < 64) {
      std::lock_guard<std::mutex> lock(mu);
      if (!per_device[dev]) e = cudaStreamCreateWithFlags(&per_device[dev], cudaStreamNonBlocking);
      copy_st = per_device[dev];
    }
    for (int k = 0; k < 4 && e == cudaSuccess; ++k) e = cudaEventCreateWithFlags(&ev_done[k], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_copied, cudaEventDisableTiming);
    if (e != cudaSuccess || !copy_st) { mp_set_error("copy stream: %s", cudaGetErrorString(e)); rc = MP_E_CUDA; }
  }
  for (int k = 0; k < n_chunks && rc == MP_OK; ++k) {
    const int za = (int)((long long)nz * k / n_chunks), zb = (int)((long long)nz * (k + 1) / n_chunks);
    float* d_chunk = d_out + (size_t)za * plane;
    rc = mp_query_grid(mlp, feat, R, z0 + za, zb - za, b_min3, b_max3, calib12, projection, z_scale, d_chunk, mode, stream);
    if (rc != MP_OK) break;
    cudaError_t e;
    if (n_chunks == 1) {
      e = cudaMemcpyAsync(out_host, d_out, bytes, cudaMemcpyDeviceToHost, st);
    } else {
      e = cudaEventRecord(ev_done[k], st);
      if (e == cudaSuccess) e = cudaStreamWaitEvent(copy_st, ev_done[k], 0);
      if (e == cudaSuccess) e = cudaMemcpyAsync(out_host + (size_t)za * plane, d_chunk, (size_t)(zb - za) * plane * sizeof(float),
                                                cudaMemcpyDeviceToHost, copy_st);
    }
    if (e != cudaSuccess) { mp_set_error("D2H failed: %s", cudaGetErrorString(e)); rc = MP_E_CUDA; }
  }
  if (n_chunks > 1 && copy_st && ev_copied) {
    // the caller's stream (and the free below) waits for the last copy
    cudaError_t e = cudaEventRecord(ev_copied, copy_st);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(st, ev_copied, 0);
    if (e != cudaSuccess && rc == MP_OK) { mp_set_error("D2H failed: %s", cudaGetErrorString(e)); rc = MP_E_CUDA; }
  }
  cudaFreeAsync(d_out, st);
  cudaError_t e = cudaStreamSynchronize(st);
  if (rc == MP_OK && e != cudaSuccess) { mp_set_error("sync failed: %s", cudaGetErrorString(e)); rc = MP_E_CUDA; }
  for (int k = 0; k < 4; ++k) if (ev_done[k]) cudaEventDestroy(ev_done[k]);
  if (ev_copied) cudaEventDestroy(ev_copied);
  return rc;
}
