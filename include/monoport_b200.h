/*
 * monoport_b200 -- C ABI of the H100-native occupancy-field hot path of MonoPort.
 *
 * The reference (Project-Splinter/MonoPort) is pure Python: it has no FFI.  Its boundary for this path is
 * a Python call protocol (SURVEY.md §8b).  This header is the C-ABI a binding for that protocol
 * would call; every entry point names the reference interface it replaces (paths relative to the
 * reference tree).  Plain pointers and sizes only -- no torch types.  INTEGRATION.md shows the ctypes
 * stub (monoport_b200/_lib.py is that stub).
 *
 * Conventions
 *   - every function returns MP_OK (0) or a negative MP_E_* code; mp_last_error() gives a thread-local
 *     message.  An empty reconstruction is NOT an error (RTL/recon.py:32-33 tolerates None).
 *   - "dev" pointers are CUDA device pointers of the current device, "host" pointers are host memory.
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream).  Calls are asynchronous
 *     on that stream unless stated otherwise.  No process-global mutable state: all scratch lives in
 *     the handles, so netG and netC queries may run concurrently from different threads
 *     (RTL/dataloader.py:734-751 runs every stage in its own thread).
 *   - volumes are [D,H,W] = [z,y,x] float32, x fastest (RTL/recon.py:35-38).
 */
#ifndef MONOPORT_B200_H_
#define MONOPORT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MP_OK 0
#define MP_E_INVALID (-1)   /* bad argument                                  */
#define MP_E_CUDA (-2)      /* a CUDA runtime call failed                    */
#define MP_E_UNSUPPORTED (-3) /* shape / mode not supported by this kernel   */
#define MP_E_CAPACITY (-4)  /* caller-provided output buffer too small       */
#define MP_E_NOMEM (-5)
#define MP_E_RANGE (-6)     /* inputs outside the validated range of the requested fast path; use the exact one */
#define MP_E_TRUNCATED (-7) /* a device-driven loop stopped at its cap: the result is incomplete; use the eager call */

/* last_op of the head: heads/SurfaceClassifier.py:68-69 (None / nn.Sigmoid / nn.Tanh) */
#define MP_LAST_NONE 0
#define MP_LAST_SIGMOID 1
#define MP_LAST_TANH 2

/* projection: geometry.py:19-34 (orthogonal) / :37-55 (perspective) */
#define MP_PROJ_ORTHOGONAL 0
#define MP_PROJ_PERSPECTIVE 1

/* arithmetic of the fused sample+MLP kernel */
#define MP_MODE_FP32 0   /* CUDA-core fp32 everywhere (|err| ~1e-6 vs the reference)                 */
#define MP_MODE_TC 1     /* wgmma fp16 operands / fp32 register accumulators, last layer fp32 (<=1e-4)   */
#define MP_MODE_AUTO 2   /* TC when the head/feature shape is supported by the wgmma kernel, else FP32 */
/* 3 was MP_MODE_TC_V2 (the self-contained tensor-core program, removed in round 2: 335 vs 485 Mpoints/s); rejected now */
#define MP_MODE_TC_V3 4  /* alias of MP_MODE_TC: the one tensor-core program (layer 0 hoisted to texels)                     */

const char* mp_last_error(void);
int mp_version(void);
/* sm count / compute capability of the current device */
int mp_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---------------------------------------------------------------------------------------------
 * Head weights.  Replaces the parameters of SurfaceClassifier (heads/SurfaceClassifier.py:7-37):
 * `channels` = filter_channels (n_layers+1 entries, e.g. {257,1024,512,256,128,1});
 * weights[l] is filters.l.weight as [Cout_l, Cin_l] row-major fp32 with Cin_l = channels[l] +
 * (l>0 && skip ? channels[0] : 0)  (:24-34), biases[l] is [Cout_l].  skip = !no_residual.
 * Pointers are host (on_device=0) or device (on_device=1) memory; they are only read during the call.
 * The handle owns repacked copies (fp32 K-major for the CUDA-core kernel, fp16 K-major SWIZZLE_128B tiles for the wgmma kernel).
 * ------------------------------------------------------------------------------------------- */
typedef struct mp_mlp mp_mlp_t;
int mp_mlp_create(int n_layers, const int* channels, const float* const* weights,
                  const float* const* biases, int skip, int last_op, int on_device, mp_mlp_t** out);
int mp_mlp_destroy(mp_mlp_t* h);
/* 1 if MP_MODE_TC is available for this head on this device */
int mp_mlp_tc_supported(const mp_mlp_t* h);
/* Validated range of the tensor-core program (no reference counterpart: the reference computes in fp32 throughout,
 * MonoPortNet.py:86-89).  MP_MODE_TC / MP_MODE_AUTO evaluate a frame on the tensor cores only while its largest
 * |feature| stays under `limit` (defaults: 12 geometry head, 8 colour head -- both keep |error| <= 1e-4 on what query()
 * returns); frames above it take the exact fp32 kernel.  The choice is made on the device from the frame itself.
 * +infinity disables the guard. */
int mp_mlp_set_tc_feature_limit(mp_mlp_t* h, float limit);

/* ---------------------------------------------------------------------------------------------
 * Feature volume.  Replaces the tensor index() samples (geometry.py:4-16): one [C,H,W] fp32 NCHW map
 * (the last hourglass stage in eval mode, MonoPortNet.py:63-64).  The handle keeps a channel-last fp32
 * copy so one bilinear tap is one contiguous vector (taps are always read in fp32).
 * ------------------------------------------------------------------------------------------- */
typedef struct mp_feat mp_feat_t;
int mp_feat_create(int C, int H, int W, mp_feat_t** out);
int mp_feat_upload(mp_feat_t* h, const float* nchw, int on_device, void* stream);
/* same for a map that is already channel-last ([H,W,C] fp32, device memory -- a torch.channels_last tensor): one copy, no
 * transposing kernel */
/* Zero-copy variant: the handle reads the caller's channel-last [H,W,C] fp32 device map IN PLACE for this frame (what a
 * channels_last encoder emits, HGFilters.py:158-159 / RTL/main.py:382-387: no repack kernel, no copy).  The memory must stay
 * valid and unchanged until the frame's queries have completed; the next upload / bind replaces the binding. */
int mp_feat_bind_nhwc(mp_feat_t* h, const float* nhwc_dev, void* stream);
int mp_feat_upload_nhwc(mp_feat_t* h, const float* nhwc_dev, void* stream);
int mp_feat_destroy(mp_feat_t* h);
/* A handle that holds B maps of [C,H,W] -- the features of a batch [B,C,H,W] (MonoPortNet.py:48-91 takes any B).
 * mp_feat_create(C,H,W) is the B = 1 case.  On such a handle the three calls above read B contiguous maps: mp_feat_upload a
 * [B,C,H,W] NCHW block, mp_feat_upload_nhwc / mp_feat_bind_nhwc a [B,H,W,C] block (the memory of a torch.channels_last
 * [B,C,H,W] tensor).  Only mp_query_points_batch evaluates a handle with B > 1; every other entry point that takes an
 * mp_feat_t* returns MP_E_INVALID for it.
 * Memory: besides the B fp32 maps (and a staging copy for host uploads) the tensor-core program keeps per-texel products for
 * every map -- per 128 x 128 map, G0 = 33.5 MB and the fp16 copy of the map 8.4 MB (16.8 MB for the colour head's 512
 * channels): a batch of 8 geometry maps holds about 0.34 GB of them. */
int mp_feat_create_batch(int B, int C, int H, int W, mp_feat_t** out);

/* calib: 12 host floats = rows 0..2 of the [4,4] / [3,4] calibration (R | t), or NULL for calibs=None
 * (MonoPortNet.py:66-67).  z_scale = DepthNormalizer scale (normalizers/DepthNormalizer.py:32,40). */

/* MonoPortNet.query(feats, points[1,3,N], calibs) -> [Res,N]   (MonoPortNet.py:48-91)
 * points_dev: coordinate a (0..2) of point i lives at points_dev[a*row_stride + i*point_stride]  -- (N,1) for a
 * contiguous [3,N] tensor, (1,3) for the permuted [N,3] view RTL/main.py:176-177 passes.
 * out_dev: [Res, N], row stride ld_out. */
int mp_query_points(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                    int64_t point_stride, const float* calib12, int projection, float z_scale, float* out_dev,
                    int64_t ld_out, int mode, void* stream);
/* MonoPortNet.query(feats[B,C,H,W], points[B,3,N], calibs[B,3|4,4]) -> [B,Res,N] in ONE launch (tiles of 64 points never
 * straddle two images).  B must equal the handle's batch (mp_feat_create_batch).  Coordinate a of point i of image b lives
 * at points_dev[b*batch_stride + a*row_stride + i*point_stride]; its channel c goes to out_dev[b*out_batch_stride +
 * c*ld_out + i].  calibs_dev: [B][12] fp32 in DEVICE memory (rows 0..2 of every [R|t]) or NULL for calibs=None -- nothing is
 * read back to the host, the call does not synchronise.  All modes; MP_MODE_TC / MP_MODE_AUTO take the range guard per
 * image: the tiles of an image whose largest |feature| is above the head's limit are evaluated by the exact fp32 kernel. */
int mp_query_points_batch(mp_mlp_t* mlp, mp_feat_t* feat, int B, const float* points_dev, int64_t n, int64_t batch_stride,
                          int64_t row_stride, int64_t point_stride, const float* calibs_dev, int projection, float z_scale,
                          float* out_dev, int64_t out_batch_stride, int64_t ld_out, int mode, void* stream);
/* Gradient of MonoPortNet.query (mp_query_points, MP_MODE_FP32) with respect to the points: exact fp32 on CUDA cores, one
 * fused launch (forward pass + reverse pass through the projection, the bilinear taps, the depth column and the skip MLP).
 * dpoints_dev: [3][ld_dpoints], coordinate a of point i at dpoints_dev[a*ld_dpoints + i] = d(sum_c grad_out[c,i] * out[c,i]) /
 * d points[a,i].  grad_out_dev: [Res][ld_grad], or NULL for all ones (the geometry head then gives grad sigma).
 * out_dev: [Res][ld_out], the value -- bit-identical to mp_query_points in MP_MODE_FP32 -- or NULL to skip it.  Points
 * outside the image get value 0 and gradient exactly 0 (in_img multiplies the output, MonoPortNet.py:89); at a
 * leaky-ReLU kink the derivative of the non-positive side is taken (torch's convention).  Single-map handles only. */
int mp_query_points_grad(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                         int64_t point_stride, const float* calib12, int projection, float z_scale, const float* grad_out_dev,
                         int64_t ld_grad, float* out_dev, int64_t ld_out, float* dpoints_dev, int64_t ld_dpoints, void* stream);
/* mp_query_points_grad with a precision mode and an optional point count on the device (count_dev: one int32, or NULL;
 * n is then the capacity and the points at or beyond min(*count_dev, n) are not touched).  Enqueue-only: nothing is read
 * back to the host, so the call can be captured in a CUDA graph.
 *   MP_MODE_FP32: the exact kernel, bit for bit mp_query_points_grad.
 *   MP_MODE_TC:   the tensor-core program's forward-mode derivative (three tangents per point carried as extra rows of the
 *                 wgmma program); its value is mp_query_points' MP_MODE_TC value bit for bit.  A frame whose largest
 *                 |feature| is above the head's limit is differentiated by the exact kernel instead, decided on the device
 *                 (as mp_query_points decides it).  Maps above 65536 texels are refused.
 *   MP_MODE_AUTO: MP_MODE_TC where the head and the map allow it, else MP_MODE_FP32.
 * Single-map handles only. */
int mp_query_points_grad_mode(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                              int64_t point_stride, const float* calib12, int projection, float z_scale, const float* grad_out_dev,
                              int64_t ld_grad, float* out_dev, int64_t ld_out, float* dpoints_dev, int64_t ld_dpoints,
                              const int32_t* count_dev, int mode, void* stream);
/* The vector-Jacobian product of MonoPortNet.query in MP_MODE_FP32, for training: with S = sum(grad_out * query(feats,
 * points, calibs)) over B images (the exact values, mp_query_points / mp_query_points_batch), every requested one of
 *   dfeat_dev      [B][C][H][W] = dS / d features (NCHW, like the map mp_feat_upload takes),
 *   dpoints_dev    [B][3][n]    = dS / d points (what mp_query_points_grad gives for B = 1, bit for bit),
 *   dweights_dev   n_layers device pointers, [Cout_l][Cin_l] = dS / d filters.l.weight (mp_mlp_create's layout),
 *   dbiases_dev    n_layers device pointers, [Cout_l]       = dS / d filters.l.bias
 * (NULL, or a NULL entry: not computed, and costs nothing).  Exact fp32 on CUDA cores, every head the exact kernel takes; the
 * feature handle may hold one map or B (mp_feat_create_batch).  Points as for mp_query_points_batch; calibs_dev: [B][12] fp32
 * in device memory (rows 0..2 of [R|t]) or NULL for calibs=None.  grad_out_dev: [B][Res][n] fp32 (NULL: all ones).  Points
 * outside the image contribute nothing (in_img multiplies the output, MonoPortNet.py:89).  Outputs are overwritten.
 * The weight gradients are contracted chunk by chunk from rows the kernel saves in scratch_dev; the feature gradient is
 * gathered in it before its layout step.  scratch_bytes: at least mp_query_points_vjp_scratch_bytes(...) for the same
 * requests; a larger scratch holds larger chunks.  The weight, bias and point gradients are deterministic for one scratch
 * size; the feature gradient is accumulated with atomics (like grid_sample's backward) and is not, unless it is asked for
 * in order (mp_query_points_vjp_ex, MP_VJP_DETERMINISTIC).  No range guard, no tensor-core variant.  Enqueue-only: nothing is read back to the host. */
int mp_query_points_vjp(mp_mlp_t* mlp, mp_feat_t* feat, int B, const float* points_dev, int64_t n, int64_t batch_stride,
                        int64_t row_stride, int64_t point_stride, const float* calibs_dev, int projection, float z_scale,
                        const float* grad_out_dev, float* dfeat_dev, float* dpoints_dev, float* const* dweights_dev,
                        float* const* dbiases_dev, void* scratch_dev, int64_t scratch_bytes, void* stream);
/* Scratch bytes of mp_query_points_vjp for B images of n points, the weight gradients contracted in chunks of chunk_points
 * points (<= 0: all points in one chunk; about 16 KB per point for the geometry head), want_dfeat / want_dweights: whether
 * the feature / weight gradients are requested (neither: 0 bytes).  Negative: an MP_E_* code. */
int64_t mp_query_points_vjp_scratch_bytes(mp_mlp_t* mlp, mp_feat_t* feat, int B, int64_t n, int64_t chunk_points, int want_dfeat,
                                          int want_dweights);
/* flags of mp_query_points_vjp_ex.  MP_VJP_DETERMINISTIC: the feature gradient is summed in a fixed order instead of with
 * atomics -- per chunk of chunk_points points, the points are sorted by the cell of their nw tap (stably, so in point order
 * within a cell) and each element of dfeat is summed by one thread over the four cells whose points reach it, in point
 * order, then added to the previous chunks' sum.  dfeat is then the same bits from run to run and whatever else is
 * requested, for one chunk size. */
#define MP_VJP_DETERMINISTIC 1
/* mp_query_points_vjp and its scratch size with flags (0: exactly the calls above).  With MP_VJP_DETERMINISTIC the scratch
 * also holds, per chunk, dX[:C], the tap weights and the cell key of every point and the buffers of the sort, and the
 * feature gradient is chunked by chunk_points whether or not the weight gradients are requested; B * H * W must be below
 * 2^32 - 1.  Enqueue-only. */
int mp_query_points_vjp_ex(mp_mlp_t* mlp, mp_feat_t* feat, int B, const float* points_dev, int64_t n, int64_t batch_stride,
                           int64_t row_stride, int64_t point_stride, const float* calibs_dev, int projection, float z_scale,
                           const float* grad_out_dev, float* dfeat_dev, float* dpoints_dev, float* const* dweights_dev,
                           float* const* dbiases_dev, void* scratch_dev, int64_t scratch_bytes, int flags, void* stream);
int64_t mp_query_points_vjp_scratch_bytes_ex(mp_mlp_t* mlp, mp_feat_t* feat, int B, int64_t n, int64_t chunk_points,
                                             int want_dfeat, int want_dweights, int flags);
/* mp_query_points with an optional point count on the device (count_dev: one int32, or NULL): n is then the capacity and
 * the points at or beyond min(*count_dev, n) are neither read nor written.  Enqueue-only like mp_query_points; the same
 * modes, range guard and kernels.  Single-map handles only. */
int mp_query_points_count(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                          int64_t point_stride, const float* calib12, int projection, float z_scale, float* out_dev,
                          int64_t ld_out, const int32_t* count_dev, int mode, void* stream);
/* Device-calibration twins (_dcal) of the enqueue-only calls mp_query_points_count, mp_octree_run_fused_async,
 * mp_colorize_surface_async, mp_surface_normals_async and mp_mesh_normals_async: calib_dev in place of calib12 is 12 float32
 * values in DEVICE memory, rows 0..2 of [R|t] like calib12, read by the kernels when they run -- a captured CUDA graph
 * then follows whatever camera the caller writes there before each replay.  NULL is refused (a call without a camera is
 * its twin with calib12 == NULL).  projection and z_scale stay arguments.  Everything else -- arguments, modes, range guard,
 * refusals -- is the twin's, and so are the results: bit for bit what the twin gives with the same 12 floats. */
int mp_query_points_count_dcal(mp_mlp_t* mlp, mp_feat_t* feat, const float* points_dev, int64_t n, int64_t row_stride,
                               int64_t point_stride, const float* calib_dev, int projection, float z_scale, float* out_dev,
                               int64_t ld_out, const int32_t* count_dev, int mode, void* stream);
/* Same call with HOST buffers (points [3,N], out [Res,N], feature map NCHW fp32 or NULL to reuse the
 * uploaded one): copies in, runs, copies out, synchronises.  This is what bench.py's e2e leg times. */
int mp_query_points_host(mp_mlp_t* mlp, mp_feat_t* feat, const float* feat_nchw_host, const float* points_host,
                         int64_t n, const float* calib12, int projection, float z_scale, float* out_host,
                         int mode, void* stream);

/* Dense grid query: the node centres of planes [z0, z0+nz) of an R^3 grid spanning [b_min,b_max]
 * (world = (idx+0.5)/R*(b_max-b_min)+b_min, the engine's convention, cf. RTL/main.py:204-209) are generated
 * in-kernel; out_dev is the [nz,R,R] slab, channel 0 of the head (Res==1 required).  z-slab sharding
 * across GPUs (SURVEY.md §8e) calls this with a different [z0,nz) per rank. */
int mp_query_grid(mp_mlp_t* mlp, mp_feat_t* feat, int R, int z0, int nz, const float* b_min3, const float* b_max3,
                  const float* calib12, int projection, float z_scale, float* out_dev, int mode, void* stream);
/* The same for any contiguous range [lin0, lin0+n) of the grid's z-major linear node order (a z slab is the range
 * [z0*R*R, (z0+nz)*R*R)): balanced sharding over GPUs whose boundaries need not fall on plane boundaries (257 = 8*32+1:
 * with whole planes one rank carries 33 planes and the others 32).  out_dev receives n values. */
int mp_query_grid_range(mp_mlp_t* mlp, mp_feat_t* feat, int R, int64_t lin0, int64_t n, const float* b_min3,
                        const float* b_max3, const float* calib12, int projection, float z_scale, float* out_dev, int mode,
                        void* stream);

/* Fused slab exchange (SURVEY.md §8e, instead of the all-gather): the slab [z0, z0+nz) is evaluated like mp_query_grid,
 * but every value is stored straight into the FULL [R,R,R] volumes of all n_peers ranks (peer_vols: host array of
 * device pointers, the caller's own volume included; peers' volumes are peer-memory mappings obtained through
 * mp_ipc_open) while the tiles are computed -- compute and transfer in ONE kernel over NVLink.  The caller synchronises
 * the ranks afterwards (any barrier ordered after this call on `stream`); with two alternating volume sets one barrier
 * per frame suffices.  n_peers <= 8.  mp_query_grid_range_peers: the same for a range of the linear node order. */
int mp_query_grid_peers(mp_mlp_t* mlp, mp_feat_t* feat, int R, int z0, int nz, const float* b_min3, const float* b_max3,
                        const float* calib12, int projection, float z_scale, float* const* peer_vols, int n_peers,
                        int mode, void* stream);
int mp_query_grid_range_peers(mp_mlp_t* mlp, mp_feat_t* feat, int R, int64_t lin0, int64_t n, const float* b_min3,
                              const float* b_max3, const float* calib12, int projection, float z_scale,
                              float* const* peer_vols, int n_peers, int mode, void* stream);
/* Exportable device memory for such volumes: cudaMalloc + the 64-byte cudaIpcMemHandle_t to hand to the other ranks
 * (one process per GPU), which map it with mp_ipc_open (enables peer access) and unmap it with mp_ipc_close. */
int mp_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64);
int mp_ipc_open(const unsigned char* handle64, void** dev_ptr);
int mp_ipc_close(void* dev_ptr);
int mp_ipc_free(void* dev_ptr);

/* mp_query_grid with HOST buffers: uploads the NCHW fp32 feature map (NULL = reuse), evaluates the slab, copies
 * the [nz,R,R] result to out_host, synchronises.  Slabs of 4 M nodes or more are evaluated and read back in four z-chunks,
 * the copy of one chunk (internal copy stream) overlapping the evaluation of the next: pin out_host to get the overlap.
 * bench.py's e2e leg. */
int mp_query_grid_host(mp_mlp_t* mlp, mp_feat_t* feat, const float* feat_nchw_host, int R, int z0, int nz,
                       const float* b_min3, const float* b_max3, const float* calib12, int projection, float z_scale,
                       float* out_host, int mode, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Coarse-to-fine occupancy engine.  Replaces implicit_seg.functional.Seg3dLossless / Seg3dTopk
 * (third-party, un-vendored; call sites RTL/main.py:28-29,188-195,390-395).
 *   resolutions: n_levels odd cube sizes 2^k+1 (RTL/main.py:187), coarse -> fine.
 *   faster != 0 : RTL/main.py:195 mode (box dilation 9/7/3, last level interpolated only)
 *   faster == 0 : lossless mode (k=3, every level examined, conflict loop)
 *   topk_points : NULL for the boundary engine, else n_levels ints = nodes evaluated per level (Seg3dTopk)
 * Two ways to drive it:
 *   (a) stepping API -- the binding calls back into an arbitrary Python query_func per step
 *       (mp_octree_begin -> loop { mp_octree_next -> query -> mp_octree_commit });
 *   (b) mp_octree_run_fused -- the whole pyramid with the fused sample+MLP kernel, no host round trip per level.
 * ------------------------------------------------------------------------------------------- */
typedef struct mp_octree mp_octree_t;
int mp_octree_create(int n_levels, const int* resolutions, const float* b_min3, const float* b_max3,
                     float balance_value, int faster, const int* topk_points, mp_octree_t** out);
int mp_octree_destroy(mp_octree_t* h);
int mp_octree_begin(mp_octree_t* h, void* stream);
/* Produces the next batch of nodes to evaluate.  *n_out = number of nodes (0 => reconstruction finished);
 * *level_out = level they belong to.  points_dev_out: device pointer to [n,3] world-space points (owned by
 * the handle, valid until the next call), idx_dev_out: their linear indices (z*R*R+y*R+x) at that level.
 * Synchronises the stream (the count has to reach the host). */
int mp_octree_next(mp_octree_t* h, int64_t* n_out, int* level_out, const float** points_dev_out,
                   const int32_t** idx_dev_out, void* stream);
/* Scatter the n values ([n] floats, device) returned by the query for the batch handed out by the last
 * mp_octree_next. */
int mp_octree_commit(mp_octree_t* h, const float* values_dev, void* stream);
/* After the last step: copies the final [R,R,R] volume to out_dev.  *nonempty = 0 when level 0 had no
 * value > balance (the engine then returns None, RTL/recon.py:32-33) -- synchronises. */
int mp_octree_finish(mp_octree_t* h, float* out_dev, int* nonempty, void* stream);
/* Whole pyramid on the device.  stats_host (may be NULL): n_levels int64 = nodes evaluated per level.
 * Synchronises once at the end (to report nonempty/stats). */
int mp_octree_run_fused(mp_octree_t* h, mp_mlp_t* mlp, mp_feat_t* feat, const float* calib12, int projection,
                        float z_scale, int mode, float* out_dev, int* nonempty, int64_t* stats_host, void* stream);
/* Multi-GPU list sharding of mp_octree_run_fused (SURVEY.md §8e; one process per GPU, one handle per rank, same ctor
 * arguments).  Every rank keeps the whole pyramid and runs the volume passes itself -- identical inputs give identical
 * node lists, the lossless conflict loop included -- and evaluates only its window of each level's ordered node list
 * (balanced to one 128-point tile); the fused kernel stores the values into the value lists of ALL ranks over NVLink peer
 * memory and a flag barrier between the ranks' streams replaces the collective.  Every rank ends up with the full volume.
 *   mp_octree_shard_export : 3 x 64-byte IPC handles (two value lists, the barrier flags) to hand to the other ranks;
 *   mp_octree_shard_set    : rank / world and, per rank, the peer mappings of those three blocks (mp_ipc_open; entry
 *                            [rank] is ignored).  world == 1 switches sharding off.  All ranks must then call
 *                            mp_octree_run_fused the same number of times with the same inputs. */
/* The fused run in two halves for CUDA-graph captured frame steps: _async only enqueues (no host memory is read, no
 * synchronisation: capturable, every engine mode), mp_octree_fetch reads the non-empty flag and the per-level counts back
 * afterwards (synchronises).  In the lossless mode (faster == 0, no top-k) the conflict loop of each level runs as a
 * conditional WHILE node of the graph whose body is one pass (query, scatter with conflict detection, next conflict list)
 * and whose loop-control kernel decides on the device whether another pass runs -- the same nodes, order, values and
 * counts as mp_octree_run_fused's host-driven loop.  A level stops after 8 x its resolution passes at most.  On a stream
 * that is not being captured the call records its own sequence into a graph and launches that (still enqueue-only).
 * A sharded lossless handle is refused (MP_E_UNSUPPORTED).
 * mp_octree_fetch_loops: n_levels int32 = conflict-loop passes per level of the last _async run (0 for level 0 and for
 * the other modes); MP_E_TRUNCATED when a level stopped at its cap with nodes left to evaluate (run that frame with
 * mp_octree_run_fused).  Synchronises. */
int mp_octree_run_fused_async(mp_octree_t* h, mp_mlp_t* mlp, mp_feat_t* feat, const float* calib12, int projection,
                              float z_scale, int mode, float* out_dev, void* stream);
/* mp_octree_run_fused_async with the camera in device memory (see mp_query_points_count_dcal): every query launch of the
 * run, the bodies of the lossless WHILE nodes included, reads calib_dev when it runs.  A sharded handle is refused. */
int mp_octree_run_fused_async_dcal(mp_octree_t* h, mp_mlp_t* mlp, mp_feat_t* feat, const float* calib_dev, int projection,
                                   float z_scale, int mode, float* out_dev, void* stream);
int mp_octree_fetch(mp_octree_t* h, int* nonempty, int64_t* stats_host, void* stream);
int mp_octree_fetch_loops(mp_octree_t* h, int32_t* passes_per_level, void* stream);
int mp_octree_shard_export(mp_octree_t* h, unsigned char* handles192);
int mp_octree_shard_set(mp_octree_t* h, int rank, int world, float* const* vals0, float* const* vals1,
                        uint32_t* const* flags);

/* ---------------------------------------------------------------------------------------------
 * Marching cubes (absent from the reference; PIFu-style reconstruction() asked for by the north star).
 * Two calls: count (synchronises, returns sizes) then emit into caller buffers.
 *   verts: [nV,3] float32 (x,y,z) in index space; faces: [nF,3] int32.
 * Deterministic: vertex ids follow (node, axis) order, faces follow (cell, table) order.
 * ------------------------------------------------------------------------------------------- */
typedef struct mp_mcubes mp_mcubes_t;
int mp_mcubes_create(int D, int H, int W, mp_mcubes_t** out);
int mp_mcubes_destroy(mp_mcubes_t* h);
int mp_mcubes_count(mp_mcubes_t* h, const float* vol_dev, float iso, int64_t* n_verts, int64_t* n_faces, void* stream);
int mp_mcubes_emit(mp_mcubes_t* h, const float* vol_dev, float iso, float* verts_dev, int32_t* faces_dev, void* stream);
/* Count and emission in one enqueue-only call (no host read, no allocation, no synchronisation: graph-capturable, and a
 * graph may replay it on the same handle).  The mesh is mp_mcubes_count + mp_mcubes_emit's, id for id, into caller buffers
 * of v_cap vertices [v_cap][3] and f_cap faces [f_cap][3]: a vertex with id >= v_cap and a face with index >= f_cap are not
 * written.  counts_dev (int64[2]) receives the true totals (nV, nF), so the caller can detect an overflow; count32_dev (one
 * int32) receives min(nV, v_cap), the point count of mp_query_points_count / mp_mesh_normals_async at the vertices.
 * world: NULL for index space, else 7 host floats {R, b_min[3], b_max[3]}: vertex v is stored as
 * (v + 0.5) * ((b_max - b_min) / R) + b_min with torch's fp32 roundings (reconstruction()'s vertices bit for bit).
 * Does not change what mp_mcubes_count / mp_mcubes_emit see on the handle. */
int mp_mcubes_run_async(mp_mcubes_t* h, const float* vol_dev, float iso, const float* world, int64_t v_cap, int64_t f_cap,
                        float* verts_dev, int32_t* faces_dev, int64_t* counts_dev, int32_t* count32_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Visible-surface extraction.  Replaces forward_vertices (RTL/recon.py:27-89).
 * direction: 0 front, 1 back, 2 left, 3 right.  Outputs (device, capacity R*R): X,Y int64, Z float, norm [n,3].
 * *n_out on the host (synchronises).
 * ------------------------------------------------------------------------------------------- */
int mp_forward_vertices(const float* vol_dev, int R, int direction, int64_t* x_dev, int64_t* y_dev, float* z_dev,
                        float* norm_dev, int64_t* n_out, void* stream);
/* Enqueue-only variant for CUDA-graph captured frame steps (SURVEY.md §8f-2; the reference overlaps its stages with one
 * Python thread per processor, RTL/dataloader.py:734-751): no allocation, no host read-back.  scratch_dev: at least
 * mp_forward_vertices_scratch_bytes(R) bytes of device memory; count_dev: one int64 on the device. */
int64_t mp_forward_vertices_scratch_bytes(int R);
int mp_forward_vertices_async(const float* vol_dev, int R, int direction, int64_t* x_dev, int64_t* y_dev, float* z_dev,
                              float* norm_dev, int64_t* count_dev, void* scratch_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The demo's display images (visulization, RTL/main.py:252-281), enqueue-only (graph-capturable): the [R,R,3] float32
 * canvases norm_dev / tex_dev (either may be NULL, not both) become [S,S,3] float32 images C * 255, rotated by
 * torch.rot90(k=1, dims [0,1]) and resized by nearest F.interpolate, bit for bit what torch gives (NaN stays NaN); and an
 * [S,S] uint8 mask, 0 where the three values of the reference image (the texture image if present, else the normal
 * image) all equal 255 and 1 elsewhere.  One kernel into staging_dev (3 * S*S floats per present image + S*S floats),
 * then one device-to-host copy per output into page-locked host memory (norm_host / tex_host for the present images,
 * mask_host always).  Refuses (MP_E_INVALID) NULL for both images, R < 1 or S < 1, a NULL output or staging buffer,
 * and a host output that is not page-locked.  The host outputs hold the result once the stream has reached this call.
 * ------------------------------------------------------------------------------------------- */
int mp_display_async(const float* norm_dev, const float* tex_dev, int R, int S, float* norm_host, float* tex_host,
                     uint8_t* mask_host, float* staging_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Direct rendering of the visible surface with the colour head.  Replaces colorization (RTL/main.py:212-249): vertex i =
 * (X[i], Y[i], R - Z[i]) of mp_forward_vertices -> world space by mat_color (:201-210) -> netC.query -> pred*0.5+0.5 ->
 * canvas[X[i], Y[i], :]  ([R,R,3] float32, prepared by the caller), in ONE launch without intermediate tensors.
 * Needs the tensor-core program of the colour head (MP_E_UNSUPPORTED otherwise) and a frame inside its validated feature
 * range (MP_E_RANGE otherwise, see mp_mlp_set_tc_feature_limit) -- the binding then takes the generic mp_query_points
 * route.
 * ------------------------------------------------------------------------------------------- */
int mp_colorize_surface(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev, const float* z_dev,
                        int64_t n, int R, const float* b_min3, const float* b_max3, const float* calib12, int projection,
                        float z_scale, float* canvas_dev, void* stream);
/* The same render for CUDA-graph captured frame steps: enqueue-only (no host read, no allocation, no synchronisation).
 * The vertex count is the int64 count_dev of mp_forward_vertices_async, read on the device and clamped to `capacity` (the
 * length of the x/y/z buffers, at most R*R); vertices at or beyond it are neither evaluated nor drawn.  `mode` as for
 * mp_query_points: MP_MODE_FP32 renders with the exact fp32 kernel; MP_MODE_TC / MP_MODE_AUTO with the tensor-core program
 * when the frame's largest |feature| is inside the head's limit and with the exact kernel when it is not, decided on the
 * device (MP_MODE_AUTO without a tensor-core program: the exact kernel).  Any head with 3 outputs; single-map handles. */
int mp_colorize_surface_async(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev, const float* z_dev,
                              const int64_t* count_dev, int64_t capacity, int R, const float* b_min3, const float* b_max3,
                              const float* calib12, int projection, float z_scale, int mode, float* canvas_dev, void* stream);
/* mp_colorize_surface_async with the camera in device memory (see mp_query_points_count_dcal). */
int mp_colorize_surface_async_dcal(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev, const float* z_dev,
                                   const int64_t* count_dev, int64_t capacity, int R, const float* b_min3, const float* b_max3,
                                   const float* calib_dev, int projection, float z_scale, int mode, float* canvas_dev,
                                   void* stream);
/* The normal image of the demo (RTL/main.py:212-228, colorization(norm=...)): canvas[X[i], Y[i], :] =
 * clamp((norm[i] + 1) / 2, 0, 1) for the first min(*count_dev, capacity) vertices, bit for bit what torch gives (NaN
 * normals stay NaN).  Enqueue-only like the call above; capacity <= R*R. */
int mp_render_normals_async(const int64_t* x_dev, const int64_t* y_dev, const float* norm_dev, const int64_t* count_dev,
                            int64_t capacity, int R, float* canvas_dev, void* stream);
/* Analytic normals of the visible surface, enqueue-only (graph-capturable): for the first min(*count_dev, capacity) vertices
 * (X, Y, Z) of mp_forward_vertices_async (int64 count on the device), the geometry head's gradient at the world point
 * (X, Y, R - Z) through mat_color (the points mp_colorize_surface_async renders) -> norm_dev[i] = -(g_x L_x, g_y L_y,
 * -g_z L_z) / R normalised (L = b_max - b_min), zero where the gradient vanishes: forward_vertices' frame and sign.
 * mode: as mp_query_points_grad_mode.  scratch_dev: 6 * capacity + 1 floats of device memory.  Heads with one output,
 * single-map handles; capacity <= R*R.  norm_dev can then be drawn with mp_render_normals_async. */
int mp_surface_normals_async(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev, const float* z_dev,
                             const int64_t* count_dev, int64_t capacity, int R, const float* b_min3, const float* b_max3,
                             const float* calib12, int projection, float z_scale, int mode, float* scratch_dev, float* norm_dev,
                             void* stream);
/* mp_surface_normals_async with the camera in device memory (see mp_query_points_count_dcal). */
int mp_surface_normals_async_dcal(mp_mlp_t* mlp, mp_feat_t* feat, const int64_t* x_dev, const int64_t* y_dev, const float* z_dev,
                                  const int64_t* count_dev, int64_t capacity, int R, const float* b_min3, const float* b_max3,
                                  const float* calib_dev, int projection, float z_scale, int mode, float* scratch_dev,
                                  float* norm_dev, void* stream);
/* Analytic normals at mesh vertices, enqueue-only: verts_dev = mp_mcubes_run_async's world-space [capacity][3] vertices,
 * counts_dev / count32_dev its counts (the first min(counts_dev[0], capacity) vertices are evaluated).  norm_dev[i] =
 * -g / |g| with g the geometry head's gradient at vertex i (zero where it vanishes), as reconstruction(normals=True) gives
 * it.  mode: as mp_query_points_grad_mode.  scratch_dev: 3 * capacity floats.  Heads with one output, single-map handles. */
int mp_mesh_normals_async(mp_mlp_t* mlp, mp_feat_t* feat, const float* verts_dev, const int64_t* counts_dev,
                          const int32_t* count32_dev, int64_t capacity, const float* calib12, int projection, float z_scale,
                          int mode, float* scratch_dev, float* norm_dev, void* stream);
/* mp_mesh_normals_async with the camera in device memory (see mp_query_points_count_dcal). */
int mp_mesh_normals_async_dcal(mp_mlp_t* mlp, mp_feat_t* feat, const float* verts_dev, const int64_t* counts_dev,
                               const int32_t* count32_dev, int64_t capacity, const float* calib_dev, int projection,
                               float z_scale, int mode, float* scratch_dev, float* norm_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MONOPORT_B200_H_ */
