// F3': visible-surface extraction.  Replaces forward_vertices (RTL/recon.py:27-89): for every (x,y) column of the
// view-aligned volume find the first occupied (>0.5) node along the view axis, its sub-voxel depth by linear
// interpolation with the node two steps before it, and a finite-difference normal.  At most one vertex per column,
// emitted in (x,y) row-major order == the order of keep.nonzero() in the reference (:62).
// HBM-bound: one read of the volume (columns are walked with x fastest across the warp => coalesced).
#include "mp_common.cuh"
#include "surface_kernels.cuh"

using namespace surface_k;


static size_t scratch_layout(int R, size_t* sums_off) {
  const long long n = (long long)R * R;
  size_t first = ((size_t)n * sizeof(int32_t) + 255) / 256 * 256;
  if (sums_off) *sums_off = first;
  return first + (size_t)(mpscan::num_blocks(n) + 3) * sizeof(unsigned long long);
}

extern "C" int64_t mp_forward_vertices_scratch_bytes(int R) { return R >= 2 ? (int64_t)scratch_layout(R, nullptr) : 0; }

// Enqueue-only variant (graph-capturable): no allocation, no host read-back.  `scratch_dev`: at least
// mp_forward_vertices_scratch_bytes(R) bytes; `count_dev`: one int64 on the device = number of vertices written.
extern "C" int mp_forward_vertices_async(const float* vol_dev, int R, int direction, int64_t* x_dev, int64_t* y_dev, float* z_dev,
                                         float* norm_dev, int64_t* count_dev, void* scratch_dev, void* stream) {
  MP_REQUIRE(vol_dev && x_dev && y_dev && z_dev && norm_dev && count_dev && scratch_dev, "NULL argument");
  MP_REQUIRE(R >= 2 && R <= 2048, "bad R=%d", R);
  MP_REQUIRE(direction >= 0 && direction <= 3, "bad direction %d", direction);
  MpRange nvtx("monoport_b200: F3' visible surface");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)R * R;
  size_t sums_off = 0;
  scratch_layout(R, &sums_off);
  int32_t* first_t = reinterpret_cast<int32_t*>(scratch_dev);
  unsigned long long* sums = reinterpret_cast<unsigned long long*>(reinterpret_cast<uint8_t*>(scratch_dev) + sums_off);
  unsigned long long* total = sums + mpscan::num_blocks(n) + 1;
  MP_CUDA(cudaMemsetAsync(total + 1, 0, sizeof(unsigned long long), st));   // ticket counter of the scan
  const int grid = (int)((n + kHitCols - 1) / kHitCols);
  first_hit_kernel<<<grid, kHitCols * kHitSlices, 0, st>>>(vol_dev, R, direction, first_t);
  HitF f{first_t};
  HitEmit em{vol_dev, first_t, R, direction, (long long*)x_dev, (long long*)y_dev, z_dev, norm_dev};
  MP_CUDA(mpscan::scan_emit(f, em, n, sums, total, st));
  MP_CUDA(cudaMemcpyAsync(count_dev, total, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
  return MP_OK;
}

// The normal image of the demo, enqueue-only (graph-capturable): the count is read on the device.
extern "C" int mp_render_normals_async(const int64_t* x_dev, const int64_t* y_dev, const float* norm_dev, const int64_t* count_dev,
                                       int64_t capacity, int R, float* canvas_dev, void* stream) {
  MP_REQUIRE(x_dev && y_dev && norm_dev && count_dev && canvas_dev, "NULL argument");
  MP_REQUIRE(capacity >= 0 && R >= 1 && capacity <= (int64_t)R * R, "bad sizes capacity=%lld R=%d", (long long)capacity, R);
  if (capacity == 0) return MP_OK;
  const long long blocks = (capacity + kNormThreads - 1) / kNormThreads;
  const int grid = (int)(blocks < 1024 ? blocks : 1024);
  render_normals_kernel<<<grid, kNormThreads, 0, (cudaStream_t)stream>>>(
      (const long long*)x_dev, (const long long*)y_dev, norm_dev, (const long long*)count_dev, capacity, R, canvas_dev);
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

extern "C" int mp_forward_vertices(const float* vol_dev, int R, int direction, int64_t* x_dev, int64_t* y_dev,
                                   float* z_dev, float* norm_dev, int64_t* n_out, void* stream) {
  MP_REQUIRE(vol_dev && x_dev && y_dev && z_dev && norm_dev && n_out, "NULL argument");
  MP_REQUIRE(R >= 2 && R <= 2048, "bad R=%d", R);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* scratch = nullptr;
  mp_ensure_pool();
  const size_t bytes = scratch_layout(R, nullptr) + 16;       // + the device-side count
  MP_CUDA(cudaMallocAsync(&scratch, bytes, st));
  int64_t* count_dev = reinterpret_cast<int64_t*>(scratch + bytes - 16);
  int rc = mp_forward_vertices_async(vol_dev, R, direction, x_dev, y_dev, z_dev, norm_dev, count_dev, scratch, stream);
  long long tot = 0;
  cudaError_t e = cudaSuccess;
  if (rc == MP_OK) e = cudaMemcpyAsync(&tot, count_dev, sizeof(tot), cudaMemcpyDeviceToHost, st);
  cudaFreeAsync(scratch, st);                                  // (freed on every path)
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (rc != MP_OK) return rc;
  if (e != cudaSuccess) {
    mp_set_error("mp_forward_vertices: %s", cudaGetErrorString(e));
    return MP_E_CUDA;
  }
  *n_out = (int64_t)tot;
  return MP_OK;
}
