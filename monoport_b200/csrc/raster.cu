// F3.2: the frame's mesh drawn from viewer cameras -- the normal and colour programs of the reference's GL renderer
// (NormalRender / ColorRender with shaders/normal.* and color.*) as a deterministic rasterizer (DESIGN.md §F3.2; PARITY WITH GL
// UNPINNED, bit-exact against tests/raster_ref.py).  Enqueue-only and graph-capturable: every grid is fixed from the
// capacities, the vertex and face counts and the large-face list length are read on the device.
//   memset nodes: the depth keys to all ones, the list length to 0
//   raster_setup_kernel : (view, face) -> transform, classify, snap; small faces drawn in the thread, the others listed
//   raster_large_kernel : a CTA per listed face -> clipping, then the pieces' pixel boxes tiled by the CTA
//   raster_resolve_kernel: a thread per pixel per view -> the winning face shaded into the normal and / or colour image
#include "mp_common.cuh"
#include "raster_kernels.cuh"

using namespace mraster;

static size_t raster_align(size_t b) { return (b + 255) & ~(size_t)255; }

static int raster_sm_count() {
  static const int sms = [] {
    int dev = 0, n = 148;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
  }();
  return sms;
}

// scratch layout, each part 256-byte aligned: the depth keys [views][H][W] uint64, the list length, the list [views * f_cap]
// of (view, face) uint32 pairs
extern "C" int64_t mp_render_mesh_scratch_bytes(int64_t f_cap, int views, int width, int height) {
  if (f_cap < 0 || f_cap > INT32_MAX || views < 1 || views > kMaxViews || width < 1 || width > kMaxSize || height < 1 ||
      height > kMaxSize)
    return -1;
  const size_t px = (size_t)views * (size_t)width * (size_t)height;
  return (int64_t)(raster_align(px * 8) + 256 + raster_align((size_t)views * (size_t)f_cap * 8));
}

extern "C" int mp_render_mesh_async(const float* verts_dev, const int32_t* faces_dev, const int64_t* counts_dev, int64_t v_cap,
                                    int64_t f_cap, const float* normals_dev, const float* colours_dev, const float* mats_dev,
                                    int views, int width, int height, const float* clear, float* out_normal_dev,
                                    float* out_colour_dev, void* scratch_dev, void* stream) {
  MP_REQUIRE(v_cap >= 0 && f_cap >= 0 && v_cap <= INT32_MAX && f_cap <= INT32_MAX,
             "mp_render_mesh_async: bad capacities v_cap=%lld f_cap=%lld", (long long)v_cap, (long long)f_cap);
  MP_REQUIRE(views >= 1 && views <= kMaxViews, "mp_render_mesh_async: bad view count %d (1..%d)", views, kMaxViews);
  MP_REQUIRE(width >= 1 && width <= kMaxSize && height >= 1 && height <= kMaxSize,
             "mp_render_mesh_async: bad image size %dx%d (1..%d per side)", width, height, kMaxSize);
  MP_REQUIRE(normals_dev || colours_dev, "mp_render_mesh_async: neither normals nor colours given: nothing to render");
  MP_REQUIRE(!out_normal_dev || normals_dev, "mp_render_mesh_async: a normal image asked for without normals");
  MP_REQUIRE(!out_colour_dev || colours_dev, "mp_render_mesh_async: a colour image asked for without colours");
  MP_REQUIRE(!normals_dev || out_normal_dev, "mp_render_mesh_async: normals given without a normal image to write");
  MP_REQUIRE(!colours_dev || out_colour_dev, "mp_render_mesh_async: colours given without a colour image to write");
  MP_REQUIRE(counts_dev && mats_dev && clear && scratch_dev && (verts_dev || v_cap == 0) && (faces_dev || f_cap == 0),
             "mp_render_mesh_async: NULL argument");
  MpRange nvtx("monoport_b200: F3.2 mesh render (enqueue-only)");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t npx = (size_t)width * (size_t)height;
  char* base = static_cast<char*>(scratch_dev);
  Mesh m;
  m.verts = verts_dev;
  m.faces = faces_dev;
  m.counts = reinterpret_cast<const long long*>(counts_dev);
  m.normals = normals_dev;
  m.colours = colours_dev;
  m.v_cap = (uint32_t)v_cap;
  m.f_cap = (uint32_t)f_cap;
  Target t;
  t.mats = mats_dev;
  t.views = views;
  t.W = width;
  t.H = height;
  t.keys = reinterpret_cast<unsigned long long*>(base);
  t.list_len = reinterpret_cast<uint32_t*>(base + raster_align((size_t)views * npx * 8));
  t.list = reinterpret_cast<uint2*>(base + raster_align((size_t)views * npx * 8) + 256);
  Shade s;
  s.normal = out_normal_dev;
  s.colour = out_colour_dev;
  for (int k = 0; k < 4; ++k) s.clear[k] = clear[k];
  MP_CUDA(cudaMemsetAsync(t.keys, 0xff, (size_t)views * npx * 8, st));
  MP_CUDA(cudaMemsetAsync(t.list_len, 0, sizeof(uint32_t), st));
  if (f_cap > 0) {
    // 8 CTAs per SM over the faces of each view, no more than the capacity needs
    const long long blocks = (f_cap + kSetupThreads - 1) / kSetupThreads;
    const long long cap = (long long)raster_sm_count() * 8;
    raster_setup_kernel<<<dim3((unsigned)(blocks < cap ? blocks : cap), (unsigned)views), kSetupThreads, 0, st>>>(m, t);
    MP_CUDA(cudaGetLastError());
    // a persistent grid of 4 CTAs per SM over the list, no more than it can hold
    const long long listed = f_cap * (long long)views;
    const long long cap2 = (long long)raster_sm_count() * 4;
    raster_large_kernel<<<(unsigned)(listed < cap2 ? listed : cap2), kLargeThreads, 0, st>>>(m, t);
    MP_CUDA(cudaGetLastError());
  }
  raster_resolve_kernel<<<dim3((unsigned)((npx + kResolveThreads - 1) / kResolveThreads), (unsigned)views), kResolveThreads, 0,
                          st>>>(m, t, s);
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}
