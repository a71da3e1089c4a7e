// TEST INFRASTRUCTURE ONLY -- a minimal CPU emulation of the CUDA execution model, just enough to run the integer /
// byte kernels of monoport_b200/csrc (*_kernels.cuh, mp_scan.cuh) UNMODIFIED on the build container, which has no GPU:
// one OS thread per CUDA thread, CTAs executed one after the other, __syncthreads() = a pthread barrier over the CTA,
// warp shuffles = an exchange buffer between two 32-thread barriers, `__shared__` = a static variable (valid because
// only one CTA is alive at a time).  It checks index arithmetic, scan / queue logic and table use against the oracle
// before a kernel is ever sent to an H100; it says nothing about performance or memory-model subtleties.
// Nothing under monoport_b200/ includes this file.
#pragma once
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <pthread.h>
#include <thread>
#include <vector>

#define MP_CUDA_EMU 1

#ifdef MP_EMU_CUDA_TYPES
// the including file has already pulled in the real <cuda_runtime.h> / <cuda_fp16.h> (host side): use their vector types
typedef uint3 uint3_emu;
#undef __global__
#undef __device__
#undef __host__
#undef __forceinline__
#undef __launch_bounds__
#undef __shared__
#undef __constant__
#else
struct uint3_emu { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
struct uint2 { unsigned x, y; };
struct uint4 { unsigned x, y, z, w; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
#endif

inline thread_local uint3_emu threadIdx, blockIdx;
inline thread_local dim3 blockDim, gridDim;

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __shared__ static      /* (dynamic shared memory goes through MP_DYN_SMEM: an array the harness defines) */
#define __constant__

namespace cuda_emu {
constexpr int kMaxThreads = 1024;
// A launch runs one CTA at a time -- or, for a 2-CTA cluster launch, the two CTAs of one cluster at a time: every CTA of the
// cluster has its own barriers / exchange buffers, selected by the thread's rank in the cluster.
inline thread_local int t_rank = 0;                 // %cluster_ctarank of the calling thread
inline int g_cluster = 1;                           // CTAs per cluster of the running launch
inline pthread_barrier_t g_cta_barrier_r[2];
inline pthread_barrier_t g_warp_barrier_r[2][kMaxThreads / 32];
inline unsigned long long g_shfl_r[2][kMaxThreads];
inline pthread_barrier_t g_cluster_barrier;         // all threads of the cluster
#define g_cta_barrier g_cta_barrier_r[cuda_emu::t_rank]
#define g_warp_barrier g_warp_barrier_r[cuda_emu::t_rank]
#define g_shfl g_shfl_r[cuda_emu::t_rank]
inline int linear_tid() { return (int)(threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z)); }

// run `body` once per CUDA thread of a grid x block launch.  The CTA's threads are created once per launch and walk the
// grid together (one barrier between CTAs, so the static "shared memory" is never reused while a thread is still in
// the previous CTA).  cluster = 2 (1-D grids, even size): the two CTAs of a cluster run concurrently, clusters one after
// the other; `__shared__` statics would be shared by the pair, so kernels launched this way must only use MP_DYN_SMEM.
template <class Body>
void launch(dim3 grid, dim3 block, Body body, int cluster = 1) {
  const int nt = (int)(block.x * block.y * block.z);
  if (nt > kMaxThreads || nt % 32 != 0) { fprintf(stderr, "cuda_emu: block of %d threads unsupported\n", nt); abort(); }
  if (cluster != 1 && (cluster != 2 || grid.y != 1 || grid.z != 1 || grid.x % 2)) { fprintf(stderr, "cuda_emu: unsupported cluster launch\n"); abort(); }
  g_cluster = cluster;
  for (int r = 0; r < cluster; ++r) {
    pthread_barrier_init(&g_cta_barrier_r[r], nullptr, nt);
    for (int w = 0; w < nt / 32; ++w) pthread_barrier_init(&g_warp_barrier_r[r][w], nullptr, 32);
  }
  pthread_barrier_init(&g_cluster_barrier, nullptr, nt * cluster);
  std::vector<std::thread> th;
  th.reserve((size_t)nt * cluster);
  for (int tt = 0; tt < nt * cluster; ++tt)
    th.emplace_back([=] {
      const int rank = tt / nt, t = tt % nt;
      t_rank = rank;
      threadIdx = {(unsigned)t % block.x, ((unsigned)t / block.x) % block.y, (unsigned)t / (block.x * block.y)};
      blockDim = block;
      gridDim = grid;
      for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
          for (unsigned bx = 0; bx < grid.x; bx += (unsigned)cluster) {
            blockIdx = {bx + (unsigned)rank, by, bz};
            body();
            pthread_barrier_wait(&g_cluster_barrier);
          }
    });
  for (auto& x : th) x.join();
  for (int r = 0; r < cluster; ++r) {
    pthread_barrier_destroy(&g_cta_barrier_r[r]);
    for (int w = 0; w < nt / 32; ++w) pthread_barrier_destroy(&g_warp_barrier_r[r][w]);
  }
  pthread_barrier_destroy(&g_cluster_barrier);
  g_cluster = 1;
}
}  // namespace cuda_emu

inline void __syncthreads() { pthread_barrier_wait(&cuda_emu::g_cta_barrier); }
inline void __syncwarp() { pthread_barrier_wait(&cuda_emu::g_warp_barrier[cuda_emu::linear_tid() >> 5]); }
inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }

inline unsigned long long __shfl_up_sync(unsigned, unsigned long long v, int delta) {
  const int tid = cuda_emu::linear_tid(), lane = tid & 31;
  cuda_emu::g_shfl[tid] = v;
  pthread_barrier_wait(&cuda_emu::g_warp_barrier[tid >> 5]);
  const unsigned long long r = lane >= delta ? cuda_emu::g_shfl[tid - delta] : v;
  pthread_barrier_wait(&cuda_emu::g_warp_barrier[tid >> 5]);
  return r;
}

// warp shuffles of 4- and 8-byte values (all 32 lanes take part, like every use in the kernels)
template <class T>
inline T emu_warp_exchange(T v, int src_lane) {
  static_assert(sizeof(T) <= 8, "shuffle operand");
  const int tid = cuda_emu::linear_tid(), w0 = tid & ~31;
  unsigned long long bits = 0;
  memcpy(&bits, &v, sizeof(T));
  cuda_emu::g_shfl[tid] = bits;
  pthread_barrier_wait(&cuda_emu::g_warp_barrier[tid >> 5]);
  const unsigned long long got = cuda_emu::g_shfl[w0 + (src_lane & 31)];
  pthread_barrier_wait(&cuda_emu::g_warp_barrier[tid >> 5]);
  T r;
  memcpy(&r, &got, sizeof(T));
  return r;
}
template <class T> inline T __shfl_sync(unsigned, T v, int src_lane) { return emu_warp_exchange(v, src_lane); }
template <class T> inline T __shfl_xor_sync(unsigned, T v, int lane_mask) { return emu_warp_exchange(v, (cuda_emu::linear_tid() & 31) ^ lane_mask); }

inline unsigned __ballot_sync(unsigned, bool pred) {
  const int tid = cuda_emu::linear_tid(), w0 = tid & ~31;
  cuda_emu::g_shfl[tid] = pred ? 1ull : 0ull;
  pthread_barrier_wait(&cuda_emu::g_warp_barrier[tid >> 5]);
  unsigned r = 0;
  for (int l = 0; l < 32; ++l) r |= (unsigned)cuda_emu::g_shfl[w0 + l] << l;
  pthread_barrier_wait(&cuda_emu::g_warp_barrier[tid >> 5]);
  return r;
}

// block-wide OR of a predicate (two barriers around a flag; a third before the flag is cleared for the next use)
inline int __syncthreads_or(int pred) {
  static int flag = 0;
  pthread_barrier_wait(&cuda_emu::g_cta_barrier);
  if (pred) __atomic_store_n(&flag, 1, __ATOMIC_SEQ_CST);
  pthread_barrier_wait(&cuda_emu::g_cta_barrier);
  const int r = __atomic_load_n(&flag, __ATOMIC_SEQ_CST);
  pthread_barrier_wait(&cuda_emu::g_cta_barrier);
  if (cuda_emu::linear_tid() == 0) __atomic_store_n(&flag, 0, __ATOMIC_SEQ_CST);
  pthread_barrier_wait(&cuda_emu::g_cta_barrier);
  return r;
}

inline bool __any_sync(unsigned m, bool pred) { return __ballot_sync(m, pred) != 0u; }
inline bool __all_sync(unsigned m, bool pred) { return __ballot_sync(m, pred) == 0xffffffffu; }
template <class T> inline T __ldg(const T* p) { return *p; }
template <class T> inline T __ldcg(const T* p) { return *reinterpret_cast<const volatile T*>(p); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
// low 32 bits of (hi:lo) >> (s & 31)
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { return (unsigned)(((((unsigned long long)hi) << 32) | lo) >> (s & 31u)); }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __fsqrt_rn(float a) { return sqrtf(a); }
inline int atomicOr(int* p, int v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicMax(unsigned* p, unsigned v) {
  unsigned old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}
inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
template <class T> inline T min(T a, T b) { return a < b ? a : b; }
template <class T> inline T max(T a, T b) { return a > b ? a : b; }
inline long long clock64() { return 0; }
