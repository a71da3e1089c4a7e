// TEST INFRASTRUCTURE ONLY -- functional CPU model of monoport_b200/csrc/tc_ptx.cuh (included by it under MP_CUDA_EMU):
// mbarriers with transaction counts, bulk async copies, named barriers, and the warpgroup MMA (wgmma.mma_async, fp16
// operands from SWIZZLE_128B K-major shared-memory descriptors, fp32 accumulators in the registers of the 128 threads of
// a warpgroup, commit / wait_group).
//
// Asynchrony is modelled adversarially: a bulk copy is only QUEUED when it is issued and executed when some thread is
// blocked in an mbarrier wait; a thread's wgmma is only recorded when it is issued and executed -- reading shared memory
// at that moment -- when the thread's wait_group retires its group.  So
//   * reading an accumulator before wait_group sees the old registers,
//   * overwriting a shared-memory operand (or a weight stage) before the wgmma that reads it has been waited for makes
//     that wgmma consume the new bytes,
// both of which show up as wrong results, and a broken hand-off protocol shows up as a reported deadlock (all threads
// waiting, nothing queued) instead of a hang.  Timing, bank conflicts and memory-model subtleties are NOT modelled.
#pragma once
#include <chrono>
#include <deque>
#include <mutex>

namespace tc {

namespace emu {
struct Op {                                  // a queued bulk copy
  uint8_t* dst; const uint8_t* src; uint32_t bytes; uint64_t* bar;
};
inline std::mutex g_mu;
inline std::deque<Op> g_copies;
inline uint8_t* g_smem_r[2] = {nullptr, nullptr};   // base of the dynamic shared memory (1024-B aligned)
inline uint32_t g_smem_bytes = 0;
#define g_smem g_smem_r[cuda_emu::t_rank]
inline std::atomic<unsigned long long> g_events{0};   // bumped by every state change (deadlock watchdog)
inline std::atomic<int> g_waiting{0};
// work counters (EMU_TC_STATS=1 prints them at exit)
struct Stats { std::atomic<unsigned long long> mma_flop{0}, mma_ops{0}, copy_bytes{0}, copies{0}; };
inline Stats g_stats;
inline void print_stats() {
  fprintf(stderr, "[tc emu stats] wgmma (per warpgroup): %llu ops, %.3f GFLOP | bulk copies: %llu, %.3f MB\n",
          g_stats.mma_ops.load() / 128, g_stats.mma_flop.load() * 1e-9, g_stats.copies.load(), g_stats.copy_bytes.load() * 1e-6);
}
inline void stats_init() {
  static const bool on = [] { const bool e = getenv("EMU_TC_STATS") != nullptr; if (e) atexit(print_stats); return e; }();
  (void)on;
}
inline bool eager() { static const bool e = getenv("EMU_TC_EAGER") != nullptr; return e; }   // debugging aid: no deferral

inline void set_smem(void* base, uint32_t bytes, void* base1 = nullptr) {
  stats_init();
  if (((uintptr_t)base | (uintptr_t)base1) & 1023) { fprintf(stderr, "tc emu: shared memory base must be 1024-byte aligned\n"); abort(); }
  g_smem_r[0] = (uint8_t*)base;
  g_smem_r[1] = (uint8_t*)base1;
  g_smem_bytes = bytes;
  g_copies.clear();
}

// ---- mbarrier word: [0,20) pending arrivals | [20,40) arrival count of a phase | [40,62) pending tx bytes | 63 phase
inline uint32_t mb_pending(uint64_t w) { return (uint32_t)(w & 0xFFFFF); }
inline uint32_t mb_count(uint64_t w) { return (uint32_t)((w >> 20) & 0xFFFFF); }
inline int32_t mb_tx(uint64_t w) { const uint32_t v = (uint32_t)((w >> 40) & 0x3FFFFF); return (v & 0x200000u) ? (int32_t)v - 0x400000 : (int32_t)v; }
inline uint32_t mb_phase(uint64_t w) { return (uint32_t)(w >> 63); }
inline uint64_t mb_make(uint32_t pending, uint32_t count, int32_t tx, uint32_t phase) {
  if (tx < -0x200000 || tx >= 0x200000) { fprintf(stderr, "tc emu: mbarrier tx-count out of range\n"); abort(); }
  return (uint64_t)pending | ((uint64_t)count << 20) | ((uint64_t)((uint32_t)tx & 0x3FFFFFu) << 40) | ((uint64_t)phase << 63);
}
inline void mb_check_complete(uint64_t* bar) {
  const uint64_t w = *bar;
  if (mb_pending(w) == 0 && mb_tx(w) == 0) *bar = mb_make(mb_count(w), mb_count(w), 0, mb_phase(w) ^ 1u);
  g_events++;
}
inline void mb_arrive_locked(uint64_t* bar) {
  const uint64_t w = *bar;
  if (mb_pending(w) == 0) { fprintf(stderr, "tc emu: arrival on a barrier with no pending arrivals (over-arrival)\n"); abort(); }
  *bar = mb_make(mb_pending(w) - 1, mb_count(w), mb_tx(w), mb_phase(w));
  mb_check_complete(bar);
}

inline float h2f(uint16_t h) { __half x; memcpy(&x, &h, 2); return __half2float(x); }
inline uint32_t swz(uint32_t a) { return a ^ (((a >> 7) & 7u) << 4); }       // SWIZZLE_128B on the shared-memory address
inline uint16_t smem_half(uint32_t addr) {
  const uint32_t p = swz(addr);
  if (p + 2 > g_smem_bytes) { fprintf(stderr, "tc emu: MMA operand address %u outside shared memory\n", p); abort(); }
  uint16_t h;
  memcpy(&h, g_smem + p, 2);
  return h;
}
inline void desc_fields(uint64_t d, uint32_t& start, uint32_t& sbo) {
  start = (uint32_t)(d & 0x3FFF) << 4;
  sbo = (uint32_t)((d >> 32) & 0x3FFF) << 4;
  if (((d >> 62) & 3) != 1 || ((d >> 49) & 7) != 0) { fprintf(stderr, "tc emu: only SWIZZLE_128B descriptors without base offset are modelled\n"); abort(); }
}

// one thread's share of D[64 x N] += A[64 x 16] * B[N x 16]^T: the accumulator fragment of thread t of the warpgroup
// (warp wl = t/32, lane l) is d[4j + e] = D[16 wl + l/4 + 8 (e>>1)][8 j + 2 (l%4) + (e&1)]
inline void exec_wgmma(float* d, int N, uint64_t a_desc, uint64_t b_desc) {
  const int t = cuda_emu::linear_tid() & 127, wl = t >> 5, l = t & 31;
  uint32_t as, asbo, bs, bsbo;
  desc_fields(a_desc, as, asbo);
  desc_fields(b_desc, bs, bsbo);
  float A[2][16];
  for (int h = 0; h < 2; ++h) {
    const uint32_t m = 16 * wl + l / 4 + 8 * h;
    for (uint32_t k = 0; k < 16; ++k) A[h][k] = h2f(smem_half(as + (m >> 3) * asbo + (m & 7) * 128 + k * 2));
  }
  for (int j = 0; j < N / 8; ++j)
    for (int e = 0; e < 2; ++e) {
      const uint32_t n = 8 * j + 2 * (l % 4) + e;
      float B[16];
      for (uint32_t k = 0; k < 16; ++k) B[k] = h2f(smem_half(bs + (n >> 3) * bsbo + (n & 7) * 128 + k * 2));
      for (int h = 0; h < 2; ++h) {
        float acc = 0.f;
        for (uint32_t k = 0; k < 16; ++k) acc += A[h][k] * B[k];
        d[4 * j + 2 * h + e] += acc;
      }
    }
  g_stats.mma_ops++;
  g_stats.mma_flop += 2ull * 16 * N * 16 / 4;    // (this thread's quarter-warp share, summed over the warpgroup)
}
struct Wgmma { float* d; int N; uint64_t a, b; };
inline thread_local std::vector<Wgmma> t_open;                    // issued, not yet committed
inline thread_local std::deque<std::vector<Wgmma>> t_groups;      // committed groups, oldest first

// executes ONE queued bulk copy; returns false when nothing is queued.  Caller holds g_mu.
// EMU_TC_ORDER=copies (default: in issue order), =random[:seed] (any outstanding copy may complete next).
inline bool progress_locked() {
  static const int order = [] {
    const char* v = getenv("EMU_TC_ORDER");
    if (!v || strncmp(v, "random", 6)) return 0;
    const char* c = strchr(v, ':');
    srand(c ? (unsigned)atoi(c + 1) : 1u);
    return 2;
  }();
  if (g_copies.empty()) return false;
  if (order == 2 && g_copies.size() > 1) std::swap(g_copies[0], g_copies[(size_t)rand() % g_copies.size()]);
  const Op op = g_copies.front();
  g_copies.pop_front();
  memcpy(op.dst, op.src, op.bytes);
  g_stats.copies++;
  g_stats.copy_bytes += op.bytes;
  const uint64_t w = *op.bar;
  if (mb_tx(w) < (int32_t)op.bytes) { fprintf(stderr, "tc emu: complete_tx without a matching expect_tx\n"); abort(); }
  *op.bar = mb_make(mb_pending(w), mb_count(w), mb_tx(w) - (int32_t)op.bytes, mb_phase(w));
  mb_check_complete(op.bar);
  return true;
}
}  // namespace emu

// shared::cta address of a pointer into the CALLING CTA's shared memory
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  const uintptr_t off = (uintptr_t)p - (uintptr_t)emu::g_smem;
  if (off >= emu::g_smem_bytes) { fprintf(stderr, "tc emu: pointer is not in this CTA's shared memory\n"); abort(); }
  return (uint32_t)off;
}

// ---------------------------------------------------------------- mbarrier
inline void mbar_init(uint64_t* bar, uint32_t count) { std::lock_guard<std::mutex> g(emu::g_mu); *bar = emu::mb_make(count, count, 0, 0); emu::g_events++; }
inline void fence_barrier_init() {}
inline void mbar_arrive(uint64_t* bar) { std::lock_guard<std::mutex> g(emu::g_mu); emu::mb_arrive_locked(bar); }
inline void mbar_arrive_if(uint64_t* bar, bool pred) { if (pred) mbar_arrive(bar); }
inline void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  std::lock_guard<std::mutex> g(emu::g_mu);
  const uint64_t w = *bar;
  *bar = emu::mb_make(emu::mb_pending(w), emu::mb_count(w), emu::mb_tx(w) + (int32_t)bytes, emu::mb_phase(w));
  emu::mb_arrive_locked(bar);
}
inline bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  {
    std::lock_guard<std::mutex> g(emu::g_mu);
    if (emu::mb_phase(*bar) != (parity & 1u)) return true;
    if (emu::progress_locked()) return emu::mb_phase(*bar) != (parity & 1u);
  }
  // nothing queued: somebody else has to arrive.  Deadlock watchdog: no state change anywhere for a long time.
  const unsigned long long seen = emu::g_events.load();
  emu::g_waiting++;
  static thread_local std::chrono::steady_clock::time_point last_change = std::chrono::steady_clock::now();
  static thread_local unsigned long long last_seen = ~0ull;
  if (seen != last_seen) { last_seen = seen; last_change = std::chrono::steady_clock::now(); }
  std::this_thread::sleep_for(std::chrono::microseconds(200));
  emu::g_waiting--;
  if (std::chrono::steady_clock::now() - last_change > std::chrono::seconds(20)) {
    const uint64_t w = *bar;
    fprintf(stderr, "tc emu: DEADLOCK -- thread %d of CTA %u waits on barrier +%u (parity %u; phase %u pending %u tx %d), nothing queued\n",
            cuda_emu::linear_tid(), blockIdx.x, smem_u32(bar), parity, emu::mb_phase(w), emu::mb_pending(w), emu::mb_tx(w));
    abort();
  }
  return false;
}
inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------- bulk async copy
inline void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  if (bytes % 16 || ((uintptr_t)smem_dst & 15) || ((uintptr_t)gmem_src & 15)) { fprintf(stderr, "tc emu: bulk copy alignment\n"); abort(); }
  (void)smem_u32(smem_dst);
  std::lock_guard<std::mutex> g(emu::g_mu);
  emu::Op op{};
  op.dst = (uint8_t*)smem_dst; op.src = (const uint8_t*)gmem_src; op.bytes = bytes; op.bar = bar;
  emu::g_copies.push_back(op);
  if (emu::eager()) while (emu::progress_locked()) {}
}

// named barrier over the first `threads` threads of the CTA (one CTA runs at a time)
inline void bar_sync(int id, int threads) {
  static pthread_barrier_t b[16];
  static int n[16];
  static std::mutex mu;
  {
    std::lock_guard<std::mutex> g(mu);
    if (n[id] != threads) { pthread_barrier_init(&b[id], nullptr, (unsigned)threads); n[id] = threads; }
  }
  if (cuda_emu::linear_tid() >= threads) { fprintf(stderr, "tc emu: thread outside the named barrier\n"); abort(); }
  pthread_barrier_wait(&b[id]);
}

// ---------------------------------------------------------------- fences
inline void fence_proxy_async_smem() {}

// ---------------------------------------------------------------- warpgroup MMA
inline void wgmma_fence() {}
inline void wgmma_commit() {
  emu::t_groups.push_back(std::move(emu::t_open));
  emu::t_open.clear();
}
template <int N>
inline void wgmma_wait() {
  if (!emu::t_open.empty()) { fprintf(stderr, "tc emu: wgmma issued but not committed before wait_group\n"); abort(); }
  while (emu::t_groups.size() > (size_t)N) {
    for (const emu::Wgmma& w : emu::t_groups.front()) emu::exec_wgmma(w.d, w.N, w.a, w.b);
    emu::t_groups.pop_front();
  }
}
inline uint64_t make_wdesc_sw128(uint32_t smem_addr, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
inline void wgmma_issue(float* d, int N, uint64_t a, uint64_t b) {
  emu::t_open.push_back(emu::Wgmma{d, N, a, b});
  if (emu::eager()) { wgmma_commit(); wgmma_wait<0>(); }
}
inline void wgmma_m64n256(float (&d)[128], uint64_t a, uint64_t b) { wgmma_issue(d, 256, a, b); }
inline void wgmma_m64n128(float (&d)[64], uint64_t a, uint64_t b) { wgmma_issue(d, 128, a, b); }
inline void wgmma_m64n64(float (&d)[32], uint64_t a, uint64_t b) { wgmma_issue(d, 64, a, b); }

// ---------------------------------------------------------------- operand layout helpers (as in tc_ptx.cuh)
inline uint32_t sw128_offset(uint32_t row, uint32_t k) {
  const uint32_t chunk = (k >> 3) ^ (row & 7u);
  return (row >> 3) * 1024u + (row & 7u) * 128u + chunk * 16u + (k & 7u) * 2u;
}
inline uint32_t pack_half2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  uint32_t u;
  memcpy(&u, &h, 4);
  return u;
}

}  // namespace tc
