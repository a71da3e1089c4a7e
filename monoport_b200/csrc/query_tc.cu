// F1 (tensor-core flavour): the fused  project -> mask -> bilinear gather -> z-concat -> 5-layer skip-MLP -> last op -> mask
// kernel of MonoPortNet.query (monoport/lib/modeling/MonoPortNet.py:48-91; heads/SurfaceClassifier.py:39-71) on the Hopper
// warpgroup tensor cores (wgmma).  Specialised for the two shipped heads, which share one program:
//   geometry  PIFuNetGMLP  filter_channels [257,1024,512,256,128,1], Sigmoid, on a 256-channel map;
//   colour    PIFuNetCMLP  filter_channels [513,1024,512,256,128,3], Tanh,    on a 512-channel map.
//
// Arithmetic: layers 1-3 fp16 operands x fp16 weights -> fp32 accumulators in registers; the depth column (z_feat) and the
// bias of every layer are applied in fp32 in the epilogue (so K is exactly 64-aligned, no padding); the last layer
// (128 + C + 1 -> R) runs in fp32 on CUDA cores from the fp32 layer-3 accumulators and the fp32-sampled features.
// Layer 0 is hoisted from points to texels: bilinear sampling is linear, so  W0[:, :C] . sample(F)(u,v) ==
// sample(W0[:, :C] . F)(u,v).  g0_wg_kernel builds G0 = W0f . F once per frame and head (fp16, [texel][1024]) and the
// query kernel SAMPLES the 1024-channel layer-0 pre-activation: h0 = lrelu(lerp(G0) + b0 + w0z * z).
// Colour head only: layer 3 multiplies by W3 as an fp16 PAIR (hi + lo, two MMAs per K-step on the same A operand): the
// Tanh output is four times as sensitive to the logit as the geometry head's Sigmoid, and the rounding of W3 is the largest
// single term of its error.
//
// One persistent CTA per SM; a tile = 64 points (of one image) = the M of every warpgroup MMA.  Warps 0-3 and 4-7 are two consumer
// warpgroups that split the N dimension of every layer (layer 1: 256 columns each, 128 fp32 accumulators per thread;
// layer 2: 128; layer 3: 64); both sample the operands (X, the layer-0 chunks) and run the epilogues.  Warpgroup 2 is the
// producer: one thread of it streams the weights L2 -> shared memory through a ring of 32 KB stages (cp.async.bulk on
// mbarriers), pre-packed on the host as K-major SWIZZLE_128B tiles in exactly the order the consumers take them; in layer
// 1 the ring also borrows the two halves of H1, the layer-2 operand (two more stages in flight where they matter), and in
// layer 2 the layer-0 chunk buffers (one more).  The producer gives its registers to the consumers (setmaxnreg: 40 and
// 232 per thread).  The MMAs run asynchronously: the
// role branches are warp-uniform by construction and the consumers wait for their MMAs at fixed points of a static
// schedule (see the ring below), so layer-0 chunk c+1 is generated while the MMAs of chunk c are in flight.
// query_wg_kernel and query_jvp_kernel (the point gradient, forward mode) share that producer, ring and trunk of layers
// 1-3 (run_trunk); each passes in its own layer-0 chunks, hidden-layer epilogue and layer 4.
#include "mp_common.cuh"
#include "mp_scan.cuh"
#include "tc_ptx.cuh"
#include <stdlib.h>

namespace {

constexpr int kTile = 64;                       // points per tile
constexpr int kConsumers = 256;                 // two consumer warpgroups
constexpr int kThreads = kConsumers + 128;      // + the producer warpgroup (query_wg_kernel)
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
static_assert(128 * kProducerRegs + kConsumers * kConsumerRegs <= 65536, "register file of one SM");
constexpr int kG0Threads = kConsumers + 32;     // g0_wg_kernel: two consumer warpgroups + one producer warp
constexpr int kL0 = 1024, kL1 = 512, kL2 = 256, kL3 = 128;
constexpr int kStageBytes = 32768;              // one ring stage: 256 weight rows x 64 K (or 2 x 128 rows x 64 K)
constexpr int kKb = kTile * 128;                // one 64-channel K-block of a 64-row A operand
constexpr int kSideFloats = kL0 + kL1 + kL2 + kL3;      // 1920 hidden output channels over layers 0..3
__host__ __device__ constexpr int side_off(int l) { return l == 0 ? 0 : l == 1 ? kL0 : l == 2 ? kL0 + kL1 : kL0 + kL1 + kL2; }

// C = feature channels of the head's map (256: geometry, 512: colour)
template <int C> struct Prog {
  static constexpr int XKB = C / 64;                          // K-blocks of the skip operand X
  static constexpr int RES = C == 256 ? 1 : 3;                // last-layer outputs
  static constexpr int L3Pass = C == 256 ? 1 : 2;             // colour: W3 as (hi, lo)
  // weight stream of one tile, in consumption order:
  //   L1: per K-block (16 of H0, then XKB of X) two stages = output halves [0,256), [256,512)
  //   L2: per K-block (8 of H1, then XKB of X) one stage = all 256 outputs
  //   L3: per pass, per two K-blocks (XKB of X, then 4 of H2) one stage = 2 x 128 outputs
  static constexpr int StagesL1 = 2 * (16 + XKB);
  static constexpr int StagesL2 = 8 + XKB;
  static constexpr int StagesL3 = L3Pass * (XKB + 4) / 2;
  static constexpr int StagesPerTile = StagesL1 + StagesL2 + StagesL3;
  static constexpr int Ring = C == 256 ? 3 : 2;               // slots of the weight ring proper (Wr)
  // Layer 1 streams through Slots = Ring + 2: H1 is only written by layer 1's epilogue, so until then its two 32 KB
  // halves are ring slots 0 and 1 and the ring slots proper are 2 .. Slots-1 (slot q at H1 + q x 32 KB)
  static constexpr int Slots = Ring + 2;
  // Layer 2 streams through Ring2 = Ring + 1 slots: the chunk buffers (32 KB, one stage) are dead from the end of layer 1
  // until layer 2's epilogue writes H2 there, so during layer 2 they are one more slot, SlotH0 = Slots (at H0).  Layer 2
  // keeps layer 3's wait depth (Ring - 1 groups in flight), so the extra slot lets the producer refill one step earlier.
  static constexpr int Ring2 = Ring + 1;
  static constexpr uint32_t SlotH0 = Slots;
  // SlotH0's last layer-2 stage is the one whose release waits for the next tile's end of layer 1: it must be among the
  // Ring stages still held when layer 2 ends, i.e. not the one residue of the last Ring2 steps released in the loop
  static constexpr bool H0LastHeld = (StagesL2 - 1 - Ring) % Ring2 < Ring;
  // shared memory (offsets inside the 1024-aligned dynamic block)
  static constexpr int X = 0;                                 // XKB x 8 KB
  static constexpr int H0 = X + XKB * kKb;                    // 2 chunk buffers x 2 K-blocks; H2 (4 K-blocks) after layer 2 (layer 2: ring slot SlotH0)
  static constexpr int H1 = H0 + 4 * kKb;                     // 8 K-blocks (layer 1: ring slots 0, 1); the last layer's partial sums after layer 2
  static constexpr int Wr = H1 + 8 * kKb;                     // Ring x 32 KB
  static constexpr int Small = Wr + Ring * kStageBytes;       // zf[64], inimg[64], s4[RES][64]
  static constexpr int Bars = Small + (2 + RES) * kTile * 4;  // full[Slots + 1], empty[Slots + 1]
  static constexpr int Total = Bars + 2 * (Slots + 1) * 8;
  // slot of a tile's stage: layer 1 stage s -> s % Slots; layer 2 step k -> 2 + k % Ring2 (SlotH0 = 2 + Ring: the last
  // slot of each round, the one that frees last, at the end of layer 1); layer 3 step j -> 2 + j % Ring
  __host__ __device__ static constexpr uint32_t l1_slot(uint32_t s) { return s % (uint32_t)Slots; }
  __host__ __device__ static constexpr uint32_t l2_slot(uint32_t k) { return 2u + k % (uint32_t)Ring2; }
  __host__ __device__ static constexpr uint32_t l3_slot(uint32_t j) { return 2u + j % (uint32_t)Ring; }
  __host__ __device__ static constexpr int slot_off(uint32_t q) { return q == SlotH0 ? H0 : H1 + (int)q * kStageBytes; }
  // The producer's parity bit of SlotH0 starts at 1: its first fill of a tile waits for the release at the end of that
  // tile's layer 1 (the other slots start free)
  static constexpr uint32_t ProducerPhase0 = 1u << SlotH0;
};
static_assert(Prog<256>::Total + 1024 <= 232448, "shared memory budget (227 KB per CTA)");
static_assert(Prog<512>::Total + 1024 <= 232448, "shared memory budget (227 KB per CTA)");
static_assert(Prog<256>::XKB % 2 == 0 && Prog<512>::XKB % 2 == 0, "layer-3 stages hold two K-blocks");
static_assert(Prog<256>::StagesL3 >= Prog<256>::Ring && Prog<512>::StagesL3 >= Prog<512>::Ring, "a layer ends by releasing its last Ring stages");
static_assert(Prog<256>::H1 + 2 * kStageBytes == Prog<256>::Wr && Prog<512>::H1 + 2 * kStageBytes == Prog<512>::Wr, "H1 = ring slots 0, 1");
static_assert(Prog<256>::StagesL1 % Prog<256>::Slots == 0 && Prog<512>::StagesL1 % Prog<512>::Slots == 0,
              "layer 1's last stages in slots 0 and 1 are StagesL1 - Slots and the one after it");
static_assert(Prog<256>::H0 + kStageBytes == Prog<256>::H1 && Prog<512>::H0 + kStageBytes == Prog<512>::H1, "the chunk buffers = one stage");
static_assert(Prog<256>::SlotH0 == 2 + Prog<256>::Ring && Prog<512>::SlotH0 == 2 + Prog<512>::Ring, "l2_slot maps the last step of a round to SlotH0");
static_assert(Prog<256>::H0LastHeld && Prog<512>::H0LastHeld, "SlotH0's last layer-2 stage is held to the end of layer 2");
static_assert(Prog<256>::StagesL2 >= Prog<256>::Ring2 && Prog<512>::StagesL2 >= Prog<512>::Ring2, "layer 2 ends by releasing its last Ring2 stages");

struct TcPack {
  __half* wstream;        // stage stream of a tile: Prog<C>::StagesPerTile x 32 KB
  __half* d_bias0;        // fp16 copies of the layer-0 bias / depth column for the H0 generation
  __half* d_wz0;
  uint8_t* d_w0t;         // W0[:, :C] as fp16 SWIZZLE_128B tiles [n tile 4][K block C/64][256 x 64] for g0_wg_kernel
  float h_bias[kSideFloats];   // host copies (passed by value in the kernel parameters)
  float h_wz[kSideFloats];
  float* w4h;             // [R][128]  last layer, hidden part
  float* w4s;             // [R][C]    last layer, feature part
  float* w4z;             // [R]
  float* b4;              // [R]
  int res;
  int kind;               // 0 = geometry head, 1 = colour head
};

struct TcParams {
  const __half* wstream;
  // per-channel bias and depth-column weight of layers 0..3, carried in the kernel parameter (constant) bank
  alignas(16) float bias_all[kSideFloats];
  alignas(16) float wz_all[kSideFloats];
  const float* w4h;
  const float* w4s;
  const float* w4z;
  const float* b4;
  int res;
  int last_op;
  int H, W;
  const __half* g0;       // [H*W][1024] fp16 per-texel layer-0 product
  const __half* feat16;   // NHWC fp16 copy of the map (taps of the X operand)
  const float* s4tex;     // [H*W][RES] fp32 per-texel last-layer feature part
  const __half* d_bias0;  // layer-0 bias and depth-feature column, fp16 [1024]
  const __half* d_wz0;
  const unsigned* amax;   // range guard (see mp_guard_skips): max |feature| of the frame, limit of this head, sense
  float amax_limit;
  int guard;
};

// Direct rendering of the visible surface (RTL/main.py:212-249) is fused into the colour query: MpSurfaceSrc (mp_common.cuh).

// --------------------------------------------------------------------------------------------------------------------
// sampling helpers
// --------------------------------------------------------------------------------------------------------------------
struct PointTaps {
  int off[4];       // texel indices of the four bilinear taps (0 when the point is invalid)
  float wgt[4];     // tap weights (0 for out-of-range taps, geometry.py:15 zeros padding)
  float zf;         // depth feature z * scale (DepthNormalizer.py:32)
  bool in_img;      // MonoPortNet.py:74
};

// The program's projection (geometry.py:19-55, m0 x rounded first) of the world point (x, y, z) and its mask
// (MonoPortNet.py:74): the taps below and the in-image list of a grid query (InImage) both take it, so the list holds
// exactly the nodes the dense launch does not multiply by 0.
__device__ __forceinline__ bool tc_project_in_image(const MpCalib& cal, float x, float y, float z, float& u, float& v, float& w) {
  mp_project<true>(cal, x, y, z, u, v, w);
  return (u >= -1.f) && (u <= 1.f) && (v >= -1.f) && (v <= 1.f);
}

// projection + mask + taps of point i of image b (i >= n: masked-out padding point), projected with image b's calibration;
// surface vertices when surf.X.
__device__ __forceinline__ PointTaps point_taps(const MpSurfaceSrc& surf, const MpPointSrc& src, const MpCalib& cal, const MpBatch& bt,
                                                int b, int H, int W, long long i, long long n) {
  PointTaps pt;
  float u = 0.f, v = 0.f, w = 0.f;
  const bool valid = i < n;
  bool in_img = false;
  if (valid) {
    float x, y, z;
    if (surf.X) {
      mp_surface_point(surf, i, x, y, z);
    } else {
      mp_load_point(src, bt, b, i, x, y, z);
    }
    in_img = tc_project_in_image(mp_image_calib(cal, bt, b), x, y, z, u, v, w);
  }
  pt.in_img = in_img;
  const MpTaps t = mp_taps(valid ? u : 0.f, valid ? v : 0.f, H, W);
  const bool dead = !valid || !(u == u) || !(v == v);      // NaN coordinates (perspective with w == 0): keep taps finite
#pragma unroll
  for (int a = 0; a < 4; ++a) { pt.off[a] = dead ? 0 : t.off[a]; pt.wgt[a] = dead ? 0.f : t.wgt[a]; }
  pt.zf = w * cal.z_scale;
  return pt;
}

// The skip operand X of a warp's 8 points, in two halves so that the caller can issue every gather before it uses one.
// Whole warp: the points whose taps sit in lanes 0..7 (duplicated in lanes 8..31), channels [phase*256, +256) of the
// fp16 copy of the map (feat16: the tile's image's), a lane covering 8 channels.
//   load_x8   the 8 x 4 taps of the lane's channels into raw[point][tap];
//   store_x8  the bilinear samples from raw into rows [pbase, pbase+8) of the fp16 X tile (K-major SWIZZLE_128B).
// The last layer's direct feature access is NOT derived from these samples but from S4 (fp32, per texel), which the lane
// owning the point interpolates in fp32.
template <int C>
__device__ __forceinline__ void load_x8(const __half* feat16, const PointTaps& pt, int lane, int phase, uint4 (&raw)[8][4]) {
  const int cbase = phase * 256 + lane * 8;
#pragma unroll
  for (int q = 0; q < 8; ++q)
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int off = __shfl_sync(0xffffffffu, pt.off[a], q);
      raw[q][a] = __ldg(reinterpret_cast<const uint4*>(feat16 + (size_t)off * C + cbase));
    }
}

__device__ __forceinline__ void store_x8(uint8_t* smem_x, const PointTaps& pt, const uint4 (&raw)[8][4], int pbase, int lane, int phase) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    float2 acc[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {                   // same accumulation order as grid_sample: nw, ne, sw, se
      const float w = __shfl_sync(0xffffffffu, pt.wgt[a], q);
      const __half2* h2 = reinterpret_cast<const __half2*>(&raw[q][a]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h2[j]);
        acc[j] = (a == 0) ? make_float2(__fmul_rn(f.x, w), __fmul_rn(f.y, w)) : make_float2(fmaf(f.x, w, acc[j].x), fmaf(f.y, w, acc[j].y));
      }
    }
    uint4 packed;
    packed.x = tc::pack_half2(acc[0].x, acc[0].y);
    packed.y = tc::pack_half2(acc[1].x, acc[1].y);
    packed.z = tc::pack_half2(acc[2].x, acc[2].y);
    packed.w = tc::pack_half2(acc[3].x, acc[3].y);
    *reinterpret_cast<uint4*>(smem_x + (phase * 4 + (lane >> 3)) * kKb + tc::sw128_offset(pbase + q, (lane & 7) * 8)) = packed;
  }
}

__device__ __forceinline__ uint32_t act_pack(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  const __half2 r = __hmax2(h, __hmul2(h, __float2half2_rn(MP_LEAKY_SLOPE)));
  return *reinterpret_cast<const uint32_t*>(&r);
}

__device__ __forceinline__ void sync_consumers() { tc::bar_sync(1, kConsumers); }

// ====================================================================================================================
// The weight ring and the trunk (layers 1-3) of the program, shared by query_wg_kernel and query_jvp_kernel: the same
// stream, slots, wait schedule and MMAs, so the JVP's value rows are the query's rows bit for bit.
// Hand-offs: every consumer takes EVERY stage of the stream (waits for it), uses the ones that carry its rows and
// releases a stage once the MMAs that read it have completed (one arrival per consumer warp); the operand buffers written
// by the consumers themselves are published with fence.proxy.async + a named barrier over the 256 consumer threads.

// the ring's barriers (one thread): full[q] completes with the bulk copy into slot q, empty[q] with the release of slot q
// by all 8 consumer warps
template <int C>
__device__ __forceinline__ void ring_init(uint64_t* full, uint64_t* empty) {
  for (int s = 0; s <= Prog<C>::Slots; ++s) {
    tc::mbar_init(full + s, 1);
    tc::mbar_init(empty + s, kConsumers / 32);
  }
  tc::fence_barrier_init();
}

// the producer thread: the weight stream of one tile into the ring.  phase: bit q is the parity of slot q's next refill
// (P::ProducerPhase0 before the first tile).
template <int C>
__device__ __forceinline__ void produce_tile(uint8_t* smem, uint64_t* full, uint64_t* empty, const uint8_t* wsrc, uint32_t& phase) {
  using P = Prog<C>;
  for (int s = 0; s < P::StagesPerTile; ++s) {
    const uint32_t slot = s < P::StagesL1 ? P::l1_slot(s)
                          : s < P::StagesL1 + P::StagesL2 ? P::l2_slot(s - P::StagesL1) : P::l3_slot(s - P::StagesL1 - P::StagesL2);
    tc::mbar_wait(empty + slot, ((phase >> slot) & 1u) ^ 1u);
    phase ^= 1u << slot;
    tc::mbar_arrive_expect_tx(full + slot, kStageBytes);
    tc::bulk_g2s(smem + P::slot_off(slot), wsrc + (size_t)s * kStageBytes, kStageBytes, full + slot);
  }
}

// The consumers' part of one tile: layers 1-3 on the tile's 64 A-operand rows, from X (at P::X) and layer-0 chunk 0 (in the
// first chunk buffer at P::H0), both written and published by the caller.  Register fragment of a 64 x N accumulator
// (wgmma m64nNk16, f32): thread t of the warpgroup (warp wl = t/32, lane l) holds d[4j + e] = D[16 wl + l/4 + 8 (e>>1)][8 j
// + 2 (l%4) + (e&1)].  The kernel passes in what differs between its programs:
//   gen_chunk(c)   layer-0 chunk c (two K-blocks) into chunk buffer c & 1, fenced for the async proxy;
//   epi(acc, side, col0, dst)   a hidden layer's epilogue: this warpgroup's outputs col0 .. (acc[128]: layer 1's 256, acc[64]:
//                               layer 2's 128; bias and depth column at side) -> the fp16 K-major operand at shared offset dst;
//   head(acc[32])  its 64 layer-3 outputs -> layer 4 and the stores (H1 is dead by then: scratch for the partial sums).
// fphase: bit q is the parity of slot q's next fill, kept across the tiles of the CTA.
template <int C, class GenChunk, class Epi, class Head>
__device__ __forceinline__ void run_trunk(uint8_t* smem, uint64_t* full, uint64_t* empty, uint32_t& fphase, int lane, int wg,
                                          GenChunk&& gen_chunk, Epi&& epi, Head&& head) {
  using P = Prog<C>;
  constexpr int Ring = P::Ring, XKB = P::XKB;
  const uint32_t smem_base = tc::smem_u32(smem);
  auto desc = [&](int off) { return tc::make_wdesc_sw128(smem_base + (uint32_t)off, 1024); };

  // ---- the weight ring, consumer side.  Every consumer takes every stage of a tile (56 for the geometry head, 76 for the
  // colour head) in a fixed order, so which stages a warpgroup still has in flight at any point is known at compile time:
  // each wait below is a fixed wgmma_wait<N> and each release names its stage by arithmetic on its index in the tile.
  // No stage is ever queued at run time; the parity of each slot's next fill is one bit per slot (fphase), flipped by
  // every take, as the producer flips its own bit per refill.
  // Layer 1 streams through Slots = Ring + 2 slots (H1's halves are slots 0 and 1), layer 2 through the Ring slots
  // 2 .. Slots-1 and SlotH0 (the chunk buffers), layer 3 through the Ring slots alone: the deeper ring lets the producer
  // run one more K-block ahead in layer 1, where each warpgroup waits for its K-block's MMAs before it takes the next,
  // and one step further ahead in layer 2.  H1's slots are refilled with the next tile's stages 0 and 1 only once
  // H1 is dead: their last layer-1 stages (Defer, Defer + 1) are released at the end of the tile, and the layer-1
  // epilogue writes H1 only after both warpgroups retired every MMA that read those slots.
  // Deadlock freedom: the producer refills a slot with stage s once all 8 consumer warps have released the stage that last
  // used it, so every consumer must have released that stage before it waits for s.  Where that release needs the
  // stage's MMAs complete, the wait for them comes first:
  //   layer 1 (two stages per K-block i: 2i carries output half 0 for warpgroup 0, 2i+1 half 1 for warpgroup 1; each
  //     warpgroup releases the other's stage right after taking it and its own once the K-block's MMAs completed):
  //     taking 2i+1 needs 2i+1-Slots <= 2i-3, which both warpgroups released by the end of K-block i-1's takes (its
  //     owner after its wait<0> there); taking 2i needs 2i-Slots, released a K-block earlier still.  The deferred stages
  //     are last users of slots 0 and 1, whose next stages are the next tile's 0 and 1;
  //   layers 2 and 3 (one stage per K-block step, read by both warpgroups, through R = Ring2 slots in layer 2 and Ring in
  //     layer 3): before taking step k the warpgroup lets at most Ring - 1 groups stay in flight (wait<Ring-1>) and
  //     releases k - Ring; taking step k needs k - R, which is released at step k - R + Ring <= k.  For k < R the slot's
  //     last stage came before the layer: a layer-1 stage of slots 2 .. Slots-1 (released in layer 1), a layer-2 stage
  //     (released at the end of layer 2), or, for SlotH0, the release at the end of this tile's layer 1, once no MMA
  //     reads the chunk buffers.  The last layer-2 stage in SlotH0 is not released at the end of layer 2 (H2 is written
  //     there): its release is the next tile's end of layer 1.
  // Every layer ends with wait<0> and releases its own stages still held, so a layer starts with nothing in flight.
  constexpr uint32_t Defer = P::StagesL1 - P::Slots;
  auto release_if = [&](uint32_t slot, bool pred) {
    __syncwarp();
    tc::mbar_arrive_if(empty + slot, pred && lane == 0);
  };
  auto release = [&](uint32_t slot) { release_if(slot, true); };
  auto l1_release = [&](uint32_t s) { release_if(P::l1_slot(s), s - Defer >= 2u); };
  auto take = [&](uint32_t slot) {
    tc::mbar_wait(full + slot, (fphase >> slot) & 1u);
    fphase ^= 1u << slot;
  };
  auto slot_off = [&](uint32_t slot) { return P::slot_off(slot); };
  // layer 1, K-block i (A operand at shared offset a_off): this warpgroup's 256 outputs times its stage 2i + wg
  auto l1_kblock = [&](float (&acc)[128], int i, int a_off) {
    const uint32_t s0 = 2 * i, mine = s0 + wg, prev = mine - 2;
    take(P::l1_slot(s0));
    tc::wgmma_wait<0>();
    if (i > 0) l1_release(prev);
    take(P::l1_slot(s0 + 1));
    l1_release(s0 + 1 - wg);                         // the other warpgroup's half
    const uint64_t da = desc(a_off), db = desc(slot_off(P::l1_slot(mine)));
    tc::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) tc::wgmma_m64n256(acc, da + 2 * k, db + 2 * k);
    tc::wgmma_commit();
  };
  // layers 2 and 3, step k of a layer whose slots are slot(k): retires and releases step k - Ring (see above), takes step k
  auto step_take = [&](auto slot, int k) {
    if (k >= Ring) {
      tc::wgmma_wait<Ring - 1>();
      release(slot(k - Ring));
    }
    take(slot(k));
    tc::wgmma_fence();
  };
  // end of a layer of n steps (n >= Ring): all MMAs complete, the last Ring stages released (but not SlotH0's)
  auto layer_end = [&](auto slot, int n) {
    tc::wgmma_wait<0>();
#pragma unroll
    for (int j = Ring; j > 0; --j) release_if(slot(n - j), slot(n - j) != P::SlotH0);
  };
  auto l2_slot = [](int k) { return P::l2_slot((uint32_t)k); };
  auto l3_slot = [](int j) { return P::l3_slot((uint32_t)j); };

  // ---- layer 1: 8 sampled layer-0 chunks (2 K-blocks each), then X; this warpgroup's 256 of the 512 outputs
  {
    float acc[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0.f;
#pragma unroll 1
    for (int c = 0; c < 8; ++c) {
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) l1_kblock(acc, 2 * c + kb, P::H0 + ((c & 1) * 2 + kb) * kKb);
      if (c < 7) {
        // the other chunk buffer was last read by chunk c-1, whose MMAs completed before chunk c's second K-block was
        // issued (in both warpgroups once they meet here); chunk c's second K-block stays in flight meanwhile
        sync_consumers();
        gen_chunk(c + 1);
        sync_consumers();
      }
    }
#pragma unroll 1
    for (int kb = 0; kb < XKB; ++kb) l1_kblock(acc, 16 + kb, P::X + kb * kKb);
    tc::wgmma_wait<0>();
    l1_release(2 * (16 + XKB - 1) + wg);
    release(P::SlotH0);      // this warpgroup's MMAs reading the chunk buffers have retired: layer 2 may stream into them
    sync_consumers();        // H1 was ring slots 0 and 1: every MMA that read them has retired in both warpgroups
    epi(acc, side_off(1), wg * 256, P::H1);
    tc::fence_proxy_async_smem();
    sync_consumers();
  }
  // ---- layer 2: H1 (8 K-blocks), then X; this warpgroup's 128 of the 256 outputs -> H2 (over the chunk buffers)
  {
    float acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.f;
#pragma unroll 1
    for (int kb = 0; kb < P::StagesL2; ++kb) {
      step_take(l2_slot, kb);
      const uint64_t da = desc(kb < 8 ? P::H1 + kb * kKb : P::X + (kb - 8) * kKb), db = desc(slot_off(l2_slot(kb)) + wg * 16384);
#pragma unroll
      for (int k = 0; k < 4; ++k) tc::wgmma_m64n128(acc, da + 2 * k, db + 2 * k);
      tc::wgmma_commit();
    }
    layer_end(l2_slot, P::StagesL2);
    sync_consumers();        // H2 overwrites SlotH0's last stage: every consumer warp has retired the MMAs that read it
    epi(acc, side_off(2), wg * 128, P::H0);
    tc::fence_proxy_async_smem();
    sync_consumers();
  }
  // ---- layer 3: X, then H2 (two K-blocks per stage; colour: hi then lo pass); 64 of the 128 outputs
  {
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
#pragma unroll 1
    for (int q = 0; q < P::StagesL3; ++q) {
      step_take(l3_slot, q);
#pragma unroll
      for (int sub = 0; sub < 2; ++sub) {
        const int kb = (2 * q + sub) % (XKB + 4);
        const uint64_t da = desc(kb < XKB ? P::X + kb * kKb : P::H0 + (kb - XKB) * kKb);
        const uint64_t db = desc(slot_off(l3_slot(q)) + sub * 16384 + wg * 8192);
#pragma unroll
        for (int k = 0; k < 4; ++k) tc::wgmma_m64n64(acc, da + 2 * k, db + 2 * k);
      }
      tc::wgmma_commit();
    }
    layer_end(l3_slot, P::StagesL3);
    head(acc);
  }
  sync_consumers();        // the per-point scalars and X are rewritten by the next tile
  // H1 (the layer-2 operand, then the partial sums) is dead: its slots may take the next tile's first stages
  tc::fence_proxy_async_smem();
  release(P::l1_slot(Defer));
  release(P::l1_slot(Defer + 1));
}

// ====================================================================================================================
// The fused query program: the trunk above, with the layer-0 chunks sampled from G0, the hidden epilogues and layer 4.
// PEERS: also store channel 0 into the peer volumes of dst (fused slab exchange).
// bt.B images of src.n points (more than one: MP_SRC_ROWS, [R,N] outputs); tile t is tile t % n_tiles of image t / n_tiles,
// and the range guard skips the tiles of the images outside the head's range -- the producer and the consumers skip
// exactly the same tiles (same predicate on the same amax word), so the weight-ring stage counters stay in step.
template <int C, bool PEERS>
__global__ void __launch_bounds__(kThreads, 1)
query_wg_kernel(const __grid_constant__ TcParams prm, MpPointSrc src, MpCalib cal, MpOutDst dst, MpSurfaceSrc surf, MpBatch bt) {
  using P = Prog<C>;
  constexpr int RES = P::RES;
  MP_DYN_SMEM(uint8_t, smem_raw);
  // aligned by an offset from the shared array itself (not through an integer cast), so the compiler keeps knowing that
  // every pointer below is a shared-memory pointer: 32-bit addresses and st.shared instead of 64-bit generic ones
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + P::Bars);
  uint64_t* empty = full + P::Slots + 1;
  float* s_zf = reinterpret_cast<float*>(smem + P::Small);
  float* s_in = s_zf + kTile;
  float* s_s4 = s_in + kTile;

  // Every branch that decides a role or skips work is warp-uniform by construction: the warp index and every value read
  // from memory that steers control flow come from lane 0 through a shuffle.  ptxas then knows that no wgmma sits on a
  // divergent path; otherwise it wraps every wgmma in warpgroup.arrive / wait and the MMAs run one at a time (C7520).
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0), wg = warp >> 2;

  long long n = src.n;
  if (src.count_dev) {
    const long long c = __shfl_sync(0xffffffffu, *src.count_dev, 0);
    n = c < n ? c : n;
  }
  if (surf.count) {                                  // (the vertex count of a captured frame step, read the same way)
    const long long c = __shfl_sync(0xffffffffu, *surf.count, 0);
    n = c < n ? c : n;
  }
  long long win0, win1;
  mp_shard_window(src, n, win0, win1);
  n = win1;                                          // points >= n are padding; tile 0 starts at point win0
  const long long n_tiles = (win1 - win0 + kTile - 1) / kTile;       // (per image)
  const long long all_tiles = n_tiles * bt.B;
  // the range guard of image b, read once per image a CTA meets (consecutive tiles of an image need no second read; the
  // consumer warps take lane 0's answer)
  auto image_skipped = [&](int b) { return mp_guard_skips(prm.amax + b, prm.amax_limit, prm.guard); };

  if (tid == 0) ring_init<C>(full, empty);
  __syncthreads();

  if (wg == 2) {
    // ============================== weight producer ==============================
    tc::setmaxnreg_dec<kProducerRegs>();
    if (warp == 8 && lane == 0) {
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(prm.wstream);
      uint32_t phase = P::ProducerPhase0;
      bool skip = false;
      int guard_b = -1;
      for (long long t = blockIdx.x; t < all_tiles; t += gridDim.x) {
        const int b = mp_tile_image(bt, t, n_tiles);
        if (b != guard_b) {
          skip = image_skipped(b);
          guard_b = b;
        }
        if (skip) {
          t = mp_skip_image(bt, t, b, n_tiles);
          continue;
        }
        produce_tile<C>(smem, full, empty, wsrc, phase);
      }
    }
    return;
  }

  // ============================== consumers ==============================
  tc::setmaxnreg_inc<kConsumerRegs>();
  const int wl = warp & 3;
  const int cq = 2 * (lane & 3);
  uint32_t fphase = 0;

  // ---- taps of this warp's 8 points for the layer-0 chunks: lane = (point 4 i + qw, channels 8 l8 .. and 64 + 8 l8 ..)
  const int l8 = lane & 7, qw = lane >> 3;
  uint32_t t_off[2][2], t_wgt[2][2], t_z[2];
  const __half* g0 = prm.g0;         // the tile's image's block of G0
  // The G0 taps of the next chunk are loaded one chunk ahead: chunk c+1's loads are issued as soon as chunk c is written,
  // so they are in flight under chunk c's MMAs instead of between the two barriers of the generation point.
  uint4 raw[2][4][2];                // [point][tap][K-block]: the taps of the chunk generated next
  auto load_chunk = [&](int c) {
    const int ch = c * 128 + l8 * 8;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const uint32_t off = (a & 1) ? (t_off[i][a >> 1] >> 16) : (t_off[i][a >> 1] & 0xFFFFu);
        const uint4* srcp = reinterpret_cast<const uint4*>(g0 + (size_t)off * kL0 + ch);
        raw[i][a][0] = __ldg(srcp);
        raw[i][a][1] = __ldg(srcp + 8);      // + 64 channels
      }
  };
  // chunk c from the taps load_chunk(c) left in raw; then chunk c+1's loads
  auto gen_chunk = [&](int c) {
    const int ch = c * 128 + l8 * 8;
    __half2 b8[8], z8[8];
    {
      const uint4 bA = __ldg(reinterpret_cast<const uint4*>(prm.d_bias0 + ch)), bB = __ldg(reinterpret_cast<const uint4*>(prm.d_bias0 + ch + 64));
      const uint4 zA = __ldg(reinterpret_cast<const uint4*>(prm.d_wz0 + ch)), zB = __ldg(reinterpret_cast<const uint4*>(prm.d_wz0 + ch + 64));
      *reinterpret_cast<uint4*>(&b8[0]) = bA; *reinterpret_cast<uint4*>(&b8[4]) = bB;
      *reinterpret_cast<uint4*>(&z8[0]) = zA; *reinterpret_cast<uint4*>(&z8[4]) = zB;
    }
    uint8_t* dstp = smem + P::H0 + (c & 1) * 2 * kKb;
    const __half2 slope2 = __float2half2_rn(MP_LEAKY_SLOPE);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int p = warp * 8 + 4 * i + qw;
      const __half2 zq2 = *reinterpret_cast<const __half2*>(&t_z[i]);
      __half2 acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = __hfma2(z8[j], zq2, b8[j]);
#pragma unroll
      for (int a = 0; a < 4; ++a) {          // same tap order as grid_sample: nw, ne, sw, se
        const __half2 wp = *reinterpret_cast<const __half2*>(&t_wgt[i][a >> 1]);
        const __half2 w2 = (a & 1) ? __high2half2(wp) : __low2half2(wp);
        const __half2* h0 = reinterpret_cast<const __half2*>(&raw[i][a][0]);
        const __half2* h1 = reinterpret_cast<const __half2*>(&raw[i][a][1]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[j] = __hfma2(h0[j], w2, acc[j]);
          acc[4 + j] = __hfma2(h1[j], w2, acc[4 + j]);
        }
      }
      uint32_t o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __half2 r = __hmax2(acc[j], __hmul2(acc[j], slope2));
        o[j] = *reinterpret_cast<const uint32_t*>(&r);
      }
      *reinterpret_cast<uint4*>(dstp + tc::sw128_offset(p, l8 * 8)) = make_uint4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<uint4*>(dstp + kKb + tc::sw128_offset(p, l8 * 8)) = make_uint4(o[4], o[5], o[6], o[7]);
    }
    if (c < 7) load_chunk(c + 1);
    tc::fence_proxy_async_smem();
  };

  int guard_b = -1, skip = 0;
  for (long long t = blockIdx.x; t < all_tiles; t += gridDim.x) {
    const int b = mp_tile_image(bt, t, n_tiles);
    if (b != guard_b) {
      skip = __shfl_sync(0xffffffffu, (int)image_skipped(b), 0);
      guard_b = b;
    }
    if (skip) {
      t = mp_skip_image(bt, t, b, n_tiles);
      continue;
    }
    const long long p0 = win0 + (t - (long long)b * n_tiles) * kTile;
    const size_t texel0 = (size_t)b * prm.H * prm.W;
    g0 = prm.g0 + texel0 * kL0;
    // ---- tile start, in one round of gathers: each warp projects its 8 points once (lane l8 = point warp * 8 + l8), issues
    // the X taps, the S4 taps and the taps of layer-0 chunk 0 of those points, and only then uses them.  The chunk taps
    // are shuffled into their lanes (t_off, t_wgt, t_z); X takes its taps and weights by shuffle from lanes 0..7; lanes 0..7
    // write the per-point scalars.
    {
      const int pbase = warp * 8;
      const PointTaps pt = point_taps(surf, src, cal, bt, b, prm.H, prm.W, p0 + pbase + l8, n);
      const uint32_t o01 = (uint32_t)pt.off[0] | ((uint32_t)pt.off[1] << 16), o23 = (uint32_t)pt.off[2] | ((uint32_t)pt.off[3] << 16);
      const uint32_t w01 = tc::pack_half2(pt.wgt[0], pt.wgt[1]), w23 = tc::pack_half2(pt.wgt[2], pt.wgt[3]);
      const uint32_t zz = tc::pack_half2(pt.zf, pt.zf);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int q = 4 * i + qw;
        t_off[i][0] = __shfl_sync(0xffffffffu, o01, q);
        t_off[i][1] = __shfl_sync(0xffffffffu, o23, q);
        t_wgt[i][0] = __shfl_sync(0xffffffffu, w01, q);
        t_wgt[i][1] = __shfl_sync(0xffffffffu, w23, q);
        t_z[i] = __shfl_sync(0xffffffffu, zz, q);
      }
      load_chunk(0);
      const __half* feat16 = prm.feat16 + texel0 * C;
      const float* s4tex = prm.s4tex + texel0 * RES;
      uint4 xraw[8][4];
      load_x8<C>(feat16, pt, lane, 0, xraw);
      float s4raw[RES][4], w4z[RES], b4[RES];
#pragma unroll
      for (int r = 0; r < RES; ++r) {
#pragma unroll
        for (int a = 0; a < 4; ++a) s4raw[r][a] = __ldg(s4tex + (size_t)pt.off[a] * RES + r);
        w4z[r] = __ldg(prm.w4z + r);
        b4[r] = __ldg(prm.b4 + r);
      }
      store_x8(smem + P::X, pt, xraw, pbase, lane, 0);
#pragma unroll 1
      for (int phase = 1; phase < C / 256; ++phase) {      // colour: the second 256 channels of X, one more round
        load_x8<C>(feat16, pt, lane, phase, xraw);
        store_x8(smem + P::X, pt, xraw, pbase, lane, phase);
      }
      if (lane < 8) {
#pragma unroll
        for (int r = 0; r < RES; ++r) {
          float s = 0.f;
#pragma unroll
          for (int a = 0; a < 4; ++a) s = fmaf(pt.wgt[a], s4raw[r][a], s);
          s_s4[r * kTile + pbase + lane] = s + w4z[r] * pt.zf + b4[r];
        }
        s_zf[pbase + lane] = pt.zf;
        s_in[pbase + lane] = pt.in_img ? 1.f : 0.f;
      }
    }
    tc::fence_proxy_async_smem();
    gen_chunk(0);
    sync_consumers();
    // rows r0 and r0 + 8 of the accumulator fragments.  Taken through a shuffle in every tile, so that the compiler does not
    // hoist the epilogues' shared-memory addresses out of the tile loop: held across it they would take the registers the
    // gathers of the tile start have in flight, and spill.
    const int r0 = __shfl_sync(0xffffffffu, 16 * wl + (lane >> 2), lane);
    const float zf0 = s_zf[r0], zf1 = s_zf[r0 + 8];

    // hidden epilogue: + bias + w_z z, leaky ReLU -> fp16, K-major
    auto epi = [&](const auto& acc, int side, int col0, int dst) {
#pragma unroll
      for (int j = 0; j < (int)(sizeof(acc) / sizeof(acc[0])) / 4; ++j) {
        const int col = col0 + 8 * j + cq;
        const float b0 = prm.bias_all[side + col], b1 = prm.bias_all[side + col + 1];
        const float z0 = prm.wz_all[side + col], z1 = prm.wz_all[side + col + 1];
        uint8_t* kbp = smem + dst + (col >> 6) * kKb;
        *reinterpret_cast<uint32_t*>(kbp + tc::sw128_offset(r0, col & 63)) =
            act_pack(acc[4 * j + 0] + fmaf(z0, zf0, b0), acc[4 * j + 1] + fmaf(z1, zf0, b1));
        *reinterpret_cast<uint32_t*>(kbp + tc::sw128_offset(r0 + 8, col & 63)) =
            act_pack(acc[4 * j + 2] + fmaf(z0, zf1, b0), acc[4 * j + 3] + fmaf(z1, zf1, b1));
      }
    };
    // layer 4 in fp32 and the stores
    auto head = [&](const float (&acc)[32]) {
      float lg[2][RES];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < RES; ++r) lg[h][r] = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = wg * 64 + 8 * j + cq + (e & 1);
          float o = acc[4 * j + e] + fmaf(prm.wz_all[side_off(3) + col], (e >> 1) ? zf1 : zf0, prm.bias_all[side_off(3) + col]);
          o = fmaxf(o, o * MP_LEAKY_SLOPE);
#pragma unroll
          for (int r = 0; r < RES; ++r) lg[e >> 1][r] = fmaf(__ldg(prm.w4h + r * kL3 + col), o, lg[e >> 1][r]);
        }
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < RES; ++r) {
          lg[h][r] += __shfl_xor_sync(0xffffffffu, lg[h][r], 1);
          lg[h][r] += __shfl_xor_sync(0xffffffffu, lg[h][r], 2);
        }
      // warpgroup 1's partial sums -> warpgroup 0 through the (dead) H1 buffer
      float* s_part = reinterpret_cast<float*>(smem + P::H1);
      const int mine = lane & 3;                 // lane 0 of a quad: row r0, lane 1: row r0 + 8
      const int row = r0 + 8 * (mine & 1);
      auto lg_mine = [&](int r) { return (mine & 1) ? lg[1][r] : lg[0][r]; };       // (a select: lg stays in registers)
      if (wg == 1 && mine < 2) {
#pragma unroll
        for (int r = 0; r < RES; ++r) s_part[r * kTile + row] = lg_mine(r);
      }
      sync_consumers();
      if (wg == 0 && mine < 2) {
        const long long i = p0 + row;
        if (i < n) {
          const float inimg = s_in[row];
#pragma unroll
          for (int r = 0; r < RES; ++r) {
            const float logit = s_s4[r * kTile + row] + (lg_mine(r) + s_part[r * kTile + row]);
            const float val = inimg * mp_last_op(logit, prm.last_op);
            if (surf.canvas) {
              mp_surface_store(surf, i, r, val);                   // RTL/main.py:244
              continue;
            }
            if (dst.out) dst.out[mp_tile_image(bt, t, n_tiles) * bt.out_stride + (long long)r * dst.ld + i] = val;
            if (dst.scatter_vol && r == 0) dst.scatter_vol[__ldg(src.nodes + i)] = val;
            if constexpr (PEERS) {
              if (r == 0) {
                const long long at = dst.peer_by_node ? (long long)__ldg(src.nodes + i) : dst.peer_off + i;
#pragma unroll
                for (int pp = 0; pp < MP_MAX_PEERS; ++pp)
                  if (pp < dst.n_peers) dst.peer[pp][at] = val;
              }
            }
          }
        }
      }
    };
    run_trunk<C>(smem, full, empty, fphase, lane, wg, gen_chunk, epi, head);
  }
}

// ====================================================================================================================
// F1‴: the gradient of the query program with respect to the points, forward mode (a JVP with three tangents).  The output
// depends on a point only through its texel coordinates (ix, iy) and its depth feature zf, and a tangent goes through the
// same weights as the value in the same order: so the tangents are three more rows of the A operand, and a tile of 64 rows
// is 16 points x (value, d/dix, d/diy, d/dzf).  It runs query_wg_kernel's trunk (run_trunk: the weight stream, the ring,
// the wait schedule and every MMA) with its own operands and epilogues; the value rows are the query's rows, bit for bit
// (same taps, same roundings, same layer-4 summation order).
// Row map (jvp_row): point k (0..15) of the tile has its value on row 16 (k/4) + k%4, d/dix 8 rows below, d/diy 4 rows
// below, d/dzf 12 rows below -- in the accumulator fragment, lanes 0-15 of warp k/4 hold (value, d/dix) and lanes 16-31
// the same columns of (d/diy, d/dzf), so a value's leaky-ReLU branch reaches its tangents as packed sign bits through one
// __shfl_xor_sync(.., 16) per 32 columns.
//   X:        value = the fp16 map sampled as query_wg_kernel does; d/dix, d/diy = the bilinear derivative of the map
//             (differences of the same taps), rounded once to fp16; d/dzf = 0 (the depth column is not part of X).
//   layer 0:  value = query_wg_kernel's chunk; tangents = slope(value) * (derivative of the sampled G0, or w0z for zf).
//   layers 1-3: bias and depth column on the value row, the depth column alone on the zf row, every tangent times the
//             value's slope (1 above 0, else 0.01: torch's lrelu'(0) = slope, as in query_grad_kernel).
//   layer 4:  the same fp32 hidden dot for every row, plus S4's value / x / y derivative, or w4z for the zf row.
// Per point: g = grad_out * act'(y), d/d(ix, iy, zf) = sum_r g_r * y'_r, then d/du = d/dix (W-1)/2, d/dv = d/diy (H-1)/2,
// d/dw = d/dzf z_scale and the projection's Jacobian as in query_grad_kernel.  Points outside the image get 0 for both.
// bt.B images of src.n points, as query_wg_kernel covers a batch: tile t is tile t % n_tiles of image t / n_tiles, which
// supplies its points, camera, per-texel products and output rows; the range guard skips the images outside the head's
// range, the producer and the consumers deciding it from the same amax word (so the ring's stage counters stay in step).
constexpr int kJvpPts = kTile / 4;      // points per tile
constexpr int kJvpDwBytes = kJvpPts * 8 * 4;   // d wgt / d(ix, iy) of the tile's points, after Prog<C>::Total
static_assert(Prog<256>::Total + kJvpDwBytes + 1024 <= 232448 && Prog<512>::Total + kJvpDwBytes + 1024 <= 232448,
              "shared memory budget of query_jvp_kernel (227 KB per CTA)");

struct JvpOut {
  float* out;             // image b: [Res][ld_out] value at out + b * MpBatch::out_stride, or null
  long long ld_out;
  float* dp;              // image b: [3][ld_dp] at dp + b * dp_stride
  long long ld_dp, dp_stride;
  const float* grad_out;  // image b: [Res][ld_grad] at grad_out + b * gout_stride, or null (ones)
  long long ld_grad, gout_stride;
};

// A-operand row of tangent t (0 value, 1 d/dix, 2 d/diy, 3 d/dzf) of point k of a tile
__device__ __forceinline__ int jvp_row(int k, int t) { return 16 * (k >> 2) + (k & 3) + (t == 1 ? 8 : t == 2 ? 4 : t == 3 ? 12 : 0); }

struct JvpTaps {
  PointTaps pt;           // the value's taps, as query_wg_kernel takes them
  float dx[4], dy[4];     // d wgt / d ix and d wgt / d iy of the taps (0 for the taps that are zero padding, and outside the image)
  float u, v, w;          // the projected point
};

// point i of image b
__device__ __forceinline__ JvpTaps jvp_taps(const MpPointSrc& src, const MpCalib& cal, const MpBatch& bt, int b, int H, int W,
                                            long long i, long long n) {
  JvpTaps j;
  MpSurfaceSrc nosurf;
  memset(&nosurf, 0, sizeof(nosurf));
  j.pt = point_taps(nosurf, src, cal, bt, b, H, W, i, n);
  float u = 0.f, v = 0.f, w = 0.f;
  if (i < n) {
    float x, y, z;
    mp_load_point(src, bt, b, i, x, y, z);
    mp_project<true>(mp_image_calib(cal, bt, b), x, y, z, u, v, w);
  }
  j.u = u; j.v = v; j.w = w;
  // the tap cell of mp_taps
  const float ix = ((u + 1.f) / 2.f) * (float)(W - 1), iy = ((v + 1.f) / 2.f) * (float)(H - 1);
  const float x0 = floorf(ix), y0 = floorf(iy), x1 = x0 + 1.f, y1 = y0 + 1.f;
  const bool x0ok = (x0 >= 0.f) && (x0 <= (float)(W - 1)), x1ok = (x1 >= 0.f) && (x1 <= (float)(W - 1));
  const bool y0ok = (y0 >= 0.f) && (y0 <= (float)(H - 1)), y1ok = (y1 >= 0.f) && (y1 <= (float)(H - 1));
  const bool live = j.pt.in_img;
  const bool ok[4] = {live && x0ok && y0ok, live && x1ok && y0ok, live && x0ok && y1ok, live && x1ok && y1ok};
  const float ddx[4] = {-(y1 - iy), y1 - iy, -(iy - y0), iy - y0};       // nw, ne, sw, se
  const float ddy[4] = {-(x1 - ix), -(ix - x0), x1 - ix, ix - x0};
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    j.dx[a] = ok[a] ? ddx[a] : 0.f;
    j.dy[a] = ok[a] ? ddy[a] : 0.f;
  }
  return j;
}

// epilogue of hidden layer 1 or 2 (side = its side_off): this lane's N / 4 column pairs (from col0 + cq) of rows r0 and r0 + 8
// -> the fp16 K-major operand at buf.  isv: the lane holds (value, d/dix) rows, else (d/diy, d/dzf).  Column pair by column
// pair, so that each accumulator dies at its first use (the value's signs cross to lanes 16-31 as two bits per pair).
// zt: the depth feature's tangent on row r0 + 8 (0: d/dix, 1: d/dzf), a multiplier rather than a select, so that no
// per-lane product of the weights is hoisted out of the tile loop.
template <int N>
__device__ __forceinline__ void jvp_hidden_epilogue(const TcParams& prm, const float (&acc)[N], int side, int col0, uint8_t* buf,
                                                    int r0, int cq, float zf, bool isv, float zt) {
#pragma unroll
  for (int j = 0; j < N / 4; ++j) {
    const int col = col0 + 8 * j + cq;
    const float z0 = prm.wz_all[side + col], z1 = prm.wz_all[side + col + 1];
    uint8_t* kbp = buf + (col >> 6) * kKb;
    // the value row as query_wg_kernel writes it (lanes 0-15), and the signs of its fp16 pre-activations
    const float a0 = acc[4 * j + 0] + fmaf(z0, zf, prm.bias_all[side + col]);
    const float a1 = acc[4 * j + 1] + fmaf(z1, zf, prm.bias_all[side + col + 1]);
    const float2 h = __half22float2(__floats2half2_rn(a0, a1));
    uint32_t bits = (h.x > 0.f ? 1u : 0u) | (h.y > 0.f ? 2u : 0u);
    const uint32_t other = __shfl_xor_sync(0xffffffffu, bits, 16);
    bits = isv ? bits : other;
    const float s0 = (bits & 1u) ? 1.f : MP_LEAKY_SLOPE, s1 = (bits & 2u) ? 1.f : MP_LEAKY_SLOPE;
    *reinterpret_cast<uint32_t*>(kbp + tc::sw128_offset(r0, col & 63)) =
        isv ? act_pack(a0, a1) : tc::pack_half2(acc[4 * j + 0] * s0, acc[4 * j + 1] * s1);
    *reinterpret_cast<uint32_t*>(kbp + tc::sw128_offset(r0 + 8, col & 63)) =
        tc::pack_half2(fmaf(z0, zt, acc[4 * j + 2]) * s0, fmaf(z1, zt, acc[4 * j + 3]) * s1);
  }
}

template <int C>
__global__ void __launch_bounds__(kThreads, 1)
query_jvp_kernel(const __grid_constant__ TcParams prm, MpPointSrc src, MpCalib cal, JvpOut jo, MpBatch bt) {
  using P = Prog<C>;
  constexpr int RES = P::RES, NP = kJvpPts;
  static_assert((5 + 3 * RES) * NP <= (2 + RES) * kTile, "per-point scalars of a JVP tile fit the Small block");
  MP_DYN_SMEM(uint8_t, smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + P::Bars);
  uint64_t* empty = full + P::Slots + 1;
  float* s_zf = reinterpret_cast<float*>(smem + P::Small);   // [NP]
  float* s_in = s_zf + NP;                                    // [NP]
  float* s_uvw = s_in + NP;                                   // [3][NP]
  float* s_s4 = s_uvw + 3 * NP;                               // [3][RES][NP]: S4 sampled, its d/dix, its d/diy
  float* s_dw = reinterpret_cast<float*>(smem + P::Total);   // [NP][8]: d wgt / d ix of the four taps, then d wgt / d iy

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0), wg = warp >> 2;
  long long n = src.n;
  if (src.count_dev) {
    const long long c = __shfl_sync(0xffffffffu, *src.count_dev, 0);
    n = c < n ? c : n;
  }
  const long long n_tiles = (n + NP - 1) / NP;      // (per image)
  const long long all_tiles = n_tiles * bt.B;
  // the range guard of image b, read once per image a CTA meets (the consumer warps take lane 0's answer)
  auto image_skipped = [&](int b) { return mp_guard_skips(prm.amax + b, prm.amax_limit, prm.guard); };

  if (tid == 0) ring_init<C>(full, empty);
  __syncthreads();

  if (wg == 2) {
    // ============================== weight producer ==============================
    tc::setmaxnreg_dec<kProducerRegs>();
    if (warp == 8 && lane == 0) {
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(prm.wstream);
      uint32_t phase = P::ProducerPhase0;
      bool skip = false;
      int guard_b = -1;
      for (long long t = blockIdx.x; t < all_tiles; t += gridDim.x) {
        const int b = mp_tile_image(bt, t, n_tiles);
        if (b != guard_b) {
          skip = image_skipped(b);
          guard_b = b;
        }
        if (skip) {
          t = mp_skip_image(bt, t, b, n_tiles);
          continue;
        }
        produce_tile<C>(smem, full, empty, wsrc, phase);
      }
    }
    return;
  }

  // ============================== consumers ==============================
  tc::setmaxnreg_inc<kConsumerRegs>();
  const int wl = warp & 3;
  const int r0 = 16 * wl + (lane >> 2), cq = 2 * (lane & 3);
  const bool isv = lane < 16;                         // rows r0, r0 + 8 hold (value, d/dix), else (d/diy, d/dzf)
  const int kpt = 4 * wl + ((lane >> 2) & 3);         // ... of point kpt
  const float zt = (float)(lane >> 4);                // the depth feature's tangent on row r0 + 8
  uint32_t fphase = 0;

  // ---- layer-0 chunks: lane = (point 2 warp + lane/16, K-block half (lane/8)%2, channels 8 (lane%8) ..), all four rows
  const int l8 = lane & 7, kbh = (lane >> 3) & 1, gq = 2 * warp + (lane >> 4);
  uint32_t t_off[2], t_wgt[2], t_z;
  const __half* g0 = prm.g0;
  auto gen_chunk = [&](int c) {
    const int ch = c * 128 + kbh * 64 + l8 * 8;
    __half2 b4[4], z4[4];
    *reinterpret_cast<uint4*>(&b4[0]) = __ldg(reinterpret_cast<const uint4*>(prm.d_bias0 + ch));
    *reinterpret_cast<uint4*>(&z4[0]) = __ldg(reinterpret_cast<const uint4*>(prm.d_wz0 + ch));
    uint8_t* dstp = smem + P::H0 + ((c & 1) * 2 + kbh) * kKb;
    const __half2 slope2 = __float2half2_rn(MP_LEAKY_SLOPE);
    uint4 raw[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const uint32_t off = (a & 1) ? (t_off[a >> 1] >> 16) : (t_off[a >> 1] & 0xFFFFu);
      raw[a] = __ldg(reinterpret_cast<const uint4*>(g0 + (size_t)off * kL0 + ch));
    }
    const __half2 zq2 = *reinterpret_cast<const __half2*>(&t_z);
    const float4 dxa = *reinterpret_cast<const float4*>(s_dw + gq * 8), dya = *reinterpret_cast<const float4*>(s_dw + gq * 8 + 4);
    const float t_dx[4] = {dxa.x, dxa.y, dxa.z, dxa.w}, t_dy[4] = {dya.x, dya.y, dya.z, dya.w};
    __half2 acc[4];
    float2 dx[4], dy[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = __hfma2(z4[j], zq2, b4[j]);
#pragma unroll
    for (int a = 0; a < 4; ++a) {            // same tap order as query_wg_kernel: nw, ne, sw, se
      const __half2 wp = *reinterpret_cast<const __half2*>(&t_wgt[a >> 1]);
      const __half2 w2 = (a & 1) ? __high2half2(wp) : __low2half2(wp);
      const __half2* h = reinterpret_cast<const __half2*>(&raw[a]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[j] = __hfma2(h[j], w2, acc[j]);
        const float2 f = __half22float2(h[j]);
        dx[j] = a == 0 ? make_float2(f.x * t_dx[0], f.y * t_dx[0]) : make_float2(fmaf(f.x, t_dx[a], dx[j].x), fmaf(f.y, t_dx[a], dx[j].y));
        dy[j] = a == 0 ? make_float2(f.x * t_dy[0], f.y * t_dy[0]) : make_float2(fmaf(f.x, t_dy[a], dy[j].x), fmaf(f.y, t_dy[a], dy[j].y));
      }
    }
    uint32_t o[4][4];                        // [row kind][channel pair]
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 r = __hmax2(acc[j], __hmul2(acc[j], slope2));
      o[0][j] = *reinterpret_cast<const uint32_t*>(&r);
      const float2 pre = __half22float2(acc[j]), wz = __half22float2(z4[j]);
      const float s0 = pre.x > 0.f ? 1.f : MP_LEAKY_SLOPE, s1 = pre.y > 0.f ? 1.f : MP_LEAKY_SLOPE;
      o[1][j] = tc::pack_half2(dx[j].x * s0, dx[j].y * s1);
      o[2][j] = tc::pack_half2(dy[j].x * s0, dy[j].y * s1);
      o[3][j] = tc::pack_half2(wz.x * s0, wz.y * s1);
    }
#pragma unroll
    for (int t = 0; t < 4; ++t)
      *reinterpret_cast<uint4*>(dstp + tc::sw128_offset(jvp_row(gq, t), l8 * 8)) = make_uint4(o[t][0], o[t][1], o[t][2], o[t][3]);
    tc::fence_proxy_async_smem();
  };

  int guard_b = -1, skip = 0;
  for (long long t = blockIdx.x; t < all_tiles; t += gridDim.x) {
    const int b = mp_tile_image(bt, t, n_tiles);
    if (b != guard_b) {
      skip = __shfl_sync(0xffffffffu, (int)image_skipped(b), 0);
      guard_b = b;
    }
    if (skip) {
      t = mp_skip_image(bt, t, b, n_tiles);
      continue;
    }
    const long long p0 = (t - (long long)b * n_tiles) * NP;
    const size_t texel0 = (size_t)b * prm.H * prm.W;
    g0 = prm.g0 + texel0 * kL0;
    const __half* feat16 = prm.feat16 + texel0 * C;
    const float* s4tex = prm.s4tex + texel0 * RES;
    // ---- this lane's point (lane % 16) of the tile; X and the per-point scalars: warp w samples points 2w, 2w + 1
    const JvpTaps jt = jvp_taps(src, cal, bt, b, prm.H, prm.W, p0 + (lane & 15), n);
#pragma unroll 1
    for (int qq = 0; qq < 2; ++qq) {
      const int q = 2 * warp + qq;
      int off[4];
      float wgt[4], wx[4], wy[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        off[a] = __shfl_sync(0xffffffffu, jt.pt.off[a], q);
        wgt[a] = __shfl_sync(0xffffffffu, jt.pt.wgt[a], q);
        wx[a] = __shfl_sync(0xffffffffu, jt.dx[a], q);
        wy[a] = __shfl_sync(0xffffffffu, jt.dy[a], q);
      }
#pragma unroll 1
      for (int phase = 0; phase < C / 256; ++phase) {
        const int cbase = phase * 256 + lane * 8;
        uint4 raw[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) raw[a] = __ldg(reinterpret_cast<const uint4*>(feat16 + (size_t)off[a] * C + cbase));
        float2 acc[4], ax[4], ay[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) {        // the value as store_x8 takes it: nw, ne, sw, se
          const float2 w2 = make_float2(wgt[a], wgt[a]);
          const __half2* h2 = reinterpret_cast<const __half2*>(&raw[a]);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(h2[j]);
            acc[j] = (a == 0) ? make_float2(__fmul_rn(f.x, w2.x), __fmul_rn(f.y, w2.y)) : make_float2(fmaf(f.x, w2.x, acc[j].x), fmaf(f.y, w2.y, acc[j].y));
            ax[j] = (a == 0) ? make_float2(__fmul_rn(f.x, wx[0]), __fmul_rn(f.y, wx[0])) : make_float2(fmaf(f.x, wx[a], ax[j].x), fmaf(f.y, wx[a], ax[j].y));
            ay[j] = (a == 0) ? make_float2(__fmul_rn(f.x, wy[0]), __fmul_rn(f.y, wy[0])) : make_float2(fmaf(f.x, wy[a], ay[j].x), fmaf(f.y, wy[a], ay[j].y));
          }
        }
        uint8_t* xkb = smem + P::X + (phase * 4 + (lane >> 3)) * kKb;
        const int k8 = (lane & 7) * 8;
        *reinterpret_cast<uint4*>(xkb + tc::sw128_offset(jvp_row(q, 0), k8)) =
            make_uint4(tc::pack_half2(acc[0].x, acc[0].y), tc::pack_half2(acc[1].x, acc[1].y), tc::pack_half2(acc[2].x, acc[2].y), tc::pack_half2(acc[3].x, acc[3].y));
        *reinterpret_cast<uint4*>(xkb + tc::sw128_offset(jvp_row(q, 1), k8)) =
            make_uint4(tc::pack_half2(ax[0].x, ax[0].y), tc::pack_half2(ax[1].x, ax[1].y), tc::pack_half2(ax[2].x, ax[2].y), tc::pack_half2(ax[3].x, ax[3].y));
        *reinterpret_cast<uint4*>(xkb + tc::sw128_offset(jvp_row(q, 2), k8)) =
            make_uint4(tc::pack_half2(ay[0].x, ay[0].y), tc::pack_half2(ay[1].x, ay[1].y), tc::pack_half2(ay[2].x, ay[2].y), tc::pack_half2(ay[3].x, ay[3].y));
        *reinterpret_cast<uint4*>(xkb + tc::sw128_offset(jvp_row(q, 3), k8)) = make_uint4(0u, 0u, 0u, 0u);
      }
    }
    if (lane < 16 && (lane >> 1) == warp) {          // point `lane`: its scalars (S4 as query_wg_kernel samples it)
      const PointTaps& pt = jt.pt;
#pragma unroll
      for (int r = 0; r < RES; ++r) {
        float s = 0.f, sx = 0.f, sy = 0.f;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          const float s4 = __ldg(s4tex + (size_t)pt.off[a] * RES + r);
          s = fmaf(pt.wgt[a], s4, s);
          sx = fmaf(jt.dx[a], s4, sx);
          sy = fmaf(jt.dy[a], s4, sy);
        }
        s_s4[r * NP + lane] = s + __ldg(prm.w4z + r) * pt.zf + __ldg(prm.b4 + r);
        s_s4[(RES + r) * NP + lane] = sx;
        s_s4[(2 * RES + r) * NP + lane] = sy;
      }
      s_zf[lane] = pt.zf;
      s_in[lane] = pt.in_img ? 1.f : 0.f;
      s_uvw[lane] = jt.u;
      s_uvw[NP + lane] = jt.v;
      s_uvw[2 * NP + lane] = jt.w;
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        s_dw[lane * 8 + a] = jt.dx[a];
        s_dw[lane * 8 + 4 + a] = jt.dy[a];
      }
    }
    {
      const PointTaps& pt = jt.pt;
      const uint32_t o01 = (uint32_t)pt.off[0] | ((uint32_t)pt.off[1] << 16), o23 = (uint32_t)pt.off[2] | ((uint32_t)pt.off[3] << 16);
      const uint32_t w01 = tc::pack_half2(pt.wgt[0], pt.wgt[1]), w23 = tc::pack_half2(pt.wgt[2], pt.wgt[3]);
      const uint32_t zz = tc::pack_half2(pt.zf, pt.zf);
      t_off[0] = __shfl_sync(0xffffffffu, o01, gq & 15);
      t_off[1] = __shfl_sync(0xffffffffu, o23, gq & 15);
      t_wgt[0] = __shfl_sync(0xffffffffu, w01, gq & 15);
      t_wgt[1] = __shfl_sync(0xffffffffu, w23, gq & 15);
      t_z = __shfl_sync(0xffffffffu, zz, gq & 15);
    }
    tc::fence_proxy_async_smem();
    sync_consumers();                                // s_dw
    gen_chunk(0);
    sync_consumers();
    const float zf = s_zf[kpt];
    // the epilogues' row and column, re-derived per tile: otherwise their 2 x 48 swizzled store offsets are hoisted out of
    // the tile loop, which leaves no registers for layer 1
    int r0t = r0, cqt = cq;
    asm volatile("" : "+r"(r0t), "+r"(cqt));

    auto epi = [&](const auto& acc, int side, int col0, int dst) {
      jvp_hidden_epilogue(prm, acc, side, col0, smem + dst, r0t, cqt, zf, isv, zt);
    };
    // layer 4 in fp32, the chain rule and the stores
    auto head = [&](const float (&acc)[32]) {
      // row r0: the value's hidden dot exactly as query_wg_kernel sums it (lanes < 16), and the signs of its layer-3 outputs
      float lg[2][RES], lt[RES];
#pragma unroll
      for (int r = 0; r < RES; ++r) lg[0][r] = lg[1][r] = lt[r] = 0.f;
      uint32_t m = 0u;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = wg * 64 + 8 * j + cq + e;
          float o = acc[4 * j + e] + fmaf(prm.wz_all[side_off(3) + col], zf, prm.bias_all[side_off(3) + col]);
          m |= (o > 0.f ? 1u : 0u) << (2 * j + e);
          o = fmaxf(o, o * MP_LEAKY_SLOPE);
#pragma unroll
          for (int r = 0; r < RES; ++r) lg[0][r] = fmaf(__ldg(prm.w4h + r * kL3 + col), o, lg[0][r]);
        }
      {
        const uint32_t o = __shfl_xor_sync(0xffffffffu, m, 16);
        m = isv ? m : o;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = wg * 64 + 8 * j + cq + (e & 1);
          const float s = ((m >> (2 * j + (e & 1))) & 1u) ? 1.f : MP_LEAKY_SLOPE;
          if (e < 2) {                                  // d/diy (lanes >= 16)
#pragma unroll
            for (int r = 0; r < RES; ++r) lt[r] = fmaf(__ldg(prm.w4h + r * kL3 + col), acc[4 * j + e] * s, lt[r]);
          } else {                                      // d/dix, d/dzf (+ the depth column)
            const float t3 = fmaf(prm.wz_all[side_off(3) + col], zt, acc[4 * j + e]) * s;
#pragma unroll
            for (int r = 0; r < RES; ++r) lg[1][r] = fmaf(__ldg(prm.w4h + r * kL3 + col), t3, lg[1][r]);
          }
        }
#pragma unroll
      for (int r = 0; r < RES; ++r) lg[0][r] = isv ? lg[0][r] : lt[r];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < RES; ++r) {
          lg[h][r] += __shfl_xor_sync(0xffffffffu, lg[h][r], 1);
          lg[h][r] += __shfl_xor_sync(0xffffffffu, lg[h][r], 2);
        }
      float* s_part = reinterpret_cast<float*>(smem + P::H1);
      const int mine = lane & 3;
      const int row = r0 + 8 * (mine & 1);
      auto lg_mine = [&](int r) { return (mine & 1) ? lg[1][r] : lg[0][r]; };
      if (wg == 1 && mine < 2) {
#pragma unroll
        for (int r = 0; r < RES; ++r) s_part[r * kTile + row] = lg_mine(r);
      }
      sync_consumers();
      if (wg == 0) {
        // this lane's row: 0 value, 1 d/dix, 2 d/diy, 3 d/dzf (of point kpt; lanes with mine >= 2 duplicate)
        const int kind = (isv ? 0 : 2) + (mine & 1);
        float y[RES], yx[RES], yy[RES], yz[RES];
#pragma unroll
        for (int r = 0; r < RES; ++r) {
          const float base = kind == 3 ? __ldg(prm.w4z + r) : s_s4[((kind == 0 ? 0 : kind == 1 ? RES : 2 * RES) + r) * NP + kpt];
          y[r] = base + (lg_mine(r) + s_part[r * kTile + row]);
        }
        // the point's four rows meet in its value lane 4k: d/dix from lane 4k + 1, d/diy from 4k + 16, d/dzf from 4k + 17
        const int lv = lane & 12;
#pragma unroll
        for (int r = 0; r < RES; ++r) {
          yx[r] = __shfl_sync(0xffffffffu, y[r], lv + 1);
          yy[r] = __shfl_sync(0xffffffffu, y[r], lv + 16);
          yz[r] = __shfl_sync(0xffffffffu, y[r], lv + 17);
        }
        const long long i = p0 + kpt;
        if (isv && mine == 0 && i < n) {
          const int b = mp_tile_image(bt, t, n_tiles);       // (re-derived: not held across the trunk)
          const float inimg = s_in[kpt];
          float gx = 0.f, gy = 0.f, gz = 0.f;
#pragma unroll
          for (int r = 0; r < RES; ++r) {
            const float act = mp_last_op(y[r], prm.last_op);
            if (jo.out) jo.out[b * bt.out_stride + (long long)r * jo.ld_out + i] = inimg * act;
            const float d = prm.last_op == MP_LAST_SIGMOID ? act * (1.f - act) : (prm.last_op == MP_LAST_TANH ? 1.f - act * act : 1.f);
            const float g = (jo.grad_out ? __ldg(jo.grad_out + b * jo.gout_stride + (long long)r * jo.ld_grad + i) : 1.f) * d;
            gx = fmaf(g, yx[r], gx);
            gy = fmaf(g, yy[r], gy);
            gz = fmaf(g, yz[r], gz);
          }
          const float du = gx * (0.5f * (float)(prm.W - 1)), dv = gy * (0.5f * (float)(prm.H - 1)), dw = cal.z_scale * gz;
          float gp[3];
          if (!cal.has) {
            gp[0] = du; gp[1] = dv; gp[2] = dw;
          } else {
            // the camera jvp_taps projected with (image b's, in device memory when bt.calibs is set), read where the
            // Jacobian needs it
            const MpCalib c = mp_image_calib(cal, bt, b);
            if (!c.perspective) {                        // J = R
#pragma unroll
              for (int a = 0; a < 3; ++a) gp[a] = c.m[a] * du + c.m[4 + a] * dv + c.m[8 + a] * dw;
            } else {                                     // J rows: (R0 - u R2) / w, (R1 - v R2) / w, R2
              const float u = s_uvw[kpt], v = s_uvw[NP + kpt], w = s_uvw[2 * NP + kpt];
              const float su = du / w, sv = dv / w;
              const float s2 = dw - su * u - sv * v;
#pragma unroll
              for (int a = 0; a < 3; ++a) gp[a] = c.m[a] * su + c.m[4 + a] * sv + c.m[8 + a] * s2;
            }
          }
#pragma unroll
          for (int a = 0; a < 3; ++a) jo.dp[b * jo.dp_stride + a * jo.ld_dp + i] = inimg != 0.f ? gp[a] : 0.f;   // outside the image: exactly 0
        }
      }
    };
    run_trunk<C>(smem, full, empty, fphase, lane, wg, gen_chunk, epi, head);
  }
}

// G0[texel][n] = sum_k F[texel][k] * W0f[n][k] on the tensor cores: fp16 operands (F rounded once while staging, W0f
// pre-packed on the host as SWIZZLE_128B tiles [n tile][K block][256 x 64]) and fp32 accumulation in registers.
// One CTA = 128 texels of one map (grid: texel blocks x maps of the handle) x all 1024 outputs: the A operand (128 x C) is staged ONCE by the two consumer warpgroups (fp32
// global -> fp16 swizzled smem), the B tiles stream through a 2-stage bulk-copy ring (warp 8), and each warpgroup multiplies
// its 64 rows by the four 256-wide output tiles.  The staging pass also publishes what it has in hand: the fp16 copy of the
// map (F16, taps of the X operand) and S4 = W4s . F per texel in fp32 (the last layer's direct access to the features:
// sampling S4 in fp32 keeps that path out of the fp16 roundings -- bilinear sampling commutes with the dot product).
constexpr int kG0TileN = 256;
constexpr int kG0NT = kL0 / kG0TileN;                 // 4 output tiles
constexpr int kG0Stages = 2;
template <int C> struct G0Cfg {
  static constexpr int KB = C / 64;
  static constexpr uint32_t SmemA = KB * 16384, SmemB = kG0Stages * 32768;
  static constexpr uint32_t Smem = SmemA + SmemB + 1024 /*align*/ + 64 /*barriers*/;
};

template <int C>
__global__ void __launch_bounds__(kG0Threads, 1)
g0_wg_kernel(const float* __restrict__ F, const uint8_t* __restrict__ Wt, __half* __restrict__ G, int M,
             __half* __restrict__ F16, float* __restrict__ S4, const float* __restrict__ w4s, unsigned* __restrict__ amax,
             unsigned* __restrict__ nonfinite) {
  using Cfg = G0Cfg<C>;
  constexpr int RES = Prog<C>::RES, KB = Cfg::KB;
  MP_DYN_SMEM(uint8_t, g0_smem_raw);
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(g0_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = base;
  uint8_t* sB = base + Cfg::SmemA;
  uint64_t* b_full = reinterpret_cast<uint64_t*>(base + Cfg::SmemA + Cfg::SmemB);
  uint64_t* b_empty = b_full + kG0Stages;
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);       // provably warp-uniform (see query_wg_kernel)
  const int m0 = blockIdx.x * 128;
  {
    // blockIdx.y = the image of a batch handle: its own blocks of every per-texel array and its own amax entry (a CTA never
    // straddles two images, whatever M % 128)
    const size_t img = blockIdx.y;
    F += img * M * C;
    G += img * M * kL0;
    F16 += img * M * C;
    S4 += img * M * RES;
    if (amax) amax += img;
    if (nonfinite) nonfinite += img;
  }
  if (tid == 0) {
    for (int i = 0; i < kG0Stages; ++i) { tc::mbar_init(&b_full[i], 1); tc::mbar_init(&b_empty[i], kConsumers / 32); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumers / 32) {
    // ---- B producer: kG0NT x KB tiles in (nt, kb) order through the ring
    if (lane == 0) {
      for (int s = 0; s < kG0NT * KB; ++s) {
        const int slot = s % kG0Stages;
        tc::mbar_wait(&b_empty[slot], ((s / kG0Stages) & 1) ^ 1);
        tc::mbar_arrive_expect_tx(&b_full[slot], 32768);
        tc::bulk_g2s(sB + slot * 32768, Wt + (size_t)s * 32768, 32768, &b_full[slot]);
      }
    }
    return;
  }
  // ---- stage A (thread -> row = tid / 2, 32-column half of each 64-wide K-block)
  {
    const int row = tid >> 1, half = tid & 1;
    const bool live = (m0 + row) < M;
    const float* frow = F + (size_t)(live ? m0 + row : 0) * C + half * 32;
    float s4acc[RES];
    float fmax_abs = 0.f;             // range guard: the largest |feature| this thread stages
    float nf_probe = 0.f;             // x - x summed over the same features: NaN once one of them is a NaN or an infinity
#pragma unroll
    for (int r = 0; r < RES; ++r) s4acc[r] = 0.f;
#pragma unroll 1
    for (int kb = 0; kb < KB; ++kb) {
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = live ? __ldg(reinterpret_cast<const float4*>(frow + kb * 64) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < 8; ++j) fmax_abs = fmaxf(fmax_abs, fmaxf(fmaxf(fabsf(v[j].x), fabsf(v[j].y)), fmaxf(fabsf(v[j].z), fabsf(v[j].w))));
#pragma unroll
      for (int j = 0; j < 8; ++j) nf_probe += ((v[j].x - v[j].x) + (v[j].y - v[j].y)) + ((v[j].z - v[j].z) + (v[j].w - v[j].w));
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint4 pk;
        pk.x = tc::pack_half2(v[2 * j].x, v[2 * j].y);
        pk.y = tc::pack_half2(v[2 * j].z, v[2 * j].w);
        pk.z = tc::pack_half2(v[2 * j + 1].x, v[2 * j + 1].y);
        pk.w = tc::pack_half2(v[2 * j + 1].z, v[2 * j + 1].w);
        *reinterpret_cast<uint4*>(sA + kb * 16384 + tc::sw128_offset(row, half * 32 + j * 8)) = pk;
        if (live) *reinterpret_cast<uint4*>(F16 + (size_t)(m0 + row) * C + kb * 64 + half * 32 + j * 8) = pk;
      }
#pragma unroll
      for (int r = 0; r < RES; ++r) {
        const float4* wv = reinterpret_cast<const float4*>(w4s + r * C + kb * 64 + half * 32);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 w = __ldg(wv + j);
          s4acc[r] = fmaf(w.x, v[j].x, s4acc[r]); s4acc[r] = fmaf(w.y, v[j].y, s4acc[r]);
          s4acc[r] = fmaf(w.z, v[j].z, s4acc[r]); s4acc[r] = fmaf(w.w, v[j].w, s4acc[r]);
        }
      }
    }
    tc::fence_proxy_async_smem();
    if (amax) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) fmax_abs = fmaxf(fmax_abs, __shfl_xor_sync(0xffffffffu, fmax_abs, o));
      if (lane == 0) atomicMax(amax, __float_as_uint(fmax_abs));       // non-negative floats order like their bit patterns
    }
    // (fmaxf drops a NaN, so the maximum above cannot tell a map with a NaN: this flag can)
    if (nonfinite && __any_sync(0xffffffffu, !(nf_probe == 0.f)) && lane == 0) atomicMax(nonfinite, 1u);
#pragma unroll
    for (int r = 0; r < RES; ++r) {
      const float tot = s4acc[r] + __shfl_xor_sync(0xffffffffu, s4acc[r], 1);
      if (live && half == 0) S4[(size_t)(m0 + row) * RES + r] = tot;
    }
  }
  tc::bar_sync(1, kConsumers);
  // ---- MMAs + epilogue: warpgroup wg owns rows [64 wg, 64 wg + 64) of the CTA's 128
  const int wg = warp >> 2, wl = warp & 3;
  const int r0 = 16 * wl + (lane >> 2), cq = 2 * (lane & 3);
  const uint32_t a_base = tc::smem_u32(sA) + wg * 8192, b_base = tc::smem_u32(sB);
#pragma unroll 1
  for (int nt = 0; nt < kG0NT; ++nt) {
    float acc[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0.f;
    tc::wgmma_fence();
#pragma unroll 1
    for (int kb = 0; kb < KB; ++kb) {
      const int s = nt * KB + kb, slot = s % kG0Stages;
      tc::mbar_wait(&b_full[slot], (s / kG0Stages) & 1);
      const uint64_t da = tc::make_wdesc_sw128(a_base + kb * 16384, 1024), db = tc::make_wdesc_sw128(b_base + slot * 32768, 1024);
#pragma unroll
      for (int k = 0; k < 4; ++k) tc::wgmma_m64n256(acc, da + 2 * k, db + 2 * k);
      tc::wgmma_commit();
      tc::wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&b_empty[slot]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + 64 * wg + r0 + 8 * h;
      if (m < M) {
        __half* grow = G + (size_t)m * kL0 + nt * kG0TileN + cq;
#pragma unroll
        for (int j = 0; j < 32; ++j)
          *reinterpret_cast<uint32_t*>(grow + 8 * j) = tc::pack_half2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
  }
}

// --------------------------------------------------------------------------------------------------------------------
// host side: weight packing
// --------------------------------------------------------------------------------------------------------------------
// writes the [nrows x 64] fp16 K-major SWIZZLE_128B image of W[row0.., col0..col0+64) (W row-major [cout][cin])
// (lo = true: the fp16 rounding of what the first rounding lost, W - float(half(W)): the low half of an fp16 pair)
void pack_tile(uint8_t* dst, const float* W, int cin, int row0, int nrows, int col0, bool lo = false) {
  for (int r = 0; r < nrows; ++r)
    for (int k = 0; k < 64; ++k) {
      const float w = W[(size_t)(row0 + r) * cin + col0 + k];
      __half h = __float2half_rn(w);
      if (lo) h = __float2half_rn(w - __half2float(h));
      memcpy(dst + tc::sw128_offset(r, k), &h, 2);
    }
}

// the head's feature channels when one of the two shipped shapes, else 0
int head_channels(const mp_mlp* m) {
  if (m->n_layers != 5 || !m->skip) return 0;
  const int C = m->channels[0] - 1;
  if (C != 256 && C != 512) return 0;
  const int want[5] = {C + 1, kL0, kL1, kL2, kL3};
  for (int l = 0; l < 5; ++l)
    if (m->channels[l] != want[l]) return 0;
  return m->channels[5] == (C == 256 ? Prog<256>::RES : Prog<512>::RES) ? C : 0;
}

// weight stream of one tile in the order query_wg_kernel<C> takes it (see Prog)
template <int C>
std::vector<uint8_t> build_stream(const std::vector<std::vector<float>>& W, const mp_mlp* mlp) {
  using P = Prog<C>;
  std::vector<uint8_t> out((size_t)P::StagesPerTile * kStageBytes, 0);
  size_t st = 0;
  auto stage_ptr = [&]() { return out.data() + (st++) * kStageBytes; };
  const int cin1 = mlp->cin[1], cin2 = mlp->cin[2], cin3 = mlp->cin[3];
  for (int kb = 0; kb < 16 + P::XKB; ++kb)                  // L1: H0, then X (the z column is applied in the epilogue)
    for (int nh = 0; nh < 2; ++nh) pack_tile(stage_ptr(), W[1].data(), cin1, nh * 256, 256, kb * 64);
  for (int kb = 0; kb < 8 + P::XKB; ++kb) pack_tile(stage_ptr(), W[2].data(), cin2, 0, 256, kb * 64);     // L2: H1, then X
  for (int pass = 0; pass < P::L3Pass; ++pass)              // L3: X, then H2; colour: hi(W3), then lo(W3)
    for (int q = 0; q < (P::XKB + 4) / 2; ++q) {
      uint8_t* p = stage_ptr();
      for (int sub = 0; sub < 2; ++sub) {
        const int kb = 2 * q + sub;
        const int col0 = kb < P::XKB ? kL2 + kb * 64 : (kb - P::XKB) * 64;
        pack_tile(p + sub * 16384, W[3].data(), cin3, 0, 128, col0, pass == 1);
      }
    }
  if ((int)st != P::StagesPerTile) out.clear();
  return out;
}

template <int C>
int tc_prepare(mp_mlp* mlp) {
  using P = Prog<C>;
  std::vector<std::vector<float>> W(5), Bv(5);
  for (int l = 0; l < 5; ++l) {
    W[l].resize((size_t)mlp->cin[l] * mlp->cout[l]);
    Bv[l].resize(mlp->cout[l]);
    MP_CUDA(cudaMemcpy(W[l].data(), mlp->w[l], W[l].size() * sizeof(float), cudaMemcpyDeviceToHost));
    MP_CUDA(cudaMemcpy(Bv[l].data(), mlp->bias[l], Bv[l].size() * sizeof(float), cudaMemcpyDeviceToHost));
  }
  const std::vector<uint8_t> stream = build_stream<C>(W, mlp);
  if (stream.empty()) {
    mp_set_error("internal: weight stream stage count mismatch");
    return MP_E_INVALID;
  }
  TcPack* pk = new TcPack();
  memset(pk, 0, sizeof(*pk));
  pk->res = P::RES;
  pk->kind = C == 256 ? 0 : 1;
  mlp->tc = pk;
  auto upload = [&](const void* src, size_t bytes, void** dptr) -> cudaError_t {
    cudaError_t e = cudaMalloc(dptr, bytes);
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*dptr, src, bytes, cudaMemcpyHostToDevice);
  };
  cudaError_t e = upload(stream.data(), stream.size(), (void**)&pk->wstream);
  if (e == cudaSuccess) {   // feature part of layer 0 as fp16 SWIZZLE_128B tiles, operand of the per-texel G0 GEMM
    constexpr int KB = G0Cfg<C>::KB;
    std::vector<uint8_t> w0t((size_t)kG0NT * KB * 32768);
    for (int nt = 0; nt < kG0NT; ++nt)
      for (int kb = 0; kb < KB; ++kb)
        pack_tile(w0t.data() + ((size_t)nt * KB + kb) * 32768, W[0].data(), mlp->cin[0], nt * kG0TileN, kG0TileN, kb * 64);
    e = upload(w0t.data(), w0t.size(), (void**)&pk->d_w0t);
  }
  const int hid[4] = {0, kL0, kL1, kL2};
  for (int l = 0; l < 4 && e == cudaSuccess; ++l) {
    std::vector<float> wz(mlp->cout[l]);
    const int zcol = hid[l] + C;
    for (int co = 0; co < mlp->cout[l]; ++co) wz[co] = W[l][(size_t)co * mlp->cin[l] + zcol];
    memcpy(pk->h_bias + side_off(l), Bv[l].data(), Bv[l].size() * sizeof(float));
    memcpy(pk->h_wz + side_off(l), wz.data(), wz.size() * sizeof(float));
    if (l == 0) {
      std::vector<__half> b0h(Bv[0].size()), wz0h(wz.size());
      for (size_t i = 0; i < b0h.size(); ++i) { b0h[i] = __float2half_rn(Bv[0][i]); wz0h[i] = __float2half_rn(wz[i]); }
      e = upload(b0h.data(), b0h.size() * sizeof(__half), (void**)&pk->d_bias0);
      if (e == cudaSuccess) e = upload(wz0h.data(), wz0h.size() * sizeof(__half), (void**)&pk->d_wz0);
    }
  }
  if (e == cudaSuccess) {
    const int R = P::RES, cin4 = mlp->cin[4];
    std::vector<float> w4h((size_t)R * kL3), w4s((size_t)R * C), w4z(R);
    for (int r = 0; r < R; ++r) {
      for (int j = 0; j < kL3; ++j) w4h[(size_t)r * kL3 + j] = W[4][(size_t)r * cin4 + j];
      for (int j = 0; j < C; ++j) w4s[(size_t)r * C + j] = W[4][(size_t)r * cin4 + kL3 + j];
      w4z[r] = W[4][(size_t)r * cin4 + kL3 + C];
    }
    e = upload(w4h.data(), w4h.size() * sizeof(float), (void**)&pk->w4h);
    if (e == cudaSuccess) e = upload(w4s.data(), w4s.size() * sizeof(float), (void**)&pk->w4s);
    if (e == cudaSuccess) e = upload(w4z.data(), w4z.size() * sizeof(float), (void**)&pk->w4z);
    if (e == cudaSuccess) e = upload(Bv[4].data(), Bv[4].size() * sizeof(float), (void**)&pk->b4);
  }
  if (e == cudaSuccess) e = cudaFuncSetAttribute(query_wg_kernel<C, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, P::Total + 1024);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(query_wg_kernel<C, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, P::Total + 1024);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(g0_wg_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G0Cfg<C>::Smem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(query_jvp_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, P::Total + kJvpDwBytes + 1024);
  if (e != cudaSuccess) {
    mp_set_error("mp_tc_prepare: %s", cudaGetErrorString(e));
    mp_tc_release(mlp);
    return MP_E_CUDA;
  }
  mlp->tc_ok = 1;
  return MP_OK;
}

// per-frame per-texel products of the head (G0, the fp16 copy of the map, S4) for every map of the handle, when stale
template <int C>
int frame_products(const mp_mlp* mlp, const TcPack* pk, mp_feat* feat, cudaStream_t st) {
  using P = Prog<C>;
  const long long HW = (long long)feat->H * feat->W;
  const int maps = feat->B > 1 ? feat->B : 1;
  if (!feat->g0 || feat->g0_n != kL0) {     // (a map has one channel count, so it serves one of the two heads)
    if (feat->g0) cudaFree(feat->g0);
    feat->g0 = nullptr;
    MP_CUDA(cudaMalloc(&feat->g0, (size_t)maps * HW * kL0 * sizeof(__half)));
    if (!feat->f16) MP_CUDA(cudaMalloc(&feat->f16, (size_t)maps * HW * C * sizeof(__half)));
    if (!feat->s4tex) MP_CUDA(cudaMalloc(&feat->s4tex, (size_t)maps * HW * P::RES * sizeof(float)));
    feat->g0_n = kL0;
    feat->g0_owner = 0;
  }
  if (feat->g0_owner != mlp->gen || feat->g0_version != feat->version) {
    const dim3 g0_grid((unsigned)((HW + 127) / 128), (unsigned)maps);
#ifndef MP_CUDA_EMU
    g0_wg_kernel<C><<<g0_grid, kG0Threads, G0Cfg<C>::Smem, st>>>(feat->nhwc32, pk->d_w0t, feat->g0, (int)HW, feat->f16, feat->s4tex, pk->w4s,
                                                              feat->amax, feat->nonfinite);
#else
    // (a 2-D grid: the CPU model's launcher of tests/emu takes the dim3 itself)
    cuda_emu::launch(g0_grid, dim3((unsigned)kG0Threads),
                     [&] { g0_wg_kernel<C>(feat->nhwc32, pk->d_w0t, feat->g0, (int)HW, feat->f16, feat->s4tex, pk->w4s, feat->amax,
                                          feat->nonfinite); });
#endif
    MP_CUDA(cudaGetLastError());
    feat->g0_owner = mlp->gen;
    feat->g0_version = feat->version;
  }
  return MP_OK;
}

// the per-frame products, the kernel parameters of the head's program on the current frame of feat and the persistent
// grid (one CTA per SM, at most one per tile) of a launch over `tiles` tiles
template <int C>
int launch_setup(const mp_mlp* mlp, const TcPack* pk, mp_feat* feat, cudaStream_t st, int guard, long long tiles, TcParams& prm,
                 int& grid) {
  const int rp = frame_products<C>(mlp, pk, feat, st);
  if (rp != MP_OK) return rp;
  memset(&prm, 0, sizeof(prm));
  prm.amax = feat->amax; prm.amax_limit = mlp->tc_amax_limit; prm.guard = guard;
  prm.wstream = pk->wstream;
  memcpy(prm.bias_all, pk->h_bias, sizeof(prm.bias_all));
  memcpy(prm.wz_all, pk->h_wz, sizeof(prm.wz_all));
  prm.w4h = pk->w4h; prm.w4s = pk->w4s; prm.w4z = pk->w4z; prm.b4 = pk->b4;
  prm.res = pk->res;
  prm.last_op = mlp->last_op;
  prm.H = feat->H; prm.W = feat->W;
  prm.g0 = feat->g0;
  prm.feat16 = feat->f16;
  prm.s4tex = feat->s4tex;
  prm.d_bias0 = pk->d_bias0;
  prm.d_wz0 = pk->d_wz0;
  int dev = 0, sms = 132;
  MP_CUDA(cudaGetDevice(&dev));
  MP_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  grid = (int)(tiles < (long long)sms ? tiles : sms);
  return MP_OK;
}

// the per-frame products, then the fused query over the images of bt
template <int C>
int launch(const mp_mlp* mlp, const TcPack* pk, mp_feat* feat, const MpPointSrc& src, const MpCalib& cal, const MpOutDst& dst,
           cudaStream_t st, const MpSurfaceSrc& surf, int guard, const MpBatch& bt) {
  using P = Prog<C>;
  TcParams prm;
  int grid = 0;
  const int rs = launch_setup<C>(mlp, pk, feat, st, guard, bt.B * ((src.n + kTile - 1) / kTile), prm, grid);
  if (rs != MP_OK) return rs;
  if (surf.X && guard == MP_GUARD_NONE && isfinite(mlp->tc_amax_limit)) {
    // the eager rendering (mp_colorize_surface): check the frame's feature range on the host (one 4-byte read-back per
    // frame) and let the caller take the unfused path when it is outside the validated range.  (The enqueue-only render,
    // mp_colorize_surface_async, passes MP_GUARD_IN_RANGE instead and launches the exact twin beside this one.)
    unsigned bits = 0;
    MP_CUDA(cudaMemcpyAsync(&bits, feat->amax, sizeof(bits), cudaMemcpyDeviceToHost, st));
    MP_CUDA(cudaStreamSynchronize(st));
    float a;
    memcpy(&a, &bits, sizeof(a));
    if (a > mlp->tc_amax_limit) {
      mp_set_error("feature magnitude %.3g is outside the validated range of the tensor-core colour program (limit %.3g)", a, mlp->tc_amax_limit);
      return MP_E_RANGE;
    }
  }
#ifndef MP_CUDA_EMU
  if (dst.n_peers > 0) query_wg_kernel<C, true><<<grid, kThreads, P::Total + 1024, st>>>(prm, src, cal, dst, surf, bt);      // fused slab exchange
  else query_wg_kernel<C, false><<<grid, kThreads, P::Total + 1024, st>>>(prm, src, cal, dst, surf, bt);
#else
  if (dst.n_peers > 0) MP_EMU_LAUNCH(grid, kThreads, (query_wg_kernel<C, true>(prm, src, cal, dst, surf, bt)));
  else MP_EMU_LAUNCH(grid, kThreads, (query_wg_kernel<C, false>(prm, src, cal, dst, surf, bt)));
#endif
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

// the per-frame products, then the JVP program over the images of bt, src.n points each (16 points per tile)
template <int C>
int launch_jvp(const mp_mlp* mlp, const TcPack* pk, mp_feat* feat, const MpPointSrc& src, const MpCalib& cal, const JvpOut& jo,
               cudaStream_t st, int guard, const MpBatch& bt) {
  using P = Prog<C>;
  TcParams prm;
  int grid = 0;
  const int rs = launch_setup<C>(mlp, pk, feat, st, guard, bt.B * ((src.n + kJvpPts - 1) / kJvpPts), prm, grid);
  if (rs != MP_OK) return rs;
#ifndef MP_CUDA_EMU
  query_jvp_kernel<C><<<grid, kThreads, P::Total + kJvpDwBytes + 1024, st>>>(prm, src, cal, jo, bt);
#else
  MP_EMU_LAUNCH(grid, kThreads, (query_jvp_kernel<C>(prm, src, cal, jo, bt)));
#endif
  MP_CUDA(cudaGetLastError());
  return MP_OK;
}

// ---- the in-image list of a grid range (mp_launch_query_tc_grid), on the ordered scan of mp_scan.cuh
// The scan runs over a brick-major index space j: the 4x4x4 bricks of the brick layers that the range's z planes cross,
// x fastest inside a brick, then the bricks along x, y and z.  So a 64-point tile of the program is one brick wherever a
// brick lies wholly in the image, and its bilinear taps touch about 3x fewer texels than a run of 64 nodes along an x row
// (DESIGN.md §F1; tools/tile_texels.py counts them).  The program stores by node, so the order changes no value.
constexpr int kBrick = 4;   // the edge of a brick, in nodes (kBrick^3 = 64 = the program's tile)
static_assert(kBrick * kBrick * kBrick == kTile, "a brick is one tile of the program");

struct BrickSpace {
  int R, rb, bz0;           // nodes per axis, bricks per axis, the first brick layer
  long long lin0, n, size;  // the range [lin0, lin0 + n) and the number of indices j
  static BrickSpace of(int R, long long lin0, long long n) {
    BrickSpace s;
    s.R = R;
    s.rb = (R + kBrick - 1) / kBrick;
    const long long plane = (long long)R * R;
    s.bz0 = (int)(lin0 / plane) / kBrick;
    const int layers = (int)((lin0 + n - 1) / plane) / kBrick - s.bz0 + 1;
    s.lin0 = lin0;
    s.n = n;
    s.size = (long long)layers * s.rb * s.rb * (kBrick * kBrick * kBrick);
    return s;
  }
  // the range index (node - lin0) of index j, or -1 for padding past R and for nodes outside the range
  __device__ __forceinline__ long long node(long long j) const {
    const int b = (int)(j / (kBrick * kBrick * kBrick)), w = (int)(j % (kBrick * kBrick * kBrick));
    const int t = b / rb;
    const int ix = (b - t * rb) * kBrick + w % kBrick;
    const int iy = (t % rb) * kBrick + (w / kBrick) % kBrick;
    const int iz = (bz0 + t / rb) * kBrick + w / (kBrick * kBrick);
    if (ix >= R || iy >= R || iz >= R) return -1;
    const long long i = ((long long)iz * R + iy) * R + ix - lin0;
    return i >= 0 && i < n ? i : -1;
  }
};

// f(j) = 1 when j's node is in the range and projects into the image.  When the map holds a NaN or an infinity every
// node of the range counts: the range guard does not send every such frame to the exact kernel (its maximum ignores a
// NaN), and then 0 * act need not be +0 outside the image.
struct InImage {
  static constexpr bool kVec8 = false;
  BrickSpace bs;
  MpPointSrc grid;
  MpCalib cal;
  const unsigned* nonfinite;
  __device__ unsigned long long operator()(long long j) const {
    const long long i = bs.node(j);
    if (i < 0) return 0ull;
    if (nonfinite && *nonfinite) return 1ull;
    float x, y, z, u, v, w;
    mp_load_point(grid, MpBatch(), 0, i, x, y, z);
    return tc_project_in_image(cal, x, y, z, u, v, w) ? 1ull : 0ull;
  }
};

// a listed node goes to the list at its prefix (brick order: the program's stores by node are 16-byte runs); any other
// node of the range gets the value the dense launch gives it, +0
struct ListOrZero {
  BrickSpace bs;
  int32_t* list;
  float* out;                       // the range's outputs, or null
  float* peer[MP_MAX_PEERS];
  int n_peers;
  long long peer_off;
  __device__ void operator()(long long j, unsigned long long in, unsigned long long at) const {
    const long long i = bs.node(j);
    if (in) {
      list[at] = (int32_t)(bs.lin0 + i);
      return;
    }
    if (i < 0) return;
    if (out) out[i] = 0.f;
#pragma unroll
    for (int p = 0; p < MP_MAX_PEERS; ++p)
      if (p < n_peers) peer[p][peer_off + i] = 0.f;
  }
};

struct StoreCount {
  int32_t* count;
  __device__ void operator()(unsigned long long total) const { *count = (int32_t)total; }
};

// what the query and the gradient launches both need: the head's program prepared, a map of the head's channel count C
// and of at most 65536 texels (texel indices travel as 16-bit pairs in registers, per map of a batch)
int check_query(const mp_mlp* mlp, const mp_feat* feat, int& C) {
  const TcPack* pk = static_cast<const TcPack*>(mlp->tc);
  if (!pk || !mlp->tc_ok) {
    mp_set_error("tensor-core path not prepared for this head");
    return MP_E_UNSUPPORTED;
  }
  C = pk->kind == 1 ? 512 : 256;
  if (feat->C != C) {
    mp_set_error("head expects %d input channels but the feature map has %d (+1 depth)", mlp->channels[0], feat->C);
    return MP_E_INVALID;
  }
  if ((long long)feat->H * feat->W > 65536) {
    mp_set_error("the tensor-core program handles feature maps of at most 65536 texels (got %d x %d); use MP_MODE_FP32", feat->H, feat->W);
    return MP_E_UNSUPPORTED;
  }
  return MP_OK;
}

}  // namespace

int mp_tc_prepare(mp_mlp* mlp) {
  mlp->tc = nullptr;
  mlp->tc_ok = 0;
  const int C = head_channels(mlp);
  if (!C) return MP_OK;
  int dev = 0, major = 0, max_smem = 0;
  MP_CUDA(cudaGetDevice(&dev));
  MP_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  MP_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  // wgmma is sm_90a only (the library is built for exactly that target)
  if (major != 9 || max_smem < (C == 256 ? Prog<256>::Total : Prog<512>::Total) + 1024) return MP_OK;
  return C == 256 ? tc_prepare<256>(mlp) : tc_prepare<512>(mlp);
}

void mp_tc_release(mp_mlp* mlp) {
  TcPack* pk = static_cast<TcPack*>(mlp->tc);
  if (!pk) return;
  if (pk->wstream) cudaFree(pk->wstream);
  if (pk->d_bias0) cudaFree(pk->d_bias0);
  if (pk->d_wz0) cudaFree(pk->d_wz0);
  if (pk->d_w0t) cudaFree(pk->d_w0t);
  if (pk->w4h) cudaFree(pk->w4h);
  if (pk->w4s) cudaFree(pk->w4s);
  if (pk->w4z) cudaFree(pk->w4z);
  if (pk->b4) cudaFree(pk->b4);
  delete pk;
  mlp->tc = nullptr;
  mlp->tc_ok = 0;
}

int mp_launch_surface_tc(const mp_mlp* mlp, mp_feat* feat, const MpSurfaceSrc& surf, long long n, const MpCalib& cal,
                         cudaStream_t st, int guard, const MpBatch* bt) {
  if (n <= 0) return MP_OK;
  const TcPack* pk = static_cast<const TcPack*>(mlp->tc);
  if (!pk || !mlp->tc_ok || pk->kind != 1) {
    mp_set_error("fused surface colourisation needs the tensor-core program of the colour head");
    return MP_E_UNSUPPORTED;
  }
  if (bt && bt->B != 1) {
    mp_set_error("the surface render takes one map");
    return MP_E_UNSUPPORTED;
  }
  if (feat->C != 512 || (long long)feat->H * feat->W > 65536) {
    mp_set_error("colour head: needs a 512-channel map of at most 65536 texels (got %d channels, %d x %d)", feat->C, feat->H, feat->W);
    return MP_E_INVALID;
  }
  MpPointSrc src;
  memset(&src, 0, sizeof(src));
  src.kind = MP_SRC_ROWS;
  src.n = n;
  MpOutDst dst;
  dst.out = nullptr; dst.ld = 0; dst.scatter_vol = nullptr;
  return launch<512>(mlp, pk, feat, src, cal, dst, st, surf, guard, bt ? *bt : MpBatch());
}

int mp_launch_colour_surface(const mp_mlp* mlp, mp_feat* feat, const long long* X, const long long* Y, const float* Z, long long n,
                             int R, const float* b_min3, const float* b_max3, const MpCalib& cal, float* canvas, cudaStream_t st) {
  if (n <= 0) return MP_OK;
  return mp_launch_surface_tc(mlp, feat, mp_surface_src(X, Y, Z, nullptr, R, b_min3, b_max3, canvas), n, cal, st, MP_GUARD_NONE);
}

int mp_launch_query_tc(const mp_mlp* mlp, mp_feat* feat, const MpPointSrc& src, const MpCalib& cal,
                       const MpOutDst& dst, cudaStream_t st, int guard, const MpBatch* bt) {
  if (src.n <= 0) return MP_OK;
  int C = 0;
  const int rc = check_query(mlp, feat, C);
  if (rc != MP_OK) return rc;
  const TcPack* pk = static_cast<const TcPack*>(mlp->tc);
  if (dst.n_peers > MP_MAX_PEERS) {
    mp_set_error("at most %d peer volumes", MP_MAX_PEERS);
    return MP_E_UNSUPPORTED;
  }
  if (C == 512 && (dst.scatter_vol || dst.n_peers > 0 || !dst.out)) {
    mp_set_error("colour head: [3,N] output or surface canvas only");
    return MP_E_UNSUPPORTED;
  }
  MpSurfaceSrc surf;
  memset(&surf, 0, sizeof(surf));
  if (bt && bt->B > 1 && (src.kind != MP_SRC_ROWS || dst.scatter_vol || dst.n_peers > 0 || !dst.out)) {
    mp_set_error("batched launches take point rows and write [R,N] outputs");
    return MP_E_UNSUPPORTED;
  }
  const MpBatch& b = bt ? *bt : MpBatch();
  return C == 256 ? launch<256>(mlp, pk, feat, src, cal, dst, st, surf, guard, b)
                  : launch<512>(mlp, pk, feat, src, cal, dst, st, surf, guard, b);
}

// scratch of mp_launch_query_tc_grid: total[2] (grand total, ticket), the chunk sums, the count, the list.  The chunk
// sums cover the brick space, whose size depends on R and lin0 as well as n; this bounds it for every range of n nodes
// with R^3 < 2^31 (so R <= 1290): at most ((n - 1) / R^2 + 8) / 4 brick layers of at most 4 (R + 3)^2 indices each,
// which is under 16 n + 8 * 1293^2 (the factor (R + 3)^2 / R^2 is largest, 16, at R = 1).  That is 1.6 % more than the
// list, plus 52 KB.
static size_t grid_list_offset(long long n) {
  return 16 + 8 * (size_t)mpscan::num_blocks(16 * n + 8ll * 1293 * 1293) + 16;
}

size_t mp_tc_grid_scratch_bytes(long long n) { return grid_list_offset(n) + 4 * (size_t)n; }

// Three launches: the compaction's two (its zero stores first on the stream), then the program over the list.  Node
// coordinates are integers, so MP_SRC_NODES gives each node the world point MP_SRC_GRID gives it, bit for bit.
int mp_launch_query_tc_grid(const mp_mlp* mlp, mp_feat* feat, const MpPointSrc& grid, const MpCalib& cal, const MpOutDst& dst,
                            void* scratch, cudaStream_t st, int guard) {
  const long long n = grid.n;
  if (n <= 0) return MP_OK;
  int C = 0;
  int rc = check_query(mlp, feat, C);
  if (rc != MP_OK) return rc;
  if (C != 256 || mlp->last_op != MP_LAST_SIGMOID || grid.kind != MP_SRC_GRID || grid.lin0 < 0 ||
      grid.lin0 + n > (long long)grid.res * grid.res * grid.res || (long long)grid.res * grid.res * grid.res >= (1ll << 31) ||
      dst.n_peers > MP_MAX_PEERS || (dst.n_peers > 0 && dst.peer_off != grid.lin0) || dst.scatter_vol || dst.peer_by_node) {
    mp_set_error("the in-image grid launch takes a grid range of int32 node indices and a single-output Sigmoid head");
    return MP_E_UNSUPPORTED;
  }
  const TcPack* pk = static_cast<const TcPack*>(mlp->tc);
  // the map's non-finite flag, which the compaction reads, comes with the per-frame products
  rc = frame_products<256>(mlp, pk, feat, st);
  if (rc != MP_OK) return rc;
  const BrickSpace bs = BrickSpace::of(grid.res, grid.lin0, n);
  unsigned long long* total = static_cast<unsigned long long*>(scratch);
  int32_t* list = reinterpret_cast<int32_t*>(static_cast<uint8_t*>(scratch) + grid_list_offset(n));
  int32_t* count = list - 4;                     // (the 16 bytes before the list)
  const InImage f{bs, grid, cal, feat->nonfinite};
  ListOrZero em;
  em.bs = bs;
  em.list = list;
  em.out = dst.out;
  for (int p = 0; p < MP_MAX_PEERS; ++p) em.peer[p] = dst.peer[p];
  em.n_peers = dst.n_peers;
  em.peer_off = dst.peer_off;
#ifndef MP_CUDA_EMU
  MP_CUDA(mpscan::scan_emit(f, em, bs.size, total + 2, total, st, StoreCount{count}));
#else
  const int nb = mpscan::num_blocks(bs.size);
  MP_EMU_LAUNCH(nb, mpscan::kThreads, (mpscan::block_sums_kernel<InImage, StoreCount>(f, bs.size, total + 2, nb, total, StoreCount{count})));
  MP_EMU_LAUNCH(nb, mpscan::kThreads, (mpscan::emit_kernel<InImage, ListOrZero>(f, em, bs.size, total + 2)));
#endif
  MpPointSrc src = grid;                         // (n stays the upper bound of the device-side count)
  src.kind = MP_SRC_NODES;
  src.nodes = list;
  src.count_dev = count;
  MpOutDst ldst = dst;                           // values by node index: out through the node scatter, the peers by peer_by_node
  ldst.out = nullptr;
  ldst.ld = 0;
  ldst.scatter_vol = dst.out ? dst.out - grid.lin0 : nullptr;
  ldst.peer_by_node = 1;
  MpSurfaceSrc surf;
  memset(&surf, 0, sizeof(surf));
  return launch<256>(mlp, pk, feat, src, cal, ldst, st, surf, guard, MpBatch());
}

int mp_launch_query_jvp_tc(const mp_mlp* mlp, mp_feat* feat, const MpPointSrc& src, const MpCalib& cal, const float* grad_out,
                           long long ld_grad, float* out, long long ld_out, float* dpoints, long long ld_dp, cudaStream_t st, int guard,
                           const MpBatch* bt) {
  if (src.n <= 0) return MP_OK;
  int C = 0;
  const int rc = check_query(mlp, feat, C);
  if (rc != MP_OK) return rc;
  const TcPack* pk = static_cast<const TcPack*>(mlp->tc);
  MpBatch b = bt ? *bt : MpBatch();
  if (src.kind != MP_SRC_ROWS || feat->B != b.B) {
    mp_set_error("the gradient program takes point rows, one set per map of the handle");
    return MP_E_UNSUPPORTED;
  }
  // (the kernel finds a tile's image with a 32-bit division)
  if (b.B > 1 && b.B * ((src.n + kJvpPts - 1) / kJvpPts) >= (1ll << 31)) {
    mp_set_error("batch too large for the gradient program: %d x %lld points", b.B, src.n);
    return MP_E_UNSUPPORTED;
  }
  const long long res = pk->res;
  b.out_stride = res * ld_out;
  JvpOut jo;
  jo.out = out; jo.ld_out = ld_out;
  jo.dp = dpoints; jo.ld_dp = ld_dp; jo.dp_stride = 3 * ld_dp;
  jo.grad_out = grad_out; jo.ld_grad = ld_grad; jo.gout_stride = res * ld_grad;
  return C == 256 ? launch_jvp<256>(mlp, pk, feat, src, cal, jo, st, guard, b) : launch_jvp<512>(mlp, pk, feat, src, cal, jo, st, guard, b);
}
