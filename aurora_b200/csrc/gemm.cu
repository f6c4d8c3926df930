// Persistent, warp-specialised wgmma GEMM for sm_90a:  out = act(A · Wᵀ + bias) + residual.
//
//   A [M,K] bf16 (K contiguous), W [N,K] bf16 (K contiguous, nn.Linear layout), fp32 accumulation.
//
//   warpgroup 0    : TMA producer (one lane) — 128B-swizzled {64 x 128} A tiles and {64 x BN} W tiles into a ring of
//                    shared-memory stages; gives its registers up (setmaxnreg) to the math warpgroups
//   warpgroups 1-2 : math + epilogue — wgmma.mma_async m64nBNk16 straight from the swizzled stages into fp32
//                    register accumulators; bias / erf-GELU / residual on the registers, 16-bit-only outputs through
//                    two alternating swizzled shared-memory boxes per warp and TMA stores, with the tile's bias
//                    copied into shared memory when the tile starts
//
// Pipelines: full / empty mbarriers per stage (TMA <-> wgmma) and the static persistent tile schedule
// (tile = blockIdx.x + i * gridDim.x, N-blocks fastest so that the CTAs running concurrently share the same A rows in
// L2 while W stays L2-resident), loaded by the producer in order.  Three ways to share it (see the kernel):
//   cooperative : both math warpgroups work on every 128 x BN tile, 64 rows each (BN = 64 / 128 / 256)
//   ping-pong   : warpgroup w takes the positions i = w, w + 2, ... and all 128 rows of each 128 x 128 tile (two
//                 m64n128k16 per k16 sharing the W descriptor); it starts a main loop only once the other has issued
//                 the last k-block of its previous tile (two "order" mbarriers), so that one warpgroup's epilogue runs
//                 while the other's wgmmas keep the tensor pipe busy
//   staggered   : the cooperative 128 x 256 tile, with warpgroup 1 kept 1-2 k-blocks behind warpgroup 0 (two rings of
//                 "issued" mbarriers), so that each warpgroup's epilogue runs under the other's wgmmas for that long
// ab_gemm_bf16 runs every shape cooperative (see the reason there); AB_GEMM_SCHEDULE forces one of the three for tools
// and tests.  One wgmma group stays in flight while the next stage is waited for.
//
// Phase trace: built with -DAB_GEMM_TRACE (tools/gemm_trace.py does that into build/trace/), the kernel sums
// clock64() cycles per warp role and phase in registers and writes them once per CTA into a device buffer set with
// ab_gemm_trace(); without the switch the trace code compiles to nothing.
//
// Replaces: every nn.Linear on Aurora's forward path (see include/aurora_b200.h).
#include <stdlib.h>
#include <string.h>

#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace ab {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int kWgmmaK = 16;
constexpr int kMathWarps = 8;  // two warpgroups, one tile each
constexpr int kNumThreads = 128 + kMathWarps * 32;
constexpr int kBoxRows = 16;   // rows of one epilogue box = rows of one m64 accumulator that one warp holds
constexpr int kBoxBytes = kBoxRows * 128;

enum Schedule { kCooperative, kPingPong, kStaggered };

// Staggered schedule: warpgroup 1 issues ring position p only once warpgroup 0 has issued p + kLagMin (or the last
// k-block of p's tile), and warpgroup 0 issues p only once warpgroup 1 has issued p - kLagMax.  kLagMax = 2 of the
// 4 stages leaves the producer one stage of prefetch ahead of warpgroup 0.
constexpr int kLagMin = 1;
constexpr int kLagMax = 2;

template <int BN, int kSched>
struct GemmCfg {
  static constexpr int kStageBytesA = kBlockM * kBlockK * 2;
  static constexpr int kStageBytesB = BN * kBlockK * 2;
  static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
  static constexpr int kStages = BN >= 256 ? 4 : (BN >= 128 ? 6 : 8);
  // full + empty per stage, 2 order (ping-pong); staggered adds one "issued" ring per warpgroup
  static constexpr int kBarriers = 2 * kStages + 2 + (kSched == kStaggered ? 2 * kStages : 0);
  static constexpr int kBarrierBytes = kBarriers * 8;
  static constexpr int kStagingBytes = kMathWarps * 2 * kBoxBytes;  // two 16-row x 128-byte store boxes per math warp
  // the tile's BN bias values: one copy per warpgroup where the two warpgroups reach their epilogues at different
  // times (ping-pong: different tiles; staggered: the same tile, k-blocks apart), one for cooperative
  static constexpr int kBiasGroups = kSched == kCooperative ? 1 : 2;
  static constexpr int kBiasThreads = kMathWarps * 32 / kBiasGroups;  // the math threads that share a copy
  static constexpr int kBiasBytes = kBiasGroups * BN * 4;
  // no alignment slack: smem_raw is declared 1024-byte aligned (staggered BN = 256 needs all but 880 bytes of 227 KB)
  static constexpr int kSmemBytes = kStages * kStageBytes + kStagingBytes + kBiasBytes + kBarrierBytes;
  static_assert(kSched != kStaggered || (kStages > kLagMax + 1 && kLagMin < kLagMax), "lag bounds (see the kernel)");
  static_assert(kSmemBytes <= 227 * 1024, "shared memory");
};

// Phase trace slots (see Trace).  A CTA's record is kTrCta 64-bit words, then kTrSlots per math warp.
enum TraceCta { kTrTimerStart, kTrTimerEnd, kTrClockStart, kTrClockEnd, kTrEmptyWait, kTrProducerTiles, kTrCta };
enum TraceSlot {
  kTrFullFirst,  // full_bar wait of a tile's first k-block (producer: empty_bar waits)
  kTrFullRest,   // full_bar waits of its other k-blocks
  kTrOrder,      // order_bar wait (ping-pong), lead_bar / follow_bar waits (staggered)
  kTrWait1,      // wgmma_wait<1> in the main loop
  kTrWait0,      // wgmma_wait<0> after it
  kTrEpi,        // the whole epilogue
  kTrEpiStore,   // of which: waits for a store buffer
  kTrEpiBias,    // of which: waits for the bias values
  kTrTiles,      // tiles taken
  kTrSlots
};
#ifdef AB_GEMM_TRACE
constexpr int kTrWords = kTrCta + kMathWarps * kTrSlots;
#endif

// Per-thread cycle sums of the phase trace; without AB_GEMM_TRACE every member is empty and compiles away.
struct Trace {
#ifdef AB_GEMM_TRACE
  uint32_t c[kTrSlots] = {};
  __device__ __forceinline__ long long now() const { return clock64(); }
  __device__ __forceinline__ void add(int slot, long long t0) { c[slot] += static_cast<uint32_t>(clock64() - t0); }
  __device__ __forceinline__ void tick(int slot) { ++c[slot]; }
#else
  __device__ __forceinline__ long long now() const { return 0; }
  __device__ __forceinline__ void add(int, long long) {}
  __device__ __forceinline__ void tick(int) {}
#endif
};

// Rows of the 16-bit output that are ALSO stored into a neighbouring GPU's memory by the epilogue (the K | V halo rows of
// a latitude-sharded forecast: the QKV projection pushes them over NVLink itself, fused compute + exchange, instead of
// a separate copy kernel; protocol and buffer layout: csrc/halo.cu).  Up to 8 row ranges = 2 sides x 4 levels.
struct PeerRows {
  int n_ranges;         // 0 = off
  int col_from;         // only boxes whose first column is >= col_from are sent (multiple of 64)
  int dst_ld;           // destination row pitch in elements
  int expected;         // number of 16-row x 64-column epilogue boxes of this launch that carry peer rows
  int row_begin[8], row_end[8];
  uint16_t* dst[8];     // peer address of (row_begin[i], col_from)
  uint32_t* flag[2];    // the neighbours' "rows landed" flags
  uint32_t* ctrl;       // this rank's control words: [2] round, [3] completion counter
};

struct GemmArgs {
  const float* bias;
  const float* residual;
  float* out_f32;
  uint16_t* out_bf16;  // 16-bit output (bf16 or fp16, see out_half)
  int m, n, k;
  int ldr, ld_f32, ld_bf16;
  int act;
  int vec_ok;    // all leading dimensions / pointers allow 16-byte vector access
  int out_half;  // 16-bit output is fp16 instead of bf16
  int tma_out;   // 16-bit-only output written through swizzled smem + TMA store (tmap_out valid), bias staged in smem
  PeerRows peer;
#ifdef AB_GEMM_TRACE
  unsigned long long* trace;  // kTrWords per CTA
#endif
};

// Destination in a neighbour's memory of columns col .. col + 64 of output row `row`, or nullptr.
__device__ __forceinline__ uint16_t* peer_row_ptr(const GemmArgs& g, int row, int col) {
  uint16_t* p = nullptr;
  if (g.peer.n_ranges > 0 && col >= g.peer.col_from && row < g.m) {
#pragma unroll 1
    for (int i = 0; i < g.peer.n_ranges; ++i)
      if (row >= g.peer.row_begin[i] && row < g.peer.row_end[i])
        p = g.peer.dst[i] + static_cast<size_t>(row - g.peer.row_begin[i]) * g.peer.dst_ld + (col - g.peer.col_from);
  }
  return p;
}

// After a box with peer rows: make the stores visible system-wide, count the box, and let the LAST box of the launch
// publish the new round in both neighbours' flags (same hand-over as halo_push_kernel).
__device__ __forceinline__ void peer_box_done(const GemmArgs& g, int lane) {
  __threadfence_system();
  __syncwarp();
  if (lane == 0) {
    const unsigned done = atomicAdd(&g.peer.ctrl[3], 1u);
    if (done == static_cast<unsigned>(g.peer.expected) - 1u) {
      __threadfence_system();
      const uint32_t round = g.peer.ctrl[2] + 1u;
      g.peer.ctrl[2] = round;
      g.peer.ctrl[3] = 0u;
      asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(g.peer.flag[0]), "r"(round) : "memory");
      asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(g.peer.flag[1]), "r"(round) : "memory");
    }
  }
}

// Bias and activation on two adjacent accumulator columns (col, col + 1; col is even).
__device__ __forceinline__ void bias_act2(const GemmArgs& g, int col, float& x0, float& x1) {
  if (g.bias != nullptr) {
    if (col + 1 < g.n) {
      x0 += __ldg(g.bias + col);
      x1 += __ldg(g.bias + col + 1);
    } else if (col < g.n) {
      x0 += __ldg(g.bias + col);
    }
  }
  if (g.act == AB_ACT_GELU_ERF) {
    x0 = gelu_erf(x0);
    x1 = gelu_erf(x1);
  }
}

// General epilogue: this thread's two rows (row0, row0 + 8) x BN / 4 columns of the accumulator straight to global
// memory.  A quad of lanes covers 8 consecutive columns: 32 bytes of the fp32 output, 16 bytes of the 16-bit one.
// Row-major order keeps one row's addresses live at a time (the register budget is set by the accumulators).
template <int BN>
__device__ __forceinline__ void epilogue_direct(const GemmArgs& g, float (&acc)[BN / 2], int row0, int col0) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 8 * h;
    if (row >= g.m) continue;
    const float* const res = g.residual + static_cast<size_t>(row) * g.ldr;
    float* const o32 = g.out_f32 + static_cast<size_t>(row) * g.ld_f32;
    uint16_t* const o16 = g.out_bf16 + static_cast<size_t>(row) * g.ld_bf16;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = col0 + 8 * j;
      if (col >= g.n) continue;
      float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
      bias_act2(g, col, x0, x1);
      if (g.vec_ok && col + 1 < g.n) {
        if (g.residual != nullptr) {
          const float2 r = __ldg(reinterpret_cast<const float2*>(res + col));
          x0 += r.x;
          x1 += r.y;
        }
        if (g.out_f32 != nullptr) *reinterpret_cast<float2*>(o32 + col) = make_float2(x0, x1);
        if (g.out_bf16 != nullptr)
          *reinterpret_cast<uint32_t*>(o16 + col) = g.out_half ? pack_f16x2(x0, x1) : pack_bf16x2(x0, x1);
      } else {
        const float x[2] = {x0, x1};
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (col + e >= g.n) continue;
          float v = x[e];
          if (g.residual != nullptr) v += __ldg(res + col + e);
          if (g.out_f32 != nullptr) o32[col + e] = v;
          if (g.out_bf16 != nullptr) o16[col + e] = to16(v, g.out_half);
        }
      }
    }
  }
}

// Copy of the tile's bias values n0 .. n0 + BN into the group's shared-memory slice, asynchronously (cp.async, 16 bytes
// per thread, waited for at the epilogue); columns past N read 0.  Issued at the start of a tile so that the epilogue
// has no global load: a bias __ldg there waits on L2 once per box.  kThreads: the math threads that share the slice.
template <int BN, int kThreads>
__device__ __forceinline__ void stage_bias(const GemmArgs& g, float* bias_s, int n0, int tid) {
  static_assert(BN / 4 <= kThreads, "one 16-byte copy per thread");
  if (tid < BN / 4) {
    const int col = n0 + 4 * tid;
    const int bytes = col >= g.n ? 0 : (g.n - col >= 4 ? 16 : 4 * (g.n - col));
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(bias_s + 4 * tid)),
                 "l"(g.bias + (bytes > 0 ? col : 0)), "r"(bytes)
                 : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// Named barrier of the kThreads math threads that share a bias slice (id 0 is __syncthreads).
template <int kThreads>
__device__ __forceinline__ void group_sync(int id) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(kThreads) : "memory");
}

// 16-bit-only epilogue of one 16-row x 64-column box (rows row0 .. row0 + 15 of the output, columns colb ..): bias (from
// the group's shared-memory copy) / activation on the registers, 16-bit pairs into one of this warp's two staging boxes
// (16 rows x 128 bytes, 128B swizzle: chunk ^= row & 7, the layout a CU_TENSOR_MAP_SWIZZLE_128B store expects), then
// one asynchronous TMA store: full 128-byte rows, M / N tails clipped by the tensor map.  The staging stores are
// stmatrix, 4 per box where 32-bit stores would take 16: in ping-pong they queue for shared memory behind the other
// warpgroup's wgmma operand reads, and fewer of them shorten the epilogue (4.8 against 5.0 µs per tile, stage-1 qkv).  The two buffers alternate per issued
// store, so filling one only waits for the store issued two boxes ago.  Rows that a neighbouring GPU needs are copied
// out of the staging box into its halo slot, 16 bytes per lane.
template <int BN>
__device__ __forceinline__ void epilogue_tma_box(const GemmArgs& g, const CUtensorMap* tmap_out, const float (&acc)[BN / 2],
                                                 const float* bias_s, int c, uint8_t* staging, uint32_t& nst,
                                                 int row0, int colb, int lane, Trace& tr) {
  if (row0 >= g.m) return;  // warp-uniform: the box lies below the matrix
  uint8_t* const stage = staging + (nst & 1u) * kBoxBytes;
  const int t = lane & 3;
  const long long t0 = tr.now();
  if (lane == 0) tma_store_wait_read<1>();  // the store that last read this buffer is done with it
  __syncwarp();
  tr.add(kTrEpiStore, t0);
  // stmatrix: four 8 x 8 16-bit matrices per instruction, (jj, rows 0-7), (jj, rows 8-15), (jj + 1, rows 0-7),
  // (jj + 1, rows 8-15), in the accumulator's fragment layout; lane l gives the address of row l & 7 of matrix l >> 3
  const int mi = lane >> 3, rr = lane & 7;
  const uint32_t row_addr = smem_u32(stage) + (rr + 8 * (mi & 1)) * 128;
#pragma unroll
  for (int jj = 0; jj < 8; jj += 2) {
    uint32_t v[4];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int j = 8 * c + jj + q;
      float x0 = acc[4 * j], x1 = acc[4 * j + 1], y0 = acc[4 * j + 2], y1 = acc[4 * j + 3];
      if (g.bias != nullptr) {  // one load for both rows; columns past N hold 0 (the tensor map clips them)
        const float2 b = *reinterpret_cast<const float2*>(bias_s + 8 * j + 2 * t);
        x0 += b.x;
        x1 += b.y;
        y0 += b.x;
        y1 += b.y;
      }
      if (g.act == AB_ACT_GELU_ERF) {
        x0 = gelu_erf(x0);
        x1 = gelu_erf(x1);
        y0 = gelu_erf(y0);
        y1 = gelu_erf(y1);
      }
      v[2 * q] = g.out_half ? pack_f16x2(x0, x1) : pack_bf16x2(x0, x1);
      v[2 * q + 1] = g.out_half ? pack_f16x2(y0, y1) : pack_bf16x2(y0, y1);
    }
    const uint32_t addr = row_addr + (((jj + (mi >> 1)) ^ rr) << 4);
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v[0]), "r"(v[1]),
                 "r"(v[2]), "r"(v[3])
                 : "memory");
  }
  if (g.peer.n_ranges > 0) {
    __syncwarp();
    bool any = false;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int lr = 4 * i + (lane >> 3), chunk = lane & 7;
      uint16_t* const dst = peer_row_ptr(g, row0 + lr, colb);
      if (dst != nullptr) {
        any = true;
        *reinterpret_cast<uint4*>(dst + chunk * 8) =
            *reinterpret_cast<const uint4*>(stage + lr * 128 + ((chunk ^ (lr & 7)) << 4));
      }
    }
    if (__any_sync(0xffffffffu, any)) peer_box_done(g, lane);
  }
  fence_proxy_async_smem();
  __syncwarp();
  if (lane == 0) {
    tma_store_2d(tmap_out, stage, colb, row0);
    tma_store_commit();
  }
  ++nst;
}

// 16-bit-only epilogue of a warpgroup's kRB x 64 rows: per 64-column box, each 64-row block in turn.
template <int BN, int kRB>
__device__ __forceinline__ void epilogue_tma(const GemmArgs& g, const CUtensorMap* tmap_out, const float (&acc)[kRB][BN / 2],
                                             const float* bias_s, uint8_t* staging, uint32_t& nst, int warp_row0,
                                             int n0, int lane, Trace& tr) {
#pragma unroll
  for (int c = 0; c < BN / 64; ++c) {
    const int colb = n0 + 64 * c;
    if (colb >= g.n) continue;  // warp-uniform
#pragma unroll
    for (int rb = 0; rb < kRB; ++rb)
      epilogue_tma_box<BN>(g, tmap_out, acc[rb], bias_s, c, staging, nst, warp_row0 + 64 * rb, colb, lane, tr);
  }
}

// kCooperative: both math warpgroups work on every tile of the CTA, warpgroup w on rows [64 w, 64 w + 64) (one
//   m64nBNk16 accumulator each, BN up to 256).
// kPingPong: warpgroup w takes the tiles at positions w, w + 2, ... of the CTA's sequence and all 128 rows of each (two
//   m64nBNk16 accumulators, BN = 128); it starts a main loop only once the other warpgroup has issued the last k-block
//   of the tile before, so that one warpgroup's epilogue runs under the other's wgmmas.
// kStaggered: the cooperative tile and stage ring (every stage is freed by all 8 math warps), with warpgroup 0 ("the
//   leader") kept between kLagMin and kLagMax k-blocks ahead of warpgroup 1 ("the follower").  Ring position p is
//   the CTA's p-th k-block, the same sequence for both warpgroups; after issuing p each warpgroup arrives on its own
//   "issued" ring (lead_bar / follow_bar [p mod S], one arrival per warp, phase p / S).  Before issuing p:
//     leader   waits until the follower has issued p - kLagMax (the upper bound: the follower's releases keep the
//              producer kLagMax - 1 stages ahead of the leader, so the leader does not wait on TMA latency);
//     follower waits until the leader has issued min(p + kLagMin, last k-block of p's tile) (the lower bound, clamped
//              to the tile: the follower never waits for the leader's epilogue).
//   So the follower's last k-blocks of a tile run under the leader's epilogue, and the leader's first kLagMax
//   k-blocks of the next tile under the follower's epilogue.  Each warpgroup stages its own bias copy, with its own
//   named barrier: the two never synchronise except through the rings.
//   No deadlock (S = kStages, kLagMin < kLagMax < S - 1; a warpgroup frees p right after issuing p + 1, or after its
//   wgmma_wait<0> when p ends its tile, with no wait in between).  Let the leader wait at a, the follower at b:
//     - leader on the follower (b <= a - kLagMax): the follower needs the leader at b + kLagMin < a, issued, and
//       stage b, which needs b - S freed by both: the leader issued up to a - 1 > b - S + 1, the follower up to b - 1.
//     - leader on stage a: needs a - S freed by the follower, so b <= a - S + 1; the follower needs the leader at
//       <= b + kLagMin < a (issued) and stage b (b - S freed by both, as above).
//     - follower on the leader (a <= min(b + kLagMin, end)): the leader needs the follower at a - kLagMax < b
//       (issued) and stage a: a - S <= b + kLagMin - S < b - 1 is freed by both.
//   Each case names a wait that the blocked warpgroup's partner or the producer can satisfy without waiting on the
//   first, so the three always progress.  Both take every tile of the CTA, so the sequence is the same whatever the
//   tile count, K (one k-block included: the lower bound then points inside the same tile) or M tail (rows past M are
//   zero-filled by TMA and computed as usual).  Parity: when the follower waits on lead_bar for q, the leader has
//   issued q - S (the follower's previous wait) and cannot issue q + S (stage q + S needs the follower to free q);
//   symmetrically for follow_bar, so the wait never sees a phase too early or too late.
template <int BN, int kSched, bool kHalfIn>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                    const __grid_constant__ CUtensorMap tmap_out, const GemmArgs g) {
  using Cfg = GemmCfg<BN, kSched>;
  constexpr bool kPP = kSched == kPingPong;
  constexpr bool kStag = kSched == kStaggered;
  constexpr int kRB = kPP ? 2 : 1;  // 64-row accumulator blocks per warpgroup
  extern __shared__ __align__(1024) uint8_t smem_raw[];  // 128B-swizzled tiles need 1024-byte alignment
  uint8_t* smem = smem_raw;
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kStageBytesA;
  uint8_t* smem_stage_out = smem + Cfg::kStages * Cfg::kStageBytes;  // 1024-byte aligned (stages are)
  float* smem_bias = reinterpret_cast<float*>(smem_stage_out + Cfg::kStagingBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_stage_out + Cfg::kStagingBytes + Cfg::kBiasBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;
  uint64_t* order_bar = empty_bar + Cfg::kStages;  // ping-pong, [w]: math warpgroup w may start its next main loop
  uint64_t* lead_bar = order_bar + 2;               // staggered, [p mod S]: the leader has issued ring position p
  uint64_t* follow_bar = lead_bar + Cfg::kStages;   // staggered: the follower has issued p

  const int warp = threadIdx.x >> 5;  // warp-uniform
  const int lane = threadIdx.x & 31;
  Trace tr;
#ifdef AB_GEMM_TRACE
  unsigned long long* const trace = g.trace + static_cast<size_t>(blockIdx.x) * kTrWords;
  if (threadIdx.x == 0) {
    trace[kTrTimerStart] = global_timer_ns();
    trace[kTrClockStart] = clock64();
  }
#endif

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_w);
    if (g.tma_out) prefetch_tmap(&tmap_out);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kPP ? 4 : kMathWarps);  // the warps that consume the stage
      if (kStag) {
        mbar_init(&lead_bar[s], 4);
        mbar_init(&follow_bar[s], 4);
      }
    }
    mbar_init(&order_bar[0], 4);
    mbar_init(&order_bar[1], 4);
    fence_mbar_init();
  }
  __syncthreads();

  const int num_n = (g.n + BN - 1) / BN;
  const int num_m = (g.m + kBlockM - 1) / kBlockM;
  const int num_tiles = num_m * num_n;
  const int num_kb = (g.k + kBlockK - 1) / kBlockK;

  if (warp < 4) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      // ===== TMA producer =====
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / num_n) * kBlockM;
        const int n0 = (tile % num_n) * BN;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const uint32_t s = it % Cfg::kStages;
          const uint32_t ph = (it / Cfg::kStages) & 1u;
          const long long t0 = tr.now();
          mbar_wait(&empty_bar[s], ph ^ 1u);
          tr.add(kTrFullFirst, t0);
          mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
          tma_load_2d(smem_a + s * Cfg::kStageBytesA, &tmap_a, &full_bar[s], kb * kBlockK, m0);
          tma_load_2d(smem_b + s * Cfg::kStageBytesB, &tmap_w, &full_bar[s], kb * kBlockK, n0);
        }
        tr.tick(kTrTiles);
      }
#ifdef AB_GEMM_TRACE
      trace[kTrEmptyWait] = tr.c[kTrFullFirst];
      trace[kTrProducerTiles] = tr.c[kTrTiles];
#endif
    }
  } else {
    // ===== math warpgroups =====
    reg_alloc<232>();
    const int wg = (warp >> 2) - 1;
    // first of this warp's 16 rows inside the tile (inside each 64-row block for ping-pong)
    const int warp_row = (kPP ? 0 : wg * 64) + (warp & 3) * kBoxRows;
    uint8_t* const staging = smem_stage_out + (warp - 4) * (2 * kBoxBytes);
    // the bias copy of this warp's group (ping-pong / staggered: its warpgroup; cooperative: both) and the group's
    // named barrier
    const int bias_group = kSched == kCooperative ? 0 : wg;
    float* const bias_s = smem_bias + bias_group * BN;
    const int bias_tid = threadIdx.x - 128 - bias_group * Cfg::kBiasThreads;
    // staggered: the ring this warpgroup signals after issuing a k-block, and the one it waits on
    uint64_t* const issued_bar = wg == 0 ? lead_bar : follow_bar;
    uint64_t* const partner_bar = wg == 0 ? follow_bar : lead_bar;
    float acc[kRB][BN / 2];
    uint32_t nst = 0;  // TMA stores this warp has issued: picks the staging buffer
    constexpr int kStep = kPP ? 2 : 1;
    uint32_t j = 0;  // tiles this warpgroup has taken
    for (int i = kPP ? wg : 0;; i += kStep, ++j) {
      const int tile = blockIdx.x + i * gridDim.x;
      if (tile >= num_tiles) break;
      const int m0 = (tile / num_n) * kBlockM;
      const int n0 = (tile % num_n) * BN;
      if (g.tma_out && g.bias != nullptr) {
        group_sync<Cfg::kBiasThreads>(1 + bias_group);  // the group's previous epilogue has read the old values
        stage_bias<BN, Cfg::kBiasThreads>(g, bias_s, n0, bias_tid);
      }
      // ping-pong: tile i - 1 (the other warpgroup's) has issued all its wgmmas
      if (kPP && i > 0) {
        const long long t0 = tr.now();
        mbar_wait(&order_bar[wg], (wg == 0 ? j - 1 : j) & 1u);
        tr.add(kTrOrder, t0);
      }
      uint32_t it = static_cast<uint32_t>(i) * num_kb;  // the ring position of this tile's first k-block
      const uint32_t it_last = it + num_kb - 1;
      int prev_s = -1;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const uint32_t s = it % Cfg::kStages;
        if (kStag && (wg == 1 || it >= kLagMax)) {  // the lag bounds (see the kernel comment)
          const uint32_t q = wg == 0 ? it - kLagMax : min(it + kLagMin, it_last);
          const long long t0 = tr.now();
          mbar_wait(&partner_bar[q % Cfg::kStages], (q / Cfg::kStages) & 1u);
          tr.add(kTrOrder, t0);
        }
        const long long t0 = tr.now();
        mbar_wait(&full_bar[s], (it / Cfg::kStages) & 1u);
        if (kb == 0) tr.add(kTrFullFirst, t0);
        else tr.add(kTrFullRest, t0);
        const uint32_t a_addr = smem_u32(smem_a + s * Cfg::kStageBytesA) + (kPP ? 0 : wg * (64 * 128));
        const uint32_t b_addr = smem_u32(smem_b + s * Cfg::kStageBytesB);
#pragma unroll
        for (int rb = 0; rb < kRB; ++rb) wgmma_fence_regs(acc[rb]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
          const uint64_t desc_b = wgmma_desc_sw128(b_addr + k * kWgmmaK * 2);
#pragma unroll
          for (int rb = 0; rb < kRB; ++rb)
            wgmma_ss<BN, kHalfIn>(acc[rb], wgmma_desc_sw128(a_addr + rb * (64 * 128) + k * kWgmmaK * 2), desc_b,
                                  (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        if (kPP && kb == num_kb - 1 && lane == 0) mbar_arrive(&order_bar[wg ^ 1]);  // hand the tensor pipe over
        if (kStag && lane == 0) mbar_arrive(&issued_bar[s]);
        if (prev_s >= 0) {
          const long long t1 = tr.now();
          wgmma_wait<1>();  // the previous stage's wgmmas have retired: hand its shared memory back to the producer
          tr.add(kTrWait1, t1);
          if (lane == 0) mbar_arrive(&empty_bar[prev_s]);
        }
        prev_s = static_cast<int>(s);
      }
      long long t0 = tr.now();
      wgmma_wait<0>();
#pragma unroll
      for (int rb = 0; rb < kRB; ++rb) wgmma_fence_regs(acc[rb]);
      tr.add(kTrWait0, t0);
      if (lane == 0) mbar_arrive(&empty_bar[prev_s]);
      t0 = tr.now();
      if (g.tma_out) {
        if (g.bias != nullptr) {
          const long long t1 = tr.now();
          asm volatile("cp.async.wait_all;" ::: "memory");
          group_sync<Cfg::kBiasThreads>(1 + bias_group);  // every thread's copy has landed
          tr.add(kTrEpiBias, t1);
        }
        epilogue_tma<BN, kRB>(g, &tmap_out, acc, bias_s, staging, nst, m0 + warp_row, n0, lane, tr);
      } else {
#pragma unroll
        for (int rb = 0; rb < kRB; ++rb)
          epilogue_direct<BN>(g, acc[rb], m0 + 64 * rb + warp_row + (lane >> 2), n0 + 2 * (lane & 3));
      }
      tr.add(kTrEpi, t0);
      tr.tick(kTrTiles);
    }
    if (g.tma_out && lane == 0) tma_store_wait_all<0>();  // smem must outlive the bulk stores
#ifdef AB_GEMM_TRACE
    if (lane == 0)
      for (int s = 0; s < kTrSlots; ++s) trace[kTrCta + (warp - 4) * kTrSlots + s] = tr.c[s];
#endif
  }
#ifdef AB_GEMM_TRACE
  __syncthreads();
  if (threadIdx.x == 0) {
    trace[kTrClockEnd] = clock64();
    trace[kTrTimerEnd] = global_timer_ns();
  }
#endif
}

#ifdef AB_GEMM_TRACE
static unsigned long long* g_trace_buf = nullptr;
#endif

template <int BN, int kSched, bool kHalfIn>
static int launch_gemm(const AbGemm* p, GemmArgs& args, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, kSched>;
  CUtensorMap ta, tw;
  int rc = make_tmap_16bit_2d(&ta, p->a, p->m, p->k, p->lda, kBlockM, kBlockK, kHalfIn);
  if (rc != AB_OK) return rc;
  rc = make_tmap_16bit_2d(&tw, p->w, p->n, p->k, p->ldw, BN, kBlockK, kHalfIn);
  if (rc != AB_OK) return rc;
  CUtensorMap tout = ta;  // placeholder when unused
  if (args.tma_out) {
    rc = make_tmap_16bit_2d(&tout, p->out_bf16, p->m, p->n, p->ld_bf16, kBoxRows, 64, args.out_half != 0);
    if (rc != AB_OK) return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_tn_kernel<BN, kSched, kHalfIn>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_error("ab_gemm_bf16: cudaFuncSetAttribute(smem=%d) failed: %s", Cfg::kSmemBytes, cudaGetErrorString(e));
      return AB_ERR_CUDA;
    }
    attr_set = true;
  }
  const long long tiles = ceil_div_ll(p->m, kBlockM) * ceil_div_ll(p->n, BN);
  const int grid = static_cast<int>(tiles < sm_count() ? tiles : sm_count());
#ifdef AB_GEMM_TRACE
  AB_CHECK_ARG(g_trace_buf != nullptr, "ab_gemm_bf16: traced build without a trace buffer (ab_gemm_trace)");
  args.trace = g_trace_buf;
#endif
  gemm_bf16_tn_kernel<BN, kSched, kHalfIn><<<grid, kNumThreads, Cfg::kSmemBytes, stream>>>(ta, tw, tout, args);
  AB_COUNT_LAUNCH(1);
  AB_CHECK_LAUNCH("ab_gemm_bf16");
  return AB_OK;
}

// The tile shape of each schedule: 128 x 128 per warpgroup for ping-pong, 128 x 256 per CTA for cooperative and
// staggered while N > 128, 128 x 128 / 128 x 64 cooperative for the narrower decoder heads.
template <bool kHalfIn>
static int launch_for(const AbGemm* p, GemmArgs& args, cudaStream_t stream, int sched) {
  if (p->n > 128) {
    if (sched == kPingPong) return launch_gemm<128, kPingPong, kHalfIn>(p, args, stream);
    if (sched == kStaggered) return launch_gemm<256, kStaggered, kHalfIn>(p, args, stream);
    return launch_gemm<256, kCooperative, kHalfIn>(p, args, stream);
  }
  if (p->n > 64) return launch_gemm<128, kCooperative, kHalfIn>(p, args, stream);
  return launch_gemm<64, kCooperative, kHalfIn>(p, args, stream);
}

// AB_GEMM_SCHEDULE=pingpong|cooperative|staggered, read once: every GEMM with N > 128 takes that schedule instead of
// the rule in ab_gemm_bf16, so that tools and tests can compare the schedules on the same shapes.  The model never
// sets it.  -1: unset.
constexpr int kBadSchedule = -2;
static int forced_schedule() {
  static const int forced = [] {
    const char* e = getenv("AB_GEMM_SCHEDULE");
    if (e == nullptr || *e == 0) return -1;
    if (strcmp(e, "pingpong") == 0) return static_cast<int>(kPingPong);
    if (strcmp(e, "cooperative") == 0) return static_cast<int>(kCooperative);
    if (strcmp(e, "staggered") == 0) return static_cast<int>(kStaggered);
    return kBadSchedule;
  }();
  return forced;
}

#ifdef AB_GEMM_TRACE
// Traced builds only: every later launch writes its phase record (kTrWords 64-bit words per CTA, at most one CTA per
// SM) into buf.  Returns kTrWords.
extern "C" int ab_gemm_trace(unsigned long long* buf) {
  ab::g_trace_buf = buf;
  return ab::kTrWords;
}
#endif

}  // namespace ab

extern "C" int ab_gemm_bf16(const AbGemm* p, void* stream) {
  using namespace ab;
  AB_CHECK_ARG(p != nullptr, "ab_gemm_bf16: null descriptor");
  AB_CHECK_ARG(p->m > 0 && p->n > 0 && p->k > 0, "ab_gemm_bf16: bad shape m=%d n=%d k=%d", p->m, p->n, p->k);
  AB_CHECK_ARG(p->a != nullptr && p->w != nullptr, "ab_gemm_bf16: null operand");
  AB_CHECK_ARG(p->out_f32 != nullptr || p->out_bf16 != nullptr, "ab_gemm_bf16: no output requested");
  AB_CHECK_ARG(p->k % 8 == 0 && p->lda % 8 == 0 && p->ldw % 8 == 0 && p->lda >= p->k && p->ldw >= p->k,
               "ab_gemm_bf16: K/lda/ldw must be multiples of 8 and ld >= K (k=%d lda=%d ldw=%d)", p->k, p->lda,
               p->ldw);
  AB_CHECK_ARG(p->act == AB_ACT_NONE || p->act == AB_ACT_GELU_ERF, "ab_gemm_bf16: unknown activation %d", p->act);
  AB_CHECK_ARG((p->in_dtype == AB_DT_BF16 || p->in_dtype == AB_DT_F16) &&
                   (p->out_dtype == AB_DT_BF16 || p->out_dtype == AB_DT_F16),
               "ab_gemm_bf16: dtypes must be AB_DT_BF16 or AB_DT_F16");
  AB_CHECK_ARG(p->out_f32 == nullptr || p->ld_f32 >= p->n, "ab_gemm_bf16: ld_f32 < n");
  AB_CHECK_ARG(p->out_bf16 == nullptr || p->ld_bf16 >= p->n, "ab_gemm_bf16: ld_bf16 < n");
  AB_CHECK_ARG(p->residual == nullptr || p->ldr >= p->n, "ab_gemm_bf16: ldr < n");

  GemmArgs a;
  a.bias = p->bias;
  a.residual = p->residual;
  a.out_f32 = p->out_f32;
  a.out_bf16 = reinterpret_cast<uint16_t*>(p->out_bf16);
  a.out_half = p->out_dtype == AB_DT_F16;
  a.m = p->m;
  a.n = p->n;
  a.k = p->k;
  a.ldr = p->ldr;
  a.ld_f32 = p->ld_f32;
  a.ld_bf16 = p->ld_bf16;
  a.act = p->act;
  auto al16 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
  a.vec_ok = al16(p->bias) && al16(p->residual) && al16(p->out_f32) && al16(p->out_bf16) &&
             (p->residual == nullptr || p->ldr % 4 == 0) && (p->out_f32 == nullptr || p->ld_f32 % 4 == 0) &&
             (p->out_bf16 == nullptr || p->ld_bf16 % 8 == 0);

  memset(&a.peer, 0, sizeof(a.peer));
  // TMA-store epilogue: 16-bit output only, no residual, 16-byte aligned rows and bias.
  a.tma_out = p->out_bf16 != nullptr && p->out_f32 == nullptr && p->residual == nullptr && al16(p->out_bf16) &&
              p->ld_bf16 % 8 == 0 && (p->bias == nullptr || (reinterpret_cast<uintptr_t>(p->bias) & 15u) == 0);
  if (p->peer_push != nullptr) {
    const AbHaloPush* h = p->peer_push;
    AB_CHECK_ARG(a.tma_out && p->out_dtype == AB_DT_BF16, "ab_gemm_bf16: peer_push needs a 16-bit-only bf16 output");
    AB_CHECK_ARG(h->c > 0 && 2 * h->c <= 8 && static_cast<long long>(h->c) * h->rows * h->w == p->m &&
                     h->src_tok_bytes == 2ll * p->n && h->tok_off_bytes % 128 == 0 &&
                     h->tok_off_bytes + h->tok_bytes == h->src_tok_bytes && h->rows_to_above <= h->rows &&
                     h->rows_to_below <= h->rows && h->rows_to_above <= h->slot_rows && h->rows_to_below <= h->slot_rows,
                 "ab_gemm_bf16: peer_push does not describe this output (c=%d rows=%d w=%d, m=%d n=%d)", h->c, h->rows,
                 h->w, p->m, p->n);
    PeerRows& pr = a.peer;
    pr.col_from = static_cast<int>(h->tok_off_bytes / 2);
    pr.dst_ld = static_cast<int>(h->tok_bytes / 2);
    pr.flag[0] = h->above_flag;
    pr.flag[1] = h->below_flag;
    pr.ctrl = h->ctrl;
    const long long slot_row_elems = static_cast<long long>(h->w) * pr.dst_ld;
    for (int c = 0; c < h->c; ++c) {
      if (h->rows_to_above > 0) {  // my first rows -> rows [0, n) of the slot of the rank above
        const int i = pr.n_ranges++;
        pr.row_begin[i] = (c * h->rows) * h->w;
        pr.row_end[i] = pr.row_begin[i] + h->rows_to_above * h->w;
        pr.dst[i] = reinterpret_cast<uint16_t*>(h->above_slot) + static_cast<long long>(c) * h->slot_rows * slot_row_elems;
      }
      if (h->rows_to_below > 0) {  // my last rows -> rows [slot_rows - n, slot_rows) of the slot of the rank below
        const int i = pr.n_ranges++;
        pr.row_begin[i] = (c * h->rows + h->rows - h->rows_to_below) * h->w;
        pr.row_end[i] = pr.row_begin[i] + h->rows_to_below * h->w;
        pr.dst[i] = reinterpret_cast<uint16_t*>(h->below_slot) +
                    (static_cast<long long>(c) * h->slot_rows + h->slot_rows - h->rows_to_below) * slot_row_elems;
      }
    }
    AB_CHECK_ARG(pr.n_ranges > 0, "ab_gemm_bf16: peer_push with nothing to send (use ab_halo_push, which still publishes)");
    // boxes of this launch that carry peer rows: distinct 16-row groups touched by any range x 64-column boxes sent
    int groups = 0, last_group = -1;
    for (int pass = 0; pass < 1; ++pass) {
      // ranges are emitted in increasing row order per level, and levels increase: a sweep over sorted begins suffices
      int order[8];
      for (int i = 0; i < pr.n_ranges; ++i) order[i] = i;
      for (int i = 1; i < pr.n_ranges; ++i)
        for (int j = i; j > 0 && pr.row_begin[order[j]] < pr.row_begin[order[j - 1]]; --j) {
          const int t = order[j];
          order[j] = order[j - 1];
          order[j - 1] = t;
        }
      for (int k = 0; k < pr.n_ranges; ++k) {
        const int i = order[k];
        int g0 = pr.row_begin[i] / kBoxRows;
        const int g1 = (pr.row_end[i] - 1) / kBoxRows;
        if (g0 <= last_group) g0 = last_group + 1;
        if (g1 >= g0) groups += g1 - g0 + 1;
        if (g1 > last_group) last_group = g1;
      }
    }
    pr.expected = groups * ((p->n - pr.col_from + 63) / 64);
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  // Every shape takes the cooperative tile (128 x 256 for N > 128).  Since the epilogue no longer waits on global loads
  // or on its stores (3.3 us per 128 x 256 tile, 4.9-5.3 us with GELU), the cooperative main loop, whose wgmmas read
  // fewer shared-memory bytes per FLOP (48 KB of operands per 128 x 256 x 64 step against 32 KB per 128 x 128 x 64),
  // costs less than the ping-pong tile's hidden epilogue saves: with every shape cooperative the 0.25-degree step ran
  // 3 % faster than with ping-pong at K <= 1024, and ping-pong at K <= 1024 for N <= 1024 only was no better (DESIGN
  // §6).  Staggered loses to both: its lag waits cost more than the epilogue time it hides.  Both stay for
  // AB_GEMM_SCHEDULE.
  int sched = kCooperative;
  const int forced = forced_schedule();
  AB_CHECK_ARG(forced != kBadSchedule, "ab_gemm_bf16: AB_GEMM_SCHEDULE must be pingpong, cooperative or staggered");
  if (forced >= 0 && p->n > 128) sched = forced;
  if (p->in_dtype == AB_DT_F16) return launch_for<true>(p, a, s, sched);
  return launch_for<false>(p, a, s, sched);
}
