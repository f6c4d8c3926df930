// Windowed multi-head self-attention over the FLAT token stream (aurora/model/swin3d.py:136-171 with the
// partition / shift / mask logic of :470-503 and :303-360 folded into addressing).
//
//   qkv  : bf16 [B*L, 3*D]   row = token of the (C,H,W) grid, columns = [q | k | v], head-major, d = 64
//   out  : bf16 [B*L, D]     merged heads, written back at the SOURCE token (reverse + crop + un-roll)
//
// One CTA per (batch, window, head), nine warps; warp w owns query rows [16w, 16w+16).
//   1. cp.async gather of the window's q/k/v rows (128 B each) into XOR-swizzled shared memory; the
//      cyclic shift, the zero padding and the window partition are index arithmetic
//      (window_index.cuh), zero-padded tokens read `pad_qkv` (= the projection bias: x = 0 there);
//   2. S = Q K^T on mma.sync m16n8k16 (bf16 in, fp32 out), 48 keys at a time with an online softmax;
//      scale 1/sqrt(64); the shifted-window mask (0 / -100) is generated in registers from one byte
//      of group id per token; an optional dense additive bias [heads, N, N] can be added too;
//   3. O += P V, normalise, stage through shared memory, 128-byte coalesced scatter to the source rows.
//
// Bound: HBM (reads 3D, writes D bf16 per token: arithmetic intensity ~72 FLOP/B, SURVEY.md §8(d)).
#include <stdlib.h>
#include <string.h>

#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"
#include "window_index.cuh"

namespace ab {

constexpr int kHeadDim = 64;
constexpr int kMaxTok = 144;
constexpr int kAttnWarps = 9;
constexpr int kAttnThreads = kAttnWarps * 32;
constexpr int kKeyBlock = 48;
constexpr int kRowBytes = kHeadDim * 2;  // 128

struct AttnArgs {
  const __nv_bfloat16* qkv;
  const __nv_bfloat16* pad_qkv;
  __nv_bfloat16* out;
  const float* bias;
  WinGeom g;
  int batch, num_heads, dim;
  long long tokens_per_batch;
  int box_rows;  // tc kernel: consecutive window-row tokens moved by one TMA box (0 = cp.async gather)
  // Latitude slab (multi-GPU sharding of one forecast): qkv / out hold only rows [h_begin, h_begin + h_rows) of the
  // global (C, H, W) grid; `halo` rows above and below (cyclic in H) come from halo_kv [2][C][halo][W][2D] (K | V columns only).
  int slab, h_begin, h_rows, halo, kh_begin, kh_count;
  const __nv_bfloat16* halo_kv;
  // Peer-memory halo transport (csrc/halo.cu): control words of this rank's halo buffer.  When set, the loaders wait
  // (ld.acquire.sys) until both neighbours' pushes of the current round have landed before they touch a foreign row —
  // and in any case before the kernel ends, which keeps neighbouring ranks at most one exchange apart.
  const uint32_t* halo_ctrl;
};

__device__ __forceinline__ void cp_async_16(uint32_t smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                              uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Byte offset of 16-byte chunk `chunk` (0..7) of row `row` in a [rows][128 B] XOR-swizzled tile.
__device__ __forceinline__ uint32_t swz(int row, int chunk) {
  return static_cast<uint32_t>(row * kRowBytes + ((chunk ^ (row & 7)) << 4));
}

struct AttnItem {
  int head, win, b;
};

__device__ __forceinline__ AttnItem decode_item(const AttnArgs& a, long long item) {
  AttnItem it;
  it.head = static_cast<int>(item % a.num_heads);
  item /= a.num_heads;
  it.win = static_cast<int>(item % a.g.nwindows);
  it.b = static_cast<int>(item / a.g.nwindows);
  return it;
}

// Persistent CTAs (two per SM), two shared-memory buffers each: while the nine warps run the attention
// math of item i out of buffer i&1, the cp.async gather of item i+1 is already in flight into the other.
__global__ void __launch_bounds__(kAttnThreads, 2) window_attention_kernel(const AttnArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const WinGeom& g = a.g;
  const int ntok = g.ntok;
  const int npad = (ntok + 15) & ~15;
  const int tile_bytes = npad * kRowBytes;
  const int buf_bytes = 3 * tile_bytes + npad * static_cast<int>(sizeof(int)) + npad;
  const int buf_stride = (buf_bytes + 127) & ~127;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int ld = 3 * a.dim;
  const long long n_items = static_cast<long long>(a.batch) * g.nwindows * a.num_heads;

  // ---- stage 1 of the pipeline: index map + asynchronous gather of one item into buffer `buf` ----
  auto prefetch = [&](long long item, int buf) -> bool {
    uint8_t* base = smem + buf * buf_stride;
    int* sSrc = reinterpret_cast<int*>(base + 3 * tile_bytes);
    uint8_t* sGrp = reinterpret_cast<uint8_t*>(sSrc + npad);
    const AttnItem it = decode_item(a, item);
    int grp0 = 0;
    win_source_token(g, it.win, 0, &grp0);
    int differs = 0;
    for (int t = tid; t < npad; t += kAttnThreads) {
      int grp = kPadGroup;
      int src = -2;  // rows in [ntok, npad): not part of the window at all
      if (t < ntok) {
        src = win_source_token(g, it.win, t, &grp);
        differs |= (grp != grp0);
      }
      sSrc[t] = src;
      sGrp[t] = static_cast<uint8_t>(grp);
    }
    // Most windows of a shifted block hold a single group: the mask is then all zeros and is skipped.
    const bool masked = __syncthreads_or(differs) != 0 && g.shifted;
    const long long row_base = static_cast<long long>(it.b) * a.tokens_per_batch;
    const uint32_t sq = smem_u32(base), sk = sq + tile_bytes, sv = sk + tile_bytes;
    for (int idx = tid; idx < npad * 8; idx += kAttnThreads) {  // 8 lanes move one 128-byte row of q, k, v
      const int t = idx >> 3;
      const int chunk = idx & 7;
      const int src = sSrc[t];
      const uint32_t off = swz(t, chunk);
      if (src >= 0) {
        const __nv_bfloat16* p = a.qkv + (row_base + src) * ld + it.head * kHeadDim + chunk * 8;
        cp_async_16(sq + off, p);
        cp_async_16(sk + off, p + a.dim);
        cp_async_16(sv + off, p + 2 * a.dim);
      } else if (src == -1) {
        // zero-padded token: x = 0, so q|k|v equal the projection bias (swin3d.py:476-482)
        const __nv_bfloat16* p = a.pad_qkv + it.head * kHeadDim + chunk * 8;
        cp_async_16(sq + off, p);
        cp_async_16(sk + off, p + a.dim);
        cp_async_16(sv + off, p + 2 * a.dim);
      } else {
        const uint4 z = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(base + off) = z;
        *reinterpret_cast<uint4*>(base + tile_bytes + off) = z;
        *reinterpret_cast<uint4*>(base + 2 * tile_bytes + off) = z;
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    return masked;
  };

  long long item = blockIdx.x;
  if (item >= n_items) return;
  bool masked_cur = prefetch(item, 0);
  int buf = 0;
  for (; item < n_items; item += gridDim.x, buf ^= 1) {
    const long long next = item + gridDim.x;
    bool masked_next = false;
    if (next < n_items) {
      masked_next = prefetch(next, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");  // this item's rows have landed; next stays in flight
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const bool masked = masked_cur;
    uint8_t* sQ = smem + buf * buf_stride;
    uint8_t* sK = sQ + tile_bytes;
    uint8_t* sV = sK + tile_bytes;
    const int* sSrc = reinterpret_cast<const int*>(sV + tile_bytes);
    const uint8_t* sGrp = reinterpret_cast<const uint8_t*>(sSrc + npad);
    const AttnItem it = decode_item(a, item);
    const int head = it.head;
    const long long row_base = static_cast<long long>(it.b) * a.tokens_per_batch;

  const int r0 = warp * 16;
  if (r0 < npad) {
    // ---- 2. attention for query rows [r0, r0+16) -------------------------------------------------
    const uint32_t sq = smem_u32(sQ), sk = smem_u32(sK), sv = smem_u32(sV);
    uint32_t qf[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      ldsm_x4(sq + swz(r0 + (lane & 15), kk * 2 + (lane >> 4)), qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);

    // 1/sqrt(64) = 2^-3 is exact in bf16: fold it into the Q fragments once.
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&qf[kk][r]);
        v = __hmul2(v, __float2bfloat162_rn(0.125f));
        qf[kk][r] = *reinterpret_cast<uint32_t*>(&v);
      }

    const int qrow0 = r0 + (lane >> 2);  // this thread's two query rows: qrow0, qrow0 + 8
    const int qrow1 = qrow0 + 8;
    const int gq0 = sGrp[qrow0], gq1 = sGrp[qrow1];
    constexpr float kLog2e = 1.4426950408889634f;
    const bool ragged = ntok != npad;

    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // running max (logit domain) and sum

    for (int kb = 0; kb < npad; kb += kKeyBlock) {
      float s[6][4];
#pragma unroll
      for (int j = 0; j < 6; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
      for (int jp = 0; jp < 3; ++jp) {
        const int n0 = kb + jp * 16;
        if (n0 < npad) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            uint32_t b0, b1, b2, b3;
            ldsm_x4(sk + swz(n0 + (lane & 7) + ((lane >> 4) << 3), kk * 2 + ((lane >> 3) & 1)), b0, b1, b2, b3);
            mma_bf16_16816(s[2 * jp], qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], b0, b1);
            mma_bf16_16816(s[2 * jp + 1], qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], b2, b3);
          }
        }
      }
      const int kcol = kb + (lane & 3) * 2;  // this thread's first key column inside tile j: kcol + 8 j
      if (a.bias != nullptr) {  // optional dense additive bias (never set by Aurora checkpoints)
#pragma unroll
        for (int j = 0; j < 6; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int key = kcol + j * 8 + (e & 1), qrow = (e < 2) ? qrow0 : qrow1;
            if (key < ntok && qrow < ntok)
              s[j][e] += __ldg(a.bias + (static_cast<size_t>(head) * ntok + qrow) * ntok + key);
          }
      }
      if (masked) {  // shifted-window mask from one byte of group id per token (0 / -100, swin3d.py:357-358)
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          const int key = kcol + j * 8;
          if (key < npad) {
            const uint16_t gk2 = *reinterpret_cast<const uint16_t*>(sGrp + key);  // two adjacent keys
            const int gk_a = gk2 & 0xff, gk_b = gk2 >> 8;
            if (gk_a != gq0) s[j][0] -= 100.f;
            if (gk_b != gq0) s[j][1] -= 100.f;
            if (gk_a != gq1) s[j][2] -= 100.f;
            if (gk_b != gq1) s[j][3] -= 100.f;
          }
        }
      }
      if (ragged || kb + kKeyBlock > npad) {  // key columns past the window (clamped windows / last block)
#pragma unroll
        for (int j = 0; j < 6; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (kcol + j * 8 + (e & 1) >= ntok) s[j][e] = -INFINITY;
      }
      float mx0 = m0, mx1 = m1;
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
        mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float alpha0 = ex2_approx((m0 - mx0) * kLog2e), alpha1 = ex2_approx((m1 - mx1) * kLog2e);
      m0 = mx0;
      m1 = mx1;
      const float nm0 = -mx0 * kLog2e, nm1 = -mx1 * kLog2e;
      float sum0 = 0.f, sum1 = 0.f;
      uint32_t pf[3][4];
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        const float p0 = ex2_approx(fmaf(s[j][0], kLog2e, nm0)), p1 = ex2_approx(fmaf(s[j][1], kLog2e, nm0));
        const float p2 = ex2_approx(fmaf(s[j][2], kLog2e, nm1)), p3 = ex2_approx(fmaf(s[j][3], kLog2e, nm1));
        sum0 += p0 + p1;
        sum1 += p2 + p3;
        pf[j >> 1][(j & 1) * 2 + 0] = pack_bf16x2(p0, p1);
        pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
      }
      l0 = l0 * alpha0 + sum0;
      l1 = l1 * alpha1 + sum1;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j][0] *= alpha0;
        o[j][1] *= alpha0;
        o[j][2] *= alpha1;
        o[j][3] *= alpha1;
      }
      // O += P V
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const int k0 = kb + t * 16;
        if (k0 < npad) {
#pragma unroll
          for (int jp = 0; jp < 4; ++jp) {
            uint32_t b0, b1, b2, b3;
            ldsm_x4_trans(sv + swz(k0 + (lane & 7) + (((lane >> 3) & 1) << 3), jp * 2 + (lane >> 4)), b0, b1, b2, b3);
            mma_bf16_16816(o[2 * jp], pf[t][0], pf[t][1], pf[t][2], pf[t][3], b0, b1);
            mma_bf16_16816(o[2 * jp + 1], pf[t][0], pf[t][1], pf[t][2], pf[t][3], b2, b3);
          }
        }
      }
    }
    // ---- 3. normalise, stage in this warp's own Q rows, coalesced scatter -----------------------
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.f / l0, inv1 = 1.f / l1;
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // columns j*8 + (lane&3)*2 .. +1  -> chunk j, byte offset (lane&3)*4 inside the chunk
      *reinterpret_cast<uint32_t*>(sQ + swz(qrow0, j) + (lane & 3) * 4) = pack_bf16x2(o[j][0] * inv0, o[j][1] * inv0);
      *reinterpret_cast<uint32_t*>(sQ + swz(qrow1, j) + (lane & 3) * 4) = pack_bf16x2(o[j][2] * inv1, o[j][3] * inv1);
    }
    __syncwarp();
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int row = r0 + it * 4 + (lane >> 3);
      const int chunk = lane & 7;
      const int src = sSrc[row];
      if (src >= 0) {
        const uint4 v = *reinterpret_cast<const uint4*>(sQ + swz(row, chunk));
        *reinterpret_cast<uint4*>(a.out + (row_base + src) * a.dim + head * kHeadDim + chunk * 8) = v;
      }
    }
  }
    masked_cur = masked_next;
    __syncthreads();  // every warp is done with this buffer before the prefetch two items ahead refills it
  }
}


// ================================================================================================
// wgmma attention for FULL windows (2 x 6 x 12 = 144 tokens, head_dim 64): the production case.
//
// Persistent CTA per SM, warp-specialised, one (window, head) item per pipeline slot:
//   warpgroup 0    : loaders (warps 0-1; registers handed to the math warpgroups).  Warp w handles items n = w (mod 2):
//                    index map + group ids by closed form (window_index.cuh), then a TMA ROW-BOX GATHER of the window's
//                    q / k / v rows into a FOUR-stage 128B-swizzled ring (bias rows for zero-padded tokens are filled
//                    by the warp itself).
//   warpgroups 1-3 : math.  Warpgroup g owns query rows [64 g, 64 g + 64) (wgmma's M is 64: rows >= 144 of the third
//                    warpgroup are don't-care and never stored; the kernel is HBM-bound, the idle tensor rows are free).
//                    S = Q K^T as four m64n144k16 wgmmas, both operands straight from the swizzled stage, the 64 x 144
//                    logits in registers; 0 / -100 shifted-window mask from one byte of group id per key, max / exp2 /
//                    sum with two quad shuffles per row; P stays IN REGISTERS — the fp32 accumulator fragment of S,
//                    packed to bf16 pairs, is exactly the A fragment of the next wgmma — and O = P V runs as nine
//                    m64n64k16 wgmmas with A from registers and V as the transposed (MN-major) B operand straight from
//                    the gathered [key][d] rows.  O is scaled by 1 / sum, staged in the warp's own (now dead) Q rows and
//                    stored as 128-byte rows at the source tokens (reverse + crop + un-roll).
// The three warpgroups run the same item on different rows without synchronising with each other, so one warpgroup's
// softmax overlaps the others' tensor work; the ring lets the loaders run up to three items ahead.
// ================================================================================================
namespace tc {

constexpr int kTok = 144;
constexpr int kTileBytes = kTok * kRowBytes;       // 18 KB per q / k / v tile
constexpr int kStageBytes = 3 * kTileBytes;        // 54 KB
constexpr int kStages = 4;                         // q/k/v ring: a stage is only released after P V, loads must run ahead
constexpr int kOffMeta = kStages * kStageBytes;    // 216 KB
constexpr int kMetaBytes = 6144;
constexpr int kSmemBytes = kOffMeta + kMetaBytes + 1024;
static_assert(kSmemBytes <= 227 * 1024, "shared memory");
constexpr int kMathWarps = 12;    // three warpgroups x 64 query rows
constexpr int kThreads = 128 + kMathWarps * 32;

// win_source_token() for the fixed (2, 6, 12) window with the window already decoded to (k0, k1, k2):
// compile-time divisors only (the generic routine's runtime divisions made the single loader warp the
// bottleneck of the whole pipeline).
__device__ __forceinline__ int tc_source_token(const WinGeom& g, int k0, int k1, int k2, int tok, int* group) {
  const int i[3] = {tok / 72, (tok / 12) % 6, tok % 12};
  const int k[3] = {k0, k1, k2};
  constexpr int kWs[3] = {2, 6, 12};
  int src[3];
  int grp = 0;
  bool valid = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int q = k[a] * kWs[a] + i[a] - g.lo[a];
    valid = valid && (q >= 0) && (q < g.res[a]);
    int sft = q + g.ss[a];
    if (sft >= g.res[a]) sft -= g.res[a];
    src[a] = sft;
    int b;
    if (g.ss[a] == 0) b = 2;
    else b = (q < g.res[a] - kWs[a]) ? 0 : ((q < g.res[a] - g.ss[a]) ? 1 : 2);
    if (a == 2 && g.warped && b == 1) b = 2;
    grp = grp * 3 + b;
  }
  if (!valid) {
    *group = kPadGroup;
    return -1;
  }
  *group = grp;
  return (src[0] * g.res[1] + src[1]) * g.res[2] + src[2];
}

// Window of pipeline item `item` as (head, k0, k1, k2); with a latitude slab only the `kh_count` window rows that
// touch the slab are enumerated (cyclically from kh_begin).
struct TcItem {
  int head, k0, k1, k2, b;
};
__device__ __forceinline__ TcItem tc_decode(const AttnArgs& a, long long item) {
  TcItem it;
  it.head = static_cast<int>(item % a.num_heads);
  item /= a.num_heads;
  const WinGeom& g = a.g;
  if (a.slab) {
    // Window rows are the SLOWEST index and the band's first / last window row — the only ones that can hold a
    // neighbour's rows — come last: every CTA works through interior windows first, so the neighbours' halo pushes land
    // under that work and the loaders' wait for them (below) is normally over before it starts.
    it.k2 = static_cast<int>(item % g.nwin[2]);
    item /= g.nwin[2];
    it.k0 = static_cast<int>(item % g.nwin[0]);
    const int j = static_cast<int>(item / g.nwin[0]);  // 0 .. kh_count - 1 in processing order
    const int idx = a.kh_count <= 2 ? j : (j < a.kh_count - 2 ? j + 1 : (j == a.kh_count - 2 ? 0 : a.kh_count - 1));
    it.k1 = (a.kh_begin + idx) % g.nwin[1];
    it.b = 0;
  } else {
    const int win = static_cast<int>(item % g.nwindows);
    it.b = static_cast<int>(item / g.nwindows);
    it.k2 = win % g.nwin[2];
    it.k1 = (win / g.nwin[2]) % g.nwin[1];
    it.k0 = win / (g.nwin[2] * g.nwin[1]);
  }
  return it;
}

constexpr int kHaloFlag = 1 << 30;

// Global source token -> (row to LOAD from, row to STORE to).  Whole grid: both are the token itself.  Slab: own
// rows live in the local buffer, halo rows in the halo buffer (load only: their outputs belong to a neighbour).
__device__ __forceinline__ void tc_translate(const AttnArgs& a, int src, int* load_row, int* store_row) {
  if (src < 0 || !a.slab) {
    *load_row = src;
    *store_row = src;
    return;
  }
  const WinGeom& g = a.g;
  const int w = src % g.res[2];
  const int t = src / g.res[2];
  const int h = t % g.res[1];
  const int c = t / g.res[1];
  int dh = h - a.h_begin;
  if (dh < 0) dh += g.res[1];
  if (dh < a.h_rows) {
    *load_row = (c * a.h_rows + dh) * g.res[2] + w;
    *store_row = *load_row;
    return;
  }
  *store_row = -1;
  // A foreign row is taken from the NEARER side of the band (ties: above) — the same rule as sharding.halo_needs, which
  // decides which rows the neighbours send: on a small grid a row can be within reach both ways round the cyclic axis.
  int up = (a.h_begin - h) % g.res[1];                 // 1 = the row just above the band
  if (up < 0) up += g.res[1];
  int down = (h - (a.h_begin + a.h_rows)) % g.res[1];  // 0 = the row just below
  if (down < 0) down += g.res[1];
  if (up <= down + 1) {
    *load_row = kHaloFlag | ((c * a.halo + (a.halo - up)) * g.res[2] + w);  // host guarantees up <= halo
    return;
  }
  *load_row = kHaloFlag | (((g.res[0] + c) * a.halo + down) * g.res[2] + w);  // host guarantees down < halo
}

struct Meta {
  int lsrc[kStages][kTok];
  int src[kStages][kTok];
  alignas(16) uint8_t grp[kStages][kTok + 16];
  int masked[kStages];
  int head[kStages];
  int batch[kStages];
  uint64_t full[kStages], empty[kStages];
};
static_assert(sizeof(Meta) <= kMetaBytes, "meta area");

// Wait until both neighbours' halo pushes of the current round have landed (protocol: csrc/halo.cu).  ctrl[0] / ctrl[1]
// are written by the ranks above / below with st.release.sys, ctrl[2] is this rank's own round (its push precedes this
// kernel on the stream).  The rows then arrive through TMA (async proxy): fence the proxies after the acquire.
__device__ __forceinline__ void halo_wait_flags(const uint32_t* ctrl, int lane) {
  if (lane < 2) {
    const uint32_t want = ctrl[2];
    uint64_t t0 = 0;
    for (uint32_t spin = 1;; ++spin) {
      uint32_t v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(ctrl + lane) : "memory");
      if (static_cast<int32_t>(v - want) >= 0) break;
      if ((spin & 0xFFFu) == 0) {
        const uint64_t now = global_timer_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > 20000000000ull) __trap();  // 20 s: a neighbour died
      }
    }
  }
  asm volatile("fence.proxy.async;" ::: "memory");
  __syncwarp();
}

__global__ void __launch_bounds__(kThreads, 1)
window_attention_tc_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_halo,
                           const AttnArgs a) {
  // warps: 0-1 loaders (2-3 idle), 4-15 math: warp w holds query rows [16 (w - 4), 16 (w - 4) + 16).
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  Meta* meta = reinterpret_cast<Meta*>(smem + kOffMeta);
  const WinGeom& g = a.g;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int ld = 3 * a.dim;
  const long long n_windows = a.slab ? static_cast<long long>(g.nwin[0]) * a.kh_count * g.nwin[2]
                                     : static_cast<long long>(a.batch) * g.nwindows;
  const long long n_items = n_windows * a.num_heads;
  const int cnt = static_cast<int>((n_items - blockIdx.x + gridDim.x - 1) / gridDim.x);  // items of this CTA

  if (warp == 0 && lane == 0 && a.box_rows > 0) prefetch_tmap(&tmap_qkv);
  if (warp == 2 && lane == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&meta->full[i], 1);
      mbar_init(&meta->empty[i], kMathWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (warp < 4) reg_dealloc<40>();
  else reg_alloc<152>();

  if (warp < 2) {
    // ===== loaders: warp w takes items n = w (mod 2); item n lives in ring stage n % kStages =====
    bool halo_ok = a.halo_ctrl == nullptr;
    if (!halo_ok && warp >= cnt) {  // a loader without work still holds the kernel until the neighbours' pushes landed
      halo_wait_flags(a.halo_ctrl, lane);
      halo_ok = true;
    }
    for (int n = warp; n < cnt; n += 2) {
      const int st = n % kStages;
      uint8_t* stage = smem + st * kStageBytes;
      const uint32_t sq = smem_u32(stage), sk = sq + kTileBytes, sv = sk + kTileBytes;
      mbar_wait(&meta->empty[st], ((((n / kStages) & 1)) ^ 1));
      const TcItem it = tc_decode(a, blockIdx.x + static_cast<long long>(n) * gridDim.x);
      int grp0 = 0;
      tc_source_token(g, it.k0, it.k1, it.k2, 0, &grp0);
      int differs = 0;
      for (int t = lane; t < kTok; t += 32) {
        int grp, lrow, srow;
        const int src = tc_source_token(g, it.k0, it.k1, it.k2, t, &grp);
        tc_translate(a, src, &lrow, &srow);
        differs |= (grp != grp0);
        meta->lsrc[st][t] = lrow;
        meta->src[st][t] = srow;
        meta->grp[st][t] = static_cast<uint8_t>(grp);
      }
      const int masked = (__any_sync(0xffffffffu, differs) && g.shifted) ? 1 : 0;
      if (lane == 0) {
        meta->masked[st] = masked;
        meta->head[st] = it.head;   // the epilogue takes (batch, head) from here instead of re-decoding the item
        meta->batch[st] = it.b;
      }
      __syncwarp();
      if (!halo_ok) {
        // does this item read a neighbour's row?  (or is it this loader's last item: then wait regardless)
        int foreign = 0;
        for (int t = lane; t < kTok; t += 32) foreign |= (meta->lsrc[st][t] >= 0 && (meta->lsrc[st][t] & kHaloFlag)) ? 1 : 0;
        if (__any_sync(0xffffffffu, foreign) || n + 2 >= cnt) {
          halo_wait_flags(a.halo_ctrl, lane);
          halo_ok = true;
        }
      }
      const long long row_base = static_cast<long long>(it.b) * a.tokens_per_batch;
      if (a.box_rows > 0) {
        // TMA gather: every run of `box_rows` consecutive in-window tokens along W is either all padding or one
        // contiguous piece of the token stream (the host picked box_rows as the gcd of all run boundaries), so
        // it is ONE 2-D box {64 columns, box_rows rows} of the [tokens, 3D] qkv matrix per q / k / v.  The
        // 128B swizzle is applied by the TMA unit, completion is counted on the stage's mbarrier.
        const int r = a.box_rows;
        const int groups_per_row = g.ws[2] / r;
        const int units = g.ws[0] * g.ws[1] * groups_per_row;  // (ic, ih, group)
        uint32_t bytes = 0;
        for (int u = lane; u < units; u += 32) {
          const int t0 = (u / groups_per_row) * g.ws[2] + (u % groups_per_row) * r;  // first window token of the run
          const int src = meta->lsrc[st][t0];
          const uint32_t off = static_cast<uint32_t>(t0) * kRowBytes;
          if (src >= 0) {
            const int col = it.head * kHeadDim;
            if (src & kHaloFlag) {
              // a neighbour's row: only its K and V are here (its query belongs to the neighbour's own output rows;
              // the Q slot keeps stale bytes, whose score / output rows are never stored)
              const int grow = src & ~kHaloFlag;
              tma_load_2d(stage + kTileBytes + off, &tmap_halo, &meta->full[st], col, grow);
              tma_load_2d(stage + 2 * kTileBytes + off, &tmap_halo, &meta->full[st], col + a.dim, grow);
              bytes += 2u * r * kRowBytes;
            } else {
              const int grow = static_cast<int>(row_base + src);
              tma_load_2d(stage + off, &tmap_qkv, &meta->full[st], col, grow);
              tma_load_2d(stage + kTileBytes + off, &tmap_qkv, &meta->full[st], col + a.dim, grow);
              tma_load_2d(stage + 2 * kTileBytes + off, &tmap_qkv, &meta->full[st], col + 2 * a.dim, grow);
              bytes += 3u * r * kRowBytes;
            }
          }
        }
        if (g.nwindows * kTok != g.res[0] * g.res[1] * g.res[2]) {
          // zero-padded tokens (x = 0): q | k | v are the projection bias; filled by the whole warp, 16 B per lane
          for (int idx = lane; idx < kTok * 8; idx += 32) {
            const int t = idx >> 3, chunk = idx & 7;
            if (meta->lsrc[st][t] < 0) {
              const uint4* pb = reinterpret_cast<const uint4*>(a.pad_qkv + it.head * kHeadDim + chunk * 8);
              const uint32_t o2 = swz(t, chunk);
              *reinterpret_cast<uint4*>(stage + o2) = __ldg(pb);
              *reinterpret_cast<uint4*>(stage + kTileBytes + o2) = __ldg(pb + a.dim / 8);
              *reinterpret_cast<uint4*>(stage + 2 * kTileBytes + o2) = __ldg(pb + 2 * a.dim / 8);
            }
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
        fence_proxy_async_smem();  // bias fills (generic proxy) -> wgmma (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive_expect_tx(&meta->full[st], bytes);
        continue;
      }
      for (int idx = lane; idx < kTok * 8; idx += 32) {
        const int t = idx >> 3, chunk = idx & 7;
        const int src = meta->lsrc[st][t];
        const uint32_t off = swz(t, chunk);
        if (src >= 0 && (src & kHaloFlag)) {  // a neighbour's row: K | V only (row pitch 2D)
          const __nv_bfloat16* pk = a.halo_kv + static_cast<long long>(src & ~kHaloFlag) * (2 * a.dim) + it.head * kHeadDim + chunk * 8;
          cp_async_16(sk + off, pk);
          cp_async_16(sv + off, pk + a.dim);
          continue;
        }
        const __nv_bfloat16* p;
        if (src < 0) p = a.pad_qkv + it.head * kHeadDim + chunk * 8;  // zero-padded token: bias
        else p = a.qkv + (row_base + src) * ld + it.head * kHeadDim + chunk * 8;
        cp_async_16(sq + off, p);
        cp_async_16(sk + off, p + a.dim);
        cp_async_16(sv + off, p + 2 * a.dim);
      }
      cp_async_wait_all();
      fence_proxy_async_smem();  // generic-proxy writes -> visible to wgmma (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(&meta->full[st]);
    }
  } else if (warp >= 4) {
    // ===== math warpgroups =====
    const int wg = (warp >> 2) - 1;
    const int row_w = (warp - 4) * 16;      // first query row of this warp
    const bool active = row_w < kTok;       // warp-uniform; 144 = 9 x 16, so an active warp holds 16 real rows
    const int t = lane & 3;
    const int qrow0 = row_w + (lane >> 2), qrow1 = qrow0 + 8;
    constexpr float kC = 0.125f * 1.4426950408889634f;  // 1/sqrt(64) in the exp2 domain
    for (int n = 0; n < cnt; ++n) {
      const int st = n % kStages;
      uint8_t* const stage = smem + st * kStageBytes;
      mbar_wait(&meta->full[st], (n / kStages) & 1);
      const uint32_t qa = smem_u32(stage) + wg * (64 * kRowBytes);
      const uint32_t ka = smem_u32(stage) + kTileBytes, va = ka + kTileBytes;
      float sv[kTok / 2];  // [4 j + 2 h + e]: row qrow_h, key 8 j + 2 t + e
      wgmma_fence_regs(sv);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss<kTok, false>(sv, wgmma_desc_sw128(qa + k * 32), wgmma_desc_sw128(ka + k * 32), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sv);
      uint32_t pa[kTok / 16][4];
      float inv0 = 0.f, inv1 = 0.f;
      if (active) {
        if (meta->masked[st]) {
          // 0 / -100 on the scaled logits == 0 / -800 on the raw q.k products (scale 1/8)
          const uint8_t* grp = meta->grp[st];
          const int gq0 = grp[qrow0], gq1 = grp[qrow1];
#pragma unroll
          for (int j = 0; j < kTok / 8; ++j) {
            const uint16_t gk2 = *reinterpret_cast<const uint16_t*>(grp + 8 * j + 2 * t);  // two adjacent keys
            const int gk_a = gk2 & 0xff, gk_b = gk2 >> 8;
            if (gk_a != gq0) sv[4 * j + 0] -= 800.f;
            if (gk_b != gq0) sv[4 * j + 1] -= 800.f;
            if (gk_a != gq1) sv[4 * j + 2] -= 800.f;
            if (gk_b != gq1) sv[4 * j + 3] -= 800.f;
          }
        }
        float mx0 = fmaxf(sv[0], sv[1]), mx1 = fmaxf(sv[2], sv[3]);
#pragma unroll
        for (int j = 1; j < kTok / 8; ++j) {
          mx0 = fmaxf(mx0, fmaxf(sv[4 * j + 0], sv[4 * j + 1]));
          mx1 = fmaxf(mx1, fmaxf(sv[4 * j + 2], sv[4 * j + 3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float nm0 = -mx0 * kC, nm1 = -mx1 * kC;
        float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
        for (int j = 0; j < kTok / 8; ++j) {
          const float p0 = ex2_approx(fmaf(sv[4 * j + 0], kC, nm0)), p1 = ex2_approx(fmaf(sv[4 * j + 1], kC, nm0));
          const float p2 = ex2_approx(fmaf(sv[4 * j + 2], kC, nm1)), p3 = ex2_approx(fmaf(sv[4 * j + 3], kC, nm1));
          sum0 += p0 + p1;
          sum1 += p2 + p3;
          // the accumulator fragment of key tiles 2 kk, 2 kk + 1 is the A fragment of k-step kk
          pa[j >> 1][(j & 1) * 2 + 0] = pack_bf16x2(p0, p1);
          pa[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
        }
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1);
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
        inv0 = 1.f / sum0;
        inv1 = 1.f / sum1;
      } else {
#pragma unroll
        for (int kk = 0; kk < kTok / 16; ++kk) pa[kk][0] = pa[kk][1] = pa[kk][2] = pa[kk][3] = 0u;
      }
      // O = P V: wgmma is warpgroup-wide, the warps without real rows multiply zeros
      float o[kHeadDim / 2];
      wgmma_fence_regs(o);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kTok / 16; ++kk)
        wgmma_rs_bt_n64(o, pa[kk], wgmma_desc_sw128(va + kk * 16 * kRowBytes), kk != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      if (active) {
        // normalise, stage in this warp's own Q rows (read for the last time by S above), 128-byte coalesced scatter
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          *reinterpret_cast<uint32_t*>(stage + swz(qrow0, j) + t * 4) = pack_bf16x2(o[4 * j] * inv0, o[4 * j + 1] * inv0);
          *reinterpret_cast<uint32_t*>(stage + swz(qrow1, j) + t * 4) = pack_bf16x2(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1);
        }
        __syncwarp();
        const long long row_base = static_cast<long long>(meta->batch[st]) * a.tokens_per_batch;
        const int head = meta->head[st];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = row_w + i * 4 + (lane >> 3);
          const int chunk = lane & 7;
          const int src = meta->src[st][row];
          if (src >= 0) {
            const uint4 v = *reinterpret_cast<const uint4*>(stage + swz(row, chunk));
            *reinterpret_cast<uint4*>(a.out + (row_base + src) * a.dim + head * kHeadDim + chunk * 8) = v;
          }
        }
        fence_proxy_async_smem();  // the staged rows (generic proxy) are overwritten by the next TMA gather
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&meta->empty[st]);  // q / k / v and the index map of this stage are consumed
    }
  }
}

}  // namespace tc

__global__ void window_index_dump_kernel(const WinGeom g, int* idx, uint8_t* grp) {
  const int total = g.nwindows * g.ntok;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int gr;
    idx[i] = win_source_token(g, i / g.ntok, i % g.ntok, &gr);
    grp[i] = static_cast<uint8_t>(gr);
  }
}

static size_t attn_smem_bytes(int ntok) {
  const int npad = (ntok + 15) & ~15;
  const size_t buf = static_cast<size_t>(npad) * kRowBytes * 3 + npad * sizeof(int) + npad;
  return 2 * ((buf + 127) & ~static_cast<size_t>(127));  // two pipeline buffers
}

}  // namespace ab

extern "C" int ab_window_geometry(const int32_t res[3], const int32_t window[3], const int32_t shift[3],
                                  int32_t* n_windows, int32_t* n_tokens, int32_t* shifted) {
  using namespace ab;
  AB_CHECK_ARG(res && window && shift, "ab_window_geometry: null argument");
  for (int a = 0; a < 3; ++a)
    AB_CHECK_ARG(res[a] > 0 && window[a] > 0 && shift[a] >= 0 && shift[a] < window[a],
                 "ab_window_geometry: bad res/window/shift on axis %d", a);
  WinGeom g = make_win_geom(res, window, shift, 1);
  if (n_windows) *n_windows = g.nwindows;
  if (n_tokens) *n_tokens = g.ntok;
  if (shifted) *shifted = g.shifted;
  return AB_OK;
}

extern "C" int ab_window_index_map_host(const int32_t res[3], const int32_t window[3], const int32_t shift[3],
                                        int32_t warped, int32_t* idx_out, uint8_t* group_out) {
  using namespace ab;
  AB_CHECK_ARG(res && window && shift && idx_out && group_out, "ab_window_index_map_host: null argument");
  for (int a = 0; a < 3; ++a)
    AB_CHECK_ARG(res[a] > 0 && window[a] > 0 && shift[a] >= 0 && shift[a] < window[a],
                 "ab_window_index_map_host: bad res/window/shift on axis %d", a);
  const WinGeom g = make_win_geom(res, window, shift, warped);
  for (int i = 0; i < g.nwindows * g.ntok; ++i) {
    int gr;
    idx_out[i] = win_source_token(g, i / g.ntok, i % g.ntok, &gr);
    group_out[i] = static_cast<uint8_t>(gr);
  }
  return AB_OK;
}

extern "C" int ab_window_index_map(const int32_t res[3], const int32_t window[3], const int32_t shift[3],
                                   int32_t warped, int32_t* idx_out, uint8_t* group_out, void* stream) {
  using namespace ab;
  AB_CHECK_ARG(res && window && shift && idx_out && group_out, "ab_window_index_map: null argument");
  for (int a = 0; a < 3; ++a)
    AB_CHECK_ARG(res[a] > 0 && window[a] > 0 && shift[a] >= 0 && shift[a] < window[a],
                 "ab_window_index_map: bad res/window/shift on axis %d", a);
  WinGeom g = make_win_geom(res, window, shift, warped);
  const int total = g.nwindows * g.ntok;
  window_index_dump_kernel<<<ceil_div(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(g, idx_out,
                                                                                                   group_out);
  AB_COUNT_LAUNCH(1);
  AB_CHECK_LAUNCH("ab_window_index_map");
  return AB_OK;
}

extern "C" int ab_window_attention(const AbWindowAttention* p, void* stream) {
  using namespace ab;
  AB_CHECK_ARG(p != nullptr && p->qkv != nullptr && p->out != nullptr, "ab_window_attention: null argument");
  AB_CHECK_ARG(p->head_dim == kHeadDim, "ab_window_attention: head_dim must be 64 (got %d)", p->head_dim);
  AB_CHECK_ARG(p->num_heads > 0 && p->batch > 0, "ab_window_attention: bad batch/heads");
  for (int a = 0; a < 3; ++a)
    AB_CHECK_ARG(p->res[a] > 0 && p->window[a] > 0 && p->shift[a] >= 0 && p->shift[a] < p->window[a],
                 "ab_window_attention: bad res/window/shift on axis %d", a);
  AttnArgs a;
  a.box_rows = 0;
  a.g = make_win_geom(p->res, p->window, p->shift, p->warped);
  AB_CHECK_ARG(a.g.ntok <= kMaxTok, "ab_window_attention: window of %d tokens exceeds the supported %d", a.g.ntok,
               kMaxTok);
  const bool has_pad = a.g.nwindows * a.g.ntok != p->res[0] * p->res[1] * p->res[2];
  AB_CHECK_ARG(!has_pad || p->pad_qkv != nullptr,
               "ab_window_attention: the window grid is zero-padded; pad_qkv (bf16 projection bias) is required");
  a.slab = p->slab_h_rows > 0 ? 1 : 0;
  a.h_begin = p->slab_h_begin;
  a.h_rows = p->slab_h_rows;
  a.halo = p->slab_halo;
  a.kh_begin = 0;
  a.kh_count = a.g.nwin[1];
  a.halo_kv = reinterpret_cast<const __nv_bfloat16*>(p->halo_kv);
  a.halo_ctrl = p->halo_ctrl;
  if (a.slab) {
    AB_CHECK_ARG(p->batch == 1, "ab_window_attention: a latitude slab needs batch == 1");
    AB_CHECK_ARG(a.g.ntok == tc::kTok && p->bias == nullptr,
                 "ab_window_attention: latitude slabs are supported for full 144-token windows only");
    AB_CHECK_ARG(a.h_begin >= 0 && a.h_begin < p->res[1] && a.h_rows <= p->res[1],
                 "ab_window_attention: bad slab rows [%d, +%d) of %d", a.h_begin, a.h_rows, p->res[1]);
    AB_CHECK_ARG(a.h_rows == p->res[1] || (a.halo >= a.g.ws[1] - 1 && p->halo_kv != nullptr),
                 "ab_window_attention: a slab needs halo_kv with at least %d halo rows", a.g.ws[1] - 1);
    // window rows (cyclic range) that contain at least one owned source row
    const int nk = a.g.nwin[1], hh = p->res[1];
    int first = -1, count = 0;
    bool any_gap = false;
    auto touches = [&](int kh) {
      for (int i = 0; i < a.g.ws[1]; ++i) {
        const int q = kh * a.g.ws[1] + i - a.g.lo[1];
        if (q < 0 || q >= hh) continue;
        int d = (q + a.g.ss[1]) % hh - a.h_begin;
        if (d < 0) d += hh;
        if (d < a.h_rows) return true;
      }
      return false;
    };
    for (int kh = 0; kh < nk; ++kh) {
      if (touches(kh)) ++count;
      else any_gap = true;
    }
    if (!any_gap) {
      first = 0;
    } else {
      for (int kh = 0; kh < nk; ++kh)
        if (touches(kh) && !touches((kh + nk - 1) % nk)) first = kh;
    }
    AB_CHECK_ARG(first >= 0 && count > 0, "ab_window_attention: the slab touches no window row");
    for (int j = 0; j < count; ++j)
      AB_CHECK_ARG(touches((first + j) % nk), "ab_window_attention: window rows of the slab are not contiguous");
    a.kh_begin = first;
    a.kh_count = count;
  }
  a.qkv = reinterpret_cast<const __nv_bfloat16*>(p->qkv);
  a.pad_qkv = reinterpret_cast<const __nv_bfloat16*>(p->pad_qkv);
  a.out = reinterpret_cast<__nv_bfloat16*>(p->out);
  a.bias = p->bias;
  a.batch = p->batch;
  a.num_heads = p->num_heads;
  a.dim = p->num_heads * kHeadDim;
  a.tokens_per_batch = static_cast<long long>(p->res[0]) * p->res[1] * p->res[2];
  // Full 144-token windows (every production resolution) run on the wgmma kernel.
  static const bool tc_disabled = getenv("AB_ATTN_NO_TC") != nullptr;
  if (!tc_disabled && a.g.ntok == tc::kTok && a.bias == nullptr) {
    static bool tc_attr_set = false;
    if (!tc_attr_set) {
      cudaError_t e = cudaFuncSetAttribute(tc::window_attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           tc::kSmemBytes);
      if (e != cudaSuccess) {
        set_error("ab_window_attention: cudaFuncSetAttribute(tc) failed: %s", cudaGetErrorString(e));
        return AB_ERR_CUDA;
      }
      tc_attr_set = true;
    }
    // Largest run length R such that every run of R in-window tokens along W is all-padding or contiguous.
    static const bool tma_disabled = getenv("AB_ATTN_NO_TMA") != nullptr;
    a.box_rows = 0;
    CUtensorMap tq, th;
    memset(&tq, 0, sizeof(tq));
    memset(&th, 0, sizeof(th));
    if (!tma_disabled) {
      auto gcd = [](int x, int y) { while (y) { int t = x % y; x = y; y = t; } return x; };
      int r = a.g.ws[2];
      for (int kw = 0; kw < a.g.nwin[2]; ++kw) {
        int prev_valid = -1, prev_src = 0;
        for (int i = 0; i < a.g.ws[2]; ++i) {
          const int q = kw * a.g.ws[2] + i - a.g.lo[2];
          const int valid = q >= 0 && q < a.g.res[2];
          const int src = valid ? (q + a.g.ss[2]) % a.g.res[2] : -1;
          if (i > 0 && (valid != prev_valid || (valid && src != prev_src + 1))) r = gcd(r, i);
          prev_valid = valid;
          prev_src = src;
        }
      }
      const long long rows = a.slab ? static_cast<long long>(p->res[0]) * a.h_rows * p->res[2]
                                    : static_cast<long long>(p->batch) * a.tokens_per_batch;
      if (make_tmap_16bit_2d(&tq, p->qkv, rows, 3ll * a.dim, 3ll * a.dim, r, kHeadDim, false) == AB_OK) a.box_rows = r;
      if (a.box_rows > 0 && a.slab && a.halo > 0 && a.halo_kv != nullptr) {
        const long long hrows = 2ll * p->res[0] * a.halo * p->res[2];
        if (make_tmap_16bit_2d(&th, p->halo_kv, hrows, 2ll * a.dim, 2ll * a.dim, r, kHeadDim, false) != AB_OK)
          a.box_rows = 0;
      }
    }
    const long long tc_windows = a.slab ? static_cast<long long>(a.g.nwin[0]) * a.kh_count * a.g.nwin[2]
                                        : static_cast<long long>(p->batch) * a.g.nwindows;
    const long long tc_items = tc_windows * p->num_heads;
    const unsigned tc_grid = static_cast<unsigned>(tc_items < sm_count() ? tc_items : sm_count());
    // pad_qkv may be NULL when the grid has no padding: the loader then never dereferences it
    tc::window_attention_tc_kernel<<<tc_grid, tc::kThreads, tc::kSmemBytes, reinterpret_cast<cudaStream_t>(stream)>>>(tq, th, a);
    AB_COUNT_LAUNCH(1);
    AB_CHECK_LAUNCH("ab_window_attention(tc)");
    return AB_OK;
  }
  if (a.slab) {
    set_error("ab_window_attention: latitude slabs need the wgmma kernel (AB_ATTN_NO_TC is set?)");
    return AB_ERR_UNSUPPORTED;
  }
  const size_t smem = attn_smem_bytes(a.g.ntok);
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(window_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(attn_smem_bytes(kMaxTok)));
    if (e != cudaSuccess) {
      set_error("ab_window_attention: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return AB_ERR_CUDA;
    }
    attr_set = true;
  }
  const long long items = static_cast<long long>(p->batch) * a.g.nwindows * p->num_heads;
  AB_CHECK_ARG(items < (1ll << 31), "ab_window_attention: too many work items");
  const long long max_ctas = 2ll * sm_count();  // persistent: two CTAs per SM
  const unsigned grid = static_cast<unsigned>(items < max_ctas ? items : max_ctas);
  window_attention_kernel<<<grid, kAttnThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  AB_COUNT_LAUNCH(1);
  AB_CHECK_LAUNCH("ab_window_attention");
  return AB_OK;
}
