// GEMM with the AdaptiveLayerNorm + residual of a Swin block fused into its epilogue:
//
//   out[m, :] = residual[m, :] + LN( A[m, :] · W^T + bias ) * scale + shift          (fp32 stream + 16-bit copy)
//
// i.e. `x = shortcut + norm1(attn.proj(.), c)` and `x = x + norm2(mlp.fc2(.), c)` of aurora/model/swin3d.py:507-508
// with film.py:48-49 (LN without affine, eps 1e-5; scale = scale_bias + scale(c), shift = shift(c), both precomputed
// per model time step).  Unfused, the projection writes y in 16 bit and a row kernel reads y + the fp32 stream back and
// writes the stream + its 16-bit copy: 14 B of HBM traffic per element; fused it is 10 B and one launch less.
//
// LayerNorm needs whole rows, so a CLUSTER owns whole rows: N = D = 256 * C columns, C = 2 or 4 CTAs per cluster, every
// CTA running the wgmma pipeline of gemm.cu on ITS 256 columns of the cluster's 128 rows (two math warpgroups x 64 rows,
// the 64 x 256 fp32 accumulator in registers).  Epilogue, all on the registers:
//   1. y = acc + bias; sum(y), sum(y^2) over the thread's 2 x 64 values, reduced over the quad of lanes that shares a row;
//   2. every CTA stores its per-row partial sums into the other CTAs' shared memory (st.shared::cluster) and arrives on
//      their mbarrier (release.cluster); after the acquire every CTA holds the statistics of the whole row.  The slots
//      are double-buffered by tile parity: a CTA can run at most one tile ahead of a neighbour that has not read yet;
//   3. residual + (y - mean) * rstd * scale + shift -> fp32 stream (may alias the residual) + 16-bit copy.  A quad of
//      lanes covers 8 consecutive columns: 32-byte sectors of the fp32 stream, 16 bytes of the 16-bit copy.
// The accumulator is read once and never leaves the registers.
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace ab {
namespace gln {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kWgmmaK = 16;
constexpr int kCtaN = 256;           // columns per CTA = one wgmma N
constexpr int kMaxCluster = 4;
constexpr int kMathWarps = 8;
constexpr int kThreads = 128 + kMathWarps * 32;
constexpr int kStageBytesA = kBlockM * kBlockK * 2;  // 16 KB
constexpr int kStageBytesB = kCtaN * kBlockK * 2;    // 32 KB
constexpr int kStageBytes = kStageBytesA + kStageBytesB;
constexpr int kStages = 4;
constexpr int kOffVec = kStages * kStageBytes;         // bias | scale | shift of this CTA's 256 columns (f32)
constexpr int kVecBytes = 3 * kCtaN * 4;
constexpr int kOffStat = kOffVec + kVecBytes;          // rem[2][kMaxCluster][128] float2 (sum, sum of squares)
constexpr int kStatBytes = 2 * kMaxCluster * kBlockM * 8;
constexpr int kOffBar = kOffStat + kStatBytes;
constexpr int kBarrierBytes = 256;
constexpr int kSmemBytes = kOffBar + kBarrierBytes + 1024;
static_assert(kSmemBytes <= 227 * 1024, "shared memory");

struct Args {
  const float* bias;
  const float* scale;
  const float* shift;
  const float* residual;
  float* out_f32;
  uint16_t* out_16;
  int m, n, k;
  int ldr, ld_f32, ld_16;
  int out_half;
  float eps;
};

// Remote (DSMEM) float2 store into CTA `cta` of this cluster at the same shared-memory offset as `p`.
__device__ __forceinline__ void st_remote_f32x2(float2* p, uint32_t cta, float2 v) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "st.shared::cluster.v2.f32 [ra], {%2, %3};\n\t"
      "}\n" ::"r"(smem_u32(p)),
      "r"(cta), "f"(v.x), "f"(v.y)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive_remote_release(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}
__device__ __forceinline__ void mbar_wait_acquire_cluster(uint64_t* bar, uint32_t parity) {
  uint64_t t0 = 0;
  for (uint32_t spin = 1;; ++spin) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (ok) return;
    if ((spin & 0x3FFu) == 0) {
      const uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ull) __trap();
    }
  }
}

template <bool kHalfIn, int C>
__global__ void __cluster_dims__(C, 1, 1) __launch_bounds__(kThreads, 1)
gemm_ln_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w, const Args g) {
  extern __shared__ uint8_t smem_raw[];
  // every CTA of the cluster carves shared memory identically: remote stores address the same offsets
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kStageBytesA;
  float* s_bias = reinterpret_cast<float*>(smem + kOffVec);
  float* s_scale = s_bias + kCtaN;
  float* s_shift = s_scale + kCtaN;
  float2* rem = reinterpret_cast<float2*>(smem + kOffStat);  // [parity][rank][row]: partial (sum, sum of squares)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* empty_bar = full_bar + kStages;
  // [tile parity]: the other CTAs' math warps arrive here once their partials are stored.  Two barriers, like the slots:
  // the next phase of a barrier needs this CTA's own arrivals of the tile in between, so no waiter can be lapped.
  uint64_t* stat_bar = empty_bar + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const int n_base = static_cast<int>(rank) * kCtaN;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_w);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kMathWarps);
    }
    mbar_init(&stat_bar[0], (C - 1) * kMathWarps);
    mbar_init(&stat_bar[1], (C - 1) * kMathWarps);
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < kCtaN; i += kThreads) {
    s_bias[i] = g.bias != nullptr ? __ldg(g.bias + n_base + i) : 0.f;
    s_scale[i] = g.scale != nullptr ? __ldg(g.scale + n_base + i) : 1.f;
    s_shift[i] = g.shift != nullptr ? __ldg(g.shift + n_base + i) : 0.f;
  }
  cluster_sync_all();  // barriers of every CTA are initialised before any remote arrive

  const int num_tiles = (g.m + kBlockM - 1) / kBlockM;
  const int num_kb = (g.k + kBlockK - 1) / kBlockK;
  const int cluster_id = blockIdx.x / C;
  const int num_clusters = gridDim.x / C;

  if (warp < 4) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      // ===== TMA producer: the cluster's 128 A rows, this CTA's 256 W rows =====
      uint32_t it = 0;
      for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const uint32_t s = it % kStages;
          mbar_wait(&empty_bar[s], ((it / kStages) & 1u) ^ 1u);
          mbar_arrive_expect_tx(&full_bar[s], kStageBytes);
          tma_load_2d(smem_a + s * kStageBytesA, &tmap_a, &full_bar[s], kb * kBlockK, tile * kBlockM);
          tma_load_2d(smem_b + s * kStageBytesB, &tmap_w, &full_bar[s], kb * kBlockK, n_base);
        }
      }
    }
  } else {
    // ===== math warpgroups =====
    reg_alloc<232>();
    const int wg = (warp >> 2) - 1;
    const int t = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows inside the tile: r0, r0 + 8
    const float inv_n = 1.f / static_cast<float>(g.n);
    float acc[kCtaN / 2];
    uint32_t it = 0, tc = 0;
    for (int tile = cluster_id; tile < num_tiles; tile += num_clusters, ++tc) {
      int prev_s = -1;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const uint32_t s = it % kStages;
        mbar_wait(&full_bar[s], (it / kStages) & 1u);
        const uint32_t a_addr = smem_u32(smem_a + s * kStageBytesA) + wg * (64 * 128);
        const uint32_t b_addr = smem_u32(smem_b + s * kStageBytesB);
        wgmma_fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k)
          wgmma_ss<kCtaN, kHalfIn>(acc, wgmma_desc_sw128(a_addr + k * kWgmmaK * 2), wgmma_desc_sw128(b_addr + k * kWgmmaK * 2),
                                   (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        if (prev_s >= 0) {
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty_bar[prev_s]);
        }
        prev_s = static_cast<int>(s);
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev_s]);

      // ---- 1. y = acc + bias, row sums over this CTA's 256 columns ----
      float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll
      for (int j = 0; j < kCtaN / 8; ++j) {
        const float2 b = *reinterpret_cast<const float2*>(s_bias + 8 * j + 2 * t);
        acc[4 * j + 0] += b.x, acc[4 * j + 1] += b.y, acc[4 * j + 2] += b.x, acc[4 * j + 3] += b.y;
        s0 += acc[4 * j + 0] + acc[4 * j + 1];
        s1 += acc[4 * j + 2] + acc[4 * j + 3];
        q0 = fmaf(acc[4 * j + 0], acc[4 * j + 0], fmaf(acc[4 * j + 1], acc[4 * j + 1], q0));
        q1 = fmaf(acc[4 * j + 2], acc[4 * j + 2], fmaf(acc[4 * j + 3], acc[4 * j + 3], q1));
      }
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        q0 += __shfl_xor_sync(0xffffffffu, q0, o);
        q1 += __shfl_xor_sync(0xffffffffu, q1, o);
      }
      // ---- 2. exchange with the CTAs that hold the other columns of these rows ----
      float2* const slot = rem + (tc & 1u) * (kMaxCluster * kBlockM);
      if (t == 0) {
#pragma unroll
        for (uint32_t c = 0; c < C; ++c)
          if (c != rank) {
            st_remote_f32x2(slot + rank * kBlockM + r0, c, make_float2(s0, q0));
            st_remote_f32x2(slot + rank * kBlockM + r0 + 8, c, make_float2(s1, q1));
          }
      }
      __syncwarp();
      if (lane == 0) {
#pragma unroll
        for (uint32_t c = 0; c < C; ++c)
          if (c != rank) mbar_arrive_remote_release(&stat_bar[tc & 1u], c);
      }
      mbar_wait_acquire_cluster(&stat_bar[tc & 1u], (tc >> 1) & 1u);
#pragma unroll
      for (uint32_t c = 0; c < C; ++c)
        if (c != rank) {
          const float2 a0 = slot[c * kBlockM + r0], a1 = slot[c * kBlockM + r0 + 8];
          s0 += a0.x, q0 += a0.y, s1 += a1.x, q1 += a1.y;
        }
      const float mean0 = s0 * inv_n, mean1 = s1 * inv_n;
      const float rstd0 = rsqrtf(fmaxf(q0 * inv_n - mean0 * mean0, 0.f) + g.eps);
      const float rstd1 = rsqrtf(fmaxf(q1 * inv_n - mean1 * mean1, 0.f) + g.eps);
      // ---- 3. normalise + modulate + residual -> fp32 stream, 16-bit copy ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = tile * kBlockM + r0 + 8 * h;
        if (row >= g.m) continue;
        const float mean = h ? mean1 : mean0, rstd = h ? rstd1 : rstd0;
#pragma unroll
        for (int j = 0; j < kCtaN / 8; ++j) {
          const int cl = 8 * j + 2 * t;
          const float2 sc = *reinterpret_cast<const float2*>(s_scale + cl);
          const float2 sh = *reinterpret_cast<const float2*>(s_shift + cl);
          float2 o;
          o.x = fmaf((acc[4 * j + 2 * h] - mean) * rstd, sc.x, sh.x);
          o.y = fmaf((acc[4 * j + 2 * h + 1] - mean) * rstd, sc.y, sh.y);
          const size_t col = static_cast<size_t>(n_base + cl);
          if (g.residual != nullptr) {
            const float2 r = *reinterpret_cast<const float2*>(g.residual + static_cast<size_t>(row) * g.ldr + col);
            o.x += r.x, o.y += r.y;
          }
          if (g.out_f32 != nullptr) *reinterpret_cast<float2*>(g.out_f32 + static_cast<size_t>(row) * g.ld_f32 + col) = o;
          if (g.out_16 != nullptr)
            *reinterpret_cast<uint32_t*>(g.out_16 + static_cast<size_t>(row) * g.ld_16 + col) =
                g.out_half ? pack_f16x2(o.x, o.y) : pack_bf16x2(o.x, o.y);
        }
      }
    }
  }
  // no CTA may exit while a neighbour can still store into its shared memory
  __syncwarp();
  cluster_sync_all();
}

template <bool kHalfIn, int C>
static int launch(const AbGemmLn* p, const Args& a, cudaStream_t stream) {
  CUtensorMap ta, tw;
  int rc = make_tmap_16bit_2d(&ta, p->a, p->m, p->k, p->lda, kBlockM, kBlockK, kHalfIn);
  if (rc != AB_OK) return rc;
  rc = make_tmap_16bit_2d(&tw, p->w, p->n, p->k, p->ldw, kCtaN, kBlockK, kHalfIn);
  if (rc != AB_OK) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_ln_kernel<kHalfIn, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) {
      set_error("ab_gemm_ln_residual: cudaFuncSetAttribute(smem=%d) failed: %s", kSmemBytes, cudaGetErrorString(e));
      return AB_ERR_CUDA;
    }
    attr_set = true;
  }
  const long long tiles = ceil_div_ll(p->m, kBlockM);
  const long long max_clusters = sm_count() / C;
  const int clusters = static_cast<int>(tiles < max_clusters ? tiles : max_clusters);
  gemm_ln_kernel<kHalfIn, C><<<C * clusters, kThreads, kSmemBytes, stream>>>(ta, tw, a);
  AB_COUNT_LAUNCH(1);
  AB_CHECK_LAUNCH("ab_gemm_ln_residual");
  return AB_OK;
}

}  // namespace gln
}  // namespace ab

extern "C" int ab_gemm_ln_supported(int32_t n) { return (n == 512 || n == 1024) ? 1 : 0; }

extern "C" int ab_gemm_ln_residual(const AbGemmLn* p, void* stream) {
  using namespace ab;
  AB_CHECK_ARG(p != nullptr && p->a != nullptr && p->w != nullptr, "ab_gemm_ln_residual: null operand");
  AB_CHECK_ARG(p->m > 0 && p->k > 0, "ab_gemm_ln_residual: bad shape m=%d k=%d", p->m, p->k);
  if (!ab_gemm_ln_supported(p->n)) {
    set_error("ab_gemm_ln_residual: N = %d is not supported (a cluster must own whole rows: N = 512 or 1024)", p->n);
    return AB_ERR_UNSUPPORTED;
  }
  AB_CHECK_ARG(p->k % 8 == 0 && p->lda % 8 == 0 && p->ldw % 8 == 0 && p->lda >= p->k && p->ldw >= p->k,
               "ab_gemm_ln_residual: K/lda/ldw must be multiples of 8 and ld >= K (k=%d lda=%d ldw=%d)", p->k, p->lda, p->ldw);
  AB_CHECK_ARG(p->out_f32 != nullptr || p->out_16 != nullptr, "ab_gemm_ln_residual: no output requested");
  AB_CHECK_ARG((p->in_dtype == AB_DT_BF16 || p->in_dtype == AB_DT_F16) && (p->out_dtype == AB_DT_BF16 || p->out_dtype == AB_DT_F16),
               "ab_gemm_ln_residual: dtypes must be AB_DT_BF16 or AB_DT_F16");
  auto al16 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
  AB_CHECK_ARG(al16(p->residual) && al16(p->out_f32) && al16(p->out_16) &&
                   (p->residual == nullptr || (p->ldr % 4 == 0 && p->ldr >= p->n)) &&
                   (p->out_f32 == nullptr || (p->ld_f32 % 4 == 0 && p->ld_f32 >= p->n)) &&
                   (p->out_16 == nullptr || (p->ld_16 % 8 == 0 && p->ld_16 >= p->n)),
               "ab_gemm_ln_residual: residual / outputs must be 16-byte aligned with 16-byte-multiple pitches >= N");
  gln::Args a;
  a.bias = p->bias, a.scale = p->scale, a.shift = p->shift, a.residual = p->residual;
  a.out_f32 = p->out_f32, a.out_16 = reinterpret_cast<uint16_t*>(p->out_16);
  a.m = p->m, a.n = p->n, a.k = p->k, a.ldr = p->ldr, a.ld_f32 = p->ld_f32, a.ld_16 = p->ld_16;
  a.out_half = p->out_dtype == AB_DT_F16;
  a.eps = p->eps;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const bool half_in = p->in_dtype == AB_DT_F16;
  if (p->n == 512) return half_in ? gln::launch<true, 2>(p, a, s) : gln::launch<false, 2>(p, a, s);
  return half_in ? gln::launch<true, 4>(p, a, s) : gln::launch<false, 4>(p, a, s);
}
