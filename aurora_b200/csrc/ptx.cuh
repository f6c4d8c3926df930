// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma descriptors, clusters.
// The wgmma.mma_async wrappers themselves are in wgmma.cuh.
// Everything here is hand-written PTX; no CUTLASS/CuTe dependency.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ab {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// Blocking wait with a deadlock watchdog: a pipeline bug traps (the launch fails with an error the
// host sees) instead of hanging the GPU until an external timeout.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint64_t t0 = 0;
  for (uint32_t spin = 1;; ++spin) {
    if (mbar_try_wait(bar, parity)) return;
    if ((spin & 0x3FFu) == 0) {
      uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ull) __trap();  // 4 s
    }
  }
}

// ---------------------------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}

// 2D tiled load global -> shared, completion signalled on an mbarrier (complete_tx::bytes).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                                 int32_t c0, int32_t c1, uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "l"(cache_hint)
      : "memory");
}

// 2D tiled store shared -> global (bulk async group).
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tmap, const void* smem_src, int32_t c0,
                                             int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// L2 eviction-priority policies (createpolicy encodings used by TMA cache hints).
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;

// ---------------------------------------------------------------------------------------------
// wgmma operand descriptors, register budget
// ---------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor for an operand tile stored as rows of 128 bytes with the 128-byte swizzle (what a
// TMA box of {64 16-bit elements, rows} with CU_TENSOR_MAP_SWIZZLE_128B produces), 1024-byte aligned.
//   start address  : bits [0,14)   (bytes >> 4)
//   leading offset : bits [16,30)  (unused for one 128-byte swizzle atom per row; canonical value 1)
//   stride offset  : bits [32,46)  (bytes >> 4 between 8-row groups = 1024 B)
//   layout type    : bits [62,64)  = 1 (SWIZZLE_128B)
// K-major operands advance along K by adding the byte offset inside the 128-byte row to the start address; an
// MN-major operand (wgmma's transposed-B form) advances along K by whole 8-row groups.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr_bytes & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Register hand-over between warpgroups: the producer warpgroup gives registers up, the math warpgroups take them.
template <int kRegs>
__device__ __forceinline__ void reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs));
}
template <int kRegs>
__device__ __forceinline__ void reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs));
}

// ---------------------------------------------------------------------------------------------
// Thread-block clusters
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------
// misc math
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// Round to nearest fp16 with finite overflow and +-inf saturated to +-65504 (fp16 overflows where bf16 would not);
// NaN stays NaN.  One F2FP.SATFINITE instruction for the pair.
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t u;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(u) : "f"(hi), "f"(lo));
  return u;
}

// fmaxf / fminf return the other operand when one is NaN; these return NaN, as torch.clamp does.
__device__ __forceinline__ float fmax_keep_nan(float a, float b) {
  float d;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}
__device__ __forceinline__ float fmin_keep_nan(float a, float b) {
  float d;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}

// 16-bit storage types selected at run time: 0 = bf16 (the backbone, as the reference's autocast),
// 1 = fp16 (encoder / decoder, which the reference keeps in fp32: 3 more mantissa bits at the same rate).
template <int kHalf>
__device__ __forceinline__ uint32_t pack16x2(float lo, float hi) {
  if constexpr (kHalf) return pack_f16x2(lo, hi);
  else return pack_bf16x2(lo, hi);
}
template <int kHalf>
__device__ __forceinline__ float2 unpack16x2(uint32_t u) {
  if constexpr (kHalf) return __half22float2(*reinterpret_cast<const __half2*>(&u));
  else return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
}
template <int kHalf>
__device__ __forceinline__ void unpack16x8(const uint4& u, float (&f)[8]) {
  float2 t;
  t = unpack16x2<kHalf>(u.x); f[0] = t.x; f[1] = t.y;
  t = unpack16x2<kHalf>(u.y); f[2] = t.x; f[3] = t.y;
  t = unpack16x2<kHalf>(u.z); f[4] = t.x; f[5] = t.y;
  t = unpack16x2<kHalf>(u.w); f[6] = t.x; f[7] = t.y;
}
template <int kHalf>
__device__ __forceinline__ uint4 pack16x8(const float (&f)[8]) {
  uint4 u;
  u.x = pack16x2<kHalf>(f[0], f[1]);
  u.y = pack16x2<kHalf>(f[2], f[3]);
  u.z = pack16x2<kHalf>(f[4], f[5]);
  u.w = pack16x2<kHalf>(f[6], f[7]);
  return u;
}
__device__ __forceinline__ uint16_t to16(float x, int half) {
  if (half) return static_cast<uint16_t>(pack_f16x2(x, 0.f));
  __nv_bfloat16 b = __float2bfloat16_rn(x);
  return *reinterpret_cast<uint16_t*>(&b);
}

// erf-form GELU as nn.GELU() (NOT the tanh approximation):
//   gelu(x) = max(x, 0) - |x| * h(z),  z = |x| / sqrt(2),  h(z) = 0.5 erfc(z) = exp(-z^2) * R(z)
// with R a degree-6 minimax fit of 0.5 * erfcx on [0, 4.5] (z clamped there; erfc(4.5) = 2e-10).
// Max abs error 1.4e-5 over all x (fit: tools/fit_gelu.py) — far below the 16-bit rounding of the stored
// activation — for 13 ALU ops + 1 MUFU, against ~30 instructions for erff(): the fc1 epilogue runs on the same
// warps that issue the next tile's wgmma, so every instruction saved here is tensor-pipe time.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fminf(fabsf(x) * 0.70710678118654752440f, 4.5f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"((z * -1.4426950408889634f) * z));
  float r = fmaf(0.003532303497195244f, z, -0.032581403851509094f);
  r = fmaf(r, z, 0.12916485965251923f);
  r = fmaf(r, z, -0.29942014813423157f);
  r = fmaf(r, z, 0.47322216629981995f);
  r = fmaf(r, z, -0.5599349141120911f);
  r = fmaf(r, z, 0.49980518221855164f);
  return fmaf(-fabsf(x), e * r, fmaxf(x, 0.f));
}

}  // namespace ab
