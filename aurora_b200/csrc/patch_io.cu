// Batch <-> token-matrix movers at the two ends of the model.
//
//   ab_patchify   : per-variable fields (physical units) -> normalised, patchified bf16 A operand of the
//                   patch-embedding GEMM.  Fuses Batch.normalise (batch.py:94-116), the positive-variable
//                   clamp and AirPollution log-combiner (aurora.py:302-319, 726-758), torch.stack of the
//                   variables (encoder.py:213-215) and conv3d's im2col (patchembed.py:100-112).
//                   K index = ((v*T + t)*P + p1)*P + p2, matching cat(weights[v][:, :, :T]) flattened.
//   ab_unpatchify : head GEMM output f32 [L, V*P*P] -> per-variable (H, W) planes in physical units.
//                   Fuses torch.stack + unpatchify (decoder.py:214-217,250-263, util.py:18-41), the
//                   AirPollution difference / clamp hooks (aurora.py:760-796), the positive clamp
//                   (aurora.py:367-388) and Batch.unnormalise (batch.py:118-140).
#include "common.h"
#include "ptx.cuh"

namespace ab {

struct PatchifyArgs {
  AbFieldIn f[AB_MAX_FIELDS];
  uint16_t* out;  // bf16 or fp16
  int nfields, t, h, w, p, ldk;
  int hp, wp;
  int out_half;
};

// torch.nan_to_num(v, nan=0): NaN -> 0, +-inf -> +-FLT_MAX
__device__ __forceinline__ float nan_to_num0(float v) {
  if (isnan(v)) return 0.f;
  if (isinf(v)) return v > 0.f ? 3.402823466e+38f : -3.402823466e+38f;
  return v;
}

__device__ __forceinline__ float transform_in(const AbFieldIn& f, float x) {
  float v = (x - f.loc) / f.scale;
  if (f.transform >= AB_IN_NAN_TO_ZERO) {
    // AuroraWave._pre_encoder_hook (aurora.py:874-892), on the normalised value
    const float kDegToRad = 0.017453292519943295f;
    switch (f.transform) {
      case AB_IN_NAN_TO_ZERO: return nan_to_num0(v);
      case AB_IN_DENSITY: return isnan(v) ? 0.f : 1.f;
      case AB_IN_SIN_DEG: return nan_to_num0(sinf(v * kDegToRad));
      default: return nan_to_num0(cosf(v * kDegToRad));
    }
  }
  // the clamps keep NaN as torch.clamp does (fmaxf would turn it into the bound)
  if (f.transform >= 1) v = fmax_keep_nan(v, 0.f);
  if (f.transform == 2) {
    // AuroraAirPollution._pre_encoder_hook: Linear(2,1)([clamp(z,0,2.5), (log(max(z,eps)) - log eps) / -log eps])
    const float eps = 1e-4f;
    const float ln_eps = -9.210340371976182f;
    const float a0 = fmin_keep_nan(fmax_keep_nan(v, 0.f), 2.5f);
    const float a1 = (logf(fmax_keep_nan(v, eps)) - ln_eps) / (-ln_eps);
    v = f.w0 * a0 + f.w1 * a1 + f.wb;
  }
  return v;
}

__global__ void __launch_bounds__(256) patchify_kernel(const __grid_constant__ PatchifyArgs a) {
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long npatch = static_cast<long long>(a.hp) * a.wp;
  const long long total = npatch * a.nfields * a.t;
  if (gid >= total) return;
  const long long l = gid % npatch;
  const int vt = static_cast<int>(gid / npatch);
  const int t = vt % a.t;
  const int v = vt / a.t;
  const int ph = static_cast<int>(l / a.wp), pw = static_cast<int>(l % a.wp);
  const AbFieldIn& f = a.f[v];
  uint16_t* o = a.out + l * a.ldk + static_cast<long long>(vt) * a.p * a.p;
  if (f.ptr == nullptr) {
    const uint16_t c = to16(f.const_value, a.out_half);
    for (int i = 0; i < a.p * a.p; ++i) o[i] = c;
    return;
  }
  const float* base = f.ptr + static_cast<long long>(t) * f.stride_t + (static_cast<long long>(ph) * a.p) * a.w + pw * a.p;
  if (a.p == 4 && (a.w & 3) == 0 && (reinterpret_cast<uintptr_t>(f.ptr) & 15u) == 0 && (f.stride_t & 3) == 0) {
    uint2 pk[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float4 x = __ldg(reinterpret_cast<const float4*>(base + static_cast<long long>(r) * a.w));
      if (a.out_half) {
        pk[r].x = pack_f16x2(transform_in(f, x.x), transform_in(f, x.y));
        pk[r].y = pack_f16x2(transform_in(f, x.z), transform_in(f, x.w));
      } else {
        pk[r].x = pack_bf16x2(transform_in(f, x.x), transform_in(f, x.y));
        pk[r].y = pack_bf16x2(transform_in(f, x.z), transform_in(f, x.w));
      }
    }
    uint4* o4 = reinterpret_cast<uint4*>(o);  // 16 bf16 = 32 bytes; ldk % 8 == 0 and vt*16 keep alignment
    o4[0] = make_uint4(pk[0].x, pk[0].y, pk[1].x, pk[1].y);
    o4[1] = make_uint4(pk[2].x, pk[2].y, pk[3].x, pk[3].y);
  } else {
    for (int r = 0; r < a.p; ++r)
      for (int c = 0; c < a.p; ++c)
        o[r * a.p + c] = to16(transform_in(f, __ldg(base + static_cast<long long>(r) * a.w + c)), a.out_half);
  }
}

struct UnpatchifyArgs {
  AbFieldOut f[AB_MAX_FIELDS];
  const float* y;
  int nfields, h, w, p, ldy;
  int hp, wp;
};

__global__ void __launch_bounds__(256) unpatchify_kernel(const __grid_constant__ UnpatchifyArgs a) {
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long npatch = static_cast<long long>(a.hp) * a.wp;
  const long long total = npatch * a.nfields * a.p;
  if (gid >= total) return;
  const long long l = gid % npatch;
  const int vp = static_cast<int>(gid / npatch);
  const int p1 = vp % a.p;
  const int v = vp / a.p;
  const int ph = static_cast<int>(l / a.wp), pw = static_cast<int>(l % a.wp);
  const AbFieldOut& f = a.f[v];
  const float* yrow = a.y + l * a.ldy;
  const long long pix = (static_cast<long long>(ph) * a.p + p1) * a.w + static_cast<long long>(pw) * a.p;
  for (int p2 = 0; p2 < a.p; ++p2) {
    float val = __ldg(yrow + f.col + p1 * a.p + p2);
    if (f.cos_col >= 0) {
      // rad2deg(atan2(sin, cos)) % 360 with torch's floored remainder (aurora.py:897-904)
      const float c = __ldg(yrow + f.cos_col + p1 * a.p + p2);
      float deg = atan2f(val, c) * 57.29577951308232f;
      float r = fmodf(deg, 360.f);
      if (r != 0.f && r < 0.f) r += 360.f;
      val = r;
    }
    if (f.mod_col >= 0) {
      // pred = model + (1 + mod) * prev   in normalised units (aurora.py:767-775)
      const float mod = __ldg(yrow + f.mod_col + p1 * a.p + p2);
      const float prev = (__ldg(f.prev + pix + p2) - f.loc) / f.scale;
      val = val + (1.f + mod) * prev;
    }
    if (f.clamp_max1) val = fmin_keep_nan(val, 1.f);  // NaN stays NaN, as with torch.clamp
    if (f.clamp_min0) val = fmax_keep_nan(val, 0.f);
    if (f.dens_col >= 0) {
      // density = sigmoid(logit) * wmb_mask; data = value * wmb_mask; data[density < 0.5] = NaN (aurora.py:906-918)
      const float m = __ldg(f.mask + pix + p2) > f.mask_min ? 1.f : 0.f;
      const float logit = __ldg(yrow + f.dens_col + p1 * a.p + p2);
      const float density = m / (1.f + expf(-logit));
      val = density < 0.5f ? __int_as_float(0x7fc00000) : val * m;
    }
    f.ptr[pix + p2] = val * f.scale + f.loc;
  }
}

}  // namespace ab

extern "C" int ab_patchify(const AbFieldIn* fields, int32_t nfields, int32_t t, int32_t h, int32_t w, int32_t p,
                           void* out_bf16, int32_t ldk, int32_t out_dtype, void* stream) {
  using namespace ab;
  AB_CHECK_ARG(fields && out_bf16, "ab_patchify: null argument");
  AB_CHECK_ARG(nfields > 0 && nfields <= AB_MAX_FIELDS, "ab_patchify: 1..%d fields supported (got %d)",
               AB_MAX_FIELDS, nfields);
  AB_CHECK_ARG(t > 0 && p > 0 && h > 0 && w > 0 && h % p == 0 && w % p == 0,
               "ab_patchify: H and W must be multiples of the patch size (h=%d w=%d p=%d)", h, w, p);
  AB_CHECK_ARG(ldk >= nfields * t * p * p && ldk % 8 == 0, "ab_patchify: ldk too small or not a multiple of 8");
  PatchifyArgs a;
  for (int i = 0; i < nfields; ++i) {
    a.f[i] = fields[i];
    AB_CHECK_ARG(fields[i].ptr == nullptr || fields[i].scale != 0.f, "ab_patchify: zero scale for field %d", i);
  }
  AB_CHECK_ARG(out_dtype == AB_DT_BF16 || out_dtype == AB_DT_F16, "ab_patchify: bad out_dtype");
  a.out = reinterpret_cast<uint16_t*>(out_bf16);
  a.out_half = out_dtype == AB_DT_F16;
  a.nfields = nfields;
  a.t = t;
  a.h = h;
  a.w = w;
  a.p = p;
  a.ldk = ldk;
  a.hp = h / p;
  a.wp = w / p;
  const long long total = static_cast<long long>(a.hp) * a.wp * nfields * t;
  patchify_kernel<<<static_cast<unsigned>(ceil_div_ll(total, 256)), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  AB_COUNT_LAUNCH(1);
  AB_CHECK_LAUNCH("ab_patchify");
  return AB_OK;
}

extern "C" int ab_unpatchify(const AbFieldOut* fields, int32_t nfields, const float* y, int32_t ldy, int32_t h,
                             int32_t w, int32_t p, void* stream) {
  using namespace ab;
  AB_CHECK_ARG(fields && y, "ab_unpatchify: null argument");
  AB_CHECK_ARG(nfields > 0 && nfields <= AB_MAX_FIELDS, "ab_unpatchify: 1..%d fields supported (got %d)",
               AB_MAX_FIELDS, nfields);
  AB_CHECK_ARG(p > 0 && h > 0 && w > 0 && h % p == 0 && w % p == 0, "ab_unpatchify: bad geometry");
  UnpatchifyArgs a;
  for (int i = 0; i < nfields; ++i) {
    a.f[i] = fields[i];
    AB_CHECK_ARG(fields[i].ptr != nullptr, "ab_unpatchify: null output plane for field %d", i);
    AB_CHECK_ARG(fields[i].mod_col < 0 || fields[i].prev != nullptr, "ab_unpatchify: modulation needs prev (field %d)", i);
    AB_CHECK_ARG(fields[i].col >= 0 && fields[i].col + p * p <= ldy, "ab_unpatchify: column out of range (field %d)", i);
    AB_CHECK_ARG(fields[i].cos_col < 0 || fields[i].cos_col + p * p <= ldy,
                 "ab_unpatchify: cosine column out of range (field %d)", i);
    AB_CHECK_ARG(fields[i].dens_col < 0 || (fields[i].dens_col + p * p <= ldy && fields[i].mask != nullptr),
                 "ab_unpatchify: density column out of range or null mask (field %d)", i);
  }
  a.y = y;
  a.nfields = nfields;
  a.h = h;
  a.w = w;
  a.p = p;
  a.ldy = ldy;
  a.hp = h / p;
  a.wp = w / p;
  const long long total = static_cast<long long>(a.hp) * a.wp * nfields * p;
  unpatchify_kernel<<<static_cast<unsigned>(ceil_div_ll(total, 256)), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  AB_COUNT_LAUNCH(1);
  AB_CHECK_LAUNCH("ab_unpatchify");
  return AB_OK;
}
