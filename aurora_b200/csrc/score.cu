// Latitude-weighted scores (ab_score_fields): the sums behind RMSE, bias, MAE and the uncentred anomaly correlation
// of a prediction against a truth and a climatology, for every level plane of up to AB_SCORE_MAX_FIELDS fields in one
// call.  The work is a streaming read of the three fields, so the kernel is bound by HBM:
//   - score_partial_kernel: one CTA per (plane, row-chunk) work item, about kChunkElems points each.  A thread keeps
//     the seven float64 sums and the count in registers, reading 16 bytes per field at a time where the field's
//     pointers, pitches and level strides allow (a scalar tail covers w % 4), then the CTA reduces them in a fixed
//     tree and writes one partial per work item to the workspace.
//   - score_reduce_kernel: one CTA per plane adds its partials, again in a fixed order.
// The partition depends only on the field shapes, and no sum is formed with atomics, so two calls on the same inputs
// give bit-identical sums.
#include <math.h>

#include "common.h"

namespace ab {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunkElems = 16384;  // points per work item: ~11 rows of a 0.25-degree plane, ~4.5 rows at 0.1 degree

struct ScoreLaunch {
  AbScoreField f[AB_SCORE_MAX_FIELDS];
  int32_t item_off[AB_SCORE_MAX_FIELDS + 1];   // first work item of each field
  int32_t plane_off[AB_SCORE_MAX_FIELDS + 1];  // first plane of each field
  int32_t chunk_rows[AB_SCORE_MAX_FIELDS];     // rows per work item
  int32_t chunks[AB_SCORE_MAX_FIELDS];         // work items per plane
  int32_t vec[AB_SCORE_MAX_FIELDS];            // 16-byte loads allowed
  int32_t n_fields;
  const double* weights;
  double* partial;  // [items][AB_SCORE_SUMS]
  double* sums;     // [planes][AB_SCORE_SUMS]
};

struct Acc {
  double s[AB_SCORE_SUMS - 1];
  int n;
};

template <bool kClim>
__device__ __forceinline__ void accumulate(Acc& a, float p, float t, float c, double w) {
  if (isnan(p) || isnan(t) || (kClim && isnan(c))) return;
  const double d = static_cast<double>(p) - static_cast<double>(t);
  a.s[0] += w;
  a.s[1] += w * d;
  a.s[2] += w * d * d;
  a.s[3] += w * fabs(d);
  if (kClim) {
    const double af = static_cast<double>(p) - static_cast<double>(c);
    const double ao = static_cast<double>(t) - static_cast<double>(c);
    a.s[4] += w * af * ao;
    a.s[5] += w * af * af;
    a.s[6] += w * ao * ao;
  }
  ++a.n;
}

// The points of rows [r0, r0 + nr) of one plane; P / T / C point at row r0.
template <bool kClim, bool kVec>
__device__ __forceinline__ void score_rows(Acc& a, const AbScoreField& f, const float* P, const float* T,
                                           const float* C, const double* wr, int nr) {
  const int w = f.w;
  int done = 0;  // columns covered by the vector loop
  if (kVec) {
    const int nv = w >> 2, n = nr * nv;
#pragma unroll 2
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const int r = i / nv, c = 4 * (i - r * nv);
      const float4 p = __ldg(reinterpret_cast<const float4*>(P + static_cast<size_t>(r) * f.ld_pred + c));
      const float4 t = __ldg(reinterpret_cast<const float4*>(T + static_cast<size_t>(r) * f.ld_truth + c));
      float4 k = make_float4(0.f, 0.f, 0.f, 0.f);
      if (kClim) k = __ldg(reinterpret_cast<const float4*>(C + static_cast<size_t>(r) * f.ld_clim + c));
      const double wt = __ldg(wr + r);
      accumulate<kClim>(a, p.x, t.x, k.x, wt);
      accumulate<kClim>(a, p.y, t.y, k.y, wt);
      accumulate<kClim>(a, p.z, t.z, k.z, wt);
      accumulate<kClim>(a, p.w, t.w, k.w, wt);
    }
    done = 4 * nv;
  }
  const int tail = w - done, n = nr * tail;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const int r = i / tail, c = done + (i - r * tail);
    const float p = __ldg(P + static_cast<size_t>(r) * f.ld_pred + c);
    const float t = __ldg(T + static_cast<size_t>(r) * f.ld_truth + c);
    const float k = kClim ? __ldg(C + static_cast<size_t>(r) * f.ld_clim + c) : 0.f;
    accumulate<kClim>(a, p, t, k, __ldg(wr + r));
  }
}

// Sum v[0..AB_SCORE_SUMS) over the CTA in a fixed order; the result is valid in thread 0.
__device__ __forceinline__ void block_sum(double (&v)[AB_SCORE_SUMS], double (*s_red)[AB_SCORE_SUMS]) {
#pragma unroll
  for (int j = 0; j < AB_SCORE_SUMS; ++j)
    for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0)
#pragma unroll
    for (int j = 0; j < AB_SCORE_SUMS; ++j) s_red[warp][j] = v[j];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < AB_SCORE_SUMS; ++j) {
      double t = s_red[0][j];
      for (int k = 1; k < kWarps; ++k) t += s_red[k][j];
      v[j] = t;
    }
}

__global__ void __launch_bounds__(kThreads) score_partial_kernel(const __grid_constant__ ScoreLaunch a) {
  __shared__ double s_red[kWarps][AB_SCORE_SUMS];
  const int item = blockIdx.x;
  int fi = 0;
  while (item >= a.item_off[fi + 1]) ++fi;
  const AbScoreField& f = a.f[fi];
  const int local = item - a.item_off[fi];
  const int level = local / a.chunks[fi], r0 = (local - level * a.chunks[fi]) * a.chunk_rows[fi];
  const int nr = min(a.chunk_rows[fi], f.h - r0);
  const float* P = f.pred + level * f.pred_level_stride + static_cast<int64_t>(r0) * f.ld_pred;
  const float* T = f.truth + level * f.truth_level_stride + static_cast<int64_t>(r0) * f.ld_truth;
  const float* C = f.clim ? f.clim + level * f.clim_level_stride + static_cast<int64_t>(r0) * f.ld_clim : nullptr;
  const double* wr = a.weights + r0;

  Acc acc;
#pragma unroll
  for (int j = 0; j < AB_SCORE_SUMS - 1; ++j) acc.s[j] = 0.0;
  acc.n = 0;
  if (C) {
    if (a.vec[fi]) score_rows<true, true>(acc, f, P, T, C, wr, nr);
    else score_rows<true, false>(acc, f, P, T, C, wr, nr);
  } else {
    if (a.vec[fi]) score_rows<false, true>(acc, f, P, T, C, wr, nr);
    else score_rows<false, false>(acc, f, P, T, C, wr, nr);
  }
  double v[AB_SCORE_SUMS];
#pragma unroll
  for (int j = 0; j < AB_SCORE_SUMS - 1; ++j) v[j] = acc.s[j];
  v[AB_SCORE_SUMS - 1] = static_cast<double>(acc.n);
  block_sum(v, s_red);
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < AB_SCORE_SUMS; ++j) a.partial[static_cast<size_t>(item) * AB_SCORE_SUMS + j] = v[j];
}

__global__ void __launch_bounds__(kThreads) score_reduce_kernel(const __grid_constant__ ScoreLaunch a) {
  __shared__ double s_red[kWarps][AB_SCORE_SUMS];
  const int plane = blockIdx.x;
  int fi = 0;
  while (plane >= a.plane_off[fi + 1]) ++fi;
  const int n = a.chunks[fi];
  const double* part = a.partial + (static_cast<size_t>(a.item_off[fi]) + static_cast<size_t>(plane - a.plane_off[fi]) * n) * AB_SCORE_SUMS;
  double v[AB_SCORE_SUMS];
#pragma unroll
  for (int j = 0; j < AB_SCORE_SUMS; ++j) v[j] = 0.0;
  for (int i = threadIdx.x; i < n; i += kThreads)
#pragma unroll
    for (int j = 0; j < AB_SCORE_SUMS; ++j) v[j] += part[static_cast<size_t>(i) * AB_SCORE_SUMS + j];
  block_sum(v, s_red);
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < AB_SCORE_SUMS; ++j) a.sums[static_cast<size_t>(plane) * AB_SCORE_SUMS + j] = v[j];
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Validate the descriptors and lay out the partition; *items / *planes receive the totals.
int plan(ScoreLaunch* l, const AbScoreField* fields, int32_t n_fields, size_t field_bytes, const char* who,
         int64_t* items, int64_t* planes) {
  AB_CHECK_ARG(field_bytes == sizeof(AbScoreField), "%s: field_bytes %zu != sizeof(AbScoreField) %zu", who,
               field_bytes, sizeof(AbScoreField));
  AB_CHECK_ARG(n_fields >= 0, "%s: n_fields %d < 0", who, n_fields);
  if (n_fields > AB_SCORE_MAX_FIELDS) {
    set_error("%s: %d fields in one call, at most %d are supported", who, n_fields, AB_SCORE_MAX_FIELDS);
    return AB_ERR_UNSUPPORTED;
  }
  AB_CHECK_ARG(n_fields == 0 || fields, "%s: null argument", who);
  int64_t n_items = 0, n_planes = 0;
  for (int i = 0; i < n_fields; ++i) {
    const AbScoreField& f = fields[i];
    AB_CHECK_ARG(f.pred && f.truth, "%s: field %d: null pred or truth", who, i);
    AB_CHECK_ARG(f.h > 0 && f.w > 0 && f.levels > 0, "%s: field %d: bad extent %d levels of %d x %d", who, i,
                 f.levels, f.h, f.w);
    AB_CHECK_ARG(f.ld_pred >= f.w && f.ld_truth >= f.w && (!f.clim || f.ld_clim >= f.w),
                 "%s: field %d: row pitch smaller than the width %d (pred %d, truth %d, clim %d)", who, i, f.w,
                 f.ld_pred, f.ld_truth, f.ld_clim);
    AB_CHECK_ARG(f.pred_level_stride >= 0 && f.truth_level_stride >= 0 && f.clim_level_stride >= 0,
                 "%s: field %d: negative level stride", who, i);
    const int rows = f.w >= kChunkElems ? 1 : (f.h < kChunkElems / f.w ? f.h : kChunkElems / f.w);
    const int chunks = ceil_div(f.h, rows);
    l->f[i] = f;
    l->chunk_rows[i] = rows;
    l->chunks[i] = chunks;
    l->vec[i] = aligned16(f.pred) && aligned16(f.truth) && (!f.clim || aligned16(f.clim)) && f.ld_pred % 4 == 0 &&
                f.ld_truth % 4 == 0 && (!f.clim || f.ld_clim % 4 == 0) && f.pred_level_stride % 4 == 0 &&
                f.truth_level_stride % 4 == 0 && (!f.clim || f.clim_level_stride % 4 == 0);
    l->item_off[i] = static_cast<int32_t>(n_items);
    l->plane_off[i] = static_cast<int32_t>(n_planes);
    n_items += static_cast<int64_t>(chunks) * f.levels;
    n_planes += f.levels;
    if (n_items > INT32_MAX) {
      set_error("%s: more than %d work items in one call", who, INT32_MAX);
      return AB_ERR_UNSUPPORTED;
    }
  }
  l->item_off[n_fields] = static_cast<int32_t>(n_items);
  l->plane_off[n_fields] = static_cast<int32_t>(n_planes);
  l->n_fields = n_fields;
  *items = n_items;
  *planes = n_planes;
  return AB_OK;
}

}  // namespace
}  // namespace ab

extern "C" int ab_score_workspace_bytes(const AbScoreField* fields, int32_t n_fields, size_t field_bytes,
                                        size_t* bytes) {
  using namespace ab;
  AB_CHECK_ARG(bytes, "ab_score_workspace_bytes: null argument");
  ScoreLaunch l;
  int64_t items = 0, planes = 0;
  const int st = plan(&l, fields, n_fields, field_bytes, "ab_score_workspace_bytes", &items, &planes);
  if (st != AB_OK) return st;
  *bytes = static_cast<size_t>(items) * AB_SCORE_SUMS * sizeof(double);
  return AB_OK;
}

extern "C" int ab_score_fields(const AbScoreField* fields, int32_t n_fields, size_t field_bytes,
                               const double* row_weights, double* sums, void* workspace, size_t workspace_bytes,
                               void* stream) {
  using namespace ab;
  ScoreLaunch l;
  int64_t items = 0, planes = 0;
  const int st = plan(&l, fields, n_fields, field_bytes, "ab_score_fields", &items, &planes);
  if (st != AB_OK) return st;
  if (n_fields == 0) return AB_OK;
  AB_CHECK_ARG(row_weights && sums && workspace, "ab_score_fields: null argument");
  const size_t need = static_cast<size_t>(items) * AB_SCORE_SUMS * sizeof(double);
  AB_CHECK_ARG(workspace_bytes >= need, "ab_score_fields: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  AB_CHECK_ARG((reinterpret_cast<uintptr_t>(row_weights) | reinterpret_cast<uintptr_t>(sums) |
                reinterpret_cast<uintptr_t>(workspace)) % alignof(double) == 0,
               "ab_score_fields: row_weights, sums and workspace must be 8-byte aligned");
  l.weights = row_weights;
  l.partial = static_cast<double*>(workspace);
  l.sums = sums;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  score_partial_kernel<<<static_cast<unsigned>(items), kThreads, 0, s>>>(l);
  AB_CHECK_LAUNCH("ab_score_fields");
  score_reduce_kernel<<<static_cast<unsigned>(planes), kThreads, 0, s>>>(l);
  AB_COUNT_LAUNCH(2);
  AB_CHECK_LAUNCH("ab_score_fields");
  return AB_OK;
}
