// Latitude-weighted scores (ab_score_fields): the sums behind RMSE, bias, MAE and the uncentred anomaly correlation
// of a prediction against a truth and a climatology, for every level plane of up to AB_SCORE_MAX_FIELDS fields in one
// call; and their ensemble counterpart (ab_ensemble_score_fields, below).  The work is a streaming read of the three
// fields, so the kernel is bound by HBM:
//   - score_partial_kernel: one CTA per (plane, row-chunk) work item, about kChunkElems points each.  A thread keeps
//     the seven float64 sums and the count in registers, reading 16 bytes per field at a time where the field's
//     pointers, pitches and level strides allow (a scalar tail covers w % 4), then the CTA reduces them in a fixed
//     tree and writes one partial per work item to the workspace.
//   - score_reduce_kernel: one CTA per plane adds its partials, again in a fixed order.
// The partition depends only on the field shapes, and no sum is formed with atomics, so two calls on the same inputs
// give bit-identical sums.
#include <math.h>

#include "score.cuh"

namespace ab {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunkElems = 16384;  // points per work item: ~11 rows of a 0.25-degree plane, ~4.5 rows at 0.1 degree

// The fixed (plane, row-chunk) partition of a call's fields into work items, shared by both kinds of score.
template <int kMaxFields>
struct Partition {
  int32_t item_off[kMaxFields + 1];   // first work item of each field
  int32_t plane_off[kMaxFields + 1];  // first plane of each field
  int32_t chunk_rows[kMaxFields];     // rows per work item
  int32_t chunks[kMaxFields];         // work items per plane
  int32_t n_fields;
};

struct WorkItem {
  int field, level, r0, nr;  // rows [r0, r0 + nr) of plane `level` of field `field`
};

template <int kMaxFields, class Field>
__device__ __forceinline__ WorkItem locate(const Partition<kMaxFields>& p, int item, const Field* fields) {
  WorkItem it;
  int fi = 0;
  while (item >= p.item_off[fi + 1]) ++fi;
  const int local = item - p.item_off[fi];
  it.field = fi;
  it.level = local / p.chunks[fi];
  it.r0 = (local - it.level * p.chunks[fi]) * p.chunk_rows[fi];
  it.nr = min(p.chunk_rows[fi], fields[fi].h - it.r0);
  return it;
}

struct ScoreLaunch {
  AbScoreField f[AB_SCORE_MAX_FIELDS];
  Partition<AB_SCORE_MAX_FIELDS> part;
  int32_t vec[AB_SCORE_MAX_FIELDS];  // 16-byte loads allowed
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

// Sum v[0..N) over the CTA in a fixed order; the result is valid in thread 0.
template <int N>
__device__ __forceinline__ void block_sum(double (&v)[N], double (*s_red)[N]) {
#pragma unroll
  for (int j = 0; j < N; ++j)
    for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0)
#pragma unroll
    for (int j = 0; j < N; ++j) s_red[warp][j] = v[j];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < N; ++j) {
      double t = s_red[0][j];
      for (int k = 1; k < kWarps; ++k) t += s_red[k][j];
      v[j] = t;
    }
}

__global__ void __launch_bounds__(kThreads) score_partial_kernel(const __grid_constant__ ScoreLaunch a) {
  __shared__ double s_red[kWarps][AB_SCORE_SUMS];
  const int item = blockIdx.x;
  const WorkItem it = locate(a.part, item, a.f);
  const int fi = it.field, level = it.level, r0 = it.r0, nr = it.nr;
  const AbScoreField& f = a.f[fi];
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

// Each plane's partials added in a fixed order: one CTA per plane.
template <int N, class Launch>
__global__ void __launch_bounds__(kThreads) reduce_kernel(const __grid_constant__ Launch a) {
  __shared__ double s_red[kWarps][N];
  const int plane = blockIdx.x;
  int fi = 0;
  while (plane >= a.part.plane_off[fi + 1]) ++fi;
  const int n = a.part.chunks[fi];
  const double* part =
      a.partial + (static_cast<size_t>(a.part.item_off[fi]) + static_cast<size_t>(plane - a.part.plane_off[fi]) * n) * N;
  double v[N];
#pragma unroll
  for (int j = 0; j < N; ++j) v[j] = 0.0;
  for (int i = threadIdx.x; i < n; i += kThreads)
#pragma unroll
    for (int j = 0; j < N; ++j) v[j] += part[static_cast<size_t>(i) * N + j];
  block_sum(v, s_red);
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < N; ++j) a.sums[static_cast<size_t>(plane) * N + j] = v[j];
}

// ---- ensemble scores ----------------------------------------------------------------------------------------------
// ens_partial_kernel<C>: one CTA per (plane, row-chunk) work item, the chunk's points taken kThreads at a time.  The
// CTA stages a tile of kThreads consecutive points of every member, the truth and the climatology in shared memory
// with cp.async (16 bytes per copy where the field allows), two tiles in flight so that the next tile's loads overlap
// this tile's arithmetic.  Each thread then takes one point: it drops the point if any of its values is NaN, sorts
// the M member values with a bitonic network over C registers (C = 8 / 16 / 32 / 64, padded with +inf that sorts
// last and is never read back), and forms every per-point quantity from the sorted values in float64.  The sums
// therefore do not depend on the order of the members, bit for bit.
constexpr int kEnsChunkFloats = 262144;  // values read per work item (1 MB): 18 rows of a 0.25-degree plane at M = 8

struct EnsLaunch {
  AbEnsembleField f[AB_ENS_MAX_FIELDS];
  Partition<AB_ENS_MAX_FIELDS> part;
  int32_t vec[AB_ENS_MAX_FIELDS];  // 16-byte loads allowed
  int32_t rows;                    // rows of kThreads floats in one staged tile: the largest M of the call + 2
  const double* weights;
  double* partial;  // [items][AB_ENS_SUMS]
  double* sums;     // [planes][AB_ENS_SUMS]
};

template <int C>
__device__ __forceinline__ void bitonic_sort(float (&v)[C]) {
#pragma unroll
  for (int k = 2; k <= C; k <<= 1)
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1)
#pragma unroll
      for (int i = 0; i < C; ++i) {
        const int l = i ^ j;
        if (l > i) {
          const float lo = fminf(v[i], v[l]), hi = fmaxf(v[i], v[l]);
          v[i] = (i & k) == 0 ? lo : hi;
          v[l] = (i & k) == 0 ? hi : lo;
        }
      }
}

__device__ __forceinline__ void cp_async16(float* dst, const float* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))),
               "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp_async4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))),
               "l"(src)
               : "memory");
}

// Start copying points [t0, t0 + kThreads) of rows [r0, r0 + nr) of one plane into the tile s_x: source s (members
// 0..M-1, then the truth and the climatology) goes to s_x[s][0..kThreads).
template <bool kVec>
__device__ __forceinline__ void stage(float* s_x, const AbEnsembleField& f, int level, int r0, int t0, int n) {
  const int m = f.n_members, ns = m + (f.clim ? 2 : 1);
  const int p = kVec ? t0 + 4 * (threadIdx.x & (kThreads / 4 - 1)) : t0 + threadIdx.x;
  if (p >= n) return;
  const int r = p / f.w, c = p - r * f.w;
  const size_t rm = static_cast<size_t>(r0 + r) * f.ld_member + c;
#pragma unroll 2
  for (int s = kVec ? threadIdx.x / (kThreads / 4) : 0; s < ns; s += kVec ? 4 : 1) {
    const float* src;
    if (s < m) src = f.members[s] + level * f.member_level_stride + rm;
    else if (s == m) src = f.truth + level * f.truth_level_stride + static_cast<size_t>(r0 + r) * f.ld_truth + c;
    else src = f.clim + level * f.clim_level_stride + static_cast<size_t>(r0 + r) * f.ld_clim + c;
    float* dst = s_x + s * kThreads + (p - t0);
    if (kVec) cp_async16(dst, src);
    else cp_async4(dst, src);
  }
}

// One point, staged in column threadIdx.x of s_x, with row weight w.
template <int C, bool kClim>
__device__ __forceinline__ void ensemble_point(double (&a)[AB_ENS_SUMS], const float* s_x, int m, double w) {
  const int t = threadIdx.x;
  const float y = s_x[m * kThreads + t];
  const float c = kClim ? s_x[(m + 1) * kThreads + t] : 0.f;
  bool nan = isnan(y) || (kClim && isnan(c));
  float v[C];
#pragma unroll
  for (int k = 0; k < C; ++k) {
    v[k] = k < m ? s_x[k * kThreads + t] : INFINITY;
    nan |= isnan(v[k]);
  }
  if (nan) return;
  bitonic_sort(v);
  // Sums of e_k = x_(k) - x_(1), exact in float64, so that the sample variance and the spread do not cancel against
  // the magnitude of the values; sk = sum (2k - M - 1) e_k, the k-th of M ascending (1-based).
  const double xr = isfinite(v[0]) ? static_cast<double>(v[0]) : 0.0, yd = y, c0 = -static_cast<double>(m + 1);
  double se = 0.0, s2 = 0.0, sk = 0.0, sa = 0.0;
#pragma unroll
  for (int k = 0; k < C; ++k) {
    if (k >= m) break;
    const double x = v[k], e = x - xr;
    se += e;
    s2 = fma(e, e, s2);
    sk = fma(c0 + 2.0 * (k + 1), e, sk);
    sa += fabs(x - yd);
  }
  const double inv_m = 1.0 / m, mean_e = se * inv_m;
  const double d = (xr - yd) + mean_e;                                        // ensemble mean - truth
  const double var = (s2 - se * mean_e) / (m - 1);                            // unbiased member variance
  a[0] += w;
  a[1] += w * d;
  a[2] += w * d * d;
  a[3] += w * var;
  a[4] += w * (sa * inv_m);                                                   // (1/M) sum_k |x_k - y|
  a[5] += w * (2.0 * sk / (static_cast<double>(m) * (m - 1)));                // sum_{k != l} |x_k - x_l| / (M (M-1))
  if (kClim) {
    const double af = (xr - static_cast<double>(c)) + mean_e, ao = yd - static_cast<double>(c);
    a[6] += w * af * ao;
    a[7] += w * af * af;
    a[8] += w * ao * ao;
  }
  a[9] += 1.0;
}

template <int C>
__global__ void __launch_bounds__(kThreads) ens_partial_kernel(const __grid_constant__ EnsLaunch a) {
  extern __shared__ __align__(16) float s_x[];  // two tiles of [a.rows][kThreads]
  __shared__ double s_red[kWarps][AB_ENS_SUMS];
  const int item = blockIdx.x;
  const WorkItem it = locate(a.part, item, a.f);
  const AbEnsembleField& f = a.f[it.field];
  const int n = it.nr * f.w, tile = a.rows * kThreads;
  const bool vec = a.vec[it.field], clim = f.clim != nullptr;
  double v[AB_ENS_SUMS];
#pragma unroll
  for (int j = 0; j < AB_ENS_SUMS; ++j) v[j] = 0.0;
  int buf = 0;
  if (vec) stage<true>(s_x, f, it.level, it.r0, 0, n);
  else stage<false>(s_x, f, it.level, it.r0, 0, n);
  asm volatile("cp.async.commit_group;" ::: "memory");
  for (int t0 = 0; t0 < n; t0 += kThreads) {
    // the next tile goes to the other buffer, which every thread finished reading before the last __syncthreads
    if (t0 + kThreads < n) {
      if (vec) stage<true>(s_x + (buf ^ 1) * tile, f, it.level, it.r0, t0 + kThreads, n);
      else stage<false>(s_x + (buf ^ 1) * tile, f, it.level, it.r0, t0 + kThreads, n);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 1;" ::: "memory");  // this thread's copies of tile t0 have landed
    __syncthreads();                                       // and every other thread's
    const int p = t0 + threadIdx.x;
    if (p < n) {
      const double w = __ldg(a.weights + it.r0 + p / f.w);
      if (clim) ensemble_point<C, true>(v, s_x + buf * tile, f.n_members, w);
      else ensemble_point<C, false>(v, s_x + buf * tile, f.n_members, w);
    }
    __syncthreads();
    buf ^= 1;
  }
  block_sum(v, s_red);
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < AB_ENS_SUMS; ++j) a.partial[static_cast<size_t>(item) * AB_ENS_SUMS + j] = v[j];
}

// ---- host side --------------------------------------------------------------------------------------------------
// Field i of the partition: whole rows, about `points` points per work item.
template <int kMaxFields>
int add_field(Partition<kMaxFields>* p, int i, int h, int w, int levels, int points, int64_t* items,
              int64_t* planes, const char* who) {
  const int rows = w >= points ? 1 : (h < points / w ? h : points / w);
  const int chunks = ceil_div(h, rows);
  p->chunk_rows[i] = rows;
  p->chunks[i] = chunks;
  p->item_off[i] = static_cast<int32_t>(*items);
  p->plane_off[i] = static_cast<int32_t>(*planes);
  *items += static_cast<int64_t>(chunks) * levels;
  *planes += levels;
  if (*items > INT32_MAX) {
    set_error("%s: more than %d work items in one call", who, INT32_MAX);
    return AB_ERR_UNSUPPORTED;
  }
  return AB_OK;
}

template <int kMaxFields>
void close_partition(Partition<kMaxFields>* p, int n_fields, int64_t items, int64_t planes) {
  p->item_off[n_fields] = static_cast<int32_t>(items);
  p->plane_off[n_fields] = static_cast<int32_t>(planes);
  p->n_fields = n_fields;
}

// The checks both entry points make on their device arguments.
int check_outputs(const double* row_weights, const double* sums, const void* workspace, size_t workspace_bytes,
                  size_t need, const char* who) {
  AB_CHECK_ARG(row_weights && sums && workspace, "%s: null argument", who);
  AB_CHECK_ARG(workspace_bytes >= need, "%s: workspace of %zu bytes, %zu needed", who, workspace_bytes, need);
  AB_CHECK_ARG((reinterpret_cast<uintptr_t>(row_weights) | reinterpret_cast<uintptr_t>(sums) |
                reinterpret_cast<uintptr_t>(workspace)) % alignof(double) == 0,
               "%s: row_weights, sums and workspace must be 8-byte aligned", who);
  return AB_OK;
}

// Validate the descriptors and lay out the partition; *items / *planes receive the totals.
int plan(ScoreLaunch* l, const AbScoreField* fields, int32_t n_fields, size_t field_bytes, const char* who,
         int64_t* items, int64_t* planes) {
  int st = check_array(fields, n_fields, field_bytes, sizeof(AbScoreField), "AbScoreField", AB_SCORE_MAX_FIELDS, who);
  if (st != AB_OK) return st;
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
    l->f[i] = f;
    l->vec[i] = aligned16(f.pred) && aligned16(f.truth) && (!f.clim || aligned16(f.clim)) && f.ld_pred % 4 == 0 &&
                f.ld_truth % 4 == 0 && (!f.clim || f.ld_clim % 4 == 0) && f.pred_level_stride % 4 == 0 &&
                f.truth_level_stride % 4 == 0 && (!f.clim || f.clim_level_stride % 4 == 0);
    st = add_field(&l->part, i, f.h, f.w, f.levels, kChunkElems, &n_items, &n_planes, who);
    if (st != AB_OK) return st;
  }
  close_partition(&l->part, n_fields, n_items, n_planes);
  *items = n_items;
  *planes = n_planes;
  return AB_OK;
}

// The same for ensemble fields; *capacity receives the sort capacity the largest ensemble needs.
int plan(EnsLaunch* l, const AbEnsembleField* fields, int32_t n_fields, size_t field_bytes, const char* who,
         int64_t* items, int64_t* planes, int* capacity) {
  int st = check_array(fields, n_fields, field_bytes, sizeof(AbEnsembleField), "AbEnsembleField", AB_ENS_MAX_FIELDS,
                       who);
  if (st != AB_OK) return st;
  int64_t n_items = 0, n_planes = 0;
  int max_m = 0;
  for (int i = 0; i < n_fields; ++i) {
    const AbEnsembleField& f = fields[i];
    const int m = f.n_members;
    AB_CHECK_ARG(m >= 2, "%s: field %d: %d members, an ensemble needs at least 2", who, i, m);
    if (m > AB_ENS_MAX_MEMBERS) {
      set_error("%s: field %d: %d members, at most %d are supported", who, i, m, AB_ENS_MAX_MEMBERS);
      return AB_ERR_UNSUPPORTED;
    }
    bool members = true, aligned = aligned16(f.truth) && (!f.clim || aligned16(f.clim));
    for (int k = 0; k < m; ++k) {
      members = members && f.members[k];
      aligned = aligned && aligned16(f.members[k]);
    }
    AB_CHECK_ARG(members && f.truth, "%s: field %d: null member or truth", who, i);
    AB_CHECK_ARG(f.h > 0 && f.w > 0 && f.levels > 0, "%s: field %d: bad extent %d levels of %d x %d", who, i,
                 f.levels, f.h, f.w);
    AB_CHECK_ARG(f.ld_member >= f.w && f.ld_truth >= f.w && (!f.clim || f.ld_clim >= f.w),
                 "%s: field %d: row pitch smaller than the width %d (members %d, truth %d, clim %d)", who, i, f.w,
                 f.ld_member, f.ld_truth, f.ld_clim);
    AB_CHECK_ARG(f.member_level_stride >= 0 && f.truth_level_stride >= 0 && f.clim_level_stride >= 0,
                 "%s: field %d: negative level stride", who, i);
    l->f[i] = f;
    // a tile of points runs across rows, so 16-byte groups need the width too to be a multiple of 4
    l->vec[i] = aligned && f.w % 4 == 0 && f.ld_member % 4 == 0 && f.ld_truth % 4 == 0 &&
                (!f.clim || f.ld_clim % 4 == 0) && f.member_level_stride % 4 == 0 && f.truth_level_stride % 4 == 0 &&
                (!f.clim || f.clim_level_stride % 4 == 0);
    st = add_field(&l->part, i, f.h, f.w, f.levels, kEnsChunkFloats / (m + 2), &n_items, &n_planes, who);
    if (st != AB_OK) return st;
    max_m = m > max_m ? m : max_m;
  }
  close_partition(&l->part, n_fields, n_items, n_planes);
  *items = n_items;
  *planes = n_planes;
  *capacity = max_m <= 8 ? 8 : max_m <= 16 ? 16 : max_m <= 32 ? 32 : 64;
  l->rows = max_m + 2;
  return AB_OK;
}

template <int C>
int launch_ensemble(const EnsLaunch& l, int64_t items, cudaStream_t s) {
  const size_t smem = 2 * static_cast<size_t>(l.rows) * kThreads * sizeof(float);
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(ens_partial_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem));
    if (e != cudaSuccess) {
      set_error("ab_ensemble_score_fields: %zu bytes of shared memory: %s", smem, cudaGetErrorString(e));
      return AB_ERR_CUDA;
    }
  }
  ens_partial_kernel<C><<<static_cast<unsigned>(items), kThreads, smem, s>>>(l);
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
  int st = plan(&l, fields, n_fields, field_bytes, "ab_score_fields", &items, &planes);
  if (st != AB_OK) return st;
  if (n_fields == 0) return AB_OK;
  st = check_outputs(row_weights, sums, workspace, workspace_bytes,
                     static_cast<size_t>(items) * AB_SCORE_SUMS * sizeof(double), "ab_score_fields");
  if (st != AB_OK) return st;
  l.weights = row_weights;
  l.partial = static_cast<double*>(workspace);
  l.sums = sums;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  score_partial_kernel<<<static_cast<unsigned>(items), kThreads, 0, s>>>(l);
  AB_CHECK_LAUNCH("ab_score_fields");
  reduce_kernel<AB_SCORE_SUMS><<<static_cast<unsigned>(planes), kThreads, 0, s>>>(l);
  AB_COUNT_LAUNCH(2);
  AB_CHECK_LAUNCH("ab_score_fields");
  return AB_OK;
}

extern "C" int ab_ensemble_score_workspace_bytes(const AbEnsembleField* fields, int32_t n_fields, size_t field_bytes,
                                                 size_t* bytes) {
  using namespace ab;
  AB_CHECK_ARG(bytes, "ab_ensemble_score_workspace_bytes: null argument");
  EnsLaunch l;
  int64_t items = 0, planes = 0;
  int capacity = 0;
  const int st = plan(&l, fields, n_fields, field_bytes, "ab_ensemble_score_workspace_bytes", &items, &planes,
                      &capacity);
  if (st != AB_OK) return st;
  *bytes = static_cast<size_t>(items) * AB_ENS_SUMS * sizeof(double);
  return AB_OK;
}

extern "C" int ab_ensemble_score_fields(const AbEnsembleField* fields, int32_t n_fields, size_t field_bytes,
                                        const double* row_weights, double* sums, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  using namespace ab;
  EnsLaunch l;
  int64_t items = 0, planes = 0;
  int capacity = 0;
  int st = plan(&l, fields, n_fields, field_bytes, "ab_ensemble_score_fields", &items, &planes, &capacity);
  if (st != AB_OK) return st;
  if (n_fields == 0) return AB_OK;
  st = check_outputs(row_weights, sums, workspace, workspace_bytes,
                     static_cast<size_t>(items) * AB_ENS_SUMS * sizeof(double), "ab_ensemble_score_fields");
  if (st != AB_OK) return st;
  l.weights = row_weights;
  l.partial = static_cast<double*>(workspace);
  l.sums = sums;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  switch (capacity) {
    case 8: st = launch_ensemble<8>(l, items, s); break;
    case 16: st = launch_ensemble<16>(l, items, s); break;
    case 32: st = launch_ensemble<32>(l, items, s); break;
    default: st = launch_ensemble<64>(l, items, s); break;
  }
  if (st != AB_OK) return st;
  AB_CHECK_LAUNCH("ab_ensemble_score_fields");
  reduce_kernel<AB_ENS_SUMS><<<static_cast<unsigned>(planes), kThreads, 0, s>>>(l);
  AB_COUNT_LAUNCH(2);
  AB_CHECK_LAUNCH("ab_ensemble_score_fields");
  return AB_OK;
}
