// Tropical-cyclone tracking boxes (ab_track_boxes): the field work of the reference's tracker
// (aurora/tracker.py:61-104 get_closest_min, :185-196 the land test, :262-282 the msl / wind crop) evaluated where the
// prediction lives.  One CTA per box; the box is gathered into shared memory through its row / column index lists,
// and only a uint8 mask (MINIMA) or one value per box is written.  The caller keeps every scalar decision.
//
// MINIMA reproduces `minimum_filter(gaussian_filter(box, 1), (8, 8)) == gaussian_filter(box, 1)` bit for bit:
//   - gaussian_filter: one correlation per axis (axis 0, then axis 1), weights exp(-x^2 / 2) / sum for |x| <= 4,
//     accumulated in float64 in SciPy's symmetric-pair order c*w0 + sum_{j=4..1} (x[-j] + x[+j])*wj and rounded to
//     float32 after each axis.  __dmul_rn / __dadd_rn keep the compiler from contracting into FMAs.
//   - minimum_filter of size 8: output i takes the minimum of inputs i-4 .. i+3 on each axis (separable).
//   - boundary mode "reflect" (half-sample symmetric, periodic with period 2n, so it repeats for boxes shorter
//     than the reach of the filter).
#include <math.h>

#include "common.h"

namespace ab {
namespace {

constexpr int kThreads = 256;
constexpr int kRadius = 4;  // int(truncate * sigma + 0.5) with SciPy's truncate 4.0, sigma 1
constexpr int kMinLo = 4;   // minimum filter of size 8, origin 0: inputs i - 4 .. i + 3
constexpr int kMinHi = 3;

// scipy.ndimage._filters._gaussian_kernel1d(1, 0, 4)[4:]: exp(-0.5 x^2) normalised by its float64 sum, printed with
// 17 significant digits (they round-trip exactly).
__constant__ double kGauss[kRadius + 1] = {0.39894346935609776, 0.24197144565660073, 0.05399112742070441,
                                           0.0044318616200312655, 0.00013383062461474175};

struct TrackLaunch {
  AbTrackBox box[AB_TRACK_MAX_BOXES];
  const int32_t* index;
  float* values;
  int32_t* counts;
  uint8_t* masks;
};

__device__ __forceinline__ int reflect(int i, int n) {
  const int p = 2 * n;
  i %= p;
  if (i < 0) i += p;
  return i < n ? i : p - 1 - i;
}

__device__ __forceinline__ float block_reduce(float v, bool is_min, float* s_red) {
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_min ? fminf(v, u) : fmaxf(v, u);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < kThreads / 32 ? s_red[lane] : (is_min ? INFINITY : -INFINITY);
    for (int o = 16; o > 0; o >>= 1) {
      const float u = __shfl_xor_sync(0xffffffffu, v, o);
      v = is_min ? fminf(v, u) : fmaxf(v, u);
    }
  }
  return v;
}

__global__ void __launch_bounds__(kThreads) track_boxes_kernel(const __grid_constant__ TrackLaunch a) {
  __shared__ int s_rows[AB_TRACK_MAX_SIDE];
  __shared__ int s_cols[AB_TRACK_MAX_SIDE];
  __shared__ float s_red[kThreads / 32];
  __shared__ int s_bad, s_nan, s_count;
  extern __shared__ float s_buf[];

  const AbTrackBox& b = a.box[blockIdx.x];
  const int nr = b.n_rows, nc = b.n_cols, n = nr * nc;
  if (threadIdx.x == 0) s_bad = s_nan = s_count = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < nr + nc; i += kThreads) {
    const bool row = i < nr;
    const int v = a.index[row ? b.rows_off + i : b.cols_off + (i - nr)];
    if (v < 0 || v >= (row ? b.h : b.w)) s_bad = 1;
    if (row) s_rows[i] = v;
    else s_cols[i - nr] = v;
  }
  __syncthreads();
  if (s_bad) {
    if (threadIdx.x == 0) {
      a.counts[blockIdx.x] = -1;
      a.values[blockIdx.x] = __int_as_float(0x7fc00000);
    }
    return;
  }

  if (b.op != AB_TRACK_MINIMA) {
    const bool is_min = b.op == AB_TRACK_MIN;
    float acc = is_min ? INFINITY : -INFINITY;
    bool nan = false;
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const size_t off = static_cast<size_t>(s_rows[i / nc]) * b.ld + s_cols[i % nc];
      float v = __ldg(b.plane + off);
      if (b.op == AB_TRACK_WINDMAX) {
        const float u = v, w = __ldg(b.plane2 + off);
        v = __fsqrt_rn(__fadd_rn(__fmul_rn(u, u), __fmul_rn(w, w)));
      }
      if (isnan(v)) nan = true;
      else acc = is_min ? fminf(acc, v) : fmaxf(acc, v);
    }
    if (nan) s_nan = 1;
    acc = block_reduce(acc, is_min, s_red);  // contains a __syncthreads after every s_nan store
    if (threadIdx.x == 0) {
      a.values[blockIdx.x] = s_nan ? __int_as_float(0x7fc00000) : acc;
      a.counts[blockIdx.x] = 0;
    }
    return;
  }

  float* x = s_buf;      // the box, then the smoothed box
  float* y = s_buf + n;  // the axis-0 pass of each filter
  for (int i = threadIdx.x; i < n; i += kThreads)
    x[i] = __ldg(b.plane + static_cast<size_t>(s_rows[i / nc]) * b.ld + s_cols[i % nc]);
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += kThreads) {  // gaussian, axis 0
    const int r = i / nc, c = i % nc;
    double acc = __dmul_rn(static_cast<double>(x[i]), kGauss[0]);
#pragma unroll
    for (int j = kRadius; j >= 1; --j) {
      const double pair = __dadd_rn(static_cast<double>(x[reflect(r - j, nr) * nc + c]),
                                    static_cast<double>(x[reflect(r + j, nr) * nc + c]));
      acc = __dadd_rn(acc, __dmul_rn(pair, kGauss[j]));
    }
    y[i] = __double2float_rn(acc);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += kThreads) {  // gaussian, axis 1
    const int r = i / nc, c = i % nc;
    double acc = __dmul_rn(static_cast<double>(y[i]), kGauss[0]);
#pragma unroll
    for (int j = kRadius; j >= 1; --j) {
      const double pair = __dadd_rn(static_cast<double>(y[r * nc + reflect(c - j, nc)]),
                                    static_cast<double>(y[r * nc + reflect(c + j, nc)]));
      acc = __dadd_rn(acc, __dmul_rn(pair, kGauss[j]));
    }
    x[i] = __double2float_rn(acc);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += kThreads) {  // minimum, axis 0
    const int r = i / nc, c = i % nc;
    float m = x[reflect(r - kMinLo, nr) * nc + c];
#pragma unroll
    for (int d = -kMinLo + 1; d <= kMinHi; ++d) m = fminf(m, x[reflect(r + d, nr) * nc + c]);
    y[i] = m;
  }
  __syncthreads();
  int count = 0;
  uint8_t* mask = a.masks + b.mask_off;
  for (int i = threadIdx.x; i < n; i += kThreads) {  // minimum, axis 1; compare; clear the border
    const int r = i / nc, c = i % nc;
    float m = y[r * nc + reflect(c - kMinLo, nc)];
#pragma unroll
    for (int d = -kMinLo + 1; d <= kMinHi; ++d) m = fminf(m, y[r * nc + reflect(c + d, nc)]);
    const bool hit = m == x[i] && r > 0 && r < nr - 1 && c > 0 && c < nc - 1;
    mask[i] = hit;
    count += hit;
  }
  if (count) atomicAdd(&s_count, count);
  __syncthreads();
  if (threadIdx.x == 0) {
    a.counts[blockIdx.x] = s_count;
    a.values[blockIdx.x] = 0.0f;
  }
}

}  // namespace
}  // namespace ab

extern "C" int ab_track_boxes(const AbTrackBox* boxes, int32_t n_boxes, size_t box_bytes, const int32_t* index,
                              float* values, int32_t* counts, uint8_t* masks, void* stream) {
  using namespace ab;
  AB_CHECK_ARG(box_bytes == sizeof(AbTrackBox), "ab_track_boxes: box_bytes %zu != sizeof(AbTrackBox) %zu", box_bytes,
               sizeof(AbTrackBox));
  AB_CHECK_ARG(n_boxes >= 0, "ab_track_boxes: n_boxes %d < 0", n_boxes);
  if (n_boxes == 0) return AB_OK;
  if (n_boxes > AB_TRACK_MAX_BOXES) {
    set_error("ab_track_boxes: %d boxes in one call, at most %d are supported", n_boxes, AB_TRACK_MAX_BOXES);
    return AB_ERR_UNSUPPORTED;
  }
  AB_CHECK_ARG(boxes && index && values && counts, "ab_track_boxes: null argument");
  TrackLaunch launch;
  int max_cells = 0;
  for (int i = 0; i < n_boxes; ++i) {
    const AbTrackBox& b = boxes[i];
    AB_CHECK_ARG(b.op >= AB_TRACK_MINIMA && b.op <= AB_TRACK_WINDMAX, "ab_track_boxes: box %d: unknown operation %d",
                 i, b.op);
    AB_CHECK_ARG(b.plane, "ab_track_boxes: box %d: null plane", i);
    AB_CHECK_ARG(b.op != AB_TRACK_WINDMAX || b.plane2, "ab_track_boxes: box %d: WINDMAX needs plane2", i);
    AB_CHECK_ARG(b.h > 0 && b.w > 0 && b.ld >= b.w, "ab_track_boxes: box %d: bad plane extent %d x %d, ld %d", i, b.h,
                 b.w, b.ld);
    AB_CHECK_ARG(b.n_rows > 0 && b.n_cols > 0 && b.rows_off >= 0 && b.cols_off >= 0,
                 "ab_track_boxes: box %d: bad index lists (%d rows at %d, %d columns at %d)", i, b.n_rows, b.rows_off,
                 b.n_cols, b.cols_off);
    if (b.n_rows > AB_TRACK_MAX_SIDE || b.n_cols > AB_TRACK_MAX_SIDE) {
      set_error("ab_track_boxes: box %d is %d x %d; boxes up to %d x %d fit in shared memory", i, b.n_rows, b.n_cols,
                AB_TRACK_MAX_SIDE, AB_TRACK_MAX_SIDE);
      return AB_ERR_UNSUPPORTED;
    }
    if (b.op == AB_TRACK_MINIMA) {
      AB_CHECK_ARG(masks && b.mask_off >= 0, "ab_track_boxes: box %d: MINIMA needs masks and mask_off >= 0", i);
      max_cells = b.n_rows * b.n_cols > max_cells ? b.n_rows * b.n_cols : max_cells;
    }
    launch.box[i] = b;
  }
  launch.index = index;
  launch.values = values;
  launch.counts = counts;
  launch.masks = masks;
  const size_t smem = 2 * sizeof(float) * static_cast<size_t>(max_cells);
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(track_boxes_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem));
    if (e != cudaSuccess) {
      set_error("ab_track_boxes: cannot reserve %zu bytes of shared memory: %s", smem, cudaGetErrorString(e));
      return AB_ERR_CUDA;
    }
  }
  track_boxes_kernel<<<n_boxes, kThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(launch);
  AB_COUNT_LAUNCH(1);
  AB_CHECK_LAUNCH("ab_track_boxes");
  return AB_OK;
}
