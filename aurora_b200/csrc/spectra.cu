// Latitude-band zonal power spectra (ab_zonal_spectra): for every level plane of up to AB_SPEC_MAX_FIELDS fields and
// up to AB_SPEC_MAX_BANDS latitude bands, the weighted sums over the band's rows of each row's one-sided variance
// spectrum, in float64.
//   - spectra_partial_kernel: one CTA per (plane, band, row-chunk) work item of up to kChunkRows rows.  The CTA builds
//     the twiddle table exp(-2 pi i n / N) (sincospi of an exact rational, no floating-point argument reduction) and
//     the mixed-radix digit-reversal permutation once, then takes the chunk's rows two at a time: the pair is staged
//     as float32 in shared memory (cp.async.bulk on an mbarrier where row address and 4 N bytes are 16-byte
//     multiples, 4-byte cp.async otherwise), the next pair's copy in flight while this pair is transformed.  A row
//     with a non-finite value is dropped (replaced by zeros in the transform and given no weight).  The pair is
//     packed as z = a + i b into digit-reversed order and transformed in place by radix-4 / 2 / 3 / 5 decimation-in-
//     time stages, and A_k = (Z_k + conj Z_{N-k}) / 2, B_k = (Z_k - conj Z_{N-k}) / 2i are separated.  Each thread
//     owns a fixed set of wavenumbers and adds w_a |A_k|^2 and w_b |B_k|^2 to them row after row, so the partial
//     sums of a work item have a fixed order; they go to the workspace scaled by c_k / N^2.
//   - spectra_reduce_kernel: one CTA per (plane, band) adds its work items' partials in chunk order.
// The partition depends only on the shapes and the bands, and no sum is formed with atomics, so two calls on the same
// inputs give bit-identical sums.
#include <math.h>

#include "ptx.cuh"
#include "score.cuh"

namespace ab {
namespace {

constexpr int kThreads = 256;
constexpr int kChunkRows = 32;  // rows per work item: the partials are ~1/32 of the bytes read
constexpr int kMaxStages = 12;  // log2(AB_SPEC_MAX_WIDTH)

struct SpecLaunch {
  AbSpectrumField f[AB_SPEC_MAX_FIELDS];
  int32_t plane_off[AB_SPEC_MAX_FIELDS + 1];  // first plane of each field
  int32_t vec[AB_SPEC_MAX_FIELDS];            // cp.async.bulk allowed
  int32_t band_r0[AB_SPEC_MAX_BANDS], band_r1[AB_SPEC_MAX_BANDS];
  int32_t band_item_off[AB_SPEC_MAX_BANDS + 1];  // first work item of each band within a plane; [n_bands]: per plane
  int32_t radix[kMaxStages];                     // stage s of the FFT has radix radix[s]
  int32_t n_stages, n, n_bands, width;           // width = n / 2 + 3 values per (plane, band)
  double inv_n, inv_nn;                          // 1 / n and 1 / n^2, rounded on the host
  const double* weights;
  double* partial;  // [items][width]
  double* out;      // [planes][n_bands][width]
};

// Dynamic shared memory of one CTA: z and the twiddles (double2 [n] each), the accumulators (double [n / 2 + 1]),
// two staging buffers of two float rows, and the permutation (uint16 [n]).
struct SmemLayout {
  size_t tw, acc, stage, perm, bytes;
  int ldw;  // floats per staged row, a multiple of 4 so that every row starts on 16 bytes
};

__host__ __device__ inline SmemLayout smem_layout(int n) {
  SmemLayout s;
  s.ldw = (n + 3) & ~3;
  s.tw = 16 * static_cast<size_t>(n);
  s.acc = s.tw + 16 * static_cast<size_t>(n);
  s.stage = (s.acc + 8 * static_cast<size_t>(n / 2 + 1) + 15) & ~static_cast<size_t>(15);
  s.perm = s.stage + 4 * sizeof(float) * static_cast<size_t>(s.ldw);
  s.bytes = s.perm + 2 * static_cast<size_t>(n);
  return s;
}

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ double2 mul_neg_i(double2 a) { return make_double2(a.y, -a.x); }  // -i a

// Forward DFT of R values in registers, y_q = sum_j v_j e^{-2 pi i j q / R}.
template <int R>
__device__ __forceinline__ void dft(double2 (&v)[R]);

template <>
__device__ __forceinline__ void dft<2>(double2 (&v)[2]) {
  const double2 a = v[0];
  v[0] = cadd(a, v[1]);
  v[1] = csub(a, v[1]);
}

template <>
__device__ __forceinline__ void dft<4>(double2 (&v)[4]) {
  const double2 t0 = cadd(v[0], v[2]), t1 = csub(v[0], v[2]);
  const double2 t2 = cadd(v[1], v[3]), t3 = mul_neg_i(csub(v[1], v[3]));
  v[0] = cadd(t0, t2);
  v[2] = csub(t0, t2);
  v[1] = cadd(t1, t3);
  v[3] = csub(t1, t3);
}

template <>
__device__ __forceinline__ void dft<3>(double2 (&v)[3]) {
  constexpr double kS = 0.86602540378443864676;  // sin(2 pi / 3)
  const double2 s = cadd(v[1], v[2]);
  const double2 t = make_double2(v[0].x - 0.5 * s.x, v[0].y - 0.5 * s.y);
  const double2 d = csub(v[1], v[2]);
  const double2 u = make_double2(kS * d.y, -kS * d.x);  // -i sin(2 pi / 3) (v1 - v2)
  v[0] = cadd(v[0], s);
  v[1] = cadd(t, u);
  v[2] = csub(t, u);
}

template <>
__device__ __forceinline__ void dft<5>(double2 (&v)[5]) {
  constexpr double kC1 = 0.30901699437494742410, kC2 = -0.80901699437494742410;  // cos(2 pi / 5), cos(4 pi / 5)
  constexpr double kS1 = 0.95105651629515357212, kS2 = 0.58778525229247312917;   // sin(2 pi / 5), sin(4 pi / 5)
  const double2 s14 = cadd(v[1], v[4]), d14 = csub(v[1], v[4]);
  const double2 s23 = cadd(v[2], v[3]), d23 = csub(v[2], v[3]);
  const double2 a1 = make_double2(v[0].x + kC1 * s14.x + kC2 * s23.x, v[0].y + kC1 * s14.y + kC2 * s23.y);
  const double2 a2 = make_double2(v[0].x + kC2 * s14.x + kC1 * s23.x, v[0].y + kC2 * s14.y + kC1 * s23.y);
  const double2 b1 = mul_neg_i(make_double2(kS1 * d14.x + kS2 * d23.x, kS1 * d14.y + kS2 * d23.y));
  const double2 b2 = mul_neg_i(make_double2(kS2 * d14.x - kS1 * d23.x, kS2 * d14.y - kS1 * d23.y));
  v[0] = cadd(v[0], cadd(s14, s23));
  v[1] = cadd(a1, b1);
  v[4] = csub(a1, b1);
  v[2] = cadd(a2, b2);
  v[3] = csub(a2, b2);
}

// One stage of the in-place decimation-in-time FFT: z holds n / L sub-transforms of length L = m R, each made of R
// transforms of length m; butterfly t combines element k = t mod m of those R, with twiddles W_L^{jk}.
template <int R>
__device__ __forceinline__ void fft_stage(double2* z, const double2* tw, int n, int m) {
  const int step = n / (m * R);  // W_L^{jk} = W_N^{jk step}
  for (int t = threadIdx.x; t < n / R; t += kThreads) {
    const int k = t % m, base = (t - k) * R + k;
    double2 v[R];
    v[0] = z[base];
#pragma unroll
    for (int j = 1; j < R; ++j) v[j] = cmul(z[base + j * m], tw[j * k * step]);
    dft<R>(v);
#pragma unroll
    for (int q = 0; q < R; ++q) z[base + q * m] = v[q];
  }
}

__device__ __forceinline__ void bulk_copy(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void cp_async4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}

// Start copying rows 2j and 2j + 1 (when below nr) of the chunk at x into the staging buffer dst (two rows of ldw).
__device__ __forceinline__ void stage_pair(float* dst, int ldw, const float* x, int64_t ld, int n, int j, int nr,
                                           bool bulk, uint64_t* bar) {
  const int rows = min(2, nr - 2 * j);
  const float* src = x + 2 * j * ld;
  if (bulk) {
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(bar, static_cast<uint32_t>(rows * n * sizeof(float)));
      for (int r = 0; r < rows; ++r) bulk_copy(dst + r * ldw, src + r * ld, n * sizeof(float), bar);
    }
  } else {
    for (int r = 0; r < rows; ++r)
      for (int i = threadIdx.x; i < n; i += kThreads) cp_async4(dst + r * ldw + i, src + r * ld + i);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
}

__global__ void __launch_bounds__(kThreads, 3) spectra_partial_kernel(const __grid_constant__ SpecLaunch a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  __shared__ uint64_t s_bar[2];
  const int n = a.n, half = n / 2;
  const SmemLayout L = smem_layout(n);
  double2* z = reinterpret_cast<double2*>(s_raw);
  double2* tw = reinterpret_cast<double2*>(s_raw + L.tw);
  double* acc = reinterpret_cast<double*>(s_raw + L.acc);
  float* stage = reinterpret_cast<float*>(s_raw + L.stage);
  uint16_t* perm = reinterpret_cast<uint16_t*>(s_raw + L.perm);

  // the work item: rows [r0, r0 + nr) of band `band` of plane `plane`
  const int item = blockIdx.x, per_plane = a.band_item_off[a.n_bands];
  const int plane = item / per_plane, local = item - plane * per_plane;
  int band = 0;
  while (local >= a.band_item_off[band + 1]) ++band;
  const int r0 = a.band_r0[band] + (local - a.band_item_off[band]) * kChunkRows;
  const int nr = min(kChunkRows, a.band_r1[band] - r0);
  int fi = 0;
  while (plane >= a.plane_off[fi + 1]) ++fi;
  const AbSpectrumField& f = a.f[fi];
  const float* x = f.x + (plane - a.plane_off[fi]) * f.level_stride + static_cast<int64_t>(r0) * f.ld;
  const bool bulk = a.vec[fi];
  const int pairs = (nr + 1) / 2;

  if (bulk && threadIdx.x == 0) {
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  stage_pair(stage, L.ldw, x, f.ld, n, 0, nr, bulk, &s_bar[0]);

  for (int i = threadIdx.x; i < n; i += kThreads) {
    // i < n: the argument 2 i / n is already reduced; one Newton step on the reciprocal's quotient makes it the
    // correctly rounded quotient (in all but rare ties), without the division's out-of-line slow path
    const double num = 2.0 * i, q0 = num * a.inv_n, quot = fma(fma(-q0, static_cast<double>(n), num), a.inv_n, q0);
    double s, c;
    sincospi(-quot, &s, &c);
    tw[i] = make_double2(c, s);
    // digit reversal: x_i goes to sum_t d_t m_t, the digits d_t of i taken last stage first, m_t = radix[0..t) product
    int pos = 0, q = i, m = n;
    for (int t = a.n_stages - 1; t >= 0; --t) {
      const int r = a.radix[t];
      m /= r;
      pos += (q % r) * m;
      q /= r;
    }
    perm[i] = static_cast<uint16_t>(pos);
  }
  for (int k = threadIdx.x; k <= half; k += kThreads) acc[k] = 0.0;

  double wsum = 0.0, rows = 0.0;  // thread 0's
  for (int j = 0; j < pairs; ++j) {
    const int buf = j & 1;
    float* ra = stage + buf * 2 * L.ldw;
    const float* rb = ra + L.ldw;
    // the other buffer was last read before the last __syncthreads of the previous pair
    if (j + 1 < pairs) stage_pair(stage + (buf ^ 1) * 2 * L.ldw, L.ldw, x, f.ld, n, j + 1, nr, bulk, &s_bar[buf ^ 1]);
    else if (!bulk) asm volatile("cp.async.commit_group;" ::: "memory");
    if (bulk) {
      mbar_wait(&s_bar[buf], (j >> 1) & 1);
    } else {
      asm volatile("cp.async.wait_group 1;" ::: "memory");
      __syncthreads();
    }
    const bool has_b = 2 * j + 1 < nr;
    bool fa = true, fb = true;
    for (int i = threadIdx.x; i < n; i += kThreads) {
      fa = fa && isfinite(ra[i]);
      fb = fb && (!has_b || isfinite(rb[i]));
    }
    const bool va = __syncthreads_and(fa), vb = has_b && __syncthreads_and(fb);
    if (!va && !vb) continue;
    for (int i = threadIdx.x; i < n; i += kThreads)
      z[perm[i]] = make_double2(va ? static_cast<double>(ra[i]) : 0.0, vb ? static_cast<double>(rb[i]) : 0.0);
    __syncthreads();
    for (int s = 0, m = 1; s < a.n_stages; m *= a.radix[s], ++s) {
      switch (a.radix[s]) {
        case 4: fft_stage<4>(z, tw, n, m); break;
        case 2: fft_stage<2>(z, tw, n, m); break;
        case 3: fft_stage<3>(z, tw, n, m); break;
        default: fft_stage<5>(z, tw, n, m); break;
      }
      __syncthreads();
    }
    const double wa = __ldg(a.weights + r0 + 2 * j), wb = has_b ? __ldg(a.weights + r0 + 2 * j + 1) : 0.0;
    for (int k = threadIdx.x; k <= half; k += kThreads) {
      const double2 p = z[k], q = z[k == 0 ? 0 : n - k];
      double s = acc[k];
      if (va) s += wa * ((p.x + q.x) * (p.x + q.x) + (p.y - q.y) * (p.y - q.y));  // 4 |A_k|^2
      if (vb) s += wb * ((p.x - q.x) * (p.x - q.x) + (p.y + q.y) * (p.y + q.y));  // 4 |B_k|^2
      acc[k] = s;
    }
    if (threadIdx.x == 0) {
      if (va) wsum += wa, rows += 1.0;
      if (vb) wsum += wb, rows += 1.0;
    }
    __syncthreads();  // z is rewritten by the next pair
  }

  double* out = a.partial + static_cast<size_t>(item) * a.width;
  if (threadIdx.x == 0) {
    out[0] = wsum;
    out[1] = rows;
  }
  for (int k = threadIdx.x; k <= half; k += kThreads) {
    const double c = (k == 0 || 2 * k == n) ? 0.25 : 0.5;  // c_k / 4
    out[2 + k] = acc[k] * c * a.inv_nn;
  }
}

// Each (plane, band)'s partials added in chunk order: one CTA per (plane, band), one thread per value.
__global__ void __launch_bounds__(kThreads) spectra_reduce_kernel(const __grid_constant__ SpecLaunch a) {
  const int pb = blockIdx.x, plane = pb / a.n_bands, band = pb - plane * a.n_bands;
  const int per_plane = a.band_item_off[a.n_bands];
  const int chunks = a.band_item_off[band + 1] - a.band_item_off[band];
  const double* part =
      a.partial + (static_cast<size_t>(plane) * per_plane + a.band_item_off[band]) * static_cast<size_t>(a.width);
  for (int j = threadIdx.x; j < a.width; j += kThreads) {
    double s = 0.0;
    for (int c = 0; c < chunks; ++c) s += part[static_cast<size_t>(c) * a.width + j];
    a.out[static_cast<size_t>(pb) * a.width + j] = s;
  }
}

// ---- host side --------------------------------------------------------------------------------------------------
// The radices of an n-point FFT (4s first, then at most one 2, then 3s and 5s); false when n has another factor.
bool factor(int n, SpecLaunch* l) {
  int s = 0;
  for (int r : {4, 2, 3, 5})
    while (n % r == 0 && n > 1) {
      l->radix[s++] = r;
      n /= r;
    }
  l->n_stages = s;
  return n == 1;
}

// Validate the descriptors and the bands and lay out the partition; *items / *planes receive the totals.
int plan(SpecLaunch* l, const AbSpectrumField* fields, int32_t n_fields, size_t field_bytes, const int32_t* band_rows,
         int32_t n_bands, const char* who, int64_t* items, int64_t* planes) {
  int st = check_array(fields, n_fields, field_bytes, sizeof(AbSpectrumField), "AbSpectrumField", AB_SPEC_MAX_FIELDS,
                       who);
  if (st != AB_OK) return st;
  AB_CHECK_ARG(n_bands >= 1, "%s: n_bands %d < 1", who, n_bands);
  if (n_bands > AB_SPEC_MAX_BANDS) {
    set_error("%s: %d bands in one call, at most %d are supported", who, n_bands, AB_SPEC_MAX_BANDS);
    return AB_ERR_UNSUPPORTED;
  }
  AB_CHECK_ARG(band_rows, "%s: null argument", who);
  int64_t n_planes = 0;
  const int h = n_fields ? fields[0].h : 0, w = n_fields ? fields[0].w : 0;
  for (int i = 0; i < n_fields; ++i) {
    const AbSpectrumField& f = fields[i];
    AB_CHECK_ARG(f.x, "%s: field %d: null x", who, i);
    AB_CHECK_ARG(f.h > 0 && f.w > 0 && f.levels > 0, "%s: field %d: bad extent %d levels of %d x %d", who, i,
                 f.levels, f.h, f.w);
    AB_CHECK_ARG(f.h == h && f.w == w, "%s: field %d is %d x %d, field 0 %d x %d; one call takes one grid", who, i,
                 f.h, f.w, h, w);
    AB_CHECK_ARG(f.ld >= f.w, "%s: field %d: row pitch %d smaller than the width %d", who, i, f.ld, f.w);
    AB_CHECK_ARG(f.level_stride >= 0, "%s: field %d: negative level stride", who, i);
    l->f[i] = f;
    l->plane_off[i] = static_cast<int32_t>(n_planes);
    n_planes += f.levels;
    l->vec[i] = aligned16(f.x) && f.w % 4 == 0 && f.ld % 4 == 0 && f.level_stride % 4 == 0;
  }
  if (n_fields) {
    if (w > AB_SPEC_MAX_WIDTH || !factor(w, l)) {
      set_error("%s: width %d: supported are widths up to %d with no prime factor above 5", who, w,
                AB_SPEC_MAX_WIDTH);
      return AB_ERR_UNSUPPORTED;
    }
  }
  int per_plane = 0;
  for (int b = 0; b < n_bands; ++b) {
    const int r0 = band_rows[2 * b], r1 = band_rows[2 * b + 1];
    AB_CHECK_ARG(0 <= r0 && r0 <= r1 && (n_fields == 0 || r1 <= h), "%s: band %d: rows [%d, %d) outside [0, %d]",
                 who, b, r0, r1, h);
    l->band_r0[b] = r0;
    l->band_r1[b] = r1;
    l->band_item_off[b] = per_plane;
    per_plane += ceil_div(r1 - r0, kChunkRows);
  }
  l->band_item_off[n_bands] = per_plane;
  l->plane_off[n_fields] = static_cast<int32_t>(n_planes);
  l->n = w;
  l->n_bands = n_bands;
  l->width = w / 2 + 3;
  l->inv_n = n_fields ? 1.0 / w : 0.0;
  l->inv_nn = n_fields ? 1.0 / (static_cast<double>(w) * w) : 0.0;
  if (n_planes * per_plane > INT32_MAX || n_planes * n_bands > INT32_MAX) {
    set_error("%s: more than %d work items in one call", who, INT32_MAX);
    return AB_ERR_UNSUPPORTED;
  }
  *items = n_planes * per_plane;
  *planes = n_planes;
  return AB_OK;
}

}  // namespace
}  // namespace ab

extern "C" int ab_zonal_spectra_workspace_bytes(const AbSpectrumField* fields, int32_t n_fields, size_t field_bytes,
                                                const int32_t* band_rows, int32_t n_bands, size_t* bytes) {
  using namespace ab;
  AB_CHECK_ARG(bytes, "ab_zonal_spectra_workspace_bytes: null argument");
  SpecLaunch l;
  int64_t items = 0, planes = 0;
  const int st = plan(&l, fields, n_fields, field_bytes, band_rows, n_bands, "ab_zonal_spectra_workspace_bytes",
                      &items, &planes);
  if (st != AB_OK) return st;
  *bytes = n_fields ? static_cast<size_t>(items) * l.width * sizeof(double) : 0;
  return AB_OK;
}

extern "C" int ab_zonal_spectra(const AbSpectrumField* fields, int32_t n_fields, size_t field_bytes,
                                const int32_t* band_rows, int32_t n_bands, const double* row_weights, double* out,
                                void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ab;
  const char* who = "ab_zonal_spectra";
  SpecLaunch l;
  int64_t items = 0, planes = 0;
  int st = plan(&l, fields, n_fields, field_bytes, band_rows, n_bands, who, &items, &planes);
  if (st != AB_OK) return st;
  if (n_fields == 0) return AB_OK;
  const size_t need = static_cast<size_t>(items) * l.width * sizeof(double);
  AB_CHECK_ARG(row_weights && out && (workspace || need == 0), "%s: null argument", who);
  AB_CHECK_ARG(workspace_bytes >= need, "%s: workspace of %zu bytes, %zu needed", who, workspace_bytes, need);
  AB_CHECK_ARG((reinterpret_cast<uintptr_t>(row_weights) | reinterpret_cast<uintptr_t>(out) |
                reinterpret_cast<uintptr_t>(workspace)) % alignof(double) == 0,
               "%s: row_weights, out and workspace must be 8-byte aligned", who);
  l.weights = row_weights;
  l.partial = static_cast<double*>(workspace);
  l.out = out;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (items > 0) {
    const size_t smem = smem_layout(l.n).bytes;
    if (smem > 48 * 1024) {
      const cudaError_t e = cudaFuncSetAttribute(spectra_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 static_cast<int>(smem));
      if (e != cudaSuccess) {
        set_error("%s: %zu bytes of shared memory: %s", who, smem, cudaGetErrorString(e));
        return AB_ERR_CUDA;
      }
    }
    spectra_partial_kernel<<<static_cast<unsigned>(items), kThreads, smem, s>>>(l);
    AB_COUNT_LAUNCH(1);
    AB_CHECK_LAUNCH(who);
  }
  spectra_reduce_kernel<<<static_cast<unsigned>(planes * n_bands), kThreads, 0, s>>>(l);
  AB_COUNT_LAUNCH(1);
  AB_CHECK_LAUNCH(who);
  return AB_OK;
}
