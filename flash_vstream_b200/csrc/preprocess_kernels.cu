// preprocess_kernels.cu — fvs_resample_plan / fvs_preprocess_workspace_bytes / fvs_preprocess: decoded uint8 RGB frames
// -> the pixels the vision towers take, bit-identical to the reference's CPU image processors.
//
// Both reference processors resize with Pillow's BICUBIC resample of an 8-bit RGB image (transformers'
// image_transforms.resize), which is fixed-point: per-axis int32 coefficients with 22 fractional bits, a horizontal pass
// into a clipped uint8 intermediate over the source rows the vertical pass reads, then the vertical pass.  Rescale and
// normalize are a function of one byte per channel, so the host hands in a float32 [3, 256] table built with the numpy
// operations of transformers, and the device only looks values up.
//
// Two launches per call: resample_rows_kernel (horizontal pass into a planar uint8 workspace [T, 3, rows, cols]) and
// resample_cols_kernel (vertical pass, table lookup, and the layout write).  Only the window of the resized image the
// caller asks for is computed (the CLIP center crop): the outputs of the window are the same integers the full resize
// computes there, because every output depends only on its own taps.
#include <cuda_fp16.h>

#include <cmath>

#include "fvs_common.h"

// The coefficients must be PIL's doubles, bit for bit: no fused multiply-add in the host arithmetic below (the pragma
// is for the host compiler; nvcc's front end does not know it).
#if defined(__GNUC__) && !defined(__clang__) && !defined(__CUDA_ARCH__)
#pragma nv_diag_suppress 1675
#pragma GCC optimize("fp-contract=off")
#endif

namespace fvs {
namespace pre {

constexpr int kThreads = 256;
constexpr int kBits = 22;                    // PIL's PRECISION_BITS for 8-bit images
constexpr int kPatch = 14, kMerge = 2, kTemporal = 2;
constexpr int kQwenCols = 3 * kTemporal * kPatch * kPatch;   // 1176
constexpr size_t kRowSmemMax = 48 * 1024;

// ---- host: PIL's precompute_coeffs + normalize_coeffs_8bpc (Pillow src/libImaging/Resample.c), BICUBIC, a = -0.5 ----
double bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

struct AxisScale {
  double scale, filterscale, support;
  int taps;
};
AxisScale axis_scale(int in_size, int out_size) {
  AxisScale s;
  s.scale = s.filterscale = double(in_size) / out_size;
  if (s.filterscale < 1.0) s.filterscale = 1.0;
  s.support = 2.0 * s.filterscale;
  s.taps = int(std::ceil(s.support)) * 2 + 1;
  return s;
}

// source window {xmin, n} of output xx
void axis_bounds(const AxisScale& s, int in_size, int xx, int* xmin_out, int* n_out) {
  const double center = (xx + 0.5) * s.scale;
  int xmin = int(center - s.support + 0.5);
  if (xmin < 0) xmin = 0;
  int xmax = int(center + s.support + 0.5);
  if (xmax > in_size) xmax = in_size;
  *xmin_out = xmin;
  *n_out = xmax - xmin;
}

void axis_coeffs(const AxisScale& s, int in_size, int xx, int32_t* bounds, int32_t* k_out) {
  int xmin, n;
  axis_bounds(s, in_size, xx, &xmin, &n);
  const double center = (xx + 0.5) * s.scale;
  const double ss = 1.0 / s.filterscale;
  std::vector<double> k(n);
  double ww = 0.0;
  for (int x = 0; x < n; ++x) {
    k[x] = bicubic((x + xmin - center + 0.5) * ss);
    ww += k[x];
  }
  for (int x = 0; x < s.taps; ++x) {
    double w = x < n ? k[x] : 0.0;
    if (x < n && ww != 0.0) w /= ww;
    k_out[x] = w < 0 ? int32_t(-0.5 + w * (1 << kBits)) : int32_t(0.5 + w * (1 << kBits));
  }
  bounds[0] = xmin;
  bounds[1] = n;
}

// the scalar fields of a window [first, first + count) of an in_size -> out_size axis
int axis_fill(int in_size, int out_size, int first, int count, fvs_resample_axis* a, const char* api) {
  FVS_REQUIRE(in_size > 0 && out_size > 0, "%s: sizes %d -> %d must be positive", api, in_size, out_size);
  FVS_REQUIRE(first >= 0 && count > 0 && int64_t(first) + count <= out_size,
              "%s: window [%d, %d + %d) is not inside the resized length %d", api, first, first, count, out_size);
  const AxisScale s = axis_scale(in_size, out_size);
  int lo, n_lo, hi, n_hi;
  axis_bounds(s, in_size, first, &lo, &n_lo);
  axis_bounds(s, in_size, first + count - 1, &hi, &n_hi);
  a->in_size = in_size;
  a->out_size = out_size;
  a->first = first;
  a->count = count;
  a->taps = s.taps;
  a->span_first = lo;
  a->span_count = hi + n_hi - lo;
  return FVS_OK;
}

int check_axis(const fvs_resample_axis* a, int in_size, const char* which, const char* api) {
  FVS_REQUIRE(a->bounds && a->coeffs, "%s: null %s-axis tables", api, which);
  FVS_REQUIRE(reinterpret_cast<uintptr_t>(a->bounds) % 8 == 0, "%s: %s-axis bounds must be 8-byte aligned", api, which);
  FVS_REQUIRE(a->in_size == in_size, "%s: the %s-axis plan is for %d source pixels, the frames have %d", api, which,
              a->in_size, in_size);
  fvs_resample_axis want = {};
  int r = axis_fill(a->in_size, a->out_size, a->first, a->count, &want, api);
  if (r) return r;
  FVS_REQUIRE(a->taps == want.taps && a->span_first == want.span_first && a->span_count == want.span_count,
              "%s: the %s-axis plan does not match %d -> %d, window [%d, +%d) (use fvs_resample_plan)", api, which,
              a->in_size, a->out_size, a->first, a->count);
  return FVS_OK;
}

size_t workspace_bytes(const fvs_resample_axis& x, const fvs_resample_axis& y, int frames) {
  return size_t(frames) * 3 * size_t(y.span_count) * size_t(x.count);
}

// ---- device ----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int clip8(int acc) {
  acc >>= kBits;
  return acc < 0 ? 0 : (acc > 255 ? 255 : acc);
}

struct RowArgs {
  const uint8_t* src;       // [T, H, W, 3]
  uint8_t* tmp;             // [T, 3, rows, cols]
  const int2* bounds;       // [cols] {xmin, n}
  const int* coeffs;        // [cols, taps]
  int H, W, taps, cols, rows, row0, span0, span;
};

// Horizontal pass: block (r, t) stages source row row0 + r of frame t (the columns the window reads) in shared memory
// and writes its `cols` outputs per channel, clipped to uint8, channel-planar.
__global__ void __launch_bounds__(kThreads) resample_rows_kernel(const __grid_constant__ RowArgs a) {
  extern __shared__ uint8_t row[];
  const int r = blockIdx.x, t = blockIdx.y;
  const uint8_t* src = a.src + ((size_t(t) * a.H + a.row0 + r) * a.W + a.span0) * 3;
  for (int i = threadIdx.x; i < a.span * 3; i += blockDim.x) row[i] = src[i];
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * a.cols; i += blockDim.x) {
    const int c = i / a.cols, x = i - c * a.cols;
    const int2 b = a.bounds[x];
    const int* k = a.coeffs + size_t(x) * a.taps;
    const uint8_t* p = row + (b.x - a.span0) * 3 + c;
    int acc = 1 << (kBits - 1);
    for (int j = 0; j < b.y; ++j) acc += int(p[3 * j]) * k[j];
    a.tmp[((size_t(t) * 3 + c) * a.rows + r) * a.cols + x] = uint8_t(clip8(acc));
  }
}

struct ColArgs {
  const uint8_t* tmp;       // [T, 3, rows, cols]
  void* out;
  const int2* bounds;       // [out_rows] {ymin, n}
  const int* coeffs;        // [out_rows, taps]
  const float* table;       // [3, 256]
  int T, taps, cols, rows, row0, out_rows;
};

// Vertical pass over output row y of frame t, then the table lookup and the layout write:
//   FVS_PRE_CLIP  f16 [T, 3, out_rows, cols];
//   FVS_PRE_QWEN  fp32 [T/2 * gh * gw, 1176], row ((ti*gh/2 + bh)*gw/2 + bw)*4 + mh*2 + mw, column ((c*2 + tp)*14 + py)*14
//                 + px; a one-frame clip fills both temporal slots.
template <int kLayout>
__global__ void __launch_bounds__(kThreads) resample_cols_kernel(const __grid_constant__ ColArgs a) {
  __shared__ float lut[3 * 256];
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) lut[i] = a.table[i];
  __syncthreads();
  const int y = blockIdx.x, t = blockIdx.y;
  const int2 b = a.bounds[y];
  const int* k = a.coeffs + size_t(y) * a.taps;
  for (int i = threadIdx.x; i < 3 * a.cols; i += blockDim.x) {
    const int c = i / a.cols, x = i - c * a.cols;
    const uint8_t* p = a.tmp + ((size_t(t) * 3 + c) * a.rows + (b.x - a.row0)) * a.cols + x;
    int acc = 1 << (kBits - 1);
    for (int j = 0; j < b.y; ++j) acc += int(p[size_t(j) * a.cols]) * k[j];
    const float v = lut[c * 256 + clip8(acc)];
    if (kLayout == FVS_PRE_CLIP) {
      static_cast<__half*>(a.out)[((size_t(t) * 3 + c) * a.out_rows + y) * a.cols + x] = __float2half_rn(v);
    } else {
      const int hy = y / kPatch, py = y - hy * kPatch, hx = x / kPatch, px = x - hx * kPatch;
      const int gh2 = a.out_rows / (kPatch * kMerge), gw2 = a.cols / (kPatch * kMerge);
      const size_t orow = ((size_t(t / kTemporal) * gh2 + hy / kMerge) * gw2 + hx / kMerge) * (kMerge * kMerge) +
                          (hy % kMerge) * kMerge + (hx % kMerge);
      float* o = static_cast<float*>(a.out) + orow * kQwenCols + (c * kTemporal * kPatch + py) * kPatch + px;
      const int tp = t % kTemporal;
      o[tp * kPatch * kPatch] = v;
      if (a.T == 1) o[(1 - tp) * kPatch * kPatch] = v;
    }
  }
}

}  // namespace pre
}  // namespace fvs

using namespace fvs;
using namespace fvs::pre;

extern "C" {

int fvs_resample_plan(int in_size, int out_size, int first, int count, fvs_resample_axis* axis_h, int32_t* bounds_h,
                      int32_t* coeffs_h) {
  const char* api = "fvs_resample_plan";
  FVS_REQUIRE(axis_h, "%s: null axis", api);
  FVS_REQUIRE(!bounds_h == !coeffs_h, "%s: bounds and coeffs are filled together", api);
  fvs_resample_axis a = {};
  int r = axis_fill(in_size, out_size, first, count, &a, api);
  if (r) return r;
  if (bounds_h) {
    const AxisScale s = axis_scale(in_size, out_size);
    for (int i = 0; i < count; ++i) axis_coeffs(s, in_size, first + i, bounds_h + 2 * i, coeffs_h + size_t(i) * s.taps);
  }
  a.bounds = axis_h->bounds;      // the device copies are the caller's to set
  a.coeffs = axis_h->coeffs;
  *axis_h = a;
  return FVS_OK;
}

size_t fvs_preprocess_workspace_bytes(const fvs_resample_axis* x_h, const fvs_resample_axis* y_h, int frames) {
  if (!x_h || !y_h || frames <= 0) return 0;
  return workspace_bytes(*x_h, *y_h, frames);
}

int fvs_preprocess(const uint8_t* frames, int T, int H, int W, int C, const fvs_resample_axis* x_h,
                   const fvs_resample_axis* y_h, const float* table, int layout, int pool, void* out, void* workspace,
                   size_t workspace_bytes_, fvs_stream_t stream) {
  const char* api = "fvs_preprocess";
  FVS_REQUIRE(frames && x_h && y_h && table && out && workspace, "%s: null pointer", api);
  FVS_REQUIRE(C == 3, "%s: %d channels (RGB frames have 3)", api, C);
  FVS_REQUIRE(T > 0 && H > 0 && W > 0, "%s: empty input [%d, %d, %d, 3]", api, T, H, W);
  FVS_REQUIRE(T <= 65535, "%s: %d frames in one call (at most 65535)", api, T);
  int r;
  if ((r = check_axis(x_h, W, "x", api)) || (r = check_axis(y_h, H, "y", api))) return r;
  const size_t need = workspace_bytes(*x_h, *y_h, T);
  FVS_REQUIRE(workspace_bytes_ >= need, "%s: workspace of %zu bytes < %zu", api, workspace_bytes_, need);
  const size_t row_smem = size_t(x_h->span_count) * 3;
  FVS_REQUIRE(row_smem <= kRowSmemMax, "%s: a window reading %d source columns is wider than the %zu supported", api,
              x_h->span_count, kRowSmemMax / 3);
  FVS_REQUIRE(layout == FVS_PRE_CLIP || layout == FVS_PRE_QWEN, "%s: unknown layout %d", api, layout);
  if (layout == FVS_PRE_QWEN) {
    FVS_REQUIRE(T == 1 || T % kTemporal == 0, "%s: Qwen2-VL clips hold 1 or an even number of frames, not %d", api, T);
    FVS_REQUIRE(pool >= 1, "%s: pool %d < 1", api, pool);
    const int f = kPatch * kMerge * pool;
    FVS_REQUIRE(x_h->first == 0 && x_h->count == x_h->out_size && y_h->first == 0 && y_h->count == y_h->out_size,
                "%s: the Qwen2-VL layout takes the whole resized frame (no crop)", api);
    FVS_REQUIRE(y_h->count % f == 0 && x_h->count % f == 0, "%s: resized %dx%d is not a multiple of %d (patch %d x merge %d x pool %d)",
                api, y_h->count, x_h->count, f, kPatch, kMerge, pool);
  }
  RowArgs ra = {};
  ra.src = frames;
  ra.tmp = static_cast<uint8_t*>(workspace);
  ra.bounds = reinterpret_cast<const int2*>(x_h->bounds);
  ra.coeffs = x_h->coeffs;
  ra.H = H;
  ra.W = W;
  ra.taps = x_h->taps;
  ra.cols = x_h->count;
  ra.rows = y_h->span_count;
  ra.row0 = y_h->span_first;
  ra.span0 = x_h->span_first;
  ra.span = x_h->span_count;
  cudaStream_t st = (cudaStream_t)stream;
  resample_rows_kernel<<<dim3(ra.rows, T), kThreads, row_smem, st>>>(ra);
  FVS_CHECK_LAUNCH("resample_rows_kernel");
  ColArgs ca = {};
  ca.tmp = ra.tmp;
  ca.out = out;
  ca.bounds = reinterpret_cast<const int2*>(y_h->bounds);
  ca.coeffs = y_h->coeffs;
  ca.table = table;
  ca.T = T;
  ca.taps = y_h->taps;
  ca.cols = x_h->count;
  ca.rows = y_h->span_count;
  ca.row0 = y_h->span_first;
  ca.out_rows = y_h->count;
  if (layout == FVS_PRE_CLIP) {
    resample_cols_kernel<FVS_PRE_CLIP><<<dim3(ca.out_rows, T), kThreads, 0, st>>>(ca);
  } else {
    resample_cols_kernel<FVS_PRE_QWEN><<<dim3(ca.out_rows, T), kThreads, 0, st>>>(ca);
  }
  FVS_CHECK_LAUNCH("resample_cols_kernel");
  return FVS_OK;
}

}  // extern "C"
