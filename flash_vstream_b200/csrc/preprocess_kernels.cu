// preprocess_kernels.cu — fvs_resample_plan / fvs_preprocess_workspace_bytes / fvs_preprocess / fvs_preprocess_plan /
// fvs_preprocess_multi: decoded uint8 RGB frames -> the pixels the vision towers take, bit-identical to the reference's
// CPU image processors.
//
// Both reference processors resize with Pillow's BICUBIC resample of an 8-bit RGB image (transformers'
// image_transforms.resize), which is fixed-point: per-axis int32 coefficients with 22 fractional bits, a horizontal pass
// into a clipped uint8 intermediate over the source rows the vertical pass reads, then the vertical pass.  Rescale and
// normalize are a function of one byte per channel, so the host hands in a float32 [3, 256] table built with the numpy
// operations of transformers, and the device only looks values up.
//
// A call is a table of jobs (clips of any size; fvs_preprocess is the one-job case) and two launches per 32 jobs:
// resample_rows_kernel (horizontal pass into a planar uint8 workspace [T, 3, rows, cols] per job) and resample_cols_kernel
// (vertical pass, table lookup, and the layout write).  A two-stage job (Qwen2-VL's fetch_video resize, then its image
// processor's) runs its first stage as an FVS_PRE_RGB8 job into its own workspace, in a launch pair of its own ahead of
// the final one: that 8-bit image is exactly the PIL image the first resize returns, and the second stage reads it as
// a single-stage job reads decoded frames.  Both grids are flat: a block finds its job in the block-offset
// table, so the per-element code is the same whatever the jobs next to it.  Only the window of the resized image the
// caller asks for is computed (the CLIP center crop): the outputs of the window are the same integers the full resize
// computes there, because every output depends only on its own taps.
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <type_traits>
#include <vector>

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

// One clip of a launch: its frames, its slice of the workspace and of the output, and its two axis plans.
struct Job {
  const uint8_t* src;       // [T, H, W, 3]
  uint8_t* tmp;             // [T, 3, rows, cols]
  void* out;
  const int2* xb;           // [cols] {xmin, n}
  const int* xk;            // [cols, xtaps]
  const int2* yb;           // [out_rows] {ymin, n}
  const int* yk;            // [out_rows, ytaps]
  int H, W, T, xtaps, ytaps, cols, rows, row0, span0, span, out_rows;
};

// Up to kMaxJobs clips per launch pair, in a kernel parameter (no allocation, no copy).  Block b of the rows launch
// belongs to the job j with row_block0[j] <= b < row_block0[j + 1]; likewise for the cols launch.
constexpr int kMaxJobs = 32;
struct MultiArgs {
  Job job[kMaxJobs];
  int row_block0[kMaxJobs + 1];
  int col_block0[kMaxJobs + 1];
  const float* table;       // [3, 256]
  int n;
};

__device__ __forceinline__ int find_job(const int* block0, int n, int b) {
  int j = 0;
  while (j + 1 < n && b >= block0[j + 1]) ++j;
  return j;
}

// Horizontal pass: row row0 + r of frame t (the columns the window reads) staged in shared memory, `cols` outputs per
// channel, clipped to uint8, channel-planar.
__device__ __forceinline__ void resample_row(const Job& a, int r, int t, uint8_t* row) {
  const uint8_t* src = a.src + ((size_t(t) * a.H + a.row0 + r) * a.W + a.span0) * 3;
  for (int i = threadIdx.x; i < a.span * 3; i += blockDim.x) row[i] = src[i];
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * a.cols; i += blockDim.x) {
    const int c = i / a.cols, x = i - c * a.cols;
    const int2 b = a.xb[x];
    const int* k = a.xk + size_t(x) * a.xtaps;
    const uint8_t* p = row + (b.x - a.span0) * 3 + c;
    int acc = 1 << (kBits - 1);
    for (int j = 0; j < b.y; ++j) acc += int(p[3 * j]) * k[j];
    a.tmp[((size_t(t) * 3 + c) * a.rows + r) * a.cols + x] = uint8_t(clip8(acc));
  }
}

// Vertical pass over output row y of frame t, then the table lookup and the layout write:
//   FVS_PRE_CLIP  f16 [T, 3, out_rows, cols];
//   FVS_PRE_QWEN  fp32 [T/2 * gh * gw, 1176], row ((ti*gh/2 + bh)*gw/2 + bw)*4 + mh*2 + mw, column ((c*2 + tp)*14 + py)*14
//                 + px; a one-frame clip fills both temporal slots;
//   FVS_PRE_QWEN_CODES  the same rows and columns as uint8: the resampled byte itself, before the table lookup;
//   FVS_PRE_RGB8  uint8 [T, out_rows, cols, 3]: the resized 8-bit image itself.
template <int kLayout>
__device__ __forceinline__ void resample_col(const Job& a, int y, int t, const float* lut) {
  const int2 b = a.yb[y];
  const int* k = a.yk + size_t(y) * a.ytaps;
  for (int i = threadIdx.x; i < 3 * a.cols; i += blockDim.x) {
    const int c = i / a.cols, x = i - c * a.cols;
    const uint8_t* p = a.tmp + ((size_t(t) * 3 + c) * a.rows + (b.x - a.row0)) * a.cols + x;
    int acc = 1 << (kBits - 1);
    for (int j = 0; j < b.y; ++j) acc += int(p[size_t(j) * a.cols]) * k[j];
    if (kLayout == FVS_PRE_RGB8) {
      static_cast<uint8_t*>(a.out)[((size_t(t) * a.out_rows + y) * a.cols + x) * 3 + c] = uint8_t(clip8(acc));
      continue;
    }
    const float v = lut[c * 256 + clip8(acc)];
    if (kLayout == FVS_PRE_CLIP) {
      static_cast<__half*>(a.out)[((size_t(t) * 3 + c) * a.out_rows + y) * a.cols + x] = __float2half_rn(v);
    } else {
      const int hy = y / kPatch, py = y - hy * kPatch, hx = x / kPatch, px = x - hx * kPatch;
      const int gh2 = a.out_rows / (kPatch * kMerge), gw2 = a.cols / (kPatch * kMerge);
      const size_t orow = ((size_t(t / kTemporal) * gh2 + hy / kMerge) * gw2 + hx / kMerge) * (kMerge * kMerge) +
                          (hy % kMerge) * kMerge + (hx % kMerge);
      using E = std::conditional_t<kLayout == FVS_PRE_QWEN, float, uint8_t>;
      const E e = kLayout == FVS_PRE_QWEN ? E(v) : E(clip8(acc));
      E* o = static_cast<E*>(a.out) + orow * kQwenCols + (c * kTemporal * kPatch + py) * kPatch + px;
      const int tp = t % kTemporal;
      o[tp * kPatch * kPatch] = e;
      if (a.T == 1) o[(1 - tp) * kPatch * kPatch] = e;
    }
  }
}

// Flat grids: job j owns blocks [block0[j], block0[j + 1]); its block (t * rows + r) is row r of frame t.
__global__ void __launch_bounds__(kThreads) resample_rows_kernel(const __grid_constant__ MultiArgs m) {
  extern __shared__ uint8_t row[];
  const int j = find_job(m.row_block0, m.n, blockIdx.x);
  const Job& a = m.job[j];
  const int b = blockIdx.x - m.row_block0[j], t = b / a.rows;
  resample_row(a, b - t * a.rows, t, row);
}

template <int kLayout>
__global__ void __launch_bounds__(kThreads) resample_cols_kernel(const __grid_constant__ MultiArgs m) {
  __shared__ float lut[3 * 256];
  if (kLayout == FVS_PRE_CLIP || kLayout == FVS_PRE_QWEN) {     // codes and images are the bytes before the lookup
    for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) lut[i] = m.table[i];
    __syncthreads();
  }
  const int j = find_job(m.col_block0, m.n, blockIdx.x);
  const Job& a = m.job[j];
  const int b = blockIdx.x - m.col_block0[j], t = b / a.out_rows;
  resample_col<kLayout>(a, b - t * a.out_rows, t, lut);
}

// ---- host: validation and the plan of a job table -------------------------------------------------------------------
struct JobPlan {
  int64_t row_block, col_block;   // first block of the job in its launch pair
  int64_t out_off, ws_off;        // output elements / workspace bytes before the job
};

bool two_stage(const fvs_preprocess_job& jb) { return jb.x2.out_size != 0 || jb.y2.out_size != 0; }

// the axes of the job's last stage, the ones its layout is written from
const fvs_resample_axis& final_x(const fvs_preprocess_job& jb) { return two_stage(jb) ? jb.x2 : jb.x; }
const fvs_resample_axis& final_y(const fvs_preprocess_job& jb) { return two_stage(jb) ? jb.y2 : jb.y; }

int check_row_span(const fvs_resample_axis& x, const char* api) {
  FVS_REQUIRE(size_t(x.span_count) * 3 <= kRowSmemMax, "%s: a window reading %d source columns is wider than the %zu "
              "supported", api, x.span_count, kRowSmemMax / 3);
  return FVS_OK;
}

// every check fvs_preprocess makes of one clip; `api` names the job
int check_job(const fvs_preprocess_job& jb, int layout, int pool, const char* api) {
  FVS_REQUIRE(jb.frames, "%s: null frames", api);
  FVS_REQUIRE(jb.C == 3, "%s: %d channels (RGB frames have 3)", api, jb.C);
  FVS_REQUIRE(jb.T > 0 && jb.H > 0 && jb.W > 0, "%s: empty input [%d, %d, %d, 3]", api, jb.T, jb.H, jb.W);
  FVS_REQUIRE(jb.T <= 65535, "%s: %d frames in one call (at most 65535)", api, jb.T);
  int r;
  if ((r = check_axis(&jb.x, jb.W, "x", api)) || (r = check_axis(&jb.y, jb.H, "y", api))) return r;
  if ((r = check_row_span(jb.x, api))) return r;
  if (two_stage(jb)) {       // the second stage resizes the first stage's window
    if ((r = check_axis(&jb.x2, jb.x.count, "second-stage x", api)) ||
        (r = check_axis(&jb.y2, jb.y.count, "second-stage y", api)) || (r = check_row_span(jb.x2, api)))
      return r;
  }
  FVS_REQUIRE(layout == FVS_PRE_CLIP || layout == FVS_PRE_QWEN || layout == FVS_PRE_QWEN_CODES || layout == FVS_PRE_RGB8,
              "%s: unknown layout %d", api, layout);
  if (layout == FVS_PRE_QWEN || layout == FVS_PRE_QWEN_CODES) {
    const fvs_resample_axis &x = final_x(jb), &y = final_y(jb);
    FVS_REQUIRE(jb.T == 1 || jb.T % kTemporal == 0, "%s: Qwen2-VL clips hold 1 or an even number of frames, not %d", api,
                jb.T);
    FVS_REQUIRE(pool >= 1, "%s: pool %d < 1", api, pool);
    const int f = kPatch * kMerge * pool;
    FVS_REQUIRE(x.first == 0 && x.count == x.out_size && y.first == 0 && y.count == y.out_size,
                "%s: the Qwen2-VL layout takes the whole resized frame (no crop)", api);
    FVS_REQUIRE(y.count % f == 0 && x.count % f == 0, "%s: resized %dx%d is not a multiple of %d (patch %d x merge "
                "%d x pool %d)", api, y.count, x.count, f, kPatch, kMerge, pool);
  }
  return FVS_OK;
}

int64_t out_elements(const fvs_preprocess_job& jb, int layout) {
  const fvs_resample_axis &x = final_x(jb), &y = final_y(jb);
  if (layout == FVS_PRE_CLIP) return int64_t(jb.T) * 3 * y.count * x.count;
  if (layout == FVS_PRE_RGB8) return int64_t(jb.T) * y.count * x.count * 3;
  return int64_t(jb.T > 1 ? jb.T / kTemporal : 1) * (y.count / kPatch) * (x.count / kPatch) * kQwenCols;
}

// A job's workspace: the planar scratch of its passes, then (two stages) the first stage's 8-bit image, which the
// second stage reads while its own passes reuse the scratch.
int64_t job_scratch_bytes(const fvs_preprocess_job& jb) {
  const int64_t one = int64_t(workspace_bytes(jb.x, jb.y, jb.T));
  return two_stage(jb) ? std::max(one, int64_t(workspace_bytes(jb.x2, jb.y2, jb.T))) : one;
}
int64_t job_workspace_bytes(const fvs_preprocess_job& jb) {
  return job_scratch_bytes(jb) + (two_stage(jb) ? int64_t(jb.T) * jb.y.count * jb.x.count * 3 : 0);
}

// Validates every job (the error names the first bad one) and lays them out; returns the number of launch groups (of
// up to 32 jobs each: one launch pair, two when a job of the group has two stages).
// `one` keeps fvs_preprocess's own messages for its single clip.
int plan_jobs(const fvs_preprocess_job* jobs, int n, int layout, int pool, JobPlan* plan, int64_t* out_total,
              int64_t* ws_total, const char* api, bool one) {
  FVS_REQUIRE(jobs && n > 0, "%s: no jobs", api);
  int64_t out = 0, ws = 0, rows = 0, cols = 0, rows1 = 0, cols1 = 0;
  char name[96];
  for (int i = 0; i < n; ++i) {
    const fvs_preprocess_job& jb = jobs[i];
    if (one) {
      std::snprintf(name, sizeof name, "%s", api);
    } else {
      std::snprintf(name, sizeof name, "%s: job %d", api, i);
    }
    int r = check_job(jb, layout, pool, name);
    if (r) return r;
    if (i % kMaxJobs == 0) rows = cols = rows1 = cols1 = 0;
    plan[i] = {rows, cols, out, ws};
    rows += int64_t(final_y(jb).span_count) * jb.T;
    cols += int64_t(final_y(jb).count) * jb.T;
    if (two_stage(jb)) {
      rows1 += int64_t(jb.y.span_count) * jb.T;
      cols1 += int64_t(jb.y.count) * jb.T;
    }
    FVS_REQUIRE(rows <= INT32_MAX && cols <= INT32_MAX && rows1 <= INT32_MAX && cols1 <= INT32_MAX,
                "%s: more than %d blocks in one launch", name, INT32_MAX);
    out += out_elements(jb, layout);
    ws += job_workspace_bytes(jb);
  }
  *out_total = out;
  *ws_total = ws;
  return (n + kMaxJobs - 1) / kMaxJobs;
}

Job make_job(const uint8_t* src, int T, int H, int W, const fvs_resample_axis& x, const fvs_resample_axis& y,
             uint8_t* tmp, void* out) {
  Job a;
  a.src = src;
  a.tmp = tmp;
  a.out = out;
  a.xb = reinterpret_cast<const int2*>(x.bounds);
  a.xk = x.coeffs;
  a.yb = reinterpret_cast<const int2*>(y.bounds);
  a.yk = y.coeffs;
  a.H = H;
  a.W = W;
  a.T = T;
  a.xtaps = x.taps;
  a.ytaps = y.taps;
  a.cols = x.count;
  a.rows = y.span_count;
  a.row0 = y.span_first;
  a.span0 = x.span_first;
  a.span = x.span_count;
  a.out_rows = y.count;
  return a;
}

// one launch pair over up to kMaxJobs jobs
int launch_pair(const Job* jobs, int n, const float* table, int layout, cudaStream_t st) {
  MultiArgs m = {};
  m.table = table;
  m.n = n;
  size_t row_smem = 0;
  for (int k = 0; k < n; ++k) {
    m.job[k] = jobs[k];
    m.row_block0[k + 1] = m.row_block0[k] + jobs[k].rows * jobs[k].T;
    m.col_block0[k + 1] = m.col_block0[k] + jobs[k].out_rows * jobs[k].T;
    row_smem = std::max(row_smem, size_t(jobs[k].span) * 3);
  }
  resample_rows_kernel<<<m.row_block0[n], kThreads, row_smem, st>>>(m);
  FVS_CHECK_LAUNCH("resample_rows_kernel");
  if (layout == FVS_PRE_CLIP) {
    resample_cols_kernel<FVS_PRE_CLIP><<<m.col_block0[n], kThreads, 0, st>>>(m);
  } else if (layout == FVS_PRE_QWEN) {
    resample_cols_kernel<FVS_PRE_QWEN><<<m.col_block0[n], kThreads, 0, st>>>(m);
  } else if (layout == FVS_PRE_QWEN_CODES) {
    resample_cols_kernel<FVS_PRE_QWEN_CODES><<<m.col_block0[n], kThreads, 0, st>>>(m);
  } else {
    resample_cols_kernel<FVS_PRE_RGB8><<<m.col_block0[n], kThreads, 0, st>>>(m);
  }
  FVS_CHECK_LAUNCH("resample_cols_kernel");
  return FVS_OK;
}

int preprocess_jobs(const fvs_preprocess_job* jobs, int n, const float* table, int layout, int pool, void* out,
                    void* workspace, size_t workspace_bytes_, cudaStream_t st, const char* api, bool one) {
  FVS_REQUIRE(jobs && table && out && workspace, "%s: null pointer", api);
  FVS_REQUIRE(n > 0 && n <= (1 << 20), "%s: %d jobs", api, n);
  std::vector<JobPlan> plan(n);
  int64_t out_total = 0, ws_total = 0;
  const int groups = plan_jobs(jobs, n, layout, pool, plan.data(), &out_total, &ws_total, api, one);
  if (groups < 0) return groups;
  FVS_REQUIRE(workspace_bytes_ >= size_t(ws_total), "%s: workspace of %zu bytes < %zu", api, workspace_bytes_,
              size_t(ws_total));
  const size_t esize = layout == FVS_PRE_CLIP ? sizeof(__half) : layout == FVS_PRE_QWEN ? sizeof(float) : 1;
  for (int g = 0; g < groups; ++g) {
    const int m = std::min(kMaxJobs, n - g * kMaxJobs);
    Job first[kMaxJobs], last[kMaxJobs];
    int n_first = 0;
    for (int k = 0; k < m; ++k) {
      const fvs_preprocess_job& jb = jobs[g * kMaxJobs + k];
      const JobPlan& p = plan[g * kMaxJobs + k];
      uint8_t* tmp = static_cast<uint8_t*>(workspace) + p.ws_off;
      void* o = static_cast<char*>(out) + p.out_off * esize;
      if (two_stage(jb)) {
        uint8_t* img = tmp + job_scratch_bytes(jb);
        first[n_first++] = make_job(jb.frames, jb.T, jb.H, jb.W, jb.x, jb.y, tmp, img);
        last[k] = make_job(img, jb.T, jb.y.count, jb.x.count, jb.x2, jb.y2, tmp, o);
      } else {
        last[k] = make_job(jb.frames, jb.T, jb.H, jb.W, jb.x, jb.y, tmp, o);
      }
    }
    int r;
    if (n_first && (r = launch_pair(first, n_first, table, FVS_PRE_RGB8, st))) return r;
    if ((r = launch_pair(last, m, table, layout, st))) return r;
  }
  return FVS_OK;
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
  fvs_preprocess_job jb = {frames, T, H, W, C, *x_h, *y_h};
  return preprocess_jobs(&jb, 1, table, layout, pool, out, workspace, workspace_bytes_, (cudaStream_t)stream, api, true);
}

int fvs_preprocess_plan(const fvs_preprocess_job* jobs_h, int n_jobs, int layout, int pool, int64_t* plan_h,
                        int64_t* totals_h) {
  const char* api = "fvs_preprocess_plan";
  FVS_REQUIRE(jobs_h && plan_h && totals_h && n_jobs > 0, "%s: null pointer or no jobs", api);
  std::vector<JobPlan> plan(n_jobs);
  const int launches = plan_jobs(jobs_h, n_jobs, layout, pool, plan.data(), &totals_h[0], &totals_h[1], api, false);
  if (launches < 0) return launches;
  for (int i = 0; i < n_jobs; ++i) {
    plan_h[4 * i + 0] = plan[i].row_block;
    plan_h[4 * i + 1] = plan[i].col_block;
    plan_h[4 * i + 2] = plan[i].out_off;
    plan_h[4 * i + 3] = plan[i].ws_off;
  }
  return launches;
}

int fvs_preprocess_multi(const fvs_preprocess_job* jobs_h, int n_jobs, const float* table, int layout, int pool, void* out,
                         void* workspace, size_t workspace_bytes_, fvs_stream_t stream) {
  return preprocess_jobs(jobs_h, n_jobs, table, layout, pool, out, workspace, workspace_bytes_, (cudaStream_t)stream,
                         "fvs_preprocess_multi", false);
}

}  // extern "C"
