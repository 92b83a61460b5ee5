// qwen_bank.cu — the feature-bank kernels of the Qwen2-VL streaming step (DESIGN.md §3.13, §3.18-§3.20): the DAM gather,
// the pick plan, the bank scatter and the pixel gather, each one job table (one stream = the one-job table).
//
// Frames [0, n_dev) of the full-resolution bank (x) and of the PatchMerger bank (merged) are contiguous HBM rows; frames
// [n_dev, n_frames) live in pinned host chunks of chunk_frames frames each, laid out [x rows of the chunk | merged rows of
// the chunk] and read through their mapped device pointers.  The picks come from the retrieval kernels and stay on the
// device: the kernel resolves every pick itself, so the step needs no host round trip to know where its frames are.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "fvs_common.h"

namespace fvs {
namespace qwen {

// The block's strided share (bx of nbx) of pick i's 16-byte words, from sources sx / sm (null: zeros): x words first,
// then merged words.
__device__ __forceinline__ void gather_copy(unsigned bx, unsigned nbx, int i, const uint4* sx, const uint4* sm,
                                            long long fx, long long fm, uint4* out_x, uint4* out_m) {
  const long long nx = out_x ? fx : 0, total = nx + (out_m ? fm : 0);
  const long long stride = (long long)nbx * blockDim.x;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  // four independent loads in flight per thread before the stores: a zero-copy read over PCIe has microseconds of latency
  for (long long w0 = (long long)bx * blockDim.x + threadIdx.x; w0 < total; w0 += 4 * stride) {
    uint4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long w = w0 + u * stride;
      v[u] = zero;
      if (w < nx) { if (sx) v[u] = sx[w]; }
      else if (w < total && sm) v[u] = sm[w - nx];
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long w = w0 + u * stride;
      if (w < nx) out_x[i * fx + w] = v[u];
      else if (w < total) out_m[i * fm + (w - nx)] = v[u];
    }
  }
}

// Frame p (0 <= p, below the bank's frame count) of a two-tier bank -> its rows x / m: the device rows dev_x / dev_m
// (null: none) for p < n_dev, else the rows in its host chunk.  Returns whether the frame is in a host chunk.
template <class T>
__device__ __forceinline__ bool tier_rows(long long p, T* dev_x, T* dev_m, long long n_dev, T* const* chunks,
                                          long long chunk_frames, long long fx, long long fm, T*& x, T*& m) {
  if (p < n_dev) {
    x = dev_x ? dev_x + p * fx : nullptr;
    m = dev_m ? dev_m + p * fm : nullptr;
    return false;
  }
  const long long q = p - n_dev, off = q % chunk_frames;
  T* c = chunks[q / chunk_frames];
  x = c + off * fx;
  m = c + chunk_frames * fx + off * fm;
  return true;
}

// the index of frame p in list[0, n), or n
__device__ __forceinline__ int find_frame(const long long* list, int n, long long p) {
  int k = 0;
  while (k < n && list[k] != p) ++k;
  return k;
}
}  // namespace qwen
}  // namespace fvs

using namespace fvs;
using namespace fvs::qwen;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

namespace {
// ---- the job-table skeleton --------------------------------------------------------------------------------------------
// One flat grid over a launch's jobs: job j owns blocks [first[j], first[j + 1]).
constexpr int kMaxJobs = FVS_QWEN_MEM_JOBS_PER_LAUNCH;
template <class Job, int K>
struct JobLaunch {
  static constexpr int kJobs = K;
  Job job[K];
  int first[K + 1];
  int n;
};

// the job of this block, and the block's index b within it
template <class Job, int K>
__device__ __forceinline__ const Job& job_of(const JobLaunch<Job, K>& L, unsigned& b) {
  int j = 0;
  if constexpr (K > 1)
    while (j + 1 < L.n && blockIdx.x >= unsigned(L.first[j + 1])) ++j;
  b = blockIdx.x - unsigned(L.first[j]);
  return L.job[j];
}

// 256-thread blocks per frame of `words` words: four words per thread, 1 to 64 blocks
int frame_blocks(long long words) {
  const long long bx = (words + 4 * 256 - 1) / (4 * 256);
  return int(bx > 64 ? 64 : bx < 1 ? 1 : bx);
}

template <class Job, int K, class In, class Dev, class Launch>
int launch_jobs(const In* jobs, int n, Dev dev, Launch launch) {
  JobLaunch<Job, K> L;
  L.n = n;
  L.first[0] = 0;
  for (int q = 0; q < n; ++q) L.first[q + 1] = L.first[q] + dev(jobs[q], L.job[q]);
  return launch(L);
}

// A checked table of n_jobs jobs in launches of at most kMaxJobs (a launch of one job: the <1> instantiation).
// dev(job, Job&) writes a job's device form and returns its blocks; launch(const JobLaunch<Job, K>&) enqueues the kernel.
template <class Job, class In, class Dev, class Launch>
int run_jobs(const In* jobs, int n_jobs, Dev dev, Launch launch) {
  for (int i0 = 0; i0 < n_jobs; i0 += kMaxJobs) {
    const int n = std::min(kMaxJobs, n_jobs - i0);
    const int r = n == 1 ? launch_jobs<Job, 1>(jobs + i0, 1, dev, launch)
                         : launch_jobs<Job, kMaxJobs>(jobs + i0, n, dev, launch);
    if (r) return r;
  }
  return FVS_OK;
}

// The outputs of a job table as address ranges: no two jobs may write the same byte.
struct Outputs {
  struct Range { uintptr_t lo, hi; int job; };
  std::vector<Range> r;
  void add(const void* p, size_t bytes, int job) {
    if (p) r.push_back({uintptr_t(p), uintptr_t(p) + bytes, job});
  }
  int check(const char* api) const {
    for (size_t a = 0; a < r.size(); ++a)
      for (size_t b = a + 1; b < r.size(); ++b)
        FVS_REQUIRE(r[a].job == r[b].job || r[a].hi <= r[b].lo || r[b].hi <= r[a].lo, "%s: jobs %d and %d share an output",
                    api, r[a].job, r[b].job);
    return FVS_OK;
  }
};

// ---- DAM gather ----------------------------------------------------------------------------------------------------------
// Job j's block b copies share b % bx of pick b / bx, read from the first source that holds the frame: the previous DAM
// (prev_picks), this step's fresh rows (fresh), the device tier [0, n_dev), a host chunk [n_dev, n_base) (counted in
// host_fetches); a pick in none of them, or outside [0, n_frames), writes zeros.
// Every source holds the same bits of a frame, so for the frames that are in more than one the order decides only which
// copy is read: a bank stream's previous DAM rows are its bank rows of the same frames (spa_x = bank_x[spa_positions],
// the DAM rows of video_embeds are bank_merged rows, and a lazy stream scatters a frame's rows before any gather reads
// them and never rewrites them).  The base bank comes last because a bank-less stream restored with a frame "not yet
// encoded" has a zero slot there; such a frame is always planned, so it is found among the fresh rows first.
struct GatherJobDev {
  const long long* picks;
  const long long* prev_picks;
  const uint4* prev_x;
  const uint4* prev_m;
  const long long* fresh;
  const uint4* fresh_x;
  const uint4* fresh_m;
  const uint4* dev_x;
  const uint4* dev_m;
  const uint4* const* chunks;
  uint4* out_x;
  uint4* out_m;
  unsigned long long* host_fetches;
  long long n_frames, n_base, n_dev, chunk_frames, fx, fm;
  int m, n_fresh, bx;
};

template <int kJobs>
__global__ void __launch_bounds__(256) dam_gather_multi_kernel(const __grid_constant__ JobLaunch<GatherJobDev, kJobs> L) {
  unsigned b;
  const GatherJobDev& J = job_of(L, b);
  const unsigned bx = b % unsigned(J.bx);
  const int i = int(b / unsigned(J.bx));
  __shared__ const uint4* src[2];
  if (threadIdx.x == 0) {
    const long long p = J.picks[i];
    const uint4 *sx = nullptr, *sm = nullptr;
    if (p >= 0 && p < J.n_frames) {
      int k;
      if ((k = find_frame(J.prev_picks, J.m, p)) < J.m) {
        sx = J.prev_x + k * J.fx;
        sm = J.prev_m ? J.prev_m + k * J.fm : nullptr;
      } else if ((k = find_frame(J.fresh, J.n_fresh, p)) < J.n_fresh) {
        sx = J.fresh_x + k * J.fx;
        sm = J.fresh_m ? J.fresh_m + k * J.fm : nullptr;
      } else if (p < J.n_base && tier_rows(p, J.dev_x, J.dev_m, J.n_dev, J.chunks, J.chunk_frames, J.fx, J.fm, sx, sm) &&
                 bx == 0 && J.host_fetches) {
        atomicAdd(J.host_fetches, 1ull);
      }
    }
    src[0] = sx;
    src[1] = sm;
  }
  __syncthreads();
  gather_copy(bx, J.bx, i, src[0], src[1], J.fx, J.fm, J.out_x, J.out_m);
}

int gather_dev(const fvs_qwen_gather_job& g, GatherJobDev& d) {
  const long long fx = g.x_frame_elems * 2 / 16, fm = g.merged_frame_elems * 2 / 16;
  const int bx = frame_blocks((g.spa_x_out ? fx : 0) + (g.merged_out ? fm : 0));
  d = GatherJobDev{(const long long*)g.picks, (const long long*)g.prev_picks, (const uint4*)g.prev_x,
                   (const uint4*)g.prev_merged, (const long long*)g.fresh_frames, (const uint4*)g.fresh_x,
                   (const uint4*)g.fresh_merged, (const uint4*)g.dev_x, (const uint4*)g.dev_merged,
                   (const uint4* const*)g.host_chunks, (uint4*)g.spa_x_out, (uint4*)g.merged_out,
                   (unsigned long long*)g.host_fetches, (long long)g.n_frames, (long long)g.n_base, (long long)g.n_dev,
                   (long long)g.chunk_frames, fx, fm, g.m, g.n_fresh, bx};
  return bx * g.n;
}

template <class In, class Dev>
int gather_jobs(const In* jobs, int n_jobs, Dev dev, cudaStream_t stream) {
  return run_jobs<GatherJobDev>(jobs, n_jobs, dev, [&](const auto& L) {
    dam_gather_multi_kernel<std::decay_t<decltype(L)>::kJobs><<<L.first[L.n], 256, 0, stream>>>(L);
    FVS_CHECK_LAUNCH("dam_gather_multi_kernel");
    return FVS_OK;
  });
}

// ---- pick plan (DESIGN.md §3.18, §3.19) --------------------------------------------------------------------------------
// One warp per job walks the picks in order, 32 at a time.  A pick is planned when it is in range, its frame's byte is
// below `stored`, it is not in prev_picks and no earlier pick names the same frame; the warp's ballot compacts the
// planned frames in pick order.  Only the lane that plans a frame (its first pick) writes the frame's byte, so the walk
// is race-free: a later pick of that frame is never planned again, whether or not it sees the byte, because it is not
// the first pick of its frame.  The plan reads prev_picks instead of a per-frame "in the previous DAM" mask, so nothing
// has to move a mask from the old picks to the new ones after the gather, and a clip that complete() redoes plans
// against the same previous DAM with nothing to undo.
struct PlanJobDev {
  const long long* picks;
  unsigned char* frames;
  const long long* prev;
  long long* plan;
  int* count;
  unsigned long long* re_encodes;
  long long n_frames;
  int n, m;
  unsigned char stored;
};

template <int kJobs>
__global__ void __launch_bounds__(32) pick_plan_kernel(const __grid_constant__ JobLaunch<PlanJobDev, kJobs> L) {
  unsigned b;
  const PlanJobDev& J = job_of(L, b);
  const unsigned lane = threadIdx.x;
  int base = 0, again = 0;
  for (int i0 = 0; i0 < J.n; i0 += 32) {
    const int i = i0 + int(lane);
    long long p = -1;
    bool first = false;
    if (i < J.n) {
      p = J.picks ? J.picks[i] : i;
      first = p >= 0 && p < J.n_frames && J.frames[p] < J.stored && find_frame(J.prev, J.m, p) == J.m;
      if (first && J.picks)
        for (int j = 0; j < i; ++j)
          if (J.picks[j] == p) { first = false; break; }
    }
    const unsigned ball = __ballot_sync(0xffffffffu, first);
    if (first) {
      J.plan[base + __popc(ball & ((1u << lane) - 1u))] = p;
      again += J.frames[p] == 1;
      J.frames[p] = 1;
    }
    base += __popc(ball);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) again += __shfl_xor_sync(0xffffffffu, again, o);
  if (lane == 0) {
    *J.count = base;
    if (J.re_encodes && again) atomicAdd(J.re_encodes, (unsigned long long)again);
  }
}

// ---- bank scatter ----------------------------------------------------------------------------------------------------
// The reverse of the DAM gather from the bank alone.  Job j's block b writes share b % bx of planned frame b / bx: x
// words first, then merged words, to the device tier or the frame's host chunk.
struct ScatterJobDev {
  const long long* plan;
  const uint4* src_x;
  const uint4* src_m;
  uint4* dev_x;
  uint4* dev_m;
  uint4* const* chunks;
  long long n_frames, n_dev, chunk_frames, fx, fm;
  int bx;
};

template <int kJobs>
__global__ void __launch_bounds__(256) bank_scatter_kernel(const __grid_constant__ JobLaunch<ScatterJobDev, kJobs> L) {
  unsigned b;
  const ScatterJobDev& J = job_of(L, b);
  const unsigned bx = b % unsigned(J.bx);
  const long long i = b / unsigned(J.bx);
  __shared__ uint4* dst[2];
  if (threadIdx.x == 0) {
    const long long p = J.plan[i];
    uint4 *dx = nullptr, *dm = nullptr;
    if (p >= 0 && p < J.n_frames) tier_rows(p, J.dev_x, J.dev_m, J.n_dev, J.chunks, J.chunk_frames, J.fx, J.fm, dx, dm);
    dst[0] = dx;
    dst[1] = J.src_m ? dm : nullptr;
  }
  __syncthreads();
  uint4 *dx = dst[0], *dm = dst[1];
  if (!dx) return;
  const long long total = J.fx + (dm ? J.fm : 0), stride = (long long)J.bx * blockDim.x;
  for (long long w = (long long)bx * blockDim.x + threadIdx.x; w < total; w += stride) {
    if (w < J.fx) dx[w] = J.src_x[i * J.fx + w];
    else dm[w - J.fx] = J.src_m[i * J.fm + (w - J.fx)];
  }
}

// ---- 8-bit pixel codes (DESIGN.md §3.20) -------------------------------------------------------------------------------
// A code row holds the resampled bytes u of one full-resolution pixel row, columns ((c*2 + tp)*14 + py)*14 + px; the
// tower reads dtype(table[c][u]).  392 = 2*14*14 columns per channel is a multiple of 8, so the 8 codes of one 8-byte
// word share a channel: word w of a row (147 words) is channel (w % 147) / 49.
constexpr long long kCodeWordsPerRow = 1176 / 8, kCodeWordsPerChannel = 392 / 8;

template <int kDtype>
__device__ __forceinline__ unsigned decode_pair(float a, float b) {
  if constexpr (kDtype == FVS_BF16) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);    // round to nearest even, as torch's fp32 -> bf16 cast
    return *reinterpret_cast<const unsigned*>(&v);
  } else {
    const __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<const unsigned*>(&v);
  }
}

// 8 codes of channel-table `lut` -> 8 tower values (16 bytes)
template <int kDtype>
__device__ __forceinline__ uint4 decode_word(uint2 c, const float* lut) {
  uint4 o;
  o.x = decode_pair<kDtype>(lut[c.x & 255], lut[(c.x >> 8) & 255]);
  o.y = decode_pair<kDtype>(lut[(c.x >> 16) & 255], lut[c.x >> 24]);
  o.z = decode_pair<kDtype>(lut[c.y & 255], lut[(c.y >> 8) & 255]);
  o.w = decode_pair<kDtype>(lut[(c.y >> 16) & 255], lut[c.y >> 24]);
  return o;
}

// the [3, 256] table into shared memory, for every thread of the block
__device__ __forceinline__ void load_lut(float* lut, const float* table) {
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) lut[i] = table[i];
  __syncthreads();
}

// words [first, total) of whole code rows, `stride` apart: out[w] = decode(src[w]) (src null: zeros).  Four loads in
// flight per thread before the stores, as gather_copy: a zero-copy read over PCIe has microseconds of latency.
template <int kDtype>
__device__ __forceinline__ void decode_words(const uint2* src, uint4* out, long long first, long long total,
                                             long long stride, const float* lut) {
  for (long long w0 = first; w0 < total; w0 += 4 * stride) {
    uint2 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long w = w0 + u * stride;
      v[u] = make_uint2(0, 0);
      if (w < total && src) v[u] = src[w];
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long w = w0 + u * stride;
      if (w < total)
        out[w] = src ? decode_word<kDtype>(v[u], lut + (w % kCodeWordsPerRow) / kCodeWordsPerChannel * 256)
                     : make_uint4(0, 0, 0, 0);
    }
  }
}

template <int kDtype>
__global__ void __launch_bounds__(256) pixel_decode_kernel(const uint2* __restrict__ codes, const float* __restrict__ table,
                                                           long long words, uint4* __restrict__ out) {
  __shared__ float lut[3 * 256];
  load_lut(lut, table);
  decode_words<kDtype>(codes, out, (long long)blockIdx.x * blockDim.x + threadIdx.x, words,
                       (long long)gridDim.x * blockDim.x, lut);
}

// The pixel gather over code chunks: job j's block b decodes share b % bx of planned frame b / bx, read in place from
// its pinned chunk (the host tier of a bank with no device tier below `base`); a frame outside [base, n_frames) yields
// zeros.
struct CodesJobDev {
  const long long* plan;
  const uint2* const* chunks;
  const float* table;
  uint4* out;
  long long n_frames, base, chunk_frames, words;    // words: 8-byte code words per frame
  int bx;
};

template <int kJobs, int kDtype>
__global__ void __launch_bounds__(256) pixel_codes_gather_kernel(const __grid_constant__ JobLaunch<CodesJobDev, kJobs> L) {
  unsigned b;
  const CodesJobDev& J = job_of(L, b);
  const unsigned bx = b % unsigned(J.bx);
  const long long i = b / unsigned(J.bx);
  __shared__ float lut[3 * 256];
  __shared__ const uint2* src;
  if (threadIdx.x == 0) {
    const long long p = J.plan[i];
    const uint2 *s = nullptr, *none;
    if (p >= 0 && p < J.n_frames)
      tier_rows<const uint2>(p, nullptr, nullptr, J.base, J.chunks, J.chunk_frames, J.words, 0, s, none);
    src = s;
  }
  load_lut(lut, J.table);
  decode_words<kDtype>(src, J.out + i * J.words, (long long)bx * blockDim.x + threadIdx.x, J.words,
                       (long long)J.bx * blockDim.x, lut);
}
}  // namespace

extern "C" {

int fvs_host_device_ptr(const void* host, void** dev_out) {
  FVS_REQUIRE(host && dev_out, "fvs_host_device_ptr: null pointer");
  cudaPointerAttributes a;
  FVS_CUDA_OK(cudaPointerGetAttributes(&a, host));
  FVS_REQUIRE(a.type == cudaMemoryTypeHost, "fvs_host_device_ptr: %p is not pinned host memory", host);
  void* d = nullptr;
  FVS_CUDA_OK(cudaHostGetDevicePointer(&d, const_cast<void*>(host), 0));
  *dev_out = d;
  return FVS_OK;
}

int fvs_qwen_dam_gather_multi(const fvs_qwen_gather_job* jobs, int n_jobs, int dtype, fvs_stream_t stream) {
  const char* api = "fvs_qwen_dam_gather_multi";
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", api);
  Outputs out;
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_gather_job& j = jobs[i];
    const int64_t fx = j.x_frame_elems, fm = j.merged_frame_elems;
    FVS_REQUIRE(j.picks && j.n > 0 && j.n <= 65535, "%s: job %d: need picks and 0 < n <= 65535 (null picks or n=%d)", api,
                i, j.n);
    FVS_REQUIRE(j.spa_x_out || j.merged_out, "%s: job %d: no output", api, i);
    FVS_REQUIRE(j.n_frames > 0 && j.n_dev >= 0 && j.n_dev <= j.n_base && j.n_base <= j.n_frames,
                "%s: job %d: need 0 <= n_dev <= n_base <= n_frames, n_frames > 0 (%lld, %lld, %lld)", api, i,
                (long long)j.n_dev, (long long)j.n_base, (long long)j.n_frames);
    FVS_REQUIRE(fx > 0 && fm >= 0, "%s: job %d: bad frame sizes", api, i);
    FVS_REQUIRE((fx * 2) % 16 == 0 && (fm * 2) % 16 == 0, "%s: job %d: frame sizes must be multiples of 16 bytes", api, i);
    FVS_REQUIRE(!j.merged_out || fm > 0, "%s: job %d: merged_out without merged rows", api, i);
    FVS_REQUIRE(j.m >= 0 && j.m <= 65535 && (j.m == 0 || (j.prev_picks && j.prev_x && (!j.merged_out || j.prev_merged))),
                "%s: job %d: bad previous DAM", api, i);
    FVS_REQUIRE(j.n_fresh >= 0 && j.n_fresh <= 65535 &&
                    (j.n_fresh == 0 || (j.fresh_frames && j.fresh_x && (!j.merged_out || j.fresh_merged))),
                "%s: job %d: bad fresh rows", api, i);
    FVS_REQUIRE(j.n_dev == 0 || (j.dev_x && (!j.merged_out || j.dev_merged)), "%s: job %d: null device tier", api, i);
    FVS_REQUIRE(j.n_dev == j.n_base || (j.host_chunks && j.chunk_frames > 0), "%s: job %d: host frames without a chunk table",
                api, i);
    for (const void* p : {j.prev_x, j.prev_merged, j.fresh_x, j.fresh_merged, j.dev_x, j.dev_merged,
                          (const void*)j.spa_x_out, (const void*)j.merged_out})
      FVS_REQUIRE(aligned16(p), "%s: job %d: row tensors must be 16-byte aligned", api, i);
    for (const void* p : {(const void*)j.picks, (const void*)j.prev_picks, (const void*)j.fresh_frames,
                          (const void*)j.host_chunks, (const void*)j.host_fetches})
      FVS_REQUIRE(aligned8(p), "%s: job %d: index tables must be 8-byte aligned", api, i);
    out.add(j.spa_x_out, size_t(j.n) * fx * 2, i);
    out.add(j.merged_out, size_t(j.n) * fm * 2, i);
    out.add(j.host_fetches, 8, i);
  }
  if (const int r = out.check(api)) return r;
  return gather_jobs(jobs, n_jobs, gather_dev, (cudaStream_t)stream);
}

int fvs_qwen_pick_plan_multi(const fvs_qwen_pick_plan_job* jobs, int n_jobs, fvs_stream_t stream) {
  const char* api = "fvs_qwen_pick_plan_multi";
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  Outputs out;
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_pick_plan_job& j = jobs[i];
    FVS_REQUIRE(j.n >= 0 && j.n <= 65535 && j.m >= 0 && j.m <= 65535 && j.n_frames >= 0,
                "%s: job %d: bad sizes (n=%d, m=%d, n_frames=%lld)", api, i, j.n, j.m, (long long)j.n_frames);
    FVS_REQUIRE((j.picks || j.n <= j.n_frames) && (j.prev_picks || j.m == 0),
                "%s: job %d: null picks or previous picks (null picks stand for frames 0..n-1, n <= n_frames)", api, i);
    FVS_REQUIRE(j.frames && j.count && (j.plan || j.n == 0), "%s: job %d: null frame bytes, plan or count", api, i);
    FVS_REQUIRE(j.stored > 0, "%s: job %d: stored must be > 0", api, i);
    FVS_REQUIRE(aligned8(j.picks) && aligned8(j.prev_picks) && aligned8(j.plan) && ((uintptr_t)j.count & 3) == 0 &&
                    aligned8(j.re_encodes),
                "%s: job %d: misaligned picks, plan, count or counter", api, i);
    out.add(j.frames, size_t(j.n_frames), i);
    out.add(j.plan, size_t(j.n) * 8, i);
    out.add(j.count, 4, i);
    out.add(j.re_encodes, 8, i);
  }
  if (const int r = out.check(api)) return r;
  const auto dev = [](const fvs_qwen_pick_plan_job& j, PlanJobDev& d) {
    d = PlanJobDev{(const long long*)j.picks, j.frames, (const long long*)j.prev_picks, (long long*)j.plan, (int*)j.count,
                   (unsigned long long*)j.re_encodes, (long long)j.n_frames, j.n, j.m, j.stored};
    return 1;
  };
  return run_jobs<PlanJobDev>(jobs, n_jobs, dev, [&](const auto& L) {
    pick_plan_kernel<std::decay_t<decltype(L)>::kJobs><<<L.n, 32, 0, (cudaStream_t)stream>>>(L);
    FVS_CHECK_LAUNCH("pick_plan_kernel");
    return FVS_OK;
  });
}

int fvs_qwen_pixel_gather_multi(const fvs_qwen_pixel_job* jobs, int n_jobs, int dtype, fvs_stream_t stream) {
  const char* api = "fvs_qwen_pixel_gather_multi";
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", api);
  const bool codes = jobs[0].table != nullptr;
  Outputs out;
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_pixel_job& j = jobs[i];
    FVS_REQUIRE(j.plan && j.out && j.n > 0 && j.n <= 65535 && (j.table != nullptr) == codes,
                "%s: job %d: need a plan, a table, an output and 0 < n <= 65535 (a table in every job or in none: code "
                "and row jobs do not mix)", api, i);
    FVS_REQUIRE(j.base >= 0 && j.base < j.n_frames && j.host_chunks && j.chunk_frames > 0,
                "%s: job %d: need 0 <= base < n_frames and a chunk table", api, i);
    if (codes)
      FVS_REQUIRE(j.frame_elems > 0 && j.frame_elems % 1176 == 0,
                  "%s: job %d: frame size %lld is not whole rows of 1176 codes", api, i, (long long)j.frame_elems);
    else
      FVS_REQUIRE(j.frame_elems > 0 && (j.frame_elems * 2) % 16 == 0,
                  "%s: job %d: frame size must be a multiple of 16 bytes", api, i);
    FVS_REQUIRE(aligned16(j.out) && aligned8(j.plan) && aligned8(j.host_chunks) && ((uintptr_t)j.table & 3) == 0,
                "%s: job %d: misaligned output or table", api, i);
    out.add(j.out, size_t(j.n) * j.frame_elems * 2, i);
  }
  if (const int r = out.check(api)) return r;
  const cudaStream_t st = (cudaStream_t)stream;
  if (!codes)      // the DAM gather with no device tier: frames below `base` have no pixel rows and read as zeros
    return gather_jobs(jobs, n_jobs, [](const fvs_qwen_pixel_job& j, GatherJobDev& d) {
      fvs_qwen_gather_job g{};
      g.picks = j.plan;
      g.n = j.n;
      g.n_frames = g.n_base = j.n_frames;
      g.n_dev = j.base;
      g.host_chunks = j.host_chunks;
      g.chunk_frames = j.chunk_frames;
      g.x_frame_elems = j.frame_elems;
      g.spa_x_out = j.out;
      return gather_dev(g, d);
    }, st);
  const auto dev = [](const fvs_qwen_pixel_job& j, CodesJobDev& d) {
    const long long words = j.frame_elems / 8;
    d = CodesJobDev{(const long long*)j.plan, (const uint2* const*)j.host_chunks, j.table, (uint4*)j.out,
                    (long long)j.n_frames, (long long)j.base, (long long)j.chunk_frames, words, frame_blocks(words)};
    return d.bx * j.n;
  };
  return run_jobs<CodesJobDev>(jobs, n_jobs, dev, [&](const auto& L) {
    constexpr int K = std::decay_t<decltype(L)>::kJobs;
    if (dtype == FVS_BF16) pixel_codes_gather_kernel<K, FVS_BF16><<<L.first[L.n], 256, 0, st>>>(L);
    else pixel_codes_gather_kernel<K, FVS_F16><<<L.first[L.n], 256, 0, st>>>(L);
    FVS_CHECK_LAUNCH("pixel_codes_gather_kernel");
    return FVS_OK;
  });
}

int fvs_qwen_bank_scatter_multi(const fvs_qwen_scatter_job* jobs, int n_jobs, int dtype, fvs_stream_t stream) {
  const char* api = "fvs_qwen_bank_scatter_multi";
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", api);
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_scatter_job& j = jobs[i];
    FVS_REQUIRE(j.plan && j.x_rows && j.n > 0 && j.n <= 65535, "%s: job %d: need a plan, x rows and 0 < n <= 65535", api, i);
    FVS_REQUIRE(j.n_frames > 0 && j.n_dev >= 0 && j.n_dev <= j.n_frames, "%s: job %d: need 0 <= n_dev <= n_frames", api, i);
    FVS_REQUIRE(j.x_frame_elems > 0 && j.merged_frame_elems >= 0 && (j.x_frame_elems * 2) % 16 == 0 &&
                    (j.merged_frame_elems * 2) % 16 == 0,
                "%s: job %d: frame sizes must be multiples of 16 bytes", api, i);
    FVS_REQUIRE(!j.merged_rows || j.merged_frame_elems > 0, "%s: job %d: merged rows without a merged bank", api, i);
    FVS_REQUIRE(j.n_dev == 0 || (j.dev_x && (!j.merged_rows || j.dev_merged)), "%s: job %d: null device tier", api, i);
    FVS_REQUIRE(j.n_dev == j.n_frames || (j.host_chunks && j.chunk_frames > 0), "%s: job %d: host frames without a chunk "
                "table", api, i);
    for (const void* p : {j.x_rows, j.merged_rows, (const void*)j.dev_x, (const void*)j.dev_merged})
      FVS_REQUIRE(aligned16(p), "%s: job %d: row tensors must be 16-byte aligned", api, i);
    FVS_REQUIRE(aligned8(j.plan) && aligned8(j.host_chunks), "%s: job %d: misaligned tables", api, i);
  }
  const auto dev = [](const fvs_qwen_scatter_job& s, ScatterJobDev& d) {
    const long long fx = s.x_frame_elems * 2 / 16, fm = s.merged_frame_elems * 2 / 16;
    d = ScatterJobDev{(const long long*)s.plan, (const uint4*)s.x_rows, (const uint4*)s.merged_rows, (uint4*)s.dev_x,
                      (uint4*)s.dev_merged, (uint4* const*)s.host_chunks, (long long)s.n_frames, (long long)s.n_dev,
                      (long long)s.chunk_frames, fx, fm, frame_blocks(fx + (s.merged_rows ? fm : 0))};
    return d.bx * s.n;
  };
  return run_jobs<ScatterJobDev>(jobs, n_jobs, dev, [&](const auto& L) {
    bank_scatter_kernel<std::decay_t<decltype(L)>::kJobs><<<L.first[L.n], 256, 0, (cudaStream_t)stream>>>(L);
    FVS_CHECK_LAUNCH("bank_scatter_kernel");
    return FVS_OK;
  });
}

int fvs_qwen_pixel_decode(const uint8_t* codes, int64_t rows, const float* table, int dtype, void* out,
                          fvs_stream_t stream) {
  const char* api = "fvs_qwen_pixel_decode";
  FVS_REQUIRE(codes && table && out, "%s: null pointer", api);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", api);
  FVS_REQUIRE(rows > 0, "%s: need rows > 0 (rows=%lld)", api, (long long)rows);
  FVS_REQUIRE(((uintptr_t)codes & 7) == 0 && aligned16(out) && ((uintptr_t)table & 3) == 0,
              "%s: codes must be 8-byte and out 16-byte aligned", api);
  const long long words = (long long)rows * kCodeWordsPerRow;
  long long blocks = (words + 4 * 256 - 1) / (4 * 256);
  if (blocks > 4096) blocks = 4096;
  if (dtype == FVS_BF16) {
    pixel_decode_kernel<FVS_BF16><<<int(blocks), 256, 0, (cudaStream_t)stream>>>((const uint2*)codes, table, words,
                                                                                   (uint4*)out);
  } else {
    pixel_decode_kernel<FVS_F16><<<int(blocks), 256, 0, (cudaStream_t)stream>>>((const uint2*)codes, table, words,
                                                                                  (uint4*)out);
  }
  FVS_CHECK_LAUNCH("pixel_decode_kernel");
  return FVS_OK;
}

}  // extern "C"
