// qwen_bank.cu — the DAM gather of the Qwen2-VL streaming step over a two-tier feature bank (DESIGN.md §3.13).
//
// Frames [0, n_dev) of the full-resolution bank (x) and of the PatchMerger bank (merged) are contiguous HBM rows; frames
// [n_dev, n_frames) live in pinned host chunks of chunk_frames frames each, laid out [x rows of the chunk | merged rows of
// the chunk] and read through their mapped device pointers.  The picks come from the retrieval kernels and stay on the
// device: the kernel resolves every pick itself, so the step needs no host round trip to know where its frames are.
#include <algorithm>
#include <vector>

#include "fvs_common.h"

namespace fvs {
namespace qwen {

// Every block copies a strided share of one pick's 16-byte words: x words first, then merged words.
// Sources, in order: the device tier, the same frame in the previous step's DAM (prev_x / prev_m), the host chunk.
// A pick outside [0, n_frames) writes zeros (the host validates nothing on the device's behalf).
// (bx, nbx, i): the block's share of pick i and the number of blocks per pick
__device__ __forceinline__ void dam_gather_body(
    unsigned bx, unsigned nbx, unsigned i_, const long long* __restrict__ picks, long long n_frames, const uint4* dev_x,
    const uint4* dev_m, long long n_dev, const uint4* const* __restrict__ chunks, long long chunk_frames,
    const long long* __restrict__ prev_picks, int m, const uint4* prev_x, const uint4* prev_m, long long fx, long long fm,
    uint4* out_x, uint4* out_m, unsigned long long* host_fetches) {
  __shared__ const uint4* src[2];
  const int i = i_;
  if (threadIdx.x == 0) {
    const long long p = picks[i];
    const uint4 *sx = nullptr, *sm = nullptr;
    if (p >= 0 && p < n_frames) {
      if (p < n_dev) {
        sx = dev_x + p * fx;
        sm = dev_m ? dev_m + p * fm : nullptr;
      } else {
        int j = 0;
        while (j < m && prev_picks[j] != p) ++j;
        if (j < m) {
          sx = prev_x + j * fx;
          sm = prev_m ? prev_m + j * fm : nullptr;
        } else {
          const long long q = p - n_dev, off = q % chunk_frames;
          const uint4* c = chunks[q / chunk_frames];
          sx = c + off * fx;
          sm = c + chunk_frames * fx + off * fm;
          if (bx == 0 && host_fetches) atomicAdd(host_fetches, 1ull);
        }
      }
    }
    src[0] = sx;
    src[1] = sm;
  }
  __syncthreads();
  const uint4 *sx = src[0], *sm = src[1];
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
}  // namespace qwen
}  // namespace fvs

using namespace fvs;
using namespace fvs::qwen;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

namespace {
constexpr int kGatherJobs = FVS_QWEN_MEM_JOBS_PER_LAUNCH;
struct GatherJobDev {
  const long long* picks;
  const uint4* dev_x;
  const uint4* dev_m;
  const uint4* const* chunks;
  const long long* prev_picks;
  const uint4* prev_x;
  const uint4* prev_m;
  uint4* out_x;
  uint4* out_m;
  unsigned long long* host_fetches;
  long long n_frames, n_dev, chunk_frames, fx, fm;
  int m, bx;
};
template <int kJobs>
struct GatherLaunch {
  GatherJobDev job[kJobs];
  int first[kJobs + 1];
  int n;
};
// one flat grid over the jobs (a single call is the one-job grid): job j's block b copies share b % bx of pick b / bx
template <int kJobs>
__global__ void __launch_bounds__(256) dam_gather_multi_kernel(const __grid_constant__ GatherLaunch<kJobs> L) {
  int j = 0;
  if constexpr (kJobs > 1)
    while (j + 1 < L.n && blockIdx.x >= unsigned(L.first[j + 1])) ++j;
  const GatherJobDev& J = L.job[j];
  const unsigned b = blockIdx.x - unsigned(L.first[j]), bx = J.bx;
  dam_gather_body(b % bx, bx, b / bx, J.picks, J.n_frames, J.dev_x, J.dev_m, J.n_dev, J.chunks, J.chunk_frames, J.prev_picks,
                  J.m, J.prev_x, J.prev_m, J.fx, J.fm, J.out_x, J.out_m, J.host_fetches);
}

GatherJobDev gather_job_dev(const fvs_qwen_gather_job& j) {
  const long long fx = j.x_frame_elems * 2 / 16, fm = j.merged_frame_elems * 2 / 16;
  const long long words = (j.spa_x_out ? fx : 0) + (j.merged_out ? fm : 0);
  long long bx = (words + 4 * 256 - 1) / (4 * 256);
  if (bx > 64) bx = 64;
  if (bx < 1) bx = 1;
  return GatherJobDev{(const long long*)j.picks, (const uint4*)j.dev_x, (const uint4*)j.dev_merged,
                      (const uint4* const*)j.host_chunks, (const long long*)j.prev_picks, (const uint4*)j.prev_x,
                      (const uint4*)j.prev_merged, (uint4*)j.spa_x_out, (uint4*)j.merged_out,
                      (unsigned long long*)j.host_fetches, (long long)j.n_frames, (long long)j.n_dev,
                      (long long)j.chunk_frames, fx, fm, j.m, int(bx)};
}

template <int kJobs>
int dam_gather_launch(const fvs_qwen_gather_job* jobs, int n, cudaStream_t stream) {
  GatherLaunch<kJobs> L;
  L.n = n;
  L.first[0] = 0;
  for (int q = 0; q < n; ++q) {
    L.job[q] = gather_job_dev(jobs[q]);
    L.first[q + 1] = L.first[q] + L.job[q].bx * jobs[q].n;
  }
  dam_gather_multi_kernel<kJobs><<<L.first[n], 256, 0, stream>>>(L);
  FVS_CHECK_LAUNCH("dam_gather_multi_kernel");
  return FVS_OK;
}

// the checks of fvs_qwen_dam_gather for every job, then (multi) no output shared by two jobs, then one flat grid per
// kGatherJobs jobs (a single call: the one-job grid)
int dam_gather_jobs(const char* api, const fvs_qwen_gather_job* jobs, int n_jobs, int dtype, cudaStream_t stream, bool multi) {
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", api);
  struct Range { uintptr_t lo, hi; int job; };
  std::vector<Range> out;
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_gather_job& j = jobs[i];
    const int n = j.n, m = j.m;
    const int64_t n_frames = j.n_frames, n_dev = j.n_dev, x_frame_elems = j.x_frame_elems,
                  merged_frame_elems = j.merged_frame_elems;
    FVS_REQUIRE(j.picks, "%s: null picks", api);
    FVS_REQUIRE(n > 0 && n <= 65535, "%s: need 0 < n <= 65535 picks (n=%d)", api, n);
    FVS_REQUIRE(j.spa_x_out || j.merged_out, "%s: no output", api);
    FVS_REQUIRE(n_frames > 0 && n_dev >= 0 && n_dev <= n_frames, "%s: need 0 <= n_dev <= n_frames, n_frames > 0 (%lld, %lld)",
                api, (long long)n_dev, (long long)n_frames);
    FVS_REQUIRE(x_frame_elems > 0 && merged_frame_elems >= 0, "%s: bad frame sizes", api);
    FVS_REQUIRE((x_frame_elems * 2) % 16 == 0 && (merged_frame_elems * 2) % 16 == 0,
                "%s: frame sizes must be multiples of 16 bytes", api);
    FVS_REQUIRE(!j.merged_out || merged_frame_elems > 0, "%s: merged_out without merged rows", api);
    FVS_REQUIRE(n_dev == 0 || (j.dev_x && (!j.merged_out || j.dev_merged)), "%s: null device tier", api);
    FVS_REQUIRE(n_dev == n_frames || (j.host_chunks && j.chunk_frames > 0), "%s: host frames without a chunk table", api);
    FVS_REQUIRE(m >= 0 && (m == 0 || (j.prev_picks && j.prev_x && (!j.merged_out || j.prev_merged))), "%s: bad previous DAM",
                api);
    for (const void* p : {j.dev_x, j.dev_merged, j.prev_x, j.prev_merged, (const void*)j.spa_x_out, (const void*)j.merged_out})
      FVS_REQUIRE(aligned16(p), "%s: row tensors must be 16-byte aligned", api);
    FVS_REQUIRE(((uintptr_t)j.picks & 7) == 0 && ((uintptr_t)j.prev_picks & 7) == 0 && ((uintptr_t)j.host_chunks & 7) == 0,
                "%s: index tables must be 8-byte aligned", api);
    if (multi) {
      if (j.spa_x_out) out.push_back({uintptr_t(j.spa_x_out), uintptr_t(j.spa_x_out) + size_t(n) * x_frame_elems * 2, i});
      if (j.merged_out)
        out.push_back({uintptr_t(j.merged_out), uintptr_t(j.merged_out) + size_t(n) * merged_frame_elems * 2, i});
      if (j.host_fetches) out.push_back({uintptr_t(j.host_fetches), uintptr_t(j.host_fetches) + 8, i});
    }
  }
  for (size_t a = 0; a < out.size(); ++a)
    for (size_t b = a + 1; b < out.size(); ++b)
      FVS_REQUIRE(out[a].job == out[b].job || out[a].hi <= out[b].lo || out[b].hi <= out[a].lo,
                  "%s: jobs %d and %d share an output", api, out[a].job, out[b].job);
  for (int i0 = 0; i0 < n_jobs; i0 += kGatherJobs) {
    const int n = std::min(kGatherJobs, n_jobs - i0);
    const int r = n == 1 ? dam_gather_launch<1>(jobs + i0, 1, stream) : dam_gather_launch<kGatherJobs>(jobs + i0, n, stream);
    if (r) return r;
  }
  return FVS_OK;
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

int fvs_qwen_dam_gather(const int64_t* picks, int n, int64_t n_frames, const void* dev_x, const void* dev_merged,
                        int64_t n_dev, const void* const* host_chunks, int chunk_frames, const int64_t* prev_picks, int m,
                        const void* prev_x, const void* prev_merged, int64_t x_frame_elems, int64_t merged_frame_elems,
                        int dtype, void* spa_x_out, void* merged_out, uint64_t* host_fetches, fvs_stream_t stream) {
  const fvs_qwen_gather_job j{picks, n, n_frames, dev_x, dev_merged, n_dev, host_chunks, chunk_frames, prev_picks, m,
                              prev_x, prev_merged, x_frame_elems, merged_frame_elems, spa_x_out, merged_out, host_fetches};
  return dam_gather_jobs("fvs_qwen_dam_gather", &j, 1, dtype, (cudaStream_t)stream, false);
}

int fvs_qwen_dam_gather_multi(const fvs_qwen_gather_job* jobs_h, int n_jobs, int dtype, fvs_stream_t stream) {
  return dam_gather_jobs("fvs_qwen_dam_gather_multi", jobs_h, n_jobs, dtype, (cudaStream_t)stream, true);
}

}  // extern "C"
