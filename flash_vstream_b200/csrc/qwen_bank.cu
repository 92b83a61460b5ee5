// qwen_bank.cu — the DAM gather of the Qwen2-VL streaming step over a two-tier feature bank (DESIGN.md §3.13).
//
// Frames [0, n_dev) of the full-resolution bank (x) and of the PatchMerger bank (merged) are contiguous HBM rows; frames
// [n_dev, n_frames) live in pinned host chunks of chunk_frames frames each, laid out [x rows of the chunk | merged rows of
// the chunk] and read through their mapped device pointers.  The picks come from the retrieval kernels and stay on the
// device: the kernel resolves every pick itself, so the step needs no host round trip to know where its frames are.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
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
        sx = dev_x ? dev_x + p * fx : nullptr;      // no device tier (the pixel store): zeros
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
  gather_copy(bx, nbx, i, src[0], src[1], fx, fm, out_x, out_m);
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

// ---- lazy full-resolution bank (DESIGN.md §3.18) --------------------------------------------------------------------
// Pick plan: one warp per job walks the picks in order, 32 at a time.  A pick is planned when it is in range, its frame's
// mask bit is clear and no earlier pick names the same frame; the warp's ballot compacts the planned frames in pick order.
// The mask bit of a planned frame is set by the lane that planned it; a later pick of that frame is never planned again,
// whether or not it sees the bit, because it is not the first pick of its frame.
struct PlanJobDev {
  const long long* picks;
  unsigned char* encoded;
  long long* plan;
  int* count;
  long long n_frames;
  int n;
};
template <int kJobs>
struct PlanLaunch {
  PlanJobDev job[kJobs];
};
template <int kJobs>
__global__ void __launch_bounds__(32) pick_plan_kernel(const __grid_constant__ PlanLaunch<kJobs> L) {
  const PlanJobDev& J = L.job[blockIdx.x];
  const unsigned lane = threadIdx.x;
  int base = 0;
  for (int i0 = 0; i0 < J.n; i0 += 32) {
    const int i = i0 + int(lane);
    long long p = -1;
    bool first = false;
    if (i < J.n) {
      p = J.picks ? J.picks[i] : i;
      first = p >= 0 && p < J.n_frames && !J.encoded[p];
      if (first && J.picks)
        for (int j = 0; j < i; ++j)
          if (J.picks[j] == p) { first = false; break; }
    }
    const unsigned ball = __ballot_sync(0xffffffffu, first);
    if (first) {
      J.plan[base + __popc(ball & ((1u << lane) - 1u))] = p;
      J.encoded[p] = 1;
    }
    base += __popc(ball);
  }
  if (lane == 0) *J.count = base;
}

template <int kJobs>
int pick_plan_launch(const fvs_qwen_pick_plan_job* jobs, int n, cudaStream_t stream) {
  PlanLaunch<kJobs> L;
  for (int q = 0; q < n; ++q)
    L.job[q] = PlanJobDev{(const long long*)jobs[q].picks, jobs[q].encoded, (long long*)jobs[q].plan, (int*)jobs[q].count,
                          (long long)jobs[q].n_frames, jobs[q].n};
  pick_plan_kernel<kJobs><<<n, 32, 0, stream>>>(L);
  FVS_CHECK_LAUNCH("pick_plan_kernel");
  return FVS_OK;
}

// Bank scatter: the reverse of the DAM gather without its previous-DAM source.  Job j's block b writes share b % bx of
// planned frame b / bx: x words first, then merged words, to the device tier or the frame's host chunk.
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
struct ScatterLaunch {
  ScatterJobDev job[kJobs];
  int first[kJobs + 1];
  int n;
};
template <int kJobs>
__global__ void __launch_bounds__(256) bank_scatter_kernel(const __grid_constant__ ScatterLaunch<kJobs> L) {
  int j = 0;
  if constexpr (kJobs > 1)
    while (j + 1 < L.n && blockIdx.x >= unsigned(L.first[j + 1])) ++j;
  const ScatterJobDev& J = L.job[j];
  const unsigned b = blockIdx.x - unsigned(L.first[j]), bx = b % unsigned(J.bx);
  const long long i = b / unsigned(J.bx);
  __shared__ uint4* dst[2];
  if (threadIdx.x == 0) {
    const long long p = J.plan[i];
    uint4 *dx = nullptr, *dm = nullptr;
    if (p >= 0 && p < J.n_frames) {
      if (p < J.n_dev) {
        dx = J.dev_x + p * J.fx;
        dm = J.dev_m ? J.dev_m + p * J.fm : nullptr;
      } else {
        const long long q = p - J.n_dev, off = q % J.chunk_frames;
        uint4* c = J.chunks[q / J.chunk_frames];
        dx = c + off * J.fx;
        dm = c + J.chunk_frames * J.fx + off * J.fm;
      }
    }
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

template <int kJobs>
int bank_scatter_launch(const fvs_qwen_scatter_job* jobs, int n, cudaStream_t stream) {
  ScatterLaunch<kJobs> L;
  L.n = n;
  L.first[0] = 0;
  for (int q = 0; q < n; ++q) {
    const fvs_qwen_scatter_job& s = jobs[q];
    const long long fx = s.x_frame_elems * 2 / 16, fm = s.merged_frame_elems * 2 / 16;
    long long bx = (fx + (s.merged_rows ? fm : 0) + 4 * 256 - 1) / (4 * 256);
    bx = bx > 64 ? 64 : bx < 1 ? 1 : bx;
    L.job[q] = ScatterJobDev{(const long long*)s.plan, (const uint4*)s.x_rows, (const uint4*)s.merged_rows, (uint4*)s.dev_x,
                             (uint4*)s.dev_merged, (uint4* const*)s.host_chunks, (long long)s.n_frames, (long long)s.n_dev,
                             (long long)s.chunk_frames, fx, fm, int(bx)};
    L.first[q + 1] = L.first[q] + int(bx) * s.n;
  }
  bank_scatter_kernel<kJobs><<<L.first[n], 256, 0, stream>>>(L);
  FVS_CHECK_LAUNCH("bank_scatter_kernel");
  return FVS_OK;
}

// ---- no full-resolution bank (DESIGN.md §3.19) ------------------------------------------------------------------------
// Pick plan against the previous DAM: the pick_plan_kernel walk, with "held" meaning "in prev_picks, or byte 2 (stored
// in the base bank)".  The plan reads prev_picks instead of a per-frame "in the previous DAM" mask, so nothing has to
// move a mask from the old picks to the new ones after the gather, and a clip that complete() redoes plans against the
// same previous DAM with nothing to undo.  The frame bytes only count re-encodes (0 -> 1 on a first encode), and only
// the lane that plans a frame (its first pick) writes its byte, so the walk stays race-free.
struct PlanPrevJobDev {
  const long long* picks;
  unsigned char* frames;
  const long long* prev;
  long long* plan;
  int* count;
  unsigned long long* re_encodes;
  long long n_frames;
  int n, m;
};
template <int kJobs>
struct PlanPrevLaunch {
  PlanPrevJobDev job[kJobs];
};
template <int kJobs>
__global__ void __launch_bounds__(32) pick_plan_prev_kernel(const __grid_constant__ PlanPrevLaunch<kJobs> L) {
  const PlanPrevJobDev& J = L.job[blockIdx.x];
  const unsigned lane = threadIdx.x;
  int base = 0, again = 0;
  for (int i0 = 0; i0 < J.n; i0 += 32) {
    const int i = i0 + int(lane);
    long long p = -1;
    bool first = false;
    if (i < J.n) {
      p = J.picks[i];
      first = p >= 0 && p < J.n_frames && J.frames[p] != 2;
      for (int j = 0; first && j < J.m; ++j)
        if (J.prev[j] == p) first = false;
      for (int j = 0; first && j < i; ++j)
        if (J.picks[j] == p) first = false;
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

template <int kJobs>
int pick_plan_prev_launch(const fvs_qwen_pick_plan_prev_job* jobs, int n, cudaStream_t stream) {
  PlanPrevLaunch<kJobs> L;
  for (int q = 0; q < n; ++q) {
    const fvs_qwen_pick_plan_prev_job& j = jobs[q];
    L.job[q] = PlanPrevJobDev{(const long long*)j.picks, j.frames, (const long long*)j.prev_picks, (long long*)j.plan,
                              (int*)j.count, (unsigned long long*)j.re_encodes, (long long)j.n_frames, j.n, j.m};
  }
  pick_plan_prev_kernel<kJobs><<<n, 32, 0, stream>>>(L);
  FVS_CHECK_LAUNCH("pick_plan_prev_kernel");
  return FVS_OK;
}

// Gather without a bank: dam_gather_body with the sources in the order previous DAM, fresh rows, stored base bank.  The
// base comes last because a frame a lazy stream had not yet encoded when its checkpoint was taken has a zero slot there
// (frame byte 0): such a frame is always planned, so it is found among the fresh rows first.
struct FreshJobDev {
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
struct FreshLaunch {
  FreshJobDev job[kJobs];
  int first[kJobs + 1];
  int n;
};
template <int kJobs>
__global__ void __launch_bounds__(256) fresh_gather_kernel(const __grid_constant__ FreshLaunch<kJobs> L) {
  int j = 0;
  if constexpr (kJobs > 1)
    while (j + 1 < L.n && blockIdx.x >= unsigned(L.first[j + 1])) ++j;
  const FreshJobDev& J = L.job[j];
  const unsigned b = blockIdx.x - unsigned(L.first[j]), bx = b % unsigned(J.bx);
  const int i = int(b / unsigned(J.bx));
  __shared__ const uint4* src[2];
  if (threadIdx.x == 0) {
    const long long p = J.picks[i];
    const uint4 *sx = nullptr, *sm = nullptr;
    if (p >= 0 && p < J.n_frames) {
      int k = 0;
      while (k < J.m && J.prev_picks[k] != p) ++k;
      if (k < J.m) {
        sx = J.prev_x + k * J.fx;
        sm = J.prev_m ? J.prev_m + k * J.fm : nullptr;
      } else {
        k = 0;
        while (k < J.n_fresh && J.fresh[k] != p) ++k;
        if (k < J.n_fresh) {
          sx = J.fresh_x + k * J.fx;
          sm = J.fresh_m ? J.fresh_m + k * J.fm : nullptr;
        } else if (p < J.n_dev) {
          sx = J.dev_x + p * J.fx;
          sm = J.dev_m ? J.dev_m + p * J.fm : nullptr;
        } else if (p < J.n_base) {
          const long long q = p - J.n_dev, off = q % J.chunk_frames;
          const uint4* c = J.chunks[q / J.chunk_frames];
          sx = c + off * J.fx;
          sm = c + J.chunk_frames * J.fx + off * J.fm;
          if (bx == 0 && J.host_fetches) atomicAdd(J.host_fetches, 1ull);
        }
      }
    }
    src[0] = sx;
    src[1] = sm;
  }
  __syncthreads();
  gather_copy(bx, J.bx, i, src[0], src[1], J.fx, J.fm, J.out_x, J.out_m);
}

template <int kJobs>
int fresh_gather_launch(const fvs_qwen_fresh_gather_job* jobs, int n, cudaStream_t stream) {
  FreshLaunch<kJobs> L;
  L.n = n;
  L.first[0] = 0;
  for (int q = 0; q < n; ++q) {
    const fvs_qwen_fresh_gather_job& g = jobs[q];
    const long long fx = g.x_frame_elems * 2 / 16, fm = g.merged_frame_elems * 2 / 16;
    long long bx = ((g.spa_x_out ? fx : 0) + (g.merged_out ? fm : 0) + 4 * 256 - 1) / (4 * 256);
    bx = bx > 64 ? 64 : bx < 1 ? 1 : bx;
    L.job[q] = FreshJobDev{(const long long*)g.picks, (const long long*)g.prev_picks, (const uint4*)g.prev_x,
                           (const uint4*)g.prev_merged, (const long long*)g.fresh_frames, (const uint4*)g.fresh_x,
                           (const uint4*)g.fresh_merged, (const uint4*)g.dev_x, (const uint4*)g.dev_merged,
                           (const uint4* const*)g.host_chunks, (uint4*)g.spa_x_out, (uint4*)g.merged_out,
                           (unsigned long long*)g.host_fetches, (long long)g.n_frames, (long long)g.n_base,
                           (long long)g.n_dev, (long long)g.chunk_frames, fx, fm, g.m, g.n_fresh, int(bx)};
    L.first[q + 1] = L.first[q] + int(bx) * g.n;
  }
  fresh_gather_kernel<kJobs><<<L.first[n], 256, 0, stream>>>(L);
  FVS_CHECK_LAUNCH("fresh_gather_kernel");
  return FVS_OK;
}

// ---- 8-bit pixel codes (DESIGN.md §3.20) -------------------------------------------------------------------------------
// A code row holds the resampled bytes u of one full-resolution pixel row, columns ((c*2 + tp)*14 + py)*14 + px; the
// tower reads dtype(table[c][u]).  392 = 2*14*14 columns per channel is a multiple of 8, so the 8 codes of one 8-byte
// word share a channel: word w of a row (147 words) is channel (w % 147) / 49.
constexpr long long kCodeWordsPerRow = 1176 / 8, kCodeWordsPerChannel = 392 / 8;
constexpr int kCodeJobs = FVS_QWEN_MEM_JOBS_PER_LAUNCH;

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

// The job table of the pixel gather over code chunks: job j's block b decodes share b % bx of planned frame b / bx,
// read in place from its pinned chunk; a frame outside [base, n_frames) yields zeros.
struct CodesJobDev {
  const long long* plan;
  const uint8_t* const* chunks;
  const float* table;
  uint4* out;
  long long n_frames, base, chunk_frames, words;    // words: 8-byte code words per frame
  int bx;
};
template <int kJobs>
struct CodesLaunch {
  CodesJobDev job[kJobs];
  int first[kJobs + 1];
  int n;
};
template <int kJobs, int kDtype>
__global__ void __launch_bounds__(256) pixel_codes_gather_kernel(const __grid_constant__ CodesLaunch<kJobs> L) {
  int j = 0;
  if constexpr (kJobs > 1)
    while (j + 1 < L.n && blockIdx.x >= unsigned(L.first[j + 1])) ++j;
  const CodesJobDev& J = L.job[j];
  const unsigned b = blockIdx.x - unsigned(L.first[j]), bx = b % unsigned(J.bx);
  const long long i = b / unsigned(J.bx);
  __shared__ float lut[3 * 256];
  __shared__ const uint2* src;
  if (threadIdx.x == 0) {
    const long long p = J.plan[i];
    const uint2* s = nullptr;
    if (p >= J.base && p < J.n_frames) {
      const long long q = p - J.base;
      s = reinterpret_cast<const uint2*>(J.chunks[q / J.chunk_frames]) + (q % J.chunk_frames) * J.words;
    }
    src = s;
  }
  load_lut(lut, J.table);
  decode_words<kDtype>(src, J.out + i * J.words, (long long)bx * blockDim.x + threadIdx.x, J.words,
                       (long long)J.bx * blockDim.x, lut);
}

template <int kJobs, int kDtype>
int codes_gather_launch(const fvs_qwen_pixel_codes_job* jobs, int n, cudaStream_t stream) {
  CodesLaunch<kJobs> L;
  L.n = n;
  L.first[0] = 0;
  for (int q = 0; q < n; ++q) {
    const fvs_qwen_pixel_codes_job& g = jobs[q];
    const long long words = g.frame_elems / 8;
    long long bx = (words + 4 * 256 - 1) / (4 * 256);
    bx = bx > 64 ? 64 : bx < 1 ? 1 : bx;
    L.job[q] = CodesJobDev{(const long long*)g.plan, (const uint8_t* const*)g.host_chunks, g.table, (uint4*)g.out,
                           (long long)g.n_frames, (long long)g.base, (long long)g.chunk_frames, words, int(bx)};
    L.first[q + 1] = L.first[q] + int(bx) * g.n;
  }
  pixel_codes_gather_kernel<kJobs, kDtype><<<L.first[n], 256, 0, stream>>>(L);
  FVS_CHECK_LAUNCH("pixel_codes_gather_kernel");
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

int fvs_qwen_pick_plan_multi(const fvs_qwen_pick_plan_job* jobs, int n_jobs, fvs_stream_t stream) {
  const char* api = "fvs_qwen_pick_plan_multi";
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_pick_plan_job& j = jobs[i];
    FVS_REQUIRE(j.n >= 0 && j.n_frames >= 0 && (j.picks || j.n <= j.n_frames), "%s: job %d: bad sizes (n=%d, n_frames=%lld)",
                api, i, j.n, (long long)j.n_frames);
    FVS_REQUIRE(j.encoded && j.count && (j.plan || j.n == 0), "%s: job %d: null mask, plan or count", api, i);
    FVS_REQUIRE(((uintptr_t)j.picks & 7) == 0 && ((uintptr_t)j.plan & 7) == 0 && ((uintptr_t)j.count & 3) == 0,
                "%s: job %d: misaligned picks, plan or count", api, i);
    for (int k = 0; k < i; ++k)
      FVS_REQUIRE(jobs[k].encoded != j.encoded && jobs[k].count != j.count && (j.n == 0 || jobs[k].plan != j.plan),
                  "%s: jobs %d and %d share an output", api, k, i);
  }
  for (int i0 = 0; i0 < n_jobs; i0 += kGatherJobs) {
    const int n = std::min(kGatherJobs, n_jobs - i0);
    const int r = n == 1 ? pick_plan_launch<1>(jobs + i0, 1, (cudaStream_t)stream)
                         : pick_plan_launch<kGatherJobs>(jobs + i0, n, (cudaStream_t)stream);
    if (r) return r;
  }
  return FVS_OK;
}

int fvs_qwen_pixel_gather_multi(const fvs_qwen_pixel_job* jobs, int n_jobs, int dtype, fvs_stream_t stream) {
  const char* api = "fvs_qwen_pixel_gather_multi";
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", api);
  std::vector<fvs_qwen_gather_job> g(n_jobs);
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_pixel_job& j = jobs[i];
    FVS_REQUIRE(j.plan && j.out && j.n > 0 && j.n <= 65535, "%s: job %d: need a plan, an output and 0 < n <= 65535", api, i);
    FVS_REQUIRE(j.base >= 0 && j.base < j.n_frames && j.host_chunks && j.chunk_frames > 0,
                "%s: job %d: need 0 <= base < n_frames and a chunk table", api, i);
    FVS_REQUIRE(j.frame_elems > 0 && (j.frame_elems * 2) % 16 == 0, "%s: job %d: frame size must be a multiple of 16 bytes",
                api, i);
    FVS_REQUIRE(aligned16(j.out) && ((uintptr_t)j.plan & 7) == 0 && ((uintptr_t)j.host_chunks & 7) == 0,
                "%s: job %d: misaligned output or table", api, i);
    // the DAM gather with no device tier: frames below `base` have no pixel rows and read as zeros
    g[i] = fvs_qwen_gather_job{j.plan, j.n, j.n_frames, nullptr, nullptr, j.base, j.host_chunks, j.chunk_frames, nullptr,
                               0, nullptr, nullptr, j.frame_elems, 0, j.out, nullptr, nullptr};
    for (int k = 0; k < i; ++k) {
      const uintptr_t a = uintptr_t(jobs[k].out), ae = a + size_t(jobs[k].n) * jobs[k].frame_elems * 2;
      const uintptr_t b = uintptr_t(j.out), be = b + size_t(j.n) * j.frame_elems * 2;
      FVS_REQUIRE(ae <= b || be <= a, "%s: jobs %d and %d share an output", api, k, i);
    }
  }
  for (int i0 = 0; i0 < n_jobs; i0 += kGatherJobs) {
    const int n = std::min(kGatherJobs, n_jobs - i0);
    const int r = n == 1 ? dam_gather_launch<1>(g.data() + i0, 1, (cudaStream_t)stream)
                         : dam_gather_launch<kGatherJobs>(g.data() + i0, n, (cudaStream_t)stream);
    if (r) return r;
  }
  return FVS_OK;
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
    FVS_REQUIRE(((uintptr_t)j.plan & 7) == 0 && ((uintptr_t)j.host_chunks & 7) == 0, "%s: job %d: misaligned tables", api, i);
  }
  for (int i0 = 0; i0 < n_jobs; i0 += kGatherJobs) {
    const int n = std::min(kGatherJobs, n_jobs - i0);
    const int r = n == 1 ? bank_scatter_launch<1>(jobs + i0, 1, (cudaStream_t)stream)
                         : bank_scatter_launch<kGatherJobs>(jobs + i0, n, (cudaStream_t)stream);
    if (r) return r;
  }
  return FVS_OK;
}

int fvs_qwen_pick_plan_prev_multi(const fvs_qwen_pick_plan_prev_job* jobs, int n_jobs, fvs_stream_t stream) {
  const char* api = "fvs_qwen_pick_plan_prev_multi";
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_pick_plan_prev_job& j = jobs[i];
    FVS_REQUIRE(j.n >= 0 && j.n <= 65535 && j.m >= 0 && j.m <= 65535 && j.n_frames >= 0,
                "%s: job %d: bad sizes (n=%d, m=%d, n_frames=%lld)", api, i, j.n, j.m, (long long)j.n_frames);
    FVS_REQUIRE((j.picks || j.n == 0) && (j.prev_picks || j.m == 0), "%s: job %d: null picks or previous picks", api, i);
    FVS_REQUIRE(j.frames && j.count && (j.plan || j.n == 0), "%s: job %d: null frame bytes, plan or count", api, i);
    FVS_REQUIRE(((uintptr_t)j.picks & 7) == 0 && ((uintptr_t)j.prev_picks & 7) == 0 && ((uintptr_t)j.plan & 7) == 0 &&
                    ((uintptr_t)j.count & 3) == 0 && ((uintptr_t)j.re_encodes & 7) == 0,
                "%s: job %d: misaligned picks, plan, count or counter", api, i);
    for (int k = 0; k < i; ++k)
      FVS_REQUIRE(jobs[k].frames != j.frames && jobs[k].count != j.count && (j.n == 0 || jobs[k].plan != j.plan) &&
                      (!j.re_encodes || jobs[k].re_encodes != j.re_encodes),
                  "%s: jobs %d and %d share an output", api, k, i);
  }
  for (int i0 = 0; i0 < n_jobs; i0 += kGatherJobs) {
    const int n = std::min(kGatherJobs, n_jobs - i0);
    const int r = n == 1 ? pick_plan_prev_launch<1>(jobs + i0, 1, (cudaStream_t)stream)
                         : pick_plan_prev_launch<kGatherJobs>(jobs + i0, n, (cudaStream_t)stream);
    if (r) return r;
  }
  return FVS_OK;
}

int fvs_qwen_dam_gather_fresh_multi(const fvs_qwen_fresh_gather_job* jobs, int n_jobs, int dtype, fvs_stream_t stream) {
  const char* api = "fvs_qwen_dam_gather_fresh_multi";
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", api);
  struct Range { uintptr_t lo, hi; int job; };
  std::vector<Range> out;
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_fresh_gather_job& j = jobs[i];
    const int64_t fx = j.x_frame_elems, fm = j.merged_frame_elems;
    FVS_REQUIRE(j.picks && j.n > 0 && j.n <= 65535, "%s: job %d: need picks and 0 < n <= 65535", api, i);
    FVS_REQUIRE(j.spa_x_out || j.merged_out, "%s: job %d: no output", api, i);
    FVS_REQUIRE(j.n_frames > 0 && j.n_dev >= 0 && j.n_dev <= j.n_base && j.n_base <= j.n_frames,
                "%s: job %d: need 0 <= n_dev <= n_base <= n_frames, n_frames > 0", api, i);
    FVS_REQUIRE(fx > 0 && fm >= 0 && (fx * 2) % 16 == 0 && (fm * 2) % 16 == 0,
                "%s: job %d: frame sizes must be multiples of 16 bytes", api, i);
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
    FVS_REQUIRE(((uintptr_t)j.picks & 7) == 0 && ((uintptr_t)j.prev_picks & 7) == 0 &&
                    ((uintptr_t)j.fresh_frames & 7) == 0 && ((uintptr_t)j.host_chunks & 7) == 0 &&
                    ((uintptr_t)j.host_fetches & 7) == 0,
                "%s: job %d: index tables must be 8-byte aligned", api, i);
    if (j.spa_x_out) out.push_back({uintptr_t(j.spa_x_out), uintptr_t(j.spa_x_out) + size_t(j.n) * fx * 2, i});
    if (j.merged_out) out.push_back({uintptr_t(j.merged_out), uintptr_t(j.merged_out) + size_t(j.n) * fm * 2, i});
    if (j.host_fetches) out.push_back({uintptr_t(j.host_fetches), uintptr_t(j.host_fetches) + 8, i});
  }
  for (size_t a = 0; a < out.size(); ++a)
    for (size_t b = a + 1; b < out.size(); ++b)
      FVS_REQUIRE(out[a].job == out[b].job || out[a].hi <= out[b].lo || out[b].hi <= out[a].lo,
                  "%s: jobs %d and %d share an output", api, out[a].job, out[b].job);
  for (int i0 = 0; i0 < n_jobs; i0 += kGatherJobs) {
    const int n = std::min(kGatherJobs, n_jobs - i0);
    const int r = n == 1 ? fresh_gather_launch<1>(jobs + i0, 1, (cudaStream_t)stream)
                         : fresh_gather_launch<kGatherJobs>(jobs + i0, n, (cudaStream_t)stream);
    if (r) return r;
  }
  return FVS_OK;
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

int fvs_qwen_pixel_gather_codes_multi(const fvs_qwen_pixel_codes_job* jobs, int n_jobs, int dtype, fvs_stream_t stream) {
  const char* api = "fvs_qwen_pixel_gather_codes_multi";
  FVS_REQUIRE(jobs && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", api);
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_pixel_codes_job& j = jobs[i];
    FVS_REQUIRE(j.plan && j.out && j.table && j.n > 0 && j.n <= 65535,
                "%s: job %d: need a plan, a table, an output and 0 < n <= 65535", api, i);
    FVS_REQUIRE(j.base >= 0 && j.base < j.n_frames && j.host_chunks && j.chunk_frames > 0,
                "%s: job %d: need 0 <= base < n_frames and a chunk table", api, i);
    FVS_REQUIRE(j.frame_elems > 0 && j.frame_elems % 1176 == 0, "%s: job %d: frame size %lld is not whole rows of 1176 "
                "codes", api, i, (long long)j.frame_elems);
    FVS_REQUIRE(aligned16(j.out) && ((uintptr_t)j.plan & 7) == 0 && ((uintptr_t)j.host_chunks & 7) == 0 &&
                    ((uintptr_t)j.table & 3) == 0,
                "%s: job %d: misaligned output or table", api, i);
    for (int k = 0; k < i; ++k) {
      const uintptr_t a = uintptr_t(jobs[k].out), ae = a + size_t(jobs[k].n) * jobs[k].frame_elems * 2;
      const uintptr_t b = uintptr_t(j.out), be = b + size_t(j.n) * j.frame_elems * 2;
      FVS_REQUIRE(ae <= b || be <= a, "%s: jobs %d and %d share an output", api, k, i);
    }
  }
  for (int i0 = 0; i0 < n_jobs; i0 += kCodeJobs) {
    const int n = std::min(kCodeJobs, n_jobs - i0);
    const cudaStream_t st = (cudaStream_t)stream;
    int r;
    if (dtype == FVS_BF16)
      r = n == 1 ? codes_gather_launch<1, FVS_BF16>(jobs + i0, 1, st) : codes_gather_launch<kCodeJobs, FVS_BF16>(jobs + i0, n, st);
    else
      r = n == 1 ? codes_gather_launch<1, FVS_F16>(jobs + i0, 1, st) : codes_gather_launch<kCodeJobs, FVS_F16>(jobs + i0, n, st);
    if (r) return r;
  }
  return FVS_OK;
}

}  // extern "C"
