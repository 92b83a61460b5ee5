// qwen_bank.cu — the DAM gather of the Qwen2-VL streaming step over a two-tier feature bank (DESIGN.md §3.13).
//
// Frames [0, n_dev) of the full-resolution bank (x) and of the PatchMerger bank (merged) are contiguous HBM rows; frames
// [n_dev, n_frames) live in pinned host chunks of chunk_frames frames each, laid out [x rows of the chunk | merged rows of
// the chunk] and read through their mapped device pointers.  The picks come from the retrieval kernels and stay on the
// device: the kernel resolves every pick itself, so the step needs no host round trip to know where its frames are.
#include "fvs_common.h"

namespace fvs {
namespace qwen {

// gridDim.y = picks; every block copies a strided share of the pick's 16-byte words: x words first, then merged words.
// Sources, in order: the device tier, the same frame in the previous step's DAM (prev_x / prev_m), the host chunk.
// A pick outside [0, n_frames) writes zeros (the host validates nothing on the device's behalf).
__global__ void __launch_bounds__(256) dam_gather_kernel(
    const long long* __restrict__ picks, long long n_frames, const uint4* dev_x, const uint4* dev_m, long long n_dev,
    const uint4* const* __restrict__ chunks, long long chunk_frames, const long long* __restrict__ prev_picks, int m,
    const uint4* prev_x, const uint4* prev_m, long long fx, long long fm, uint4* out_x, uint4* out_m,
    unsigned long long* host_fetches) {
  __shared__ const uint4* src[2];
  const int i = blockIdx.y;
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
          if (blockIdx.x == 0 && host_fetches) atomicAdd(host_fetches, 1ull);
        }
      }
    }
    src[0] = sx;
    src[1] = sm;
  }
  __syncthreads();
  const uint4 *sx = src[0], *sm = src[1];
  const long long nx = out_x ? fx : 0, total = nx + (out_m ? fm : 0);
  const long long stride = (long long)gridDim.x * blockDim.x;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  // four independent loads in flight per thread before the stores: a zero-copy read over PCIe has microseconds of latency
  for (long long w0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; w0 < total; w0 += 4 * stride) {
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
  const char* api = "fvs_qwen_dam_gather";
  FVS_REQUIRE(picks, "%s: null picks", api);
  FVS_REQUIRE(n > 0 && n <= 65535, "%s: need 0 < n <= 65535 picks (n=%d)", api, n);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", api);
  FVS_REQUIRE(spa_x_out || merged_out, "%s: no output", api);
  FVS_REQUIRE(n_frames > 0 && n_dev >= 0 && n_dev <= n_frames, "%s: need 0 <= n_dev <= n_frames, n_frames > 0 (%lld, %lld)",
              api, (long long)n_dev, (long long)n_frames);
  FVS_REQUIRE(x_frame_elems > 0 && merged_frame_elems >= 0, "%s: bad frame sizes", api);
  FVS_REQUIRE((x_frame_elems * 2) % 16 == 0 && (merged_frame_elems * 2) % 16 == 0,
              "%s: frame sizes must be multiples of 16 bytes", api);
  FVS_REQUIRE(!merged_out || merged_frame_elems > 0, "%s: merged_out without merged rows", api);
  FVS_REQUIRE(n_dev == 0 || (dev_x && (!merged_out || dev_merged)), "%s: null device tier", api);
  FVS_REQUIRE(n_dev == n_frames || (host_chunks && chunk_frames > 0), "%s: host frames without a chunk table", api);
  FVS_REQUIRE(m >= 0 && (m == 0 || (prev_picks && prev_x && (!merged_out || prev_merged))), "%s: bad previous DAM", api);
  for (const void* p : {dev_x, dev_merged, prev_x, prev_merged, (const void*)spa_x_out, (const void*)merged_out})
    FVS_REQUIRE(aligned16(p), "%s: row tensors must be 16-byte aligned", api);
  FVS_REQUIRE(((uintptr_t)picks & 7) == 0 && ((uintptr_t)prev_picks & 7) == 0 && ((uintptr_t)host_chunks & 7) == 0,
              "%s: index tables must be 8-byte aligned", api);
  const long long fx = x_frame_elems * 2 / 16, fm = merged_frame_elems * 2 / 16;
  const long long words = (spa_x_out ? fx : 0) + (merged_out ? fm : 0);
  long long bx = (words + 4 * 256 - 1) / (4 * 256);
  if (bx > 64) bx = 64;
  dam_gather_kernel<<<dim3(unsigned(bx), unsigned(n)), 256, 0, (cudaStream_t)stream>>>(
      (const long long*)picks, (long long)n_frames, (const uint4*)dev_x, (const uint4*)dev_merged, (long long)n_dev,
      (const uint4* const*)host_chunks, (long long)chunk_frames, (const long long*)prev_picks, m, (const uint4*)prev_x,
      (const uint4*)prev_merged, fx, fm, (uint4*)spa_x_out, (uint4*)merged_out, (unsigned long long*)host_fetches);
  FVS_CHECK_LAUNCH("dam_gather_kernel");
  return FVS_OK;
}

}  // extern "C"
