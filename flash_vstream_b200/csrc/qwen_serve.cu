// qwen_serve.cu — fvs_qwen_pub_layout / fvs_qwen_publish / fvs_qwen_snapshot: the Qwen2-VL streaming memory published for
// readers in other processes (CUDA IPC) or on other GPUs (peer access), under the seqlock of seqlock.cuh.
//
// The reference hands the memory to the LLM process by pickling all 13 items of `video_embedding_memory` through a
// Manager server after every clip (Flash-VStream-Qwen/cli_server_2gpu.py:197-239, vstream_qwen2vl_realtime.py:620-627).
// What the LLM reads is `video_embeds` and the positions that AM-RoPE needs (prepare_realtime_inference, :632-640), so a
// publication holds just those, in one device allocation: the writer copies them in with one launch at the end of a clip,
// a reader copies them out on its own device whenever it is asked a question.
#include <cooperative_groups.h>

#include <mutex>
#include <set>
#include <utility>

#include "fvs_common.h"
#include "seqlock.cuh"

namespace cg = cooperative_groups;

namespace fvs {
namespace qserve {

constexpr int kThreads = 256;
enum { H_SEQ, H_EPOCH, H_CLIPS, H_FRAMES, H_TEM, H_SPA, H_ROWS, H_GRID, H_WORDS };
static_assert(H_WORDS * 8 == 64, "the header is 64 bytes");

struct Layout {
  size_t ts, pos, emb, bytes;
};
inline size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline Layout layout(int tem_len, int spa_len, int64_t rows_cap, int dim) {
  Layout L;
  L.ts = 64;
  L.pos = round_up(L.ts + 4 * size_t(tem_len), 8);
  L.emb = round_up(L.pos + 8 * size_t(spa_len), 16);
  L.bytes = L.emb + size_t(rows_cap) * size_t(dim) * 2;
  return L;
}

// grid-stride copy with four independent 16-byte loads in flight per thread
template <class T>
__device__ __forceinline__ void copy_strided(T* __restrict__ dst, const T* __restrict__ src, size_t n) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n; i += 4 * stride) {
    const T a = src[i], b = src[i + stride], c = src[i + 2 * stride], d = src[i + 3 * stride];
    dst[i] = a; dst[i + stride] = b; dst[i + 2 * stride] = c; dst[i + 3 * stride] = d;
  }
  for (; i < n; i += stride) dst[i] = src[i];
}

struct PubArgs {
  unsigned long long* hdr;
  float* ts;
  long long* pos;
  uint4* emb;
  const float* src_ts;
  const long long* src_pos;
  const uint4* src_emb;
  size_t emb_vecs;
  int n_tem, n_spa;
  unsigned long long fields[H_WORDS];   // [H_EPOCH .. H_GRID] are written behind the copy
};

__global__ void __launch_bounds__(kThreads) publish_kernel(const __grid_constant__ PubArgs a) {
  cg::grid_group grid = cg::this_grid();
  if (blockIdx.x == 0 && threadIdx.x == 0) seqlock::write_begin(&a.hdr[H_SEQ]);
  grid.sync();                                   // no block writes before seq is odd
  copy_strided(a.emb, a.src_emb, a.emb_vecs);
  copy_strided(a.ts, a.src_ts, size_t(a.n_tem));
  copy_strided(a.pos, a.src_pos, size_t(a.n_spa));
  __threadfence_system();
  grid.sync();                                   // every block's writes are visible at system scope
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (int i = H_EPOCH; i < H_WORDS; ++i) a.hdr[i] = a.fields[i];
    seqlock::write_end(&a.hdr[H_SEQ]);
  }
}

struct SnapArgs {
  const unsigned long long* hdr;
  const float* ts;
  const long long* pos;
  const uint4* emb;
  float* ts_out;
  long long* pos_out;
  uint4* emb_out;
  unsigned long long* status;   // {seq0, seq1, header[1..7]}
  int tem_len, spa_len;
  long long rows_cap;
  int vecs_per_row;
};

// Block 0 reads the counter and the header once and hands them to every block through `status` (one grid sync), so
// all blocks copy the counts of one header read, and the accepted copy is the one that header describes.
__global__ void __launch_bounds__(kThreads) snapshot_kernel(const __grid_constant__ SnapArgs a) {
  cg::grid_group grid = cg::this_grid();
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.status[0] = seqlock::read_open(&a.hdr[H_SEQ]);
    const volatile unsigned long long* h = a.hdr;
    for (int i = H_EPOCH; i < H_WORDS; ++i) a.status[1 + i] = h[i];
  }
  grid.sync();
  const volatile unsigned long long* st = a.status;
  const unsigned long long n_tem = st[1 + H_TEM], n_spa = st[1 + H_SPA], rows = st[1 + H_ROWS];
  // a torn header may say anything: never beyond the capacities the publication and the outputs were sized for
  const size_t nt = n_tem < (unsigned long long)a.tem_len ? size_t(n_tem) : size_t(a.tem_len);
  const size_t ns = n_spa < (unsigned long long)a.spa_len ? size_t(n_spa) : size_t(a.spa_len);
  const size_t nr = rows < (unsigned long long)a.rows_cap ? size_t(rows) : size_t(a.rows_cap);
  copy_strided(a.emb_out, a.emb, nr * size_t(a.vecs_per_row));
  copy_strided(a.ts_out, a.ts, nt);
  copy_strided(a.pos_out, a.pos, ns);
  __threadfence_system();
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.status[1] = seqlock::read_close(&a.hdr[H_SEQ]);
}

// Blocks of a cooperative launch of `kern`: two per SM keep enough loads in flight for the copy and leave room on every
// SM for the other side's kernels (a writer's step and a reader's snapshot run concurrently).
template <class K>
int coop_blocks(K kern, int* out) {
  int per_sm = 0;
  FVS_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, 0));
  if (per_sm > 2) per_sm = 2;
  *out = (per_sm > 0 ? per_sm : 1) * device_sm_count();
  return FVS_OK;
}

// Peer access from the current device to the device that owns `p`, enabled once per pair.
int ensure_peer(const void* p, const char* api) {
  static std::mutex mu;
  static std::set<std::pair<int, int>> enabled;
  cudaPointerAttributes attr;
  FVS_CUDA_OK(cudaPointerGetAttributes(&attr, p));
  FVS_REQUIRE(attr.type == cudaMemoryTypeDevice, "%s: the publication is not device memory", api);
  int cur = 0;
  FVS_CUDA_OK(cudaGetDevice(&cur));
  if (attr.device == cur) return FVS_OK;
  std::lock_guard<std::mutex> lk(mu);
  if (enabled.count({cur, attr.device})) return FVS_OK;
  int can = 0;
  FVS_CUDA_OK(cudaDeviceCanAccessPeer(&can, cur, attr.device));
  FVS_REQUIRE(can, "%s: device %d cannot access the memory of device %d (no peer access between them)", api, cur, attr.device);
  const cudaError_t e = cudaDeviceEnablePeerAccess(attr.device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();                          // enabled elsewhere in this process (torch, another library): fine
  } else {
    FVS_CUDA_OK(e);
  }
  enabled.insert({cur, attr.device});
  return FVS_OK;
}

int check_layout(size_t pub_bytes, int tem_len, int spa_len, int64_t rows_cap, int dim, const char* api) {
  FVS_REQUIRE(tem_len >= 0 && spa_len >= 0 && rows_cap >= 0, "%s: negative capacity", api);
  FVS_REQUIRE(dim > 0 && dim % 8 == 0, "%s: dim %d must be a positive multiple of 8", api, dim);
  const Layout L = layout(tem_len, spa_len, rows_cap, dim);
  FVS_REQUIRE(pub_bytes >= L.bytes, "%s: publication of %zu bytes < %zu the layout needs", api, pub_bytes, L.bytes);
  return FVS_OK;
}

}  // namespace qserve
}  // namespace fvs

using namespace fvs;
using namespace fvs::qserve;

extern "C" {

int fvs_qwen_pub_layout(int tem_len, int spa_len, int h, int w, int hs, int ws, int dim, int64_t* layout_out) {
  FVS_REQUIRE(layout_out, "fvs_qwen_pub_layout: null argument");
  FVS_REQUIRE(tem_len >= 0 && spa_len >= 0 && dim > 0 && dim % 8 == 0, "fvs_qwen_pub_layout: bad shape");
  FVS_REQUIRE(h > 0 && w > 0 && hs > 0 && ws > 0 && h < 65536 && w < 65536 && hs < 65536 && ws < 65536 &&
                  (h * w) % 4 == 0 && (hs * ws) % 4 == 0,
              "fvs_qwen_pub_layout: grid (%d, %d) / (%d, %d) must be positive, < 65536 and hold whole 2x2 groups", h, w, hs, ws);
  const int64_t rows = int64_t(spa_len) * (h * w / 4) + int64_t(tem_len) * (hs * ws / 4);
  const Layout L = layout(tem_len, spa_len, rows, dim);
  layout_out[0] = rows;
  layout_out[1] = int64_t(L.ts);
  layout_out[2] = int64_t(L.pos);
  layout_out[3] = int64_t(L.emb);
  layout_out[4] = int64_t(L.bytes);
  return FVS_OK;
}

int fvs_qwen_publish(void* pub, size_t pub_bytes, int tem_len, int spa_len, int64_t rows_cap, int dim,
                     const void* video_embeds, int64_t rows, const float* tem_timestamp, int n_tem,
                     const int64_t* spa_positions, int n_spa, int h, int w, int hs, int ws, uint64_t epoch, uint64_t clips,
                     int64_t n_frames, fvs_stream_t stream) {
  const char* api = "fvs_qwen_publish";
  FVS_REQUIRE(pub, "%s: null publication", api);
  int r = check_layout(pub_bytes, tem_len, spa_len, rows_cap, dim, api);
  if (r) return r;
  FVS_REQUIRE(n_tem >= 0 && n_tem <= tem_len && n_spa >= 0 && n_spa <= spa_len, "%s: %d CSM / %d DAM frames exceed %d / %d",
              api, n_tem, n_spa, tem_len, spa_len);
  FVS_REQUIRE(h > 0 && w > 0 && hs > 0 && ws > 0 && h < 65536 && w < 65536 && hs < 65536 && ws < 65536 &&
                  (h * w) % 4 == 0 && (hs * ws) % 4 == 0, "%s: bad grid (%d, %d) / (%d, %d)", api, h, w, hs, ws);
  FVS_REQUIRE(rows >= 0 && rows <= rows_cap && rows == int64_t(n_spa) * (h * w / 4) + int64_t(n_tem) * (hs * ws / 4),
              "%s: %lld rows do not match %d DAM frames of %dx%d and %d CSM frames of %dx%d (capacity %lld)", api,
              (long long)rows, n_spa, h, w, n_tem, hs, ws, (long long)rows_cap);
  FVS_REQUIRE((rows == 0 || video_embeds) && (n_tem == 0 || tem_timestamp) && (n_spa == 0 || spa_positions),
              "%s: null source", api);
  FVS_REQUIRE(n_frames >= 0, "%s: n_frames %lld < 0", api, (long long)n_frames);
  FVS_REQUIRE(reinterpret_cast<uintptr_t>(pub) % 16 == 0 && reinterpret_cast<uintptr_t>(video_embeds) % 16 == 0,
              "%s: publication and video_embeds must be 16-byte aligned", api);
  const Layout L = layout(tem_len, spa_len, rows_cap, dim);
  PubArgs a = {};
  uint8_t* base = static_cast<uint8_t*>(pub);
  a.hdr = reinterpret_cast<unsigned long long*>(base);
  a.ts = reinterpret_cast<float*>(base + L.ts);
  a.pos = reinterpret_cast<long long*>(base + L.pos);
  a.emb = reinterpret_cast<uint4*>(base + L.emb);
  a.src_ts = tem_timestamp;
  a.src_pos = reinterpret_cast<const long long*>(spa_positions);
  a.src_emb = static_cast<const uint4*>(video_embeds);
  a.emb_vecs = size_t(rows) * size_t(dim) / 8;
  a.n_tem = n_tem;
  a.n_spa = n_spa;
  a.fields[H_EPOCH] = epoch;
  a.fields[H_CLIPS] = clips;
  a.fields[H_FRAMES] = (unsigned long long)n_frames;
  a.fields[H_TEM] = (unsigned long long)n_tem;
  a.fields[H_SPA] = (unsigned long long)n_spa;
  a.fields[H_ROWS] = (unsigned long long)rows;
  a.fields[H_GRID] = (unsigned long long)h | (unsigned long long)w << 16 | (unsigned long long)hs << 32 |
                     (unsigned long long)ws << 48;
  int blocks = 0;
  if ((r = coop_blocks(publish_kernel, &blocks))) return r;
  void* args[] = {&a};
  FVS_CUDA_OK(cudaLaunchCooperativeKernel((const void*)publish_kernel, dim3(blocks), dim3(kThreads), args, 0,
                                          (cudaStream_t)stream));
  FVS_CHECK_LAUNCH("qwen publish_kernel");
  return FVS_OK;
}

int fvs_qwen_snapshot(const void* pub, size_t pub_bytes, int tem_len, int spa_len, int64_t rows_cap, int dim,
                      void* embeds_out, int64_t out_rows, float* ts_out, int64_t ts_cap, int64_t* pos_out, int64_t pos_cap,
                      uint64_t* status, fvs_stream_t stream) {
  const char* api = "fvs_qwen_snapshot";
  FVS_REQUIRE(pub && embeds_out && ts_out && pos_out && status, "%s: null pointer", api);
  int r = check_layout(pub_bytes, tem_len, spa_len, rows_cap, dim, api);
  if (r) return r;
  FVS_REQUIRE(out_rows >= rows_cap && ts_cap >= tem_len && pos_cap >= spa_len,
              "%s: reader buffers ([%lld rows], [%lld], [%lld]) below the publication's capacity ([%lld], [%d], [%d])", api,
              (long long)out_rows, (long long)ts_cap, (long long)pos_cap, (long long)rows_cap, tem_len, spa_len);
  FVS_REQUIRE(reinterpret_cast<uintptr_t>(pub) % 16 == 0 && reinterpret_cast<uintptr_t>(embeds_out) % 16 == 0,
              "%s: publication and embeds_out must be 16-byte aligned", api);
  if ((r = ensure_peer(pub, api))) return r;
  const Layout L = layout(tem_len, spa_len, rows_cap, dim);
  const uint8_t* base = static_cast<const uint8_t*>(pub);
  SnapArgs a = {};
  a.hdr = reinterpret_cast<const unsigned long long*>(base);
  a.ts = reinterpret_cast<const float*>(base + L.ts);
  a.pos = reinterpret_cast<const long long*>(base + L.pos);
  a.emb = reinterpret_cast<const uint4*>(base + L.emb);
  a.ts_out = ts_out;
  a.pos_out = reinterpret_cast<long long*>(pos_out);
  a.emb_out = static_cast<uint4*>(embeds_out);
  a.status = reinterpret_cast<unsigned long long*>(status);
  a.tem_len = tem_len;
  a.spa_len = spa_len;
  a.rows_cap = rows_cap;
  a.vecs_per_row = dim / 8;
  int blocks = 0;
  if ((r = coop_blocks(snapshot_kernel, &blocks))) return r;
  void* args[] = {&a};
  FVS_CUDA_OK(cudaLaunchCooperativeKernel((const void*)snapshot_kernel, dim3(blocks), dim3(kThreads), args, 0,
                                          (cudaStream_t)stream));
  FVS_CHECK_LAUNCH("qwen snapshot_kernel");
  return FVS_OK;
}

}  // extern "C"
