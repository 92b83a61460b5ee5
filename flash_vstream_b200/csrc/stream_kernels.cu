// stream_kernels.cu — fvs_stream_step / fvs_bank_*: the reference's per-clip streaming update on a PERSISTENT bank.
//
// Behavioural spec: VStreamMetaForCausalLM.embed_video_streaming after the encoder
// (Flash-VStream-LLaVA/flash_vstream/model/vstream_arch.py:644-697; SURVEY.md Appendix B), default compressor
// 'weighted_kmeans' (model/compress_functions.py:130-169), abstract memory = attention_feature over
// VStreamMetaForCausalLM.attention (compress_functions.py:263-277, vstream_arch.py:174-183,47-52).
//
// The reference runs this as ~60 small torch ops, three torch.cat copies of the whole state and a CPU<->GPU round trip
// of the state through a Manager list per frame.  Here a step is
//   1. the three pooled STAR levels, written straight into the bank's arrays — by the encoder's tail
//      (fvs_vit_encode_pool3: pooled from the fp32 residual stream, the [t,576,D] feature map is never stored) or by
//      pool3_kernel when the caller brings finished ViT features;
//   2. ONE cooperative kernel (consolidate_kernel) that walks the whole update with block-group barriers and a DEVICE-SIDE
//      early exit: Lloyd iterations (distance partials | assign + weighted mean + refill + convergence partial), stable
//      argsort of the cluster weights, key-frame distances + argmin, the abstract-memory update (a dedicated block that
//      overlaps the Lloyd phases), and the write-back of [Turing | long | key | current] into the prefix buffer, which is
//      laid out in the reader's order (vstream_arch.py:483) so the LLM's visual prefix is a VIEW of the bank.
// Every unit of work (a row's slice partials and label, a (cluster, slice) update, a convergence term, an argsort rank, a
// key distance, an abstract-memory dot product / softmax row / output element) is a device function of mem_device.cuh that
// the op-by-op kernels of memory_kernels.cu call too; this kernel adds only the launch shape, barriers and bookkeeping.  So
// the bank is bit-identical to the op-by-op path and to oracle/fvs_oracle.py.
//
// fvs_stream_step_multi steps many banks the same way: one pooling pass for all their clips, then as few cooperative launches
// of consolidate_kernel as fit on the device, each job on its own range of blocks with its own barriers.
//
// Readers in other processes / on other GPUs (the LLM rank) map the prefix buffer through CUDA IPC and take a consistent
// snapshot with fvs_bank_snapshot: the kernel brackets its write-back with a sequence counter (odd while writing).
#include <cooperative_groups.h>

#include <cstdio>
#include <vector>

#include "fvs_common.h"
#include "fvs_kernels.h"
#include "mem_device.cuh"
#include "seqlock.cuh"

namespace cg = cooperative_groups;

namespace fvs {
namespace stream {
using namespace mem;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxT = 192;   // rows of the k-means working set (old long rows + new frames)
constexpr int kMaxK = 64;    // long-memory length
constexpr int kMaxKey = 8;
constexpr int kMaxS = 32;    // 1024-element slices per long-memory row

struct StepArgs {
  // ---- shapes (all host-known: the data-dependent part of a step is only WHICH rows win)
  int D, PDl, PDa, S;          // channel dim; elements of a long row (b*b*D) / a frame row (a*a*D); PDl / 1024
  int T, K, do_kmeans;         // k-means over T = old long rows + new frames, K = long_len; do_kmeans = T > K > 0
  int kl;                      // key frames retrieved this step = min(key_len, #sorted weights)
  int n_tur_in, tur_len, abs_chunks, H;   // Turing working rows, memory rows, number of <= tur_len-row chunks folded in
  float ratio, sqrtH;
  int cur_start;               // current-memory frames taken from the END of this clip
  long long n_frames_after;    // frames in the buffer including this clip
  int n_tur_new, n_long_new, n_cur_new;   // rows of the published state
  int max_iter;
  uint16_t tol_h;
  // ---- persistent per-stream buffers
  uint16_t* LW;                // [.., PDl] long working set: rows [0, n_long_old) old, then this clip's level-b rows
  uint16_t* TW;                // [.., D]   Turing working set, same convention
  const uint16_t* frames;      // [n_frames_after, PDa] frame buffer (level a)
  uint16_t* prefix;            // [n_tur_new + n_long_new*b*b + n_cur_new*a*a, D]  = [Turing | long | key | current]
  unsigned long long* header;  // {seq, n_tur, n_long, n_cur, n_frames, step, 0, 0}
  unsigned long long step;
  // ---- per-step inputs
  const int* init_idx;         // [K]
  const int* refill_idx;       // [max_iter * K]
  const uint16_t *Wq, *bq, *Wk, *bk;
  // ---- workspace
  uint16_t* C[2];              // [K, PDl] centroid ping-pong
  float* normpart;             // [K, S]
  uint16_t* wsum;              // [K]
  float* dist;                 // [T, kl]
  uint16_t* Mbuf[2];           // [tur_len, D] abstract-memory ping-pong
  float *absq, *absk, *abswgt, *absdecay;   // [tur_len, H] x 2, [tur_len, tur_len], [tur_len] scratch of the abstract group
  int n_abs_blocks;            // the job's last n_abs_blocks blocks form the abstract-memory group
  unsigned int *km_ctr, *abs_ctr, *job_ctr;   // arrival counters of the two block groups' and the whole job's barriers (zero at launch)
  int* labels_out;             // [T]
  int* info_out;               // {exit_step, refills, converged, kmeans_ran}
  long long* key_idx_out;      // [kl]
  unsigned int* done_ctr;
  // ---- device window of the frame buffer (fvs_bank.frames_window; read by the tiered kernel only)
  long long clip_first;        // global index of this clip's first frame
  long long window;            // frames [0, window) stay in `frames`; 0: uncapped
};

// Row of `frames` that holds global frame g of the clip starting at frame clip_first, in a bank whose device window is
// `window` frames (0: uncapped, the row is g).  Frames below the window are at their own index; the clip's frames at or
// past it follow the window in order, in the chunk_cap-row slot — so a clip's rows are contiguous whether it lies below
// the window, straddles it or lies past it.  The pooled tail writes through it (prepare_job) and the write-back reads the
// current frames through it.
__host__ __device__ __forceinline__ long long frame_row(long long g, long long clip_first, long long window) {
  return (window == 0 || g < window) ? g : window + g - (clip_first > window ? clip_first : window);
}

// ---------------------------------------------------------------------------------------------------- group barrier
// Barrier among a GROUP of co-resident blocks (the launch is cooperative, so spinning is safe): a monotonic arrival counter,
// `target` is the calling block's running count of expected arrivals.  Two groups run different programs side by side — the
// Lloyd loop (data-dependent number of phases) and the abstract-memory update — so a grid-wide barrier would serialise them.
__device__ __forceinline__ void group_sync(unsigned int* ctr, unsigned int n, unsigned int& target) {
  __syncthreads();
  target += n;
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
    // poll with plain L2 loads (an acquire load per poll would invalidate the L1 every time: CCTL.IVALL), fence once at the end
    const volatile unsigned int* vc = ctr;
    while (*vc < target) __nanosleep(32);
    __threadfence();
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------- abstract memory
// attention_feature (compress_functions.py:263-277) on a small group of blocks, concurrently with the Lloyd loop: per chunk
// of <= tur_len new rows, projections (one warp per (row, h) dot product) | softmax * ratio and row decay (one warp per
// memory row) | M' = M (1 - decay) + W F.  Result: Mbuf[(chunks-1)&1].
__device__ void abstract_group(const StepArgs& A, int gb, int ng) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T1 = A.tur_len, D = A.D, H = A.H;
  unsigned int target = 0;
  const uint16_t* M = A.TW;
  for (int c = 0; c < A.abs_chunks; ++c) {
    const int f0 = T1 + c * T1;
    const int T2 = min(T1, A.n_tur_in - f0);
    const uint16_t* F = A.TW + size_t(f0) * D;
    uint16_t* Mout = A.Mbuf[c & 1];
    for (int u = gb * kWarps + warp; u < (T1 + T2) * H; u += ng * kWarps) {   // projections: q rows of M, k rows of F
      const int r = u / H, h = u % H;
      const bool isq = r < T1;
      const uint16_t* x = isq ? M + size_t(r) * D : F + size_t(r - T1) * D;
      const float v = abs_proj_dot(x, (isq ? A.Wq : A.Wk) + size_t(h) * D, (isq ? A.bq : A.bk) + h, D, lane);
      if (lane == 0) (isq ? A.absq + r * H : A.absk + (r - T1) * H)[h] = v;
    }
    group_sync(A.abs_ctr, ng, target);
    for (int i = gb * kWarps + warp; i < T1; i += ng * kWarps) {   // softmax * ratio, row decay
      const float decay = abs_softmax_row(A.absq, A.absk, i, A.abswgt + size_t(i) * T1, T2, H, A.sqrtH, A.ratio, lane);
      if (lane == 0) A.absdecay[i] = decay;
    }
    group_sync(A.abs_ctr, ng, target);
    for (int o = gb * kThreads + threadIdx.x; o < T1 * D; o += ng * kThreads) {   // M' = M (1 - decay) + W F
      const int i = o / D, d = o % D;
      Mout[o] = abs_apply_elem(A.abswgt + size_t(i) * T1, F, T2, D, d, M[size_t(i) * D + d], A.absdecay[i]);
    }
    if (c + 1 < A.abs_chunks) group_sync(A.abs_ctr, ng, target);
    M = Mout;
  }
}

// ---------------------------------------------------------------------------------------------------- the step kernel
// One cooperative launch (a "wave") advances up to kJobs banks.  Job j owns the contiguous blocks [first[j], first[j+1]):
// its Lloyd-loop blocks, then its abstract-memory blocks.  Every barrier of a job counts that job's blocks only, so no
// stream waits for another, and every phase is a stride loop over independent units of mem_device.cuh, so a bank's bits do
// not depend on how many blocks its job gets.  fvs_stream_step is the one-job wave (kJobs = 1).  kTier: some job of the
// wave has a device window (the current frames are read through frame_row); uncapped waves run the kTier = false code.
template <int kJobs>
struct Wave {
  int n;
  int first[kJobs + 1];
  StepArgs job[kJobs];
};

template <int kJobs, bool kTier>
__global__ void __launch_bounds__(kThreads, 1) consolidate_kernel(const __grid_constant__ Wave<kJobs> W) {
  int j = 0;
  if constexpr (kJobs > 1)
    while (j + 1 < W.n && int(blockIdx.x) >= W.first[j + 1]) ++j;
  const StepArgs& A = W.job[j];
  __shared__ int s_labels[kMaxT];
  __shared__ float s_part[kMaxK * kMaxS];   // distance partials of ONE row against every centroid slice
  __shared__ float s_v[kMaxK];
  __shared__ int s_order[kMaxK];
  __shared__ long long s_idx[kMaxKey];
  __shared__ int s_flag[4];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = W.first[j + 1] - W.first[j];          // this job's blocks
  const int wb = int(blockIdx.x) - W.first[j];         // block index within the job
  const int nwork = G - A.n_abs_blocks;               // blocks [0, nwork): Lloyd loop + key distances; the rest: abstract memory
  const bool abs_block = wb >= nwork;
  unsigned int km_target = 0, job_target = 0;
  const int D = A.D, PD = A.PDl, S = A.S, T = A.T, K = A.K;

  // readers see an odd sequence number from before the first barrier until the write-back has completed
  if (wb == 0 && threadIdx.x == 0) seqlock::write_begin(&A.header[0]);
  if (abs_block) abstract_group(A, wb - nwork, A.n_abs_blocks);

  // ------------------------------------------------------------------ Lloyd loop (compress_functions.py:135-156)
  int have_c = 0, cur = 0, refill_pos = 0, exit_step = 0, converged = 0;
  if (A.do_kmeans && !abs_block) {
    for (int it = 0; it < A.max_iter; ++it) {
      const int nxt = have_c ? (cur ^ 1) : 0;
      // phase A: a block = ONE row of the working set: warp w owns the slices w, w+8, ... (x in registers), sweeps the K centroid
      // slices into shared memory, and the row's label = first-index / NaN-wins argmin of f16(sqrt(f16(sum of partials))) is
      // formed on the spot — no round trip of the [T, K, S] partials through global memory, no label pass per block.
      for (int t = wb; t < T; t += nwork) {
        for (int sl = warp; sl < S; sl += kWarps) {
          uint4 x[4];
          load_slice(x, A.LW + size_t(t) * PD + sl * SLICE, lane);
#pragma unroll 5
          for (int k = 0; k < K; ++k) {
            const uint16_t* c = have_c ? A.C[cur] + size_t(k) * PD : A.LW + size_t(A.init_idx[k]) * PD;
            const float p = slice_sqdiff(x, c + sl * SLICE, lane);
            if (lane == 0) s_part[k * S + sl] = p;
          }
        }
        __syncthreads();
        if (warp == 0) {
          const int label = km_row_label(s_part, K, S, lane);
          if (lane == 0) A.labels_out[t] = label;
        }
        __syncthreads();
      }
      group_sync(A.km_ctr, nwork, km_target);
      for (int t = threadIdx.x; t < T; t += kThreads) s_labels[t] = A.labels_out[t];
      __syncthreads();
      // phase C: one warp per (cluster j, slice s): mean of the members (unit weights), empty-cluster refill, ||dc||^2 partial
      for (int unit = wb * kWarps + warp; unit < K * S; unit += nwork * kWarps) {
        const int j = unit / S, s = unit % S;
        const uint16_t* Cold = (have_c ? A.C[cur] + size_t(j) * PD : A.LW + size_t(A.init_idx[j]) * PD) + s * SLICE;
        km_cluster_slice_update(A.LW, nullptr, s_labels, A.refill_idx + refill_pos, T, PD, S, j, s, Cold,
                                A.C[nxt] + size_t(j) * PD + s * SLICE, A.normpart, A.wsum, lane);
      }
      group_sync(A.km_ctr, nwork, km_target);
      // phase D (every block for itself, identical result): diff = f16(sum_k f16(sqrt(sum_s normpart))) < f16(tol) ?
      if (warp == 0) {
        for (int k = lane; k < K; k += 32) s_v[k] = centroid_shift(A.normpart, k, S);
        __syncwarp();
        if (lane == 0) {
          float diff = 0.f;
          int n_empty = 0;
          for (int k = 0; k < K; ++k) {
            diff = diff + s_v[k];
            if (!(h2f(A.wsum[k]) > 0.f)) n_empty++;
          }
          s_flag[0] = round_h(diff) < h2f(A.tol_h) ? 1 : 0;
          s_flag[1] = n_empty;
        }
      }
      __syncthreads();
      const int brk = s_flag[0];
      refill_pos += s_flag[1];
      exit_step = it;
      __syncthreads();
      if (brk) { converged = 1; break; }     // `if diff < tol: break` — the centroids stay the OLD ones (:154-155)
      have_c = 1;
      cur = nxt;
    }
    if (!have_c) {
      // broke at the very first iteration: the result is the initial draw X[init_idx]; materialise it so that the
      // write-back below never permutes the working set in place
      for (size_t i = size_t(wb) * kThreads + threadIdx.x; i < size_t(K) * (PD / 8); i += size_t(nwork) * kThreads) {
        const int k = int(i / (PD / 8)), v = int(i % (PD / 8));
        reinterpret_cast<uint4*>(A.C[0])[i] = reinterpret_cast<const uint4*>(A.LW + size_t(A.init_idx[k]) * PD)[v];
      }
      cur = 0;     // (the job-wide barrier below orders these writes before the write-back reads them)
    }
  }

  // ------------------------------------------------------------------ key-frame retrieval (vstream_arch.py:681-688)
  const int kl = A.kl;
  if (kl > 0 && !abs_block) {
    // stable descending argsort of the cluster weights (pass-through: all ones -> identity)
    if (A.do_kmeans) {
      for (int i = threadIdx.x; i < K; i += kThreads)
        s_order[stable_desc_rank(i, K, [&](int j) { return h2f(A.wsum[j]); })] = i;
    } else {
      for (int i = threadIdx.x; i < kl; i += kThreads) s_order[i] = i;
    }
    __syncthreads();
    // key distances, one warp per (l, k); rows of the PRE-clustering working set
    for (int unit = wb * kWarps + warp; unit < T * kl; unit += nwork * kWarps) {
      const int l = unit / kl, k = unit % kl;
      const float d = key_distance(A.LW + size_t(l) * PD, A.LW + size_t(s_order[k]) * PD, PD / D, D, lane);
      if (lane == 0) A.dist[unit] = d;
    }
  }
  if (wb == 0 && threadIdx.x == 0) {
    A.info_out[0] = exit_step; A.info_out[1] = refill_pos; A.info_out[2] = converged; A.info_out[3] = A.do_kmeans;
    A.info_out[4] = cur;       // which centroid buffer holds the result (the abstract group's blocks need it for the write-back)
  }
  // the ONE job-wide barrier: Lloyd loop, key distances and the abstract memory are all complete behind it
  group_sync(A.job_ctr, G, job_target);
  cur = A.info_out[4];
  if (kl > 0) {
    if (warp < kl) {   // first-index / NaN-wins argmin over the working-set rows (every block for itself)
      const int besti = warp_argmin_of(T, [&](int l) { return A.dist[l * kl + warp]; }, lane);
      if (lane == 0) {
        s_idx[warp] = besti;
        if (wb == 0) A.key_idx_out[warp] = besti;
      }
    }
    __syncthreads();
  }

  // ------------------------------------------------------------------ write-back: prefix = [Turing | long | key | current]
  // (vstream_arch.py:483 reader order), and the compressed state back into the working sets for the next step
  {
    const size_t vD = size_t(D) / 8, vL = size_t(PD) / 8, vA = size_t(A.PDa) / 8;
    const size_t n1 = size_t(A.n_tur_new) * vD;                          // prefix Turing rows
    const size_t n2 = n1 + size_t(A.n_long_new) * vL;                    // prefix long rows
    const size_t n3 = n2 + size_t(A.n_cur_new) * vA;                     // prefix key + current frames
    const size_t n4 = n3 + (A.do_kmeans ? size_t(K) * vL : 0);           // LW[0:K) <- centroids
    const size_t n5 = n4 + (A.abs_chunks > 0 ? size_t(A.tur_len) * vD : 0);  // TW[0:tur_len) <- updated abstract memory
    const uint4* tur_src = reinterpret_cast<const uint4*>(A.abs_chunks > 0 ? A.Mbuf[(A.abs_chunks - 1) & 1] : A.TW);
    const uint4* long_src = reinterpret_cast<const uint4*>(A.do_kmeans ? A.C[cur] : A.LW);
    const uint4* fr = reinterpret_cast<const uint4*>(A.frames);
    uint4* pre = reinterpret_cast<uint4*>(A.prefix);
    for (size_t i = size_t(wb) * kThreads + threadIdx.x; i < n5; i += size_t(G) * kThreads) {
      if (i < n1) {
        pre[i] = tur_src[i];
      } else if (i < n2) {
        pre[i] = long_src[i - n1];
      } else if (i < n3) {
        const size_t r = (i - n2) / vA, c = (i - n2) % vA;
        long long row = r < size_t(kl) ? s_idx[r] : A.n_frames_after - A.cur_start + (long long)(r - kl);
        if constexpr (kTier) {   // key rows are below the window (s_idx < T <= long_work_rows <= window): unmapped
          if (r >= size_t(kl)) row = frame_row(row, A.clip_first, A.window);
        }
        pre[i] = fr[size_t(row) * vA + c];
      } else if (i < n4) {
        reinterpret_cast<uint4*>(A.LW)[i - n3] = long_src[i - n3];
      } else {
        reinterpret_cast<uint4*>(A.TW)[i - n4] = tur_src[i - n4];
      }
    }
  }
  // the job's last block to finish publishes its counters and makes the sequence number even again
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const unsigned ticket = atomicAdd(A.done_ctr, 1u);
    if (ticket == unsigned(G) - 1u) {
      A.header[1] = A.n_tur_new; A.header[2] = A.n_long_new; A.header[3] = A.n_cur_new;
      A.header[4] = (unsigned long long)A.n_frames_after; A.header[5] = A.step;
      *A.done_ctr = 0u;
      *A.km_ctr = 0u;
      *A.abs_ctr = 0u;
      *A.job_ctr = 0u;
      seqlock::write_end(&A.header[0]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------- snapshot for readers
// out <- prefix (rows known to the reader from the header it read first).  status[0] = the sequence number seen before the
// copy, status[1] = after: a reader accepts the snapshot iff both are equal and even, else it retries.
__global__ void snapshot_kernel(const uint4* __restrict__ prefix, const unsigned long long* __restrict__ header,
                                uint4* __restrict__ out, unsigned long long* __restrict__ status, size_t max_vecs, int D,
                                int pa, int pb) {
  cg::grid_group grid = cg::this_grid();
  __shared__ unsigned long long s_hdr[6];
  if (threadIdx.x == 0) {
    s_hdr[0] = seqlock::read_open(header);
    const volatile unsigned long long* h = header;
    for (int i = 1; i < 6; ++i) s_hdr[i] = h[i];
  }
  __syncthreads();
  const size_t rows = size_t(s_hdr[1]) + size_t(s_hdr[2]) * pb + size_t(s_hdr[3]) * pa;
  size_t n = rows * size_t(D / 8);
  if (n > max_vecs) n = max_vecs;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x) out[i] = prefix[i];
  __threadfence_system();
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    status[0] = s_hdr[0];
    status[1] = seqlock::read_close(header);
    for (int i = 1; i < 6; ++i) status[1 + i] = s_hdr[i];
  }
}

// ---------------------------------------------------------------------------------------------------- restore
// prefix <- src and header words 1-5 <- the restored counters, under the writer side of the seqlock: a reader that has the
// bank mapped (a bank of a closed stream that StreamPool hands to a new one may still be) sees the old prefix or the
// restored one, never a mix.  src is a device pointer or a pinned host pointer (read over PCIe through UVA).
__global__ void __launch_bounds__(256) restore_kernel(const uint4* __restrict__ src, uint4* __restrict__ prefix,
                                                      unsigned long long* __restrict__ header, size_t n_vecs,
                                                      unsigned long long n_tur, unsigned long long n_long,
                                                      unsigned long long n_cur, unsigned long long n_frames,
                                                      unsigned long long step) {
  cg::grid_group grid = cg::this_grid();
  if (blockIdx.x == 0 && threadIdx.x == 0) seqlock::write_begin(&header[0]);
  grid.sync();
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vecs; i += size_t(gridDim.x) * blockDim.x)
    prefix[i] = src[i];
  __threadfence_system();
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    header[1] = n_tur; header[2] = n_long; header[3] = n_cur; header[4] = n_frames; header[5] = step;
    seqlock::write_end(&header[0]);
  }
}

inline size_t al(size_t v) { return (v + 255) & ~size_t(255); }

struct Carve {
  uint16_t* C[2]; float* normpart; uint16_t* wsum; float* dist; uint16_t* Mbuf[2];
  float *absq, *absk, *abswgt, *absdecay;
  int* labels; int* info; long long* key_idx; unsigned int* done_ctr;   // done_ctr[0..3] = {finished blocks, k-means group, abstract group, job}
  size_t total;
};
Carve carve(const fvs_star_config& c, int chunk_cap, void* base) {
  const int b2 = c.long_size * c.long_size;
  const size_t PDl = size_t(b2) * c.D, S = PDl / SLICE;
  const size_t Tmax = size_t(c.long_len > chunk_cap ? c.long_len : chunk_cap) + chunk_cap;
  Carve w;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? static_cast<uint8_t*>(base) + off : nullptr;
    off += al(bytes);
    return p;
  };
  const size_t K = c.long_len > 0 ? c.long_len : 1;
  w.C[0] = (uint16_t*)take(K * PDl * 2);
  w.C[1] = (uint16_t*)take(K * PDl * 2);
  w.normpart = (float*)take(K * S * 4);
  w.wsum = (uint16_t*)take(K * 2);
  w.dist = (float*)take(Tmax * kMaxKey * 4);
  const size_t tl = c.tur_len > 0 ? c.tur_len : 1;
  w.Mbuf[0] = (uint16_t*)take(tl * c.D * 2);
  w.Mbuf[1] = (uint16_t*)take(tl * c.D * 2);
  w.absq = (float*)take(tl * size_t(c.ntm_dim) * 4);
  w.absk = (float*)take(tl * size_t(c.ntm_dim) * 4);
  w.abswgt = (float*)take(tl * tl * 4);
  w.absdecay = (float*)take(tl * 4);
  w.labels = (int*)take(Tmax * 4);
  w.info = (int*)take(32);
  w.key_idx = (long long*)take(kMaxKey * 8);
  w.done_ctr = (unsigned int*)take(16);
  w.total = off;
  return w;
}

int check_config(const fvs_star_config* c, const char* who) {
  FVS_REQUIRE(c, "%s: null config", who);
  FVS_REQUIRE(c->D > 0 && c->D % 256 == 0, "%s: D (%d) must be a multiple of 256", who, c->D);
  FVS_REQUIRE(c->grid > 0 && c->cur_size > 0 && c->grid % c->cur_size == 0 && c->cur_size * c->cur_size <= 64,
              "%s: grid %d / compress_size %d unsupported", who, c->grid, c->cur_size);
  FVS_REQUIRE(c->long_size > 0 && c->cur_size % c->long_size == 0, "%s: compress_long_memory_size %d must divide %d", who,
              c->long_size, c->cur_size);
  FVS_REQUIRE((size_t(c->long_size) * c->long_size * c->D) % SLICE == 0, "%s: long rows must be whole 1024-element slices", who);
  FVS_REQUIRE(c->long_len >= 0 && c->long_len <= kMaxK && c->tur_len >= 0 && c->tur_len <= 64 && c->cur_len >= 0,
              "%s: memory lengths out of range (long %d <= %d, Turing %d <= 64)", who, c->long_len, kMaxK, c->tur_len);
  FVS_REQUIRE(c->key_len >= 0 && c->key_len <= kMaxKey, "%s: key_len %d > %d", who, c->key_len, kMaxKey);
  FVS_REQUIRE(c->ntm_dim > 0 && c->ntm_dim <= 64, "%s: ntm_dim %d out of range", who, c->ntm_dim);
  return FVS_OK;
}

// A bank's device window (fvs_bank.frames_window): 0, or at least the long working set's rows (every key frame index is
// a row of it) with room for one clip's slot behind it.
int check_window(const fvs_bank* bank, int64_t lrows, const char* who) {
  const int64_t N = bank->frames_window;
  FVS_REQUIRE(N == 0 || N >= lrows, "%s: frames_window %lld < %lld, the long working set's rows (max(long_len, chunk_cap) + "
              "chunk_cap): key frames are read from below the window", who, (long long)N, (long long)lrows);
  FVS_REQUIRE(N == 0 || N + bank->chunk_cap <= bank->frames_cap, "%s: frames_cap %lld < frames_window %lld + chunk_cap %d",
              who, (long long)bank->frames_cap, (long long)N, bank->chunk_cap);
  return FVS_OK;
}

constexpr int kWaveJobs = 32;   // jobs per cooperative launch (the per-job kernel arguments travel as kernel parameters)

// One job of a step, validated: its kernel arguments, its pooling destination and the blocks it wants.
struct JobPrep {
  StepArgs A;
  Carve w;
  Pool3Dst dst;
  int units;   // blocks of its widest Lloyd / key-distance phase
};

// Every check of one job; fills the kernel arguments without touching the bank or the device.
int prepare_job(const fvs_star_config* cfg, const fvs_stream_job& job, const char* who, JobPrep& P) {
  const fvs_bank* bank = job.bank;
  FVS_REQUIRE(bank && job.workspace, "%s: null argument", who);
  FVS_REQUIRE(bank->prefix && bank->long_work && bank->tur_work && bank->frames && bank->header, "%s: bank buffers missing", who);
  const int t = job.frames;
  FVS_REQUIRE(t > 0 && t <= bank->chunk_cap, "%s: %d frames per call, bank was sized for <= %d", who, t, bank->chunk_cap);
  int64_t lrows, trows, prows;
  fvs_bank_rows(cfg, bank->chunk_cap, &lrows, &trows, &prows);
  int r = check_window(bank, lrows, who);
  if (r) return r;
  const int64_t row0 = frame_row(bank->n_frames, bank->n_frames, bank->frames_window);   // the clip's first row in `frames`
  FVS_REQUIRE(row0 + t <= bank->frames_cap, "%s: frame buffer full (%lld + %d > %lld): grow it first", who,
              (long long)row0, t, (long long)bank->frames_cap);
  const Carve w = carve(*cfg, bank->chunk_cap, job.workspace);
  FVS_REQUIRE(job.workspace_bytes >= w.total, "%s: workspace too small (%zu < %zu)", who, job.workspace_bytes, w.total);
  const int D = cfg->D, a = cfg->cur_size, b = cfg->long_size;
  const size_t PDa = size_t(a) * a * D, PDl = size_t(b) * b * D;
  const bool has_memory = bank->step > 0;
  const int n_long_old = has_memory ? bank->n_long : 0, n_tur_old = has_memory ? bank->n_tur : 0;
  FVS_REQUIRE(n_long_old + t <= lrows && n_tur_old + t <= trows, "%s: working set overflow", who);

  // pooled levels of this clip -> frame buffer (its rows are contiguous there, see frame_row) / long working set / Turing
  // working set
  P.dst.a = static_cast<uint16_t*>(bank->frames) + size_t(row0) * PDa;
  P.dst.b = static_cast<uint16_t*>(bank->long_work) + size_t(n_long_old) * PDl;
  P.dst.c = static_cast<uint16_t*>(bank->tur_work) + size_t(n_tur_old) * D;
  P.dst.frames = t;

  StepArgs& A = P.A;
  A = {};
  A.D = D; A.PDl = int(PDl); A.PDa = int(PDa); A.S = int(PDl / SLICE);
  A.T = n_long_old + t;
  A.K = cfg->long_len;
  A.do_kmeans = (has_memory && A.K > 0 && A.T > A.K) ? 1 : 0;
  FVS_REQUIRE(A.T <= kMaxT, "%s: working set of %d rows > %d", who, A.T, kMaxT);
  FVS_REQUIRE(A.S <= kMaxS, "%s: long rows of %d slices > %d", who, A.S, kMaxS);
  const int n_sorted = A.do_kmeans ? A.K : A.T;
  A.kl = (has_memory && cfg->long_len > 0) ? (cfg->key_len < n_sorted ? cfg->key_len : n_sorted) : 0;
  A.n_tur_in = n_tur_old + t;
  A.tur_len = cfg->tur_len;
  A.abs_chunks = 0;
  if (has_memory && cfg->tur_len > 0 && A.n_tur_in > cfg->tur_len)
    A.abs_chunks = (A.n_tur_in - cfg->tur_len + cfg->tur_len - 1) / cfg->tur_len;
  FVS_REQUIRE(A.abs_chunks == 0 || job.ntm, "%s: abstract-memory weights missing", who);
  A.H = cfg->ntm_dim;
  A.ratio = cfg->ratio;
  A.sqrtH = sqrtf(float(cfg->ntm_dim));
  A.cur_start = cfg->cur_len < t ? cfg->cur_len : t;
  A.n_frames_after = bank->n_frames + t;
  // lengths of 0 switch a memory off (offline guard vstream_arch.py:253,271; the reference's streaming branch has no such
  // guard and would raise — this is the natural extension, used for the 256-token bank of SURVEY.md §8d(2))
  A.n_tur_new = cfg->tur_len == 0 ? 0 : (A.abs_chunks > 0 ? cfg->tur_len : A.n_tur_in);
  A.n_long_new = cfg->long_len == 0 ? 0 : (A.do_kmeans ? A.K : A.T);
  A.n_cur_new = A.kl + A.cur_start;
  A.max_iter = 10;                                                   // compress_functions.py:133
  A.tol_h = __half_as_ushort(__float2half_rn(1e-4f));                // tol compared in the tensor dtype
  A.LW = static_cast<uint16_t*>(bank->long_work);
  A.TW = static_cast<uint16_t*>(bank->tur_work);
  A.frames = static_cast<const uint16_t*>(bank->frames);
  A.prefix = static_cast<uint16_t*>(bank->prefix);
  A.header = static_cast<unsigned long long*>(bank->header);
  A.step = bank->step + 1;
  A.init_idx = job.init_idx;
  A.refill_idx = job.refill_idx;
  FVS_REQUIRE(!A.do_kmeans || (job.init_idx && job.refill_idx), "%s: k-means draws (init_idx, refill_idx) missing", who);
  const fvs_ntm_weights* ntm = job.ntm;
  if (ntm) { A.Wq = (const uint16_t*)ntm->q_w; A.bq = (const uint16_t*)ntm->q_b; A.Wk = (const uint16_t*)ntm->k_w; A.bk = (const uint16_t*)ntm->k_b; }
  A.C[0] = w.C[0]; A.C[1] = w.C[1]; A.normpart = w.normpart; A.wsum = w.wsum; A.dist = w.dist;
  A.Mbuf[0] = w.Mbuf[0]; A.Mbuf[1] = w.Mbuf[1]; A.labels_out = w.labels; A.info_out = w.info; A.key_idx_out = w.key_idx;
  A.done_ctr = w.done_ctr;
  A.clip_first = bank->n_frames;
  A.window = bank->frames_window;
  A.km_ctr = w.done_ctr + 1;
  A.abs_ctr = w.done_ctr + 2;
  A.job_ctr = w.done_ctr + 3;
  A.absq = w.absq; A.absk = w.absk; A.abswgt = w.abswgt; A.absdecay = w.absdecay;
  const int64_t need_rows = int64_t(A.n_tur_new) + int64_t(A.n_long_new) * b * b + int64_t(A.n_cur_new) * a * a;
  FVS_REQUIRE(need_rows <= prows, "%s: prefix of %lld rows exceeds the buffer (%lld)", who, (long long)need_rows, (long long)prows);

  // blocks for the widest phase (the abstract-memory group comes on top)
  int units = 8;
  if (A.do_kmeans) {
    units = A.T;                                            // phase A: one block per row
    const int uc = (A.K * A.S + kWarps - 1) / kWarps;        // phase C: one warp per (cluster, slice)
    if (uc > units) units = uc;
  }
  const int ue = (A.T * A.kl + kWarps - 1) / kWarps;
  if (ue > units) units = ue;
  P.units = units;
  P.w = w;
  return FVS_OK;
}

int min_blocks(const JobPrep& P) { return 1 + (P.A.abs_chunks > 0 ? 1 : 0); }

// Launch plan for `budget` co-resident blocks per launch.  A job wants blocks for its widest phase plus an abstract-memory
// group (16 blocks, 1 on small budgets) when its Turing memory folds a chunk — alone in a launch, exactly the grid of a
// single-stream step.  Jobs are packed in order into as few waves as the budget allows (at least the minimum of every job,
// at most kWaveJobs jobs); in a wave whose wants exceed the budget every job gets its minimum plus a share of the spare
// blocks in proportion to what it wants beyond it (cumulative rounding: the shares add up to exactly the spare blocks).
// Returns the number of waves, or an error when a job's minimum exceeds the budget.
int plan_waves(const JobPrep* P, int n, int budget, const char* api, int* km_out, int* abs_out, int* wave_out) {
  std::vector<int> km_want(n), abs_want(n);
  for (int i = 0; i < n; ++i) {
    FVS_REQUIRE(min_blocks(P[i]) <= budget, "%s: job %d needs at least %d blocks per launch, the budget is %d", api, i,
                min_blocks(P[i]), budget);
    abs_want[i] = P[i].A.abs_chunks > 0 ? (budget >= 64 ? 16 : 1) : 0;
    const int room = budget - abs_want[i];
    km_want[i] = P[i].units < room ? P[i].units : room;
    if (km_want[i] < 1) km_want[i] = 1;
  }
  int waves = 0;
  for (int s = 0; s < n; ++waves) {
    int e = s, need = 0;
    long long want = 0;
    while (e < n && e - s < kWaveJobs && need + min_blocks(P[e]) <= budget) {
      need += min_blocks(P[e]);
      want += km_want[e] + abs_want[e];
      ++e;
    }
    const long long spare = budget - need, excess = want - need;
    long long cum = 0, given = 0;
    auto share = [&](int extra) {
      if (want <= budget) return extra;
      cum += extra;
      const long long upto = spare * cum / excess;
      const long long g = upto - given;
      given = upto;
      return int(g);
    };
    for (int i = s; i < e; ++i) {
      const int abs_min = P[i].A.abs_chunks > 0 ? 1 : 0;
      km_out[i] = 1 + share(km_want[i] - 1);
      abs_out[i] = abs_min + share(abs_want[i] - abs_min);
      wave_out[i] = waves;
    }
    s = e;
  }
  return waves;
}

// Co-resident blocks of one cooperative launch: one per SM at most (the block groups spin on barriers).
int device_budget(int* out) {
  static int cap = 0;
  if (cap == 0) {
    int p[4] = {0, 0, 0, 0};
    FVS_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&p[0], consolidate_kernel<1, false>, kThreads, 0));
    FVS_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&p[1], consolidate_kernel<kWaveJobs, false>, kThreads, 0));
    FVS_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&p[2], consolidate_kernel<1, true>, kThreads, 0));
    FVS_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&p[3], consolidate_kernel<kWaveJobs, true>, kThreads, 0));
    int per_sm = p[0];
    for (int i = 1; i < 4; ++i) per_sm = p[i] < per_sm ? p[i] : per_sm;
    const int co = (per_sm > 0 ? per_sm : 1) * device_sm_count();
    cap = device_sm_count() < co ? device_sm_count() : co;
  }
  *out = cap;
  return FVS_OK;
}

// Validate every job (no CUDA call, nothing touched), then plan for `budget` blocks (0: query the device).
int prepare_all(const fvs_star_config* cfg, const fvs_stream_job* jobs, int n, const char* api, bool multi,
                std::vector<JobPrep>& P) {
  int r = check_config(cfg, api);
  if (r) return r;
  FVS_REQUIRE(jobs && n > 0, "%s: no jobs", api);
  P.resize(n);
  for (int i = 0; i < n; ++i) {
    char who[64];
    if (multi) snprintf(who, sizeof who, "%s: job %d", api, i);
    else snprintf(who, sizeof who, "%s", api);
    if ((r = prepare_job(cfg, jobs[i], who, P[i]))) return r;
    for (int k = 0; k < i; ++k) {
      FVS_REQUIRE(jobs[k].bank != jobs[i].bank && jobs[k].bank->header != jobs[i].bank->header,
                  "%s: jobs %d and %d step the same bank", api, k, i);
      FVS_REQUIRE(jobs[k].workspace != jobs[i].workspace, "%s: jobs %d and %d share a workspace", api, k, i);
    }
  }
  return FVS_OK;
}

template <int kJobs>
int launch_wave(const JobPrep* P, int n, const int* km, const int* ab, cudaStream_t stream) {
  Wave<kJobs> W;
  W.n = n;
  W.first[0] = 0;
  bool tier = false;
  for (int i = 0; i < n; ++i) {
    W.job[i] = P[i].A;
    W.job[i].n_abs_blocks = ab[i];
    W.first[i + 1] = W.first[i] + km[i] + ab[i];
    tier = tier || P[i].A.window > 0;
  }
  void* args[] = {&W};
  const void* fn = tier ? (const void*)consolidate_kernel<kJobs, true> : (const void*)consolidate_kernel<kJobs, false>;
  FVS_CUDA_OK(cudaLaunchCooperativeKernel(fn, dim3(W.first[n]), dim3(kThreads), args, 0, stream));
  FVS_CHECK_LAUNCH("consolidate_kernel");
  return FVS_OK;
}

// fvs_stream_step / fvs_stream_step_multi: validate everything, then pool every clip (one encoder pass / one pool3 launch
// for all jobs), then the consolidation waves; the host counters move only once every launch is enqueued.
int step_jobs(const fvs_star_config* cfg, fvs_stream_job* jobs, int n, fvs_vit_t vit, const void* input, int input_kind,
              void* vit_workspace, size_t vit_workspace_bytes, int max_blocks, cudaStream_t stream, bool multi) {
  const char* api = multi ? "fvs_stream_step_multi" : "fvs_stream_step";
  FVS_REQUIRE(input, "%s: null argument", api);
  FVS_REQUIRE(input_kind == FVS_INPUT_PIXELS || input_kind == FVS_INPUT_FEATURES, "%s: bad input_kind %d", api, input_kind);
  FVS_REQUIRE(input_kind != FVS_INPUT_PIXELS || (vit && vit_workspace), "%s: pixels need a ViT handle and its workspace", api);
  FVS_REQUIRE(max_blocks >= 0, "%s: max_blocks %d < 0", api, max_blocks);
  std::vector<JobPrep> P;
  int r = prepare_all(cfg, jobs, n, api, multi, P);
  if (r) return r;
  for (int i = 0; i < n; ++i)
    FVS_REQUIRE(max_blocks == 0 || min_blocks(P[i]) <= max_blocks, "%s: job %d needs at least %d blocks per launch, max_blocks is %d",
                api, i, min_blocks(P[i]), max_blocks);
  int budget = 0;
  if ((r = device_budget(&budget))) return r;
  if (max_blocks > 0 && max_blocks < budget) budget = max_blocks;
  std::vector<int> km(n), ab(n), wave(n);
  const int waves = plan_waves(P.data(), n, budget, api, km.data(), ab.data(), wave.data());
  if (waves < 0) return waves;

  // ---- 1. pooled levels of every clip, straight into each bank
  std::vector<Pool3Dst> dst(n);
  int total = 0;
  for (int i = 0; i < n; ++i) dst[i] = P[i].dst, total += P[i].dst.frames;
  if (input_kind == FVS_INPUT_PIXELS) {
    if ((r = vit_encode_pool3(vit, input, dst.data(), n, cfg->cur_size, cfg->long_size, vit_workspace, vit_workspace_bytes, stream)))
      return r;
  } else {
    if ((r = pool3_launch(input, false, dst.data(), n, 0, total, cfg->grid, cfg->cur_size, cfg->long_size, cfg->D, stream))) return r;
  }

  // ---- 2. the updates, one cooperative launch per wave
  for (int i = 0; i < n; ++i)
    if (jobs[i].bank->step == 0) FVS_CUDA_OK(cudaMemsetAsync(P[i].w.done_ctr, 0, 16, stream));
  for (int s = 0; s < n;) {
    int e = s;
    while (e < n && wave[e] == wave[s]) ++e;
    r = e - s == 1 ? launch_wave<1>(&P[s], 1, &km[s], &ab[s], stream)
                   : launch_wave<kWaveJobs>(&P[s], e - s, &km[s], &ab[s], stream);
    if (r) return r;
    s = e;
  }

  for (int i = 0; i < n; ++i) {
    fvs_bank* bank = jobs[i].bank;
    bank->n_frames += jobs[i].frames;
    bank->n_long = P[i].A.n_long_new;
    bank->n_tur = P[i].A.n_tur_new;
    bank->n_cur = P[i].A.n_cur_new;
    bank->step += 1;
  }
  return FVS_OK;
}

}  // namespace stream
}  // namespace fvs

using namespace fvs;
using namespace fvs::stream;

extern "C" {

size_t fvs_stream_workspace_bytes(const fvs_star_config* cfg, int chunk_cap) {
  if (!cfg || chunk_cap <= 0 || check_config(cfg, "fvs_stream_workspace_bytes")) return 0;
  return carve(*cfg, chunk_cap, nullptr).total;
}

int fvs_bank_rows(const fvs_star_config* cfg, int chunk_cap, int64_t* long_work_rows, int64_t* tur_work_rows,
                  int64_t* prefix_rows) {
  int r = check_config(cfg, "fvs_bank_rows");
  if (r) return r;
  FVS_REQUIRE(chunk_cap > 0, "fvs_bank_rows: chunk_cap must be > 0");
  const int64_t lcap = (cfg->long_len > chunk_cap ? cfg->long_len : chunk_cap), tcap = (cfg->tur_len > chunk_cap ? cfg->tur_len : chunk_cap);
  if (long_work_rows) *long_work_rows = lcap + chunk_cap;
  if (tur_work_rows) *tur_work_rows = tcap + chunk_cap;
  if (prefix_rows)
    *prefix_rows = (tcap + chunk_cap) + (lcap + chunk_cap) * cfg->long_size * cfg->long_size +
                   int64_t(cfg->key_len + (cfg->cur_len < chunk_cap ? cfg->cur_len : chunk_cap)) * cfg->cur_size * cfg->cur_size;
  return FVS_OK;
}

int fvs_bank_reset(fvs_bank* bank, fvs_stream_t stream) {
  FVS_REQUIRE(bank && bank->header, "fvs_bank_reset: null bank");
  bank->n_frames = 0;
  bank->n_long = bank->n_tur = bank->n_cur = 0;
  bank->step = 0;
  FVS_CUDA_OK(cudaMemsetAsync(bank->header, 0, 64, (cudaStream_t)stream));
  return FVS_OK;
}

int fvs_bank_restore(const fvs_star_config* cfg, fvs_bank* bank, int32_t n_tur, int32_t n_long, int32_t n_cur,
                     int64_t n_frames, uint64_t step, const void* prefix_src, const void* long_src, const void* tur_src,
                     const void* frames_src, fvs_stream_t stream) {
  const char* api = "fvs_bank_restore";
  int r = check_config(cfg, api);
  if (r) return r;
  FVS_REQUIRE(bank, "%s: null bank", api);
  FVS_REQUIRE(bank->prefix && bank->long_work && bank->tur_work && bank->frames && bank->header, "%s: bank buffers missing", api);
  FVS_REQUIRE(bank->chunk_cap > 0, "%s: chunk_cap must be > 0", api);
  int64_t lrows, trows, prows;
  if ((r = fvs_bank_rows(cfg, bank->chunk_cap, &lrows, &trows, &prows))) return r;
  // a first clip longer than a memory leaves that many rows (the k-means / abstract update only start at the second step),
  // so the working sets hold up to max(length, chunk_cap) rows between steps — lrows / trows less one clip
  const int64_t lcap = lrows - bank->chunk_cap, tcap = trows - bank->chunk_cap;
  FVS_REQUIRE(n_long >= 0 && n_long <= lcap, "%s: n_long %d > %lld (long_len %d, chunk_cap %d)", api, n_long, (long long)lcap,
              cfg->long_len, bank->chunk_cap);
  FVS_REQUIRE(n_tur >= 0 && n_tur <= tcap, "%s: n_tur %d > %lld (tur_len %d, chunk_cap %d)", api, n_tur, (long long)tcap,
              cfg->tur_len, bank->chunk_cap);
  FVS_REQUIRE(n_cur >= 0 && n_cur <= cfg->key_len + cfg->cur_len, "%s: n_cur %d > key_len + cur_len (%d)", api, n_cur,
              cfg->key_len + cfg->cur_len);
  const int a2 = cfg->cur_size * cfg->cur_size, b2 = cfg->long_size * cfg->long_size;
  const int64_t rows = int64_t(n_tur) + int64_t(n_long) * b2 + int64_t(n_cur) * a2;
  FVS_REQUIRE(rows <= prows, "%s: prefix of %lld rows exceeds the buffer (%lld)", api, (long long)rows, (long long)prows);
  if ((r = check_window(bank, lrows, api))) return r;
  const int64_t window = bank->frames_window;
  FVS_REQUIRE(n_frames >= 0 && (window > 0 || n_frames <= bank->frames_cap),
              "%s: %lld frames > frames_cap %lld: grow the frame buffer first", api, (long long)n_frames,
              (long long)bank->frames_cap);
  const int64_t dev_frames = window > 0 && n_frames > window ? window : n_frames;   // the rest stays with the caller
  FVS_REQUIRE((step == 0) == (n_frames == 0), "%s: step %llu with %lld frames (step is 0 exactly when no frame was seen)", api,
              (unsigned long long)step, (long long)n_frames);
  FVS_REQUIRE(step > 0 || (n_tur == 0 && n_long == 0 && n_cur == 0), "%s: a state at step 0 holds no memory rows", api);
  FVS_REQUIRE(rows == 0 || prefix_src, "%s: prefix_src is null", api);
  FVS_REQUIRE(n_long == 0 || long_src, "%s: long_src is null", api);
  FVS_REQUIRE(n_tur == 0 || tur_src, "%s: tur_src is null", api);
  FVS_REQUIRE(n_frames == 0 || frames_src, "%s: frames_src is null", api);

  // every source must be readable by the bank's device: its own memory or pinned host memory (a pageable pointer would
  // fault in the kernel, another device's memory needs peer mappings the caller did not ask for)
  cudaPointerAttributes at;
  FVS_CUDA_OK(cudaPointerGetAttributes(&at, bank->header));
  const int dev = at.device;
  const void* srcs[4] = {rows ? prefix_src : nullptr, n_long ? long_src : nullptr, n_tur ? tur_src : nullptr,
                         n_frames ? frames_src : nullptr};
  const char* names[4] = {"prefix_src", "long_src", "tur_src", "frames_src"};
  for (int i = 0; i < 4; ++i) {
    if (!srcs[i]) continue;
    FVS_CUDA_OK(cudaPointerGetAttributes(&at, srcs[i]));
    FVS_REQUIRE(at.type == cudaMemoryTypeHost || ((at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) &&
                                                 at.device == dev),
                "%s: %s is neither pinned host memory nor memory of the bank's device %d", api, names[i], dev);
  }

  cudaStream_t s = (cudaStream_t)stream;
  const size_t D = size_t(cfg->D);
  if (n_long) FVS_CUDA_OK(cudaMemcpyAsync(bank->long_work, long_src, size_t(n_long) * b2 * D * 2, cudaMemcpyDefault, s));
  if (n_tur) FVS_CUDA_OK(cudaMemcpyAsync(bank->tur_work, tur_src, size_t(n_tur) * D * 2, cudaMemcpyDefault, s));
  if (dev_frames) FVS_CUDA_OK(cudaMemcpyAsync(bank->frames, frames_src, size_t(dev_frames) * a2 * D * 2, cudaMemcpyDefault, s));

  static int per_sm = 0;
  if (per_sm == 0) FVS_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, restore_kernel, 256, 0));
  const uint4* src = static_cast<const uint4*>(prefix_src);
  uint4* pre = static_cast<uint4*>(bank->prefix);
  unsigned long long* hdr = static_cast<unsigned long long*>(bank->header);
  size_t n_vecs = size_t(rows) * (D / 8);
  unsigned long long w[5] = {(unsigned long long)n_tur, (unsigned long long)n_long, (unsigned long long)n_cur,
                             (unsigned long long)n_frames, (unsigned long long)step};
  const size_t want = (n_vecs + 255) / 256;
  const size_t cap = size_t(per_sm > 0 ? per_sm : 1) * device_sm_count();
  const unsigned blocks = unsigned(want < 1 ? 1 : (want < cap ? want : cap));
  void* args[] = {&src, &pre, &hdr, &n_vecs, &w[0], &w[1], &w[2], &w[3], &w[4]};
  FVS_CUDA_OK(cudaLaunchCooperativeKernel((const void*)restore_kernel, dim3(blocks), dim3(256), args, 0, s));
  FVS_CHECK_LAUNCH("restore_kernel");

  bank->n_tur = n_tur;
  bank->n_long = n_long;
  bank->n_cur = n_cur;
  bank->n_frames = n_frames;
  bank->step = step;
  return FVS_OK;
}

int fvs_bank_prefix(const fvs_star_config* cfg, const fvs_bank* bank, void** prefix_out, int64_t* rows_out) {
  FVS_REQUIRE(cfg && bank && rows_out, "fvs_bank_prefix: null argument");
  if (prefix_out) *prefix_out = bank->prefix;
  *rows_out = int64_t(bank->n_tur) + int64_t(bank->n_long) * cfg->long_size * cfg->long_size +
              int64_t(bank->n_cur) * cfg->cur_size * cfg->cur_size;
  return FVS_OK;
}

int fvs_stream_step(const fvs_star_config* cfg, fvs_bank* bank, const fvs_ntm_weights* ntm, fvs_vit_t vit,
                    const void* input, int input_kind, int frames, const int32_t* init_idx, const int32_t* refill_idx,
                    void* vit_workspace, size_t vit_workspace_bytes, void* workspace, size_t workspace_bytes,
                    fvs_stream_t stream) {
  fvs_stream_job job = {bank, ntm, frames, init_idx, refill_idx, workspace, workspace_bytes};
  return step_jobs(cfg, &job, 1, vit, input, input_kind, vit_workspace, vit_workspace_bytes, 0, (cudaStream_t)stream, false);
}

int fvs_stream_step_multi(const fvs_star_config* cfg, fvs_stream_job* jobs, int n_jobs, fvs_vit_t vit, const void* input,
                          int input_kind, void* vit_workspace, size_t vit_workspace_bytes, int max_blocks, fvs_stream_t stream) {
  return step_jobs(cfg, jobs, n_jobs, vit, input, input_kind, vit_workspace, vit_workspace_bytes, max_blocks,
                   (cudaStream_t)stream, true);
}

int fvs_stream_plan(const fvs_star_config* cfg, const fvs_stream_job* jobs, int n_jobs, int budget, int32_t* blocks_out,
                    int32_t* wave_out) {
  FVS_REQUIRE(budget > 0 && blocks_out && wave_out, "fvs_stream_plan: budget must be > 0 and outputs non-null");
  std::vector<JobPrep> P;
  int r = prepare_all(cfg, jobs, n_jobs, "fvs_stream_plan", true, P);
  if (r) return r;
  std::vector<int> km(n_jobs), ab(n_jobs), wave(n_jobs);
  const int waves = plan_waves(P.data(), n_jobs, budget, "fvs_stream_plan", km.data(), ab.data(), wave.data());
  if (waves < 0) return waves;
  for (int i = 0; i < n_jobs; ++i) {
    blocks_out[2 * i] = km[i];
    blocks_out[2 * i + 1] = ab[i];
    wave_out[i] = wave[i];
  }
  return waves;
}

int fvs_stream_step_info(const fvs_star_config* cfg, const fvs_bank* bank, void* workspace, int32_t** labels, int32_t** info,
                         int64_t** key_idx, void** wsum) {
  FVS_REQUIRE(cfg && bank && workspace, "fvs_stream_step_info: null argument");
  const Carve w = carve(*cfg, bank->chunk_cap, workspace);
  if (labels) *labels = w.labels;
  if (info) *info = w.info;
  if (key_idx) *key_idx = (int64_t*)w.key_idx;
  if (wsum) *wsum = w.wsum;
  return FVS_OK;
}

int fvs_bank_snapshot(const void* prefix, const void* header, void* out, int64_t max_rows, int D, int cur_size, int long_size,
                      uint64_t* status, fvs_stream_t stream) {
  FVS_REQUIRE(prefix && header && out && status, "fvs_bank_snapshot: null pointer");
  FVS_REQUIRE(D > 0 && D % 8 == 0 && max_rows > 0, "fvs_bank_snapshot: bad shape");
  const uint4* p = (const uint4*)prefix;
  const unsigned long long* h = (const unsigned long long*)header;
  uint4* o = (uint4*)out;
  unsigned long long* st = (unsigned long long*)status;
  size_t max_vecs = size_t(max_rows) * (D / 8);
  int pa = cur_size * cur_size, pb = long_size * long_size;
  void* args[] = {&p, &h, &o, &st, &max_vecs, &D, &pa, &pb};
  FVS_CUDA_OK(cudaLaunchCooperativeKernel((const void*)snapshot_kernel, dim3(64), dim3(256), args, 0, (cudaStream_t)stream));
  FVS_CHECK_LAUNCH("snapshot_kernel");
  return FVS_OK;
}

}  // extern "C"
