// qwen_kernels.cu — Flash-Memory kernels of the Qwen2-VL variant (Flash-VStream-Qwen/models/):
//   temporal_pool               vstream_qwen2vl_model.py:113-142   (pixel-space 2x2 average of the patchified clip)
//   weighted_kmeans_ordered     compress_functions.py:181-298      (fp32 Lloyd, GEMM-form distances, unique() init)
//   spatial_enhance (klarge)    vstream_qwen2vl_model.py:182-244   (16-bit GEMM-form distances + argmin over the bank)
//   calc_am_rope                vstream_qwen2vl_model.py:254-277   (integer 3-D position ids)
// HBM/ALU-bound integer and fp32/16-bit element work (the contractions have <= 64 rows on one side: ~0.5 flop/byte, so
// they run as split-K sweeps on the CUDA cores, not as tensor-core GEMMs).  Arithmetic follows the reference's PyTorch
// expression trees: one rounding per op in the op's dtype, fp32 accumulation inside reductions in the canonical slice order
// of mem_device.cuh (fp32 products are rounded before they are added — no FMA — and 16-bit x 16-bit products are exact,
// so oracle/qwen_oracle.py reproduces every bit with numpy).
#include <algorithm>
#include <vector>

#include "fvs_common.h"
#include "fvs_ptx.cuh"
#include "mem_device.cuh"

namespace fvs {
namespace qwen {

using mem::SLICE;
using mem::argmin_better;
using mem::butterfly_sum;
using mem::warp_argmin;

// element -> fp32 (exact widening); dt: FVS_F16 / FVS_BF16 / FVS_F32
__device__ __forceinline__ float ld_f32(const void* base, size_t i, int dt) {
  if (dt == FVS_F32) return static_cast<const float*>(base)[i];
  const uint16_t v = static_cast<const uint16_t*>(base)[i];
  if (dt == FVS_BF16) return __uint_as_float(uint32_t(v) << 16);
  return __half2float(__ushort_as_half(v));
}
__device__ __forceinline__ float round_to(float v, int dt) {
  if (dt == FVS_BF16) return __bfloat162float(__float2bfloat16_rn(v));
  if (dt == FVS_F16) return __half2float(__float2half_rn(v));
  return v;
}

// ------------------------------------------------------------------------------------------------ temporal_pool
// x rows ordered (t, h/2, w/2, 2, 2), columns (c=3, tp=2, 14, 14).  Every group of 4 rows (a 2x2 block of patches) forms
// a 28x28 image per (c, tp) plane; 2x2 average -> one 14x14 low-res patch.  Output rows ordered (t, h/4, w/4, 2, 2).
template <bool kBF16>
__global__ void __launch_bounds__(196) temporal_pool_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ out, int t,
                                                            int h, int w) {
  const int h2 = h / 2, w2 = w / 2, nh = h2 / 2, nw = w2 / 2;
  // one block = one output row (1176 pixels); one thread = two horizontally adjacent output pixels (X, X+1 with X even):
  // every source pixel pair (xx, xx+1) with xx even lies inside one 14-wide patch row, so the four 2-pixel reads and the
  // 2-pixel write are aligned 32-bit accesses and each source byte is read exactly once.
  auto cvt = [](uint32_t v16) { return kBF16 ? __uint_as_float(v16 << 16) : __half2float(__ushort_as_half((uint16_t)v16)); };
  const unsigned n_rows = unsigned(t) * h2 * w2;   // < 2^31 (checked by the host entry point)
  for (unsigned out_row = blockIdx.x; out_row < n_rows; out_row += gridDim.x) {
    unsigned r = out_row;                  // (tt, bh, bw, dy, dx)
    const int dx = int(r % 2); r /= 2;
    const int dy = int(r % 2); r /= 2;
    const int bw = int(r % nw); r /= nw;
    const int bh = int(r % nh);
    const int tt = int(r / nh);
    const int py = bh * 2 + dy, px = bw * 2 + dx;  // low-res patch coordinates in the (h/2, w/2) grid
    const uint16_t* blk = x + (((size_t(tt) * h2 + py) * w2 + px) * 4) * 1176;   // the 2x2 block of source patches
    uint16_t* orow = out + size_t(out_row) * 1176;
    const int half = threadIdx.x >= 98 ? 1 : 0, rem = 2 * (threadIdx.x - 98 * half), Y = rem / 14, X = rem - Y * 14;
#pragma unroll
    for (int it = 0; it < 3; ++it) {               // 196 threads x 3 = the row's 588 pixel pairs (98 per colour/time plane)
      const int plane = 2 * it + half, col = plane * 196 + rem;
      float acc[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int yy = 2 * Y + i;                       // row in the 28x28 image of this 2x2 patch block
        const int a = yy >= 14 ? 1 : 0, y = yy - 14 * a;
#pragma unroll
        for (int q = 0; q < 2; ++q) {                   // q-th output pixel of the pair
          const int xx = 2 * (X + q);
          const int b = xx >= 14 ? 1 : 0, xq = xx - 14 * b;
          const uint32_t v = *reinterpret_cast<const uint32_t*>(blk + (a * 2 + b) * 1176 + plane * 196 + y * 14 + xq);
          // fp32 sum in the order (i,j) = (0,0), (0,1), (1,0), (1,1)
          acc[q] = (acc[q] + cvt(v & 0xffffu)) + cvt(v >> 16);
        }
      }
      uint32_t o[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float m = acc[q] * 0.25f;
        if (kBF16) { __nv_bfloat16 hb = __float2bfloat16_rn(m); o[q] = *reinterpret_cast<uint16_t*>(&hb); }
        else o[q] = __half_as_ushort(__float2half_rn(m));
      }
      *reinterpret_cast<uint32_t*>(orow + col) = o[0] | (o[1] << 16);
    }
  }
}

// ------------------------------------------------------------------------------------------------ unique(X, dim=0)
// cmp[i*T+j] = sign of the lexicographic comparison row i vs row j (-1, 0, +1); one block per pair, early exit.
__device__ __forceinline__ void lex_compare_body(int i, int j, const void* __restrict__ X, int T, int PD, int dt,
                                                 signed char* __restrict__ cmp) {
  if (j <= i) {
    if (j == i && threadIdx.x == 0) cmp[i * T + i] = 0;
    return;
  }
  __shared__ int first_diff;
  int result = 0;
  for (int base = 0; base < PD; base += 1024) {
    if (threadIdx.x == 0) first_diff = 0x7fffffff;
    __syncthreads();
    int mine = 0x7fffffff;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int e = base + u * 256 + threadIdx.x;
      if (e < PD) {
        const float a = ld_f32(X, size_t(i) * PD + e, dt), b = ld_f32(X, size_t(j) * PD + e, dt);
        if (a != b && e < mine) mine = e;
      }
    }
    if (mine != 0x7fffffff) atomicMin(&first_diff, mine);
    __syncthreads();
    const int fd = first_diff;
    __syncthreads();
    if (fd != 0x7fffffff) {
      const float a = ld_f32(X, size_t(i) * PD + fd, dt), b = ld_f32(X, size_t(j) * PD + fd, dt);
      result = a < b ? -1 : 1;
      break;
    }
  }
  if (threadIdx.x == 0) {
    cmp[i * T + j] = (signed char)result;
    cmp[j * T + i] = (signed char)(-result);
  }
}
// single block: rows that are the first of their duplicate class, in ascending lexicographic order
__device__ __forceinline__ void unique_order_body(const signed char* __restrict__ cmp, int T, int* __restrict__ uniq_idx,
                                                  int* __restrict__ n_unique, int* is_first) {
  for (int i = threadIdx.x; i < T; i += blockDim.x) {
    int f = 1;
    for (int j = 0; j < i; ++j)
      if (cmp[j * T + i] == 0) { f = 0; break; }
    is_first[i] = f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < T; i += blockDim.x) {
    if (!is_first[i]) continue;
    int rank = 0;
    for (int j = 0; j < T; ++j)
      if (is_first[j] && cmp[j * T + i] < 0) rank++;
    uniq_idx[rank] = i;
  }
  if (threadIdx.x == 0) {
    int n = 0;
    for (int i = 0; i < T; ++i) n += is_first[i];
    *n_unique = n;
  }
}

// ------------------------------------------------------------------------------------------------ fp32 k-means
struct KO {             // device state + buffers of one weighted_kmeans_ordered call
  int* state;           // [0] done  [1] commit ticket (iter + 1)  [2] iter  [3] refill_pos  [4] converged
  float* C[2];          // [K, PD] fp32: C[0] current centroids, C[1] staging for the rows ko_update recomputes
  float* ab;            // [T*K + K, S] slice partials: rows t*K+k = x_t . c_k, rows T*K+k = |c_k|^2 (b2 = ab + T*K*S)
  float* b2;
  float* abt;           // [T*K + K]   their totals (slices added sequentially), b2t = abt + T*K
  float* b2t;
  float* a2;            // [T, S]    partial |x|^2 (computed once per call)
  float* a2t;           // [T]
  float* normpart;      // [K, S]    partial ||c_old - c_new||^2
  float* normt;         // [K]
  float* wsum;          // [K]
  int* labels;          // [T]
  int* dirty;           // [K]   set by ko_assign when a row joined or left the cluster
  float* wprev;         // [K]   weight sums of the previous iteration (<= 0: the cluster was refilled from a random draw)
  int* chg_flag;        // [K]   set by ko_update when a centroid's new value differs bitwise from the old one
  int* chg_list;        // [1 + K] count, then the centroids whose x . c partials must be recomputed this iteration
};

// tot[u] = part[u, 0] + part[u, 1] + ... sequentially (the oracle's _seq_sum over slices); one warp per unit: coalesced
// loads of 32 partials, then a broadcast chain so the dependent adds run at register speed
__device__ __forceinline__ void seq_reduce_body(unsigned bid, const float* __restrict__ part, float* __restrict__ tot, int units,
                                                int S, const int* __restrict__ done) {
  if (done && *done) return;
  const int u = bid * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (u >= units) return;
  float acc = 0.f;
  for (int base = 0; base < S; base += 32) {
    const float v = base + lane < S ? part[size_t(u) * S + base + lane] : 0.f;
    const int n = min(32, S - base);
    for (int i = 0; i < n; ++i) acc = __fadd_rn(acc, __shfl_sync(0xffffffffu, v, i));
  }
  if (lane == 0) tot[u] = acc;
}

// one 1024-element slice of a row -> 32 fp32 registers in the canonical ownership (lane l: elements i*256 + l*8 + e),
// with 16-byte loads; off = element offset of the slice (multiple of 1024)
__device__ __forceinline__ void load_slice(const void* __restrict__ X, int dt, size_t off, int lane, float (&x)[32]) {
  if (dt == FVS_F32) {
    const float4* p = reinterpret_cast<const float4*>(static_cast<const float*>(X) + off);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float4 a = p[i * 64 + lane * 2], b = p[i * 64 + lane * 2 + 1];
      x[i * 8 + 0] = a.x; x[i * 8 + 1] = a.y; x[i * 8 + 2] = a.z; x[i * 8 + 3] = a.w;
      x[i * 8 + 4] = b.x; x[i * 8 + 5] = b.y; x[i * 8 + 6] = b.z; x[i * 8 + 7] = b.w;
    }
  } else {
    const uint4* p = reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(X) + off);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint4 v = p[i * 32 + lane];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (dt == FVS_BF16) {
          x[i * 8 + 2 * q] = __uint_as_float(w[q] << 16);
          x[i * 8 + 2 * q + 1] = __uint_as_float(w[q] & 0xffff0000u);
        } else {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[q]));
          x[i * 8 + 2 * q] = f.x;
          x[i * 8 + 2 * q + 1] = f.y;
        }
      }
    }
  }
}
__device__ __forceinline__ void store_slice_f32(float* __restrict__ dst, int lane, const float (&x)[32]) {
  float4* p = reinterpret_cast<float4*>(dst);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    p[i * 64 + lane * 2] = make_float4(x[i * 8 + 0], x[i * 8 + 1], x[i * 8 + 2], x[i * 8 + 3]);
    p[i * 64 + lane * 2 + 1] = make_float4(x[i * 8 + 4], x[i * 8 + 5], x[i * 8 + 6], x[i * 8 + 7]);
  }
}

// |x_t|^2 slice partials: warp per (t, slice)
__device__ __forceinline__ void ko_xnorm_body(unsigned bid, KO B, const void* __restrict__ X, int dt, int T, int PD) {
  const int S = PD / SLICE;
  const int unit = bid * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (unit >= T * S) return;
  float x[32];
  load_slice(X, dt, size_t(unit / S) * PD + size_t(unit % S) * SLICE, lane, x);
  float acc = 0.f;
#pragma unroll
  for (int q = 0; q < 32; ++q) acc = __fadd_rn(acc, __fmul_rn(x[q], x[q]));
  acc = butterfly_sum(acc);
  if (lane == 0) B.a2[unit] = acc;
}

// initial centroids = unique_X[indices] widened to fp32, and their |c|^2 slice partials: warp per (k, slice)
__device__ __forceinline__ void ko_init_body(unsigned bid, KO B, const void* __restrict__ X, int dt, const int* __restrict__ uniq_idx,
                                                      const int* __restrict__ init_idx, int T, int K, int PD) {
  if (bid == 0) {
    if (threadIdx.x == 0) {
      B.state[0] = 0; B.state[1] = 0; B.state[2] = 0; B.state[3] = 0; B.state[4] = 0;
      B.chg_list[0] = K;
    }
    for (int k = threadIdx.x; k < K; k += blockDim.x) { B.chg_list[1 + k] = k; B.chg_flag[k] = 0; B.dirty[k] = 0; B.wprev[k] = 0.f; }
    for (int t = threadIdx.x; t < T; t += blockDim.x) B.labels[t] = -1;
  }
  const int S = PD / SLICE;
  const int unit = bid * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (unit >= K * S) return;
  const int k = unit / S, s = unit % S;
  const int src = uniq_idx ? uniq_idx[init_idx[k]] : init_idx[k];
  float x[32];
  load_slice(X, dt, size_t(src) * PD + size_t(s) * SLICE, lane, x);
  store_slice_f32(B.C[0] + size_t(k) * PD + size_t(s) * SLICE, lane, x);
  float acc = 0.f;
#pragma unroll
  for (int q = 0; q < 32; ++q) acc = __fadd_rn(acc, __fmul_rn(x[q], x[q]));
  acc = butterfly_sum(acc);
  if (lane == 0) B.b2[unit] = acc;
}

// canonical slice partial of sum(a*b): lane l owns elements i*256 + l*8 + e, products rounded, sequential adds, butterfly.
// b is a slice staged in shared memory in the conflict-free order [i][half][lane][4] (half = e / 4).
__device__ __forceinline__ float slice_dot_smem(const float (&a)[32], const float4* __restrict__ b, int lane) {
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 b0 = b[i * 64 + lane], b1 = b[i * 64 + 32 + lane];
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) acc = __fadd_rn(acc, __fmul_rn(a[i * 8 + e], bb[e]));
  }
  return butterfly_sum(acc);
}

// block = 8 warps = 8 rows t of one slice: each warp keeps its x slice (fp32) in registers; the block streams the K
// centroid slices through shared memory (cp.async, 2 stages of KO_KC slices) so that every centroid byte is fetched from
// L2 once per 8 rows and the loads overlap the dot products.  Only the centroids on the change list are swept: a centroid
// whose value did not change (bitwise) in the last update — in streaming most clusters are singletons — keeps the partials
// of the previous iteration, which are exactly what a recomputation would produce.
constexpr int KO_KC = 8;
constexpr int KO_PARTIAL_SMEM = 2 * KO_KC * SLICE * 4;
__device__ __forceinline__ void ko_partial_body(unsigned bid, float4* cs, KO B, const void* __restrict__ X, int dt, int T, int K,
                                                int PD) {
  if (B.state[0]) return;
  const int S = PD / SLICE;                                 // cs: [2][KO_KC][256] float4 of dynamic shared memory
  const int s = bid % S;
  const int t_raw = (bid / S) * 8 + (threadIdx.x >> 5);
  const int t = min(t_raw, T - 1);
  const int lane = threadIdx.x & 31;
  const float* C = B.C[0] + size_t(s) * SLICE;
  const int n_list = B.chg_list[0];
  const int* list = B.chg_list + 1;
  const int n_chunks = (n_list + KO_KC - 1) / KO_KC;
  if (n_chunks == 0) return;
  auto issue = [&](int c) {
    float4* dst = cs + (c & 1) * KO_KC * 256;
    for (int i = threadIdx.x; i < KO_KC * 256; i += 256) {
      const int kk = i >> 8, q = i & 255;                   // q-th float4 of the slice: row q/64, lane (q%64)/2, half q%2
      if (c * KO_KC + kk < n_list) {
        const int d = kk * 256 + (q >> 6) * 64 + (q & 1) * 32 + ((q & 63) >> 1);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst + d)),
                     "l"(C + size_t(list[c * KO_KC + kk]) * PD + q * 4) : "memory");
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  issue(0);
  float x[32];
  load_slice(X, dt, size_t(t) * PD + size_t(s) * SLICE, lane, x);
  for (int c = 0; c < n_chunks; ++c) {
    if (c + 1 < n_chunks) {
      issue(c + 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const float4* stage = cs + (c & 1) * KO_KC * 256;
#pragma unroll 2
    for (int kk = 0; kk < KO_KC; ++kk) {
      if (c * KO_KC + kk >= n_list) break;
      const int k = list[c * KO_KC + kk];
      const float p = slice_dot_smem(x, stage + kk * 256, lane);
      if (lane == 0 && t_raw < T) B.ab[(size_t(t) * K + k) * S + s] = p;
    }
    __syncthreads();
  }
}
// dists = sqrt((A_2 + B_2^T) - 2*AB); labels = argmin (first index, NaN wins); warp per row.  A row whose label moved marks
// both clusters dirty: only dirty clusters are recomputed by ko_update.
__device__ __forceinline__ void ko_assign_body(unsigned bid, KO B, int T, int K, int PD) {
  if (B.state[0]) return;
  const int t = bid * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const float a2 = B.a2t[t];
  float best = INFINITY;
  int besti = 0x7fffffff;
  for (int k = lane; k < K; k += 32) {
    const float ab = B.abt[size_t(t) * K + k], b2 = B.b2t[k];
    const float d = sqrtf(__fsub_rn(__fadd_rn(a2, b2), __fmul_rn(2.0f, ab)));
    if (besti == 0x7fffffff || argmin_better(d, k, best, besti)) { best = d; besti = k; }
  }
  warp_argmin(best, besti);
  if (lane == 0) {
    const int old = B.labels[t];
    if (old != besti) {
      B.dirty[besti] = 1;                 // benign races: every writer stores 1
      if (old >= 0) B.dirty[old] = 1;
      B.labels[t] = besti;
    }
  }
}
// warp per (cluster j, slice): weighted mean (sequential in t), refill of empty clusters, ||c_old - c_new||^2 partial.
// A cluster whose member set did not change since the previous iteration (and that was not empty, i.e. not refilled from
// a fresh random draw) would reproduce its centroid bit for bit: it is skipped (norm partial 0, weight sum unchanged).
// New values go to the staging buffer C[1]; ko_commit copies the changed rows into C[0] unless the loop stopped on the
// tolerance (the reference then keeps the OLD centroids).
__device__ __forceinline__ void ko_update_body(unsigned bid, KO B, const void* __restrict__ X, int dt, const float* __restrict__ w,
                                                        const int* __restrict__ refill_idx, int T, int K, int PD, int iter) {
  if (B.state[0]) return;
  const int S = PD / SLICE;
  const int unit = bid * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (unit >= K * S) return;
  const int j = unit / S, s = unit % S;
  if (iter > 0 && !B.dirty[j] && B.wprev[j] > 0.f) {
    if (lane == 0) B.normpart[unit] = 0.f;
    return;
  }
  const float* Cold = B.C[0] + size_t(j) * PD + s * SLICE;
  float* Cnew = B.C[1] + size_t(j) * PD + s * SLICE;
  float wsum_j = 0.f;
  int empties_before = 0;
  for (int c = lane; c <= j; c += 32) {
    float ws = 0.f;
    for (int t = 0; t < T; ++t)
      if (B.labels[t] == c) ws = __fadd_rn(ws, w[t]);
    if (c == j) wsum_j = ws;
    else if (!(ws > 0.f)) empties_before++;
  }
  wsum_j = butterfly_sum(wsum_j);
  empties_before = __reduce_add_sync(0xffffffffu, empties_before);
  float acc[32];
#pragma unroll
  for (int q = 0; q < 32; ++q) acc[q] = 0.f;
  if (wsum_j > 0.f) {
    for (int t = 0; t < T; ++t) {
      if (B.labels[t] != j) continue;
      const float wt = w[t];
      float x[32];
      load_slice(X, dt, size_t(t) * PD + size_t(s) * SLICE, lane, x);
#pragma unroll
      for (int q = 0; q < 32; ++q) acc[q] = __fadd_rn(acc[q], __fmul_rn(wt, x[q]));
    }
#pragma unroll
    for (int q = 0; q < 32; ++q) acc[q] = __fdiv_rn(acc[q], wsum_j);
  } else {
    load_slice(X, dt, size_t(refill_idx[B.state[3] + empties_before]) * PD + size_t(s) * SLICE, lane, acc);
  }
  float cold[32];
  load_slice(Cold, FVS_F32, 0, lane, cold);
  float nacc = 0.f;
  bool differs = false;
#pragma unroll
  for (int q = 0; q < 32; ++q) {
    const float d = __fsub_rn(cold[q], acc[q]);
    nacc = __fadd_rn(nacc, __fmul_rn(d, d));
    differs |= __float_as_uint(cold[q]) != __float_as_uint(acc[q]);
  }
  store_slice_f32(Cnew, lane, acc);
  nacc = butterfly_sum(nacc);
  differs = __any_sync(0xffffffffu, differs);
  if (lane == 0) {
    if (differs) B.chg_flag[j] = 1;      // benign race: every writer stores 1
    B.normpart[unit] = nacc;
    if (s == 0) B.wsum[j] = wsum_j;
  }
}
// one block: per-cluster norms (slices added in order: warp per cluster, coalesced loads + shuffle chain), then thread 0
// forms diff = sum_k ||c_k - c'_k||, takes the break decision and builds the change list of the next iteration
__device__ __forceinline__ void ko_converge_body(KO B, int K, int PD, int iter, int max_iter, float tol) {
  if (B.state[0]) return;
  const int S = PD / SLICE;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = warp; k < K; k += 32) {
    float acc = 0.f;
    for (int base = 0; base < S; base += 32) {
      const float v = base + lane < S ? B.normpart[size_t(k) * S + base + lane] : 0.f;
      const int n = min(32, S - base);
      for (int i = 0; i < n; ++i) acc = __fadd_rn(acc, __shfl_sync(0xffffffffu, v, i));
    }
    if (lane == 0) B.normt[k] = acc;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  float diff = 0.f;
  int n_empty = 0;
  for (int k = 0; k < K; ++k) {
    diff = __fadd_rn(diff, sqrtf(B.normt[k]));
    if (!(B.wsum[k] > 0.f)) n_empty++;
    B.wprev[k] = B.wsum[k];
    B.dirty[k] = 0;
  }
  B.state[2] = iter;
  B.state[3] += n_empty;
  int n_chg = 0;                               // rows to commit and next iteration's sweep list
  for (int k = 0; k < K; ++k)
    if (B.chg_flag[k]) { B.chg_list[1 + n_chg++] = k; B.chg_flag[k] = 0; }
  B.chg_list[0] = n_chg;
  if (diff < tol) {                            // `break` before `centroids = new_centroids`: nothing is committed
    B.state[0] = 1;
    B.state[4] = 1;
  } else {
    B.state[1] = iter + 1;                     // ko_commit of THIS iteration applies the change list
    if (iter == max_iter - 1) B.state[0] = 1;
  }
}
// centroids = new_centroids for the rows that changed, plus their |c|^2 slice partials: warp per (list entry, slice)
__device__ __forceinline__ void ko_commit_body(unsigned bid, KO B, int K, int PD, int iter, int max_iter) {
  if (B.state[1] != iter + 1) return;          // loop already over, or this iteration stopped on the tolerance
  const int S = PD / SLICE;
  const int unit = bid * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int n_list = B.chg_list[0];
  if (unit < n_list * S) {
    const int k = B.chg_list[1 + unit / S], s = unit % S;
    float x[32];
    load_slice(B.C[1] + size_t(k) * PD + size_t(s) * SLICE, FVS_F32, 0, lane, x);
    store_slice_f32(B.C[0] + size_t(k) * PD + size_t(s) * SLICE, lane, x);
    float acc = 0.f;
#pragma unroll
    for (int q = 0; q < 32; ++q) acc = __fadd_rn(acc, __fmul_rn(x[q], x[q]));
    acc = butterfly_sum(acc);
    if (lane == 0) B.b2[size_t(k) * S + s] = acc;
  }
}
// a plain copy: the result does not depend on how many blocks (nblk) share it
__device__ __forceinline__ void ko_finish_body(unsigned bid, unsigned nblk, KO B, float* __restrict__ C_out, float* __restrict__ wsum_out,
                                               int* __restrict__ labels_out, int* __restrict__ info_out, int T, int K, int PD) {
  const float4* src = reinterpret_cast<const float4*>(B.C[0]);
  float4* dst = reinterpret_cast<float4*>(C_out);
  const size_t n4 = size_t(K) * PD / 4;
  for (size_t i = bid * size_t(blockDim.x) + threadIdx.x; i < n4; i += size_t(nblk) * blockDim.x) dst[i] = src[i];
  if (bid == 0) {
    for (int i = threadIdx.x; i < K; i += blockDim.x) wsum_out[i] = B.wsum[i];
    for (int i = threadIdx.x; i < T; i += blockDim.x) labels_out[i] = B.labels[i];
    if (threadIdx.x == 0) {
      info_out[0] = B.state[2]; info_out[1] = B.state[3]; info_out[2] = B.state[4]; info_out[3] = 0;
    }
  }
}

// out[i, :] = cast(src_f32[idx[i], :]) ; idx int64; block bx of nbx covers a strided share of output row i, 4 elements per
// thread (row % 4 == 0)
__device__ __forceinline__ void gather_cast_body(unsigned bx, unsigned nbx, size_t i, const float* __restrict__ src,
                                                 const long long* __restrict__ idx, void* __restrict__ out, size_t row,
                                                 int out_dt) {
  const float4* s = reinterpret_cast<const float4*>(src + size_t(idx[i]) * row);
  for (size_t c = bx * size_t(blockDim.x) + threadIdx.x; c < row / 4; c += size_t(nbx) * blockDim.x) {
    const float4 v = s[c];
    if (out_dt == FVS_F32) {
      reinterpret_cast<float4*>(static_cast<float*>(out) + i * row)[c] = v;
    } else if (out_dt == FVS_BF16) {
      const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
      reinterpret_cast<uint2*>(static_cast<uint16_t*>(out) + i * row)[c] =
          make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
    } else {
      const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
      reinterpret_cast<uint2*>(static_cast<uint16_t*>(out) + i * row)[c] =
          make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
    }
  }
}

// ------------------------------------------------------------------------------------------------ k-means bookkeeping
// What weighted_kmeans_ordered_feature does on the host after the Lloyd loop (compress_functions.py:274-290), on the device:
// timestamp of a cluster = mean member row index, evaluated like Python's int / int (correctly rounded double) and stored as
// fp32 (torch.tensor of the list); clusters ordered by timestamp (stable, or the caller's replayed permutation); weights and
// timestamps permuted accordingly.  flags[0] = number of empty clusters (the reference raises ZeroDivisionError there).
// One block; integer atomics, so the result does not depend on thread order.
constexpr int kMaxFinalizeK = 1024;
__device__ __forceinline__ void ko_finalize_body(const int* __restrict__ labels, const float* __restrict__ wsum, int T, int K,
                                                 const long long* __restrict__ order_in, long long* __restrict__ sorted_idx,
                                                 float* __restrict__ ts_sorted, float* __restrict__ w_sorted,
                                                 int* __restrict__ flags) {
  __shared__ unsigned long long s_sum[kMaxFinalizeK];
  __shared__ int s_cnt[kMaxFinalizeK];
  __shared__ float s_ts[kMaxFinalizeK];
  __shared__ int s_empty;
  if (threadIdx.x == 0) s_empty = 0;
  for (int k = threadIdx.x; k < K; k += blockDim.x) { s_sum[k] = 0ull; s_cnt[k] = 0; }
  __syncthreads();
  for (int j = threadIdx.x; j < T; j += blockDim.x) {
    const int l = labels[j];
    atomicAdd(&s_cnt[l], 1);
    atomicAdd(&s_sum[l], (unsigned long long)j);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    if (s_cnt[k] == 0) { s_ts[k] = __int_as_float(0x7fc00000); atomicAdd(&s_empty, 1); }
    else s_ts[k] = float(double(s_sum[k]) / double(s_cnt[k]));
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    int src, dst;
    if (order_in) { dst = k; src = int(order_in[k]); }
    else {            // stable rank of cluster k (NaNs last)
      const float a = s_ts[k];
      int rank = 0;
      for (int j = 0; j < K; ++j) {
        const float b = s_ts[j];
        const bool before = (a != a) ? (b == b || j < k) : (b == b && (b < a || (b == a && j < k)));
        rank += before ? 1 : 0;
      }
      dst = rank; src = k;
    }
    sorted_idx[dst] = src;
    ts_sorted[dst] = s_ts[src];
    w_sorted[dst] = wsum[src];
  }
  if (threadIdx.x == 0) flags[0] = s_empty;
}

// ------------------------------------------------------------------------------------------------ spatial_enhance
// klarge_retrieve (vstream_qwen2vl_model.py:197-207, 231-238): for the k heaviest centroids c (rows klarge_idx of tem_x) and
// every bank frame b:  d = sqrt((|c|^2 + |b|^2) - 2 c.b), every op rounded to the features' 16-bit dtype dt, then argmin_b.
//   |v|^2 = dt( sum_f32( dt(v_i^2) ) ),  c.b = dt( sum_f32( c_i b_i ) )   (a 16-bit x 16-bit product is exact in fp32)
// Both sums run in the canonical slice order, so the oracle reproduces every bit.  The contraction is HBM-bound (k <= 64
// rows against t bank rows of P*D elements: ~0.5 flop/byte), so it runs as a split-K sweep on the CUDA cores: one block per
// 1024-element slice keeps the centroid slice in shared memory, streams the bank slice once and emits fp32 slice partials;
// seq_reduce adds the slices in order; the tail rounds, forms the distances and takes the argmin.
template <bool kBF16>
__device__ __forceinline__ void unpack8(const uint4 v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (kBF16) {
      f[2 * q] = __uint_as_float(w[q] << 16);
      f[2 * q + 1] = __uint_as_float(w[q] & 0xffff0000u);
    } else {
      const float2 p = __half22float2(*reinterpret_cast<const __half2*>(&w[q]));
      f[2 * q] = p.x;
      f[2 * q + 1] = p.y;
    }
  }
}
template <bool kBF16>
__device__ __forceinline__ float round16(float v) {
  return kBF16 ? __bfloat162float(__float2bfloat16_rn(v)) : __half2float(__float2half_rn(v));
}

// klarge_retrieve_cos (vstream_qwen2vl_model.py:208-215, 231-238): argmin_b of the cosine SIMILARITY of c and b (the
// reference takes the argmin of the similarity, i.e. the LEAST similar frame; mirrored as is):
//   |v| = dt( sqrt( sum_f32(v_i^2) ) )   (Tensor.norm accumulates the exact products in fp32),   vn_i = dt(v_i / |v|),
//   cos = dt( sum_f32( cn_i bn_i ) ),   all sums in the canonical slice order.
// Same sweep in two passes: kMode 1 emits the slice partials of the squared norms (unrounded products), the norms are
// finalised by klcos_norm, kMode 2 normalises both operands on the fly (centroids when they are staged in shared
// memory, bank rows after the unpack) and emits the dot-product partials.  kMode 0 is the Euclidean form.
//
// partial layout [units, S]: unit t*k + kk = c_kk . b_t, unit t_total*k + t = |b_t|^2, unit t_total*k + t_total + kk = |c_kk|^2
template <bool kBF16>
__device__ __forceinline__ uint32_t pack2_16(float a, float b) {
  if (kBF16) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
// kRange: the launch sweeps bank rows [t_first, t_first + rows) of the t_total, row t_first at `bank` (one tier of a
// two-tier bank, DESIGN.md §3.13: the HBM rows, or one pinned host chunk through its mapped pointer), and writes their
// partials at the rows' global indices; the launch whose range starts at row 0 writes the |c|^2 partials.  A row's
// partials do not depend on the block or launch that computes them, so any split of the rows gives the same bits.
// Without kRange the launch sweeps the whole bank (t_first 0, rows t_total) and ignores the last two arguments.
// (s, by, ny): the slice, the row split and the number of row splits of the block
template <bool kBF16, int kMode, bool kRange>
__device__ __forceinline__ void klarge_partial_body(unsigned s_, unsigned by, unsigned ny, uint4* cs,
                                                    const uint16_t* __restrict__ tem_x, const long long* __restrict__ klarge_idx,
                                                    const uint16_t* __restrict__ bank, float* __restrict__ part, int k,
                                                    int t_total, int PD, const float* __restrict__ norms, int range_first,
                                                    int range_rows) {
  const int t_first = kRange ? range_first : 0, rows = kRange ? range_rows : t_total;
  // cs: [k][128] uint4 of dynamic shared memory = k rows of 1024 16-bit elements
  const int S = PD / SLICE, s = s_;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // norms (kMode 2): [t_total] bank norms then [k] centroid norms, fp32 holding the dtype-rounded values
  for (int i = threadIdx.x; i < k * 128; i += 256) {
    const int kk = i >> 7, c = i & 127;
    uint4 v = *reinterpret_cast<const uint4*>(tem_x + size_t(klarge_idx[kk]) * PD + size_t(s) * SLICE + c * 8);
    if (kMode == 2) {
      float f[8];
      unpack8<kBF16>(v, f);
      const float n = norms[t_total + kk];
      v.x = pack2_16<kBF16>(__fdiv_rn(f[0], n), __fdiv_rn(f[1], n));
      v.y = pack2_16<kBF16>(__fdiv_rn(f[2], n), __fdiv_rn(f[3], n));
      v.z = pack2_16<kBF16>(__fdiv_rn(f[4], n), __fdiv_rn(f[5], n));
      v.w = pack2_16<kBF16>(__fdiv_rn(f[6], n), __fdiv_rn(f[7], n));
    }
    cs[i] = v;
  }
  __syncthreads();
  float* p_ab = part;
  float* p_b2 = part + size_t(t_total) * k * S;
  float* p_a2 = p_b2 + size_t(t_total) * S;
  const int rows_per = (rows + ny - 1) / ny;                       // bank rows of this block
  const int t_beg = t_first + by * rows_per, t_end = min(t_first + rows, t_beg + rows_per);
  if (kMode != 2 && by == 0 && t_first == 0) {
    for (int kk = warp; kk < k; kk += 8) {                  // |c|^2 slice partials
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float f[8];
        unpack8<kBF16>(cs[kk * 128 + i * 32 + lane], f);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          acc = kMode == 1 ? __fmaf_rn(f[e], f[e], acc) : __fadd_rn(acc, round16<kBF16>(__fmul_rn(f[e], f[e])));
      }
      acc = butterfly_sum(acc);
      if (lane == 0) p_a2[size_t(kk) * S + s] = acc;
    }
  }
  // register tile: 2 bank rows x 2 centroids per pass = 4 independent accumulation chains, each centroid unpack shared by
  // both rows
  for (int t0 = t_beg + warp * 2; t0 < t_end; t0 += 16) {
    const bool two = t0 + 1 < t_end;
    float x0[32], x1[32];
    const uint4* src0 = reinterpret_cast<const uint4*>(bank + size_t(t0 - t_first) * PD + size_t(s) * SLICE);
    const uint4* src1 = reinterpret_cast<const uint4*>(bank + size_t((two ? t0 + 1 : t0) - t_first) * PD + size_t(s) * SLICE);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      unpack8<kBF16>(src0[i * 32 + lane], x0 + i * 8);
      unpack8<kBF16>(src1[i * 32 + lane], x1 + i * 8);
    }
    if (kMode == 2) {
      const float n0 = norms[t0], n1 = norms[two ? t0 + 1 : t0];
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        x0[q] = round16<kBF16>(__fdiv_rn(x0[q], n0));
        x1[q] = round16<kBF16>(__fdiv_rn(x1[q], n1));
      }
    } else {
      float b20 = 0.f, b21 = 0.f;
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        b20 = kMode == 1 ? __fmaf_rn(x0[q], x0[q], b20) : __fadd_rn(b20, round16<kBF16>(__fmul_rn(x0[q], x0[q])));
        b21 = kMode == 1 ? __fmaf_rn(x1[q], x1[q], b21) : __fadd_rn(b21, round16<kBF16>(__fmul_rn(x1[q], x1[q])));
      }
      b20 = butterfly_sum(b20);
      b21 = butterfly_sum(b21);
      if (lane == 0) {
        p_b2[size_t(t0) * S + s] = b20;
        if (two) p_b2[size_t(t0 + 1) * S + s] = b21;
      }
    }
    if (kMode == 1) continue;
    for (int k0 = 0; k0 < k; k0 += 2) {
      const int k1 = min(k0 + 1, k - 1);
      float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float f0[8], f1[8];
        unpack8<kBF16>(cs[k0 * 128 + i * 32 + lane], f0);
        unpack8<kBF16>(cs[k1 * 128 + i * 32 + lane], f1);
#pragma unroll
        for (int e = 0; e < 8; ++e) {                        // exact 16-bit products: fma == mul then add
          a00 = __fmaf_rn(x0[i * 8 + e], f0[e], a00);
          a01 = __fmaf_rn(x0[i * 8 + e], f1[e], a01);
          a10 = __fmaf_rn(x1[i * 8 + e], f0[e], a10);
          a11 = __fmaf_rn(x1[i * 8 + e], f1[e], a11);
        }
      }
      a00 = butterfly_sum(a00); a01 = butterfly_sum(a01); a10 = butterfly_sum(a10); a11 = butterfly_sum(a11);
      if (lane == 0) {
        p_ab[(size_t(t0) * k + k0) * S + s] = a00;
        if (k0 + 1 < k) p_ab[(size_t(t0) * k + k0 + 1) * S + s] = a01;
        if (two) {
          p_ab[(size_t(t0 + 1) * k + k0) * S + s] = a10;
          if (k0 + 1 < k) p_ab[(size_t(t0 + 1) * k + k0 + 1) * S + s] = a11;
        }
      }
    }
  }
}
// one tier of a bank with host rows: bank rows [range_first, range_first + range_rows) (a bank wholly in HBM is swept by
// klarge_multi_kernel)
template <bool kBF16, int kMode>
__global__ void __launch_bounds__(256) klarge_partial_kernel(const uint16_t* __restrict__ tem_x, const long long* __restrict__ klarge_idx,
                                                             const uint16_t* __restrict__ bank, float* __restrict__ part, int k,
                                                             int t_total, int PD, const float* __restrict__ norms,
                                                             int range_first, int range_rows) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  klarge_partial_body<kBF16, kMode, true>(blockIdx.x, blockIdx.y, gridDim.y, reinterpret_cast<uint4*>(smem_raw), tem_x,
                                          klarge_idx, bank, part, k, t_total, PD, norms, range_first, range_rows);
}
// warp per centroid: distances over the bank (lane-strided) and argmin (NaN from a negative radicand wins, as in torch)
template <bool kBF16>
__device__ __forceinline__ void klarge_tail_body(unsigned kk_, const float* __restrict__ tot, int k, int t_total,
                                                 long long* __restrict__ idx, float* __restrict__ dist_out) {
  const int kk = kk_, lane = threadIdx.x;
  const float* ab = tot;
  const float* b2 = tot + size_t(t_total) * k;
  const float* a2 = b2 + t_total;
  const float a = round16<kBF16>(a2[kk]);
  float best = INFINITY;
  int besti = 0x7fffffff;
  for (int t = lane; t < t_total; t += 32) {
    const float sum = round16<kBF16>(__fadd_rn(a, round16<kBF16>(b2[t])));
    const float m = round16<kBF16>(__fmul_rn(2.0f, round16<kBF16>(ab[size_t(t) * k + kk])));
    const float d = round16<kBF16>(sqrtf(round16<kBF16>(__fsub_rn(sum, m))));
    if (dist_out) dist_out[size_t(kk) * t_total + t] = d;
    if (besti == 0x7fffffff || argmin_better(d, t, best, besti)) { best = d; besti = t; }
  }
  warp_argmin(best, besti);
  if (lane == 0) idx[kk] = besti;
}

// norms[i] = dt(sqrt(sumsq[i])) for the t bank rows followed by the k centroids (in place over the reduced totals)
template <bool kBF16>
__device__ __forceinline__ void klcos_norm_body(unsigned bid, float* __restrict__ v, int n) {
  const int i = bid * blockDim.x + threadIdx.x;
  if (i < n) v[i] = round16<kBF16>(sqrtf(v[i]));
}
// warp per centroid: similarities over the bank and their argmin (a zero row gives 0/0 = NaN, which wins as in torch)
template <bool kBF16>
__device__ __forceinline__ void klarge_cos_tail_body(unsigned kk_, const float* __restrict__ ab, int k, int t_total,
                                                     long long* __restrict__ idx, float* __restrict__ sim_out) {
  const int kk = kk_, lane = threadIdx.x;
  float best = INFINITY;
  int besti = 0x7fffffff;
  for (int t = lane; t < t_total; t += 32) {
    const float c = round16<kBF16>(ab[size_t(t) * k + kk]);
    if (sim_out) sim_out[size_t(kk) * t_total + t] = c;
    if (besti == 0x7fffffff || argmin_better(c, t, best, besti)) { best = c; besti = t; }
  }
  warp_argmin(best, besti);
  if (lane == 0) idx[kk] = besti;
}

// ------------------------------------------------------------------------------------------------ AM-RoPE
// pos[c, n] for the n-th visual token: DAM (spa) tokens first, then CSM (tem) tokens offset by spa_size
// (get_mm_index_with_positions, vstream_qwen2vl_model.py:265-271).  All int64.
__global__ void am_rope_kernel(const long long* __restrict__ spa_pos, int spa_t, int spa_h, int spa_w,
                               const long long* __restrict__ tem_pos, int tem_t, int tem_h, int tem_w, long long start_id,
                               long long* __restrict__ out, int total) {
  const int spa_size = spa_t * spa_h * spa_w;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < total; n += gridDim.x * blockDim.x) {
    long long tt, hh, ww;
    if (n < spa_size) {
      tt = spa_pos[n / (spa_h * spa_w)]; hh = (n / spa_w) % spa_h; ww = n % spa_w;
    } else {
      const int m = n - spa_size;
      tt = tem_pos[m / (tem_h * tem_w)] + spa_size; hh = (m / tem_w) % tem_h + spa_size; ww = m % tem_w + spa_size;
    }
    out[n] = start_id + tt;
    out[total + n] = start_id + hh;
    out[2 * size_t(total) + n] = start_id + ww;
  }
}

__host__ __device__ inline size_t al(size_t v) { return (v + 255) & ~size_t(255); }

// the device state of one fvs_qwen_kmeans call, carved from its workspace (fvs_qwen_kmeans_workspace_bytes)
__host__ __device__ inline KO ko_carve(void* workspace, int T, int K, int PD) {
  const size_t S = size_t(PD) / SLICE, TK = size_t(T) * K + K;
  uint8_t* p = (uint8_t*)workspace;
  KO B;
  B.state = (int*)p; p += al(32);
  B.C[0] = (float*)p; p += al(size_t(K) * PD * 4);
  B.C[1] = (float*)p; p += al(size_t(K) * PD * 4);
  B.ab = (float*)p; p += al(TK * S * 4);
  B.b2 = B.ab + size_t(T) * K * S;
  B.abt = (float*)p; p += al(TK * 4);
  B.b2t = B.abt + size_t(T) * K;
  B.a2 = (float*)p; p += al(size_t(T) * S * 4);
  B.a2t = (float*)p; p += al(size_t(T) * 4);
  B.normpart = (float*)p; p += al(size_t(K) * S * 4);
  B.normt = (float*)p; p += al(size_t(K) * 4);
  B.wsum = (float*)p; p += al(size_t(K) * 4);
  B.labels = (int*)p; p += al(size_t(T) * 4);
  B.chg_flag = (int*)p; p += al((size_t(K) + 1) * 4);
  B.chg_list = (int*)p; p += al((size_t(K) + 1) * 4);
  B.dirty = (int*)p; p += al((size_t(K) + 1) * 4);
  B.wprev = (float*)p;
  return B;
}

// ------------------------------------------------------------------------------------------------ job tables
// Every kernel of the CSM chain and of the klarge retrieval is launched over a job table (DESIGN.md §3.17): job j owns
// blocks [first[j], first[j+1]) of one flat grid and calls the per-block body with its local block index.  A job gets the
// same blocks in the same order whatever the other jobs are, so its reductions run in the same order however the jobs are
// grouped into launches.  A single call is the one-job table: kJobs = 1 has no job scan and a small parameter block; a
// group of more jobs runs the kJobs = FVS_QWEN_MEM_JOBS_PER_LAUNCH instantiation.  The table travels as a
// __grid_constant__ kernel parameter (under 4 KB).
constexpr int kMemJobs = FVS_QWEN_MEM_JOBS_PER_LAUNCH;
struct MemJobDev {
  const void* X;
  const float* w;
  const int* init_idx;
  const int* refill_idx;
  int* uniq_idx;
  int* n_unique;
  void* uniq_ws;
  float* C;
  float* wsum;
  int* labels;
  int* info;
  void* km_ws;
  const long long* order_in;
  long long* sorted_idx;
  float* ts;
  float* w_sorted;
  int* flags;
  void* out;
  int T, K, PD, dt, max_iter, out_dt;
  float tol;
  long long row_elems;     // gather: elements per row of C and out (PD in a table)
};
template <int kJobs>
struct MemLaunch {
  MemJobDev job[kJobs];
  int first[kJobs + 1];    // block offsets of the launched kernel
  int n, it, finish_blocks;
};
enum MemStage { kLex, kOrder, kInit, kXnorm, kA2, kPartial, kReduce, kAssign, kUpdate, kConverge, kCommit, kFinish, kFinalize,
                kGather };

// blocks of job J in stage st (iteration it); 0 once the job's loop is over
__host__ __device__ inline int gather_bx(long long row) { const long long bx = (row / 4 + 255) / 256; return bx > 64 ? 64 : int(bx); }
inline int mem_stage_blocks(const MemJobDev& J, int st, int it, int finish_blocks) {
  const int S = J.PD / SLICE, iters = J.max_iter == 0 ? 1 : J.max_iter;
  const bool loop = it < iters, upd = J.max_iter > 0 && it < J.max_iter;
  switch (st) {
    case kLex: return J.T * J.T;
    case kOrder: case kFinalize: return 1;
    case kInit: return (J.K * S + 7) / 8;
    case kXnorm: return (J.T * S + 7) / 8;
    case kA2: return (J.T + 7) / 8;
    case kPartial: return loop ? ((J.T + 7) / 8) * S : 0;
    case kReduce: return loop ? int((size_t(J.T) * J.K + J.K + 7) / 8) : 0;
    case kAssign: return loop ? (J.T + 7) / 8 : 0;
    case kUpdate: case kCommit: return upd ? (J.K * S + 7) / 8 : 0;
    case kConverge: return upd ? 1 : 0;
    case kFinish: return finish_blocks;
    case kGather: return gather_bx(J.row_elems) * J.K;
  }
  return 0;
}

// Blocks of 256 per SM that the heaviest one-job stages keep: without a bound a one-job kernel spends extra registers on
// its job descriptor and loses blocks per SM.  The Lloyd update runs at most 80 registers (3 blocks); the klarge bank
// sweeps are bounded by kl_min_blocks.  A minBlocks of 0 leaves an instantiation unbounded, as every many-job one is.
constexpr int mem_min_blocks(int jobs, int stage) { return jobs == 1 && stage == kUpdate ? 3 : 0; }
template <int kJobs, int kStage>
__global__ void __launch_bounds__(kStage == kConverge ? 1024 : 256, mem_min_blocks(kJobs, kStage))
    mem_multi_kernel(const __grid_constant__ MemLaunch<kJobs> L) {
  extern __shared__ __align__(16) uint8_t mm_smem[];
  int j = 0;
  if constexpr (kJobs > 1)
    while (j + 1 < L.n && blockIdx.x >= unsigned(L.first[j + 1])) ++j;
  const MemJobDev& J = L.job[j];
  const unsigned b = blockIdx.x - unsigned(L.first[j]);
  if constexpr (kStage == kLex) {
    lex_compare_body(int(b % unsigned(J.T)), int(b / unsigned(J.T)), J.X, J.T, J.PD, J.dt, (signed char*)J.uniq_ws);
  } else if constexpr (kStage == kOrder) {
    unique_order_body((const signed char*)J.uniq_ws, J.T, J.uniq_idx, J.n_unique, reinterpret_cast<int*>(mm_smem));
  } else if constexpr (kStage == kFinalize) {
    ko_finalize_body(J.labels, J.wsum, J.T, J.K, J.order_in, J.sorted_idx, J.ts, J.w_sorted, J.flags);
  } else if constexpr (kStage == kGather) {
    const unsigned bx = gather_bx(J.row_elems);
    gather_cast_body(b % bx, bx, b / bx, J.C, J.sorted_idx, J.out, size_t(J.row_elems), J.out_dt);
  } else {
    const KO B = ko_carve(J.km_ws, J.T, J.K, J.PD);
    const int S = J.PD / SLICE;
    if constexpr (kStage == kInit) ko_init_body(b, B, J.X, J.dt, J.uniq_idx, J.init_idx, J.T, J.K, J.PD);
    else if constexpr (kStage == kXnorm) ko_xnorm_body(b, B, J.X, J.dt, J.T, J.PD);
    else if constexpr (kStage == kA2) seq_reduce_body(b, B.a2, B.a2t, J.T, S, nullptr);
    else if constexpr (kStage == kPartial) ko_partial_body(b, reinterpret_cast<float4*>(mm_smem), B, J.X, J.dt, J.T, J.K, J.PD);
    else if constexpr (kStage == kReduce) seq_reduce_body(b, B.ab, B.abt, J.T * J.K + J.K, S, B.state);
    else if constexpr (kStage == kAssign) ko_assign_body(b, B, J.T, J.K, J.PD);
    else if constexpr (kStage == kUpdate) ko_update_body(b, B, J.X, J.dt, J.w, J.refill_idx, J.T, J.K, J.PD, L.it);
    else if constexpr (kStage == kConverge) ko_converge_body(B, J.K, J.PD, L.it, J.max_iter, J.tol);
    else if constexpr (kStage == kCommit) ko_commit_body(b, B, J.K, J.PD, L.it, J.max_iter);
    else if constexpr (kStage == kFinish) ko_finish_body(b, L.finish_blocks, B, J.C, J.wsum, J.labels, J.info, J.T, J.K, J.PD);
  }
}

// the klarge retrieval: a sweep of the bank, the slice reductions and the tail, each one flat grid over the jobs
struct KlJobDev {
  const uint16_t* tem_x;
  const long long* klarge_idx;
  const uint16_t* bank;
  float* part;
  float* tot;
  long long* idx;
  float* dist;
  int k, t_total, PD, nsplit;
};
template <int kJobs>
struct KlLaunch {
  KlJobDev job[kJobs];
  int first[kJobs + 1];
  int n;
};
enum KlStage { kKlSweep0, kKlSweep1, kKlSweep2, kKlReduceAll, kKlReduceNorms, kKlNorms, kKlReduceAb, kKlTail, kKlCosTail };
// launch bounds of the one-job Euclidean and cosine bank sweeps (see mem_min_blocks): bf16 Euclidean at most 64
// registers (4 blocks of 256 per SM), the others at most 96 (2 blocks of up to 320 threads per SM; a 256-thread sweep
// runs 2 blocks per SM either way, and a bound of 80 would spill)
constexpr int kl_min_blocks(int jobs, bool bf16, int stage) {
  return jobs > 1 || (stage != kKlSweep0 && stage != kKlSweep2) ? 0 : bf16 && stage == kKlSweep0 ? 4 : 2;
}
constexpr int kl_max_threads(int jobs, bool bf16, int stage) { return kl_min_blocks(jobs, bf16, stage) == 2 ? 320 : 256; }
inline int kl_stage_blocks(const KlJobDev& J, int st) {
  const int S = J.PD / SLICE;
  const size_t n_ab = size_t(J.t_total) * J.k, n_norm = size_t(J.t_total) + J.k;
  switch (st) {
    case kKlSweep0: case kKlSweep1: case kKlSweep2: return S * J.nsplit;
    case kKlReduceAll: return int((n_ab + n_norm + 7) / 8);
    case kKlReduceNorms: return int((n_norm + 7) / 8);
    case kKlNorms: return int((n_norm + 255) / 256);
    case kKlReduceAb: return int((n_ab + 7) / 8);
    case kKlTail: case kKlCosTail: return J.k;
  }
  return 0;
}
template <int kJobs, bool kBF16, int kStage>
__global__ void __launch_bounds__(kl_max_threads(kJobs, kBF16, kStage), kl_min_blocks(kJobs, kBF16, kStage))
    klarge_multi_kernel(const __grid_constant__ KlLaunch<kJobs> L) {
  extern __shared__ __align__(16) uint8_t kl_smem[];
  int j = 0;
  if constexpr (kJobs > 1)
    while (j + 1 < L.n && blockIdx.x >= unsigned(L.first[j + 1])) ++j;
  const KlJobDev& J = L.job[j];
  const unsigned b = blockIdx.x - unsigned(L.first[j]);
  const unsigned S = J.PD / SLICE;
  const size_t n_ab = size_t(J.t_total) * J.k, n_norm = size_t(J.t_total) + J.k;
  uint4* cs = reinterpret_cast<uint4*>(kl_smem);
  if constexpr (kStage == kKlSweep0 || kStage == kKlSweep1 || kStage == kKlSweep2) {
    constexpr int kMode = kStage - kKlSweep0;
    klarge_partial_body<kBF16, kMode, false>(b % S, b / S, J.nsplit, cs, J.tem_x, J.klarge_idx, J.bank, J.part, J.k,
                                             J.t_total, J.PD, kMode == 2 ? J.tot + n_ab : nullptr, 0, J.t_total);
  } else if constexpr (kStage == kKlReduceAll) {
    seq_reduce_body(b, J.part, J.tot, int(n_ab + n_norm), S, nullptr);
  } else if constexpr (kStage == kKlReduceNorms) {
    seq_reduce_body(b, J.part + n_ab * S, J.tot + n_ab, int(n_norm), S, nullptr);
  } else if constexpr (kStage == kKlNorms) {
    klcos_norm_body<kBF16>(b, J.tot + n_ab, int(n_norm));
  } else if constexpr (kStage == kKlReduceAb) {
    seq_reduce_body(b, J.part, J.tot, int(n_ab), S, nullptr);
  } else if constexpr (kStage == kKlTail) {
    klarge_tail_body<kBF16>(b, J.tot, J.k, J.t_total, J.idx, J.dist);
  } else {
    klarge_cos_tail_body<kBF16>(b, J.tot, J.k, J.t_total, J.idx, J.dist);
  }
}

}  // namespace qwen
}  // namespace fvs

using namespace fvs;
using namespace fvs::qwen;

namespace {
// the output byte ranges of a job table: no byte may belong to two jobs
struct JobOutputs {
  struct Range { uintptr_t lo, hi; int job; };
  std::vector<Range> r;
  void add(const void* p, size_t bytes, int job) { r.push_back({uintptr_t(p), uintptr_t(p) + bytes, job}); }
  int check(const char* api) const {
    for (size_t a = 0; a < r.size(); ++a)
      for (size_t b = a + 1; b < r.size(); ++b)
        FVS_REQUIRE(r[a].job == r[b].job || r[a].hi <= r[b].lo || r[b].hi <= r[a].lo, "%s: jobs %d and %d share an output",
                    api, r[a].job, r[b].job);
    return FVS_OK;
  }
};

// ---- the CSM chain
enum MemCall { kCallUnique, kCallKmeans, kCallFinalize, kCallGather };

bool known_dtype(int dt) { return dt == FVS_F16 || dt == FVS_BF16 || dt == FVS_F32; }

// the checks of one call of the chain, reported as `who` ("fvs_qwen_kmeans", or "fvs_qwen_kmeans_multi: job 3");
// ws_bytes: the call's workspace (unique rows, k-means)
int check_mem_call(const char* who, const MemJobDev& J, size_t ws_bytes, int call) {
  if (call == kCallUnique) {
    FVS_REQUIRE(J.X && J.uniq_idx && J.n_unique && J.uniq_ws, "%s: null pointer", who);
    FVS_REQUIRE(J.T > 0 && J.T <= 4096 && J.PD > 0, "%s: bad shape T=%d PD=%d", who, J.T, J.PD);
    FVS_REQUIRE(ws_bytes >= fvs_qwen_unique_workspace_bytes(J.T), "%s: workspace too small", who);
  } else if (call == kCallKmeans) {
    FVS_REQUIRE(J.X && J.w && J.init_idx && J.refill_idx && J.C && J.wsum && J.labels && J.info && J.km_ws,
                "%s: null pointer", who);
    FVS_REQUIRE(known_dtype(J.dt), "%s: bad x dtype", who);
    FVS_REQUIRE(J.T > 0 && J.K > 0 && J.K <= J.T, "%s: need 0 < K <= T (T=%d K=%d)", who, J.T, J.K);
    FVS_REQUIRE(J.PD > 0 && J.PD % SLICE == 0, "%s: PD (%d) must be a positive multiple of %d", who, J.PD, SLICE);
    FVS_REQUIRE(J.max_iter >= 0 && J.max_iter <= 1000, "%s: bad max_iter", who);
    FVS_REQUIRE(ws_bytes >= fvs_qwen_kmeans_workspace_bytes(J.T, J.K, J.PD), "%s: workspace too small", who);
  } else if (call == kCallFinalize) {
    FVS_REQUIRE(J.labels && J.wsum && J.sorted_idx && J.ts && J.w_sorted && J.flags, "%s: null pointer", who);
    FVS_REQUIRE(J.T > 0 && J.K > 0 && J.K <= kMaxFinalizeK, "%s: need T > 0, 0 < K <= %d (T=%d K=%d)", who, kMaxFinalizeK,
                J.T, J.K);
  } else {
    FVS_REQUIRE(J.C && J.sorted_idx && J.out, "%s: null pointer", who);
    FVS_REQUIRE(J.K > 0 && J.K <= 65535 && J.row_elems > 0, "%s: need 0 < n <= 65535 rows, row_elems > 0 (n=%d)", who, J.K);
    FVS_REQUIRE(J.row_elems % 4 == 0, "%s: row_elems must be a multiple of 4", who);
  }
  return FVS_OK;
}

int lloyd_blocks(const fvs_qwen_mem_job& j) { return ((j.T + 7) / 8) * (j.PD / SLICE); }

// jobs in order, at most kMemJobs per group and, with budget > 0, at most `budget` Lloyd-sweep blocks (a larger job alone)
int mem_groups(const fvs_qwen_mem_job* jobs, int n, int budget, int32_t* blocks, int32_t* groups) {
  int g = 0, in_group = 0;
  long long sum = 0;
  for (int i = 0; i < n; ++i) {
    const int b = lloyd_blocks(jobs[i]);
    if (in_group && (in_group == kMemJobs || (budget > 0 && sum + b > budget))) {
      ++g;
      in_group = 0;
      sum = 0;
    }
    blocks[i] = b;
    groups[i] = g;
    ++in_group;
    sum += b;
  }
  return g + 1;
}

MemJobDev mem_job_dev(const fvs_qwen_mem_job& j) {
  return MemJobDev{j.X, j.w, j.init_idx, j.refill_idx, j.uniq_idx, j.n_unique, j.uniq_workspace, j.C, j.wsum, j.labels,
                   j.info, j.km_workspace, (const long long*)j.order_in, (long long*)j.sorted_idx, j.ts, j.w_sorted, j.flags,
                   j.out, j.T, j.K, j.PD, j.x_dtype, j.max_iter, j.out_dtype, j.tol, j.PD};
}

// one launch of stage kStage over the group in L (skipped when no job has blocks in it)
template <int kJobs, int kStage>
int mem_launch(MemLaunch<kJobs>& L, int threads, size_t smem, cudaStream_t stream, const char* name) {
  L.first[0] = 0;
  for (int j = 0; j < L.n; ++j) L.first[j + 1] = L.first[j] + mem_stage_blocks(L.job[j], kStage, L.it, L.finish_blocks);
  if (L.first[L.n] == 0) return FVS_OK;
  if constexpr (kStage == kPartial) {
    static bool attr = false;   // per instantiation
    if (!attr) {
      FVS_CUDA_OK(cudaFuncSetAttribute(mem_multi_kernel<kJobs, kPartial>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       KO_PARTIAL_SMEM));
      attr = true;
    }
  }
  mem_multi_kernel<kJobs, kStage><<<L.first[L.n], threads, smem, stream>>>(L);
  FVS_CHECK_LAUNCH(name);
  return FVS_OK;
}

// the launch sequence of `call` for one group of n <= kJobs jobs
template <int kJobs>
int mem_group(const MemJobDev* jobs, int n, int call, cudaStream_t stream) {
  MemLaunch<kJobs> L;
  L.n = n;
  L.it = 0;
  L.finish_blocks = 1;
  int max_T = 1, iters = 0, r;
  size_t max_row4 = 1;
  for (int j = 0; j < n; ++j) {
    L.job[j] = jobs[j];
    max_T = std::max(max_T, jobs[j].T);
    iters = std::max(iters, jobs[j].max_iter == 0 ? 1 : jobs[j].max_iter);
    max_row4 = std::max(max_row4, size_t(jobs[j].K) * jobs[j].PD / 4);
  }
  if (call == kCallUnique) {
    if ((r = mem_launch<kJobs, kLex>(L, 256, 0, stream, "mem_multi_kernel<lex_compare>"))) return r;
    return mem_launch<kJobs, kOrder>(L, 256, size_t(max_T) * sizeof(int), stream, "mem_multi_kernel<unique_order>");
  }
  if (call == kCallFinalize) return mem_launch<kJobs, kFinalize>(L, 256, 0, stream, "mem_multi_kernel<ko_finalize>");
  if (call == kCallGather) return mem_launch<kJobs, kGather>(L, 256, 0, stream, "mem_multi_kernel<gather_cast>");
  if ((r = mem_launch<kJobs, kInit>(L, 256, 0, stream, "mem_multi_kernel<ko_init>"))) return r;
  if ((r = mem_launch<kJobs, kXnorm>(L, 256, 0, stream, "mem_multi_kernel<ko_xnorm>"))) return r;
  if ((r = mem_launch<kJobs, kA2>(L, 256, 0, stream, "mem_multi_kernel<seq_reduce>"))) return r;
  // 6 launches per iteration, all early-exit once a job's device-side loop is over; a job whose host-side loop is over
  // (max_iter == 0: one assignment, no update) has no blocks
  for (int it = 0; it < iters; ++it) {
    L.it = it;
    if ((r = mem_launch<kJobs, kPartial>(L, 256, KO_PARTIAL_SMEM, stream, "mem_multi_kernel<ko_partial>"))) return r;
    if ((r = mem_launch<kJobs, kReduce>(L, 256, 0, stream, "mem_multi_kernel<seq_reduce>"))) return r;
    if ((r = mem_launch<kJobs, kAssign>(L, 256, 0, stream, "mem_multi_kernel<ko_assign>"))) return r;
    if ((r = mem_launch<kJobs, kUpdate>(L, 256, 0, stream, "mem_multi_kernel<ko_update>"))) return r;
    if ((r = mem_launch<kJobs, kConverge>(L, 1024, 0, stream, "mem_multi_kernel<ko_converge>"))) return r;
    if ((r = mem_launch<kJobs, kCommit>(L, 256, 0, stream, "mem_multi_kernel<ko_commit>"))) return r;
  }
  // the result copy is split evenly: its bits do not depend on the number of blocks
  L.finish_blocks = int(std::min<size_t>(std::max(1, device_sm_count() * 8 / n), (max_row4 + 255) / 256));
  return mem_launch<kJobs, kFinish>(L, 256, 0, stream, "mem_multi_kernel<ko_finish>");
}
int mem_run(const MemJobDev* jobs, int n, int call, cudaStream_t stream) {
  return n == 1 ? mem_group<1>(jobs, 1, call, stream) : mem_group<kMemJobs>(jobs, n, call, stream);
}

// a single call of the chain: the one-job table
int mem_single(const char* who, const MemJobDev& J, size_t ws_bytes, int call, fvs_stream_t stream) {
  const int r = check_mem_call(who, J, ws_bytes, call);
  return r ? r : mem_run(&J, 1, call, (cudaStream_t)stream);
}

int mem_table(const char* api, const fvs_qwen_mem_job* jobs, int n, int budget, fvs_stream_t stream, int call) {
  FVS_REQUIRE(jobs && n > 0 && budget >= 0, "%s: need a job table, n_jobs > 0 and budget >= 0", api);
  std::vector<MemJobDev> dev(n);
  JobOutputs out;
  for (int i = 0; i < n; ++i) {
    const fvs_qwen_mem_job& j = jobs[i];
    char who[96];
    snprintf(who, sizeof who, "%s: job %d", api, i);
    // the table's own limits: the shapes fvs_qwen_mem_plan takes, and the dtypes the single calls leave unchecked
    FVS_REQUIRE(j.T > 0 && j.T <= 4096 && j.K > 0 && j.K <= j.T && j.K <= kMaxFinalizeK,
                "%s: need 0 < T <= 4096, 0 < K <= min(T, %d) (T=%d K=%d)", who, kMaxFinalizeK, j.T, j.K);
    FVS_REQUIRE(j.PD > 0 && j.PD % SLICE == 0, "%s: PD (%d) must be a positive multiple of %d", who, j.PD, SLICE);
    FVS_REQUIRE(call != kCallUnique || known_dtype(j.x_dtype), "%s: bad x dtype", who);
    FVS_REQUIRE(call != kCallGather || known_dtype(j.out_dtype), "%s: bad out dtype", who);
    dev[i] = mem_job_dev(j);
    const int r = check_mem_call(who, dev[i], call == kCallUnique ? j.uniq_workspace_bytes : j.km_workspace_bytes, call);
    if (r) return r;
    if (call == kCallUnique) {
      out.add(j.uniq_idx, size_t(j.T) * 4, i);
      out.add(j.n_unique, 4, i);
      out.add(j.uniq_workspace, fvs_qwen_unique_workspace_bytes(j.T), i);
    } else if (call == kCallKmeans) {
      out.add(j.C, size_t(j.K) * j.PD * 4, i);
      out.add(j.wsum, size_t(j.K) * 4, i);
      out.add(j.labels, size_t(j.T) * 4, i);
      out.add(j.info, 16, i);
      out.add(j.km_workspace, fvs_qwen_kmeans_workspace_bytes(j.T, j.K, j.PD), i);
    } else if (call == kCallFinalize) {
      out.add(j.sorted_idx, size_t(j.K) * 8, i);
      out.add(j.ts, size_t(j.K) * 4, i);
      out.add(j.w_sorted, size_t(j.K) * 4, i);
      out.add(j.flags, 4, i);
    } else {
      out.add(j.out, size_t(j.K) * j.PD * (j.out_dtype == FVS_F32 ? 4 : 2), i);
    }
  }
  int r = out.check(api);
  if (r) return r;
  std::vector<int32_t> blocks(n), groups(n);
  const int n_groups = mem_groups(jobs, n, budget, blocks.data(), groups.data());
  for (int g = 0, i0 = 0; g < n_groups; ++g) {
    int i1 = i0;
    while (i1 < n && groups[i1] == g) ++i1;
    if ((r = mem_run(dev.data() + i0, i1 - i0, call, (cudaStream_t)stream))) return r;
    i0 = i1;
  }
  return FVS_OK;
}

// ---- the klarge retrieval
// the bank of a klarge retrieval, in two tiers: rows [0, n_dev) are contiguous at dev (HBM), row n_dev + c*chunk_frames + r
// is row r of host chunk c (chunks: a host array of the chunks' mapped device pointers)
struct KlargeBank {
  const void* dev;
  int n_dev;
  const void* const* chunks;
  int chunk_frames, t_total;
};

// the checks of fvs_qwen_klarge_retrieve and its tiered form, reported as `who`
int check_klarge(const char* who, const void* tem_x, const int64_t* klarge_idx, const KlargeBank& b, int k, int PD, int dtype,
                 int metric, const int64_t* idx_out, const void* workspace, size_t workspace_bytes) {
  const int t_total = b.t_total;
  FVS_REQUIRE(tem_x && klarge_idx && idx_out && workspace && (b.dev || b.n_dev == 0), "%s: null pointer", who);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", who);
  FVS_REQUIRE(metric == FVS_KLARGE_EUCLIDEAN || metric == FVS_KLARGE_COSINE, "%s: unknown metric %d", who, metric);
  FVS_REQUIRE(k > 0 && k <= 64 && t_total > 0, "%s: need 0 < k <= 64, t > 0 (k=%d t=%d)", who, k, t_total);
  FVS_REQUIRE(PD > 0 && PD % SLICE == 0, "%s: PD (%d) must be a positive multiple of %d", who, PD, SLICE);
  FVS_REQUIRE(b.n_dev >= 0 && b.n_dev <= t_total, "%s: need 0 <= n_dev <= t_total (n_dev=%d t=%d)", who, b.n_dev, t_total);
  if (b.n_dev < t_total) {
    FVS_REQUIRE(b.chunks && b.chunk_frames > 0, "%s: host rows need a chunk table and chunk_frames > 0", who);
    for (int c = 0; c * int64_t(b.chunk_frames) < t_total - b.n_dev; ++c)
      FVS_REQUIRE(b.chunks[c], "%s: null pointer of host chunk %d", who, c);
  }
  FVS_REQUIRE(workspace_bytes >= fvs_qwen_klarge_workspace_bytes(k, t_total, PD), "%s: workspace too small", who);
  return FVS_OK;
}

KlJobDev kl_job_dev(const void* tem_x, const int64_t* klarge_idx, const void* bank, int k, int t_total, int PD,
                    int64_t* idx_out, float* dist_out, void* workspace) {
  const size_t units = size_t(t_total) * k + t_total + k;
  float* part = (float*)workspace;
  float* tot = (float*)((uint8_t*)workspace + al(units * (PD / SLICE) * 4));
  // <= 32 bank rows per block: enough blocks to fill every SM from t ~ 32 up
  return KlJobDev{(const uint16_t*)tem_x, (const long long*)klarge_idx, (const uint16_t*)bank, part, tot,
                  (long long*)idx_out, dist_out, k, t_total, PD, (t_total + 31) / 32};
}

template <int kJobs, bool kBF16, int kStage>
int kl_launch(KlLaunch<kJobs>& L, int threads, size_t smem, cudaStream_t stream, const char* name) {
  L.first[0] = 0;
  for (int j = 0; j < L.n; ++j) L.first[j + 1] = L.first[j] + kl_stage_blocks(L.job[j], kStage);
  if (L.first[L.n] == 0) return FVS_OK;
  if (smem > 48 * 1024) {
    static bool attr = false;   // per instantiation
    if (!attr) {
      FVS_CUDA_OK(cudaFuncSetAttribute(klarge_multi_kernel<kJobs, kBF16, kStage>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       64 * SLICE * 2));
      attr = true;
    }
  }
  klarge_multi_kernel<kJobs, kBF16, kStage><<<L.first[L.n], threads, smem, stream>>>(L);
  FVS_CHECK_LAUNCH(name);
  return FVS_OK;
}

// sweep kMode of a bank with host rows (one job): one range launch over the device rows and one per host chunk, each
// reading its rows through the chunk's mapped pointer (PCIe)
template <bool kBF16, int kMode>
int klarge_tier_sweep(const KlJobDev& J, const KlargeBank& b, cudaStream_t stream) {
  static bool attr = false;   // per instantiation
  auto kern = klarge_partial_kernel<kBF16, kMode>;
  if (!attr) { FVS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * SLICE * 2)); attr = true; }
  const float* norms = kMode == 2 ? J.tot + size_t(J.t_total) * J.k : nullptr;
  auto launch = [&](const void* rows_at, int t_first, int rows) {
    kern<<<dim3(J.PD / SLICE, (rows + 31) / 32), 256, size_t(J.k) * SLICE * 2, stream>>>(
        J.tem_x, J.klarge_idx, (const uint16_t*)rows_at, J.part, J.k, J.t_total, J.PD, norms, t_first, rows);
    FVS_CHECK_LAUNCH("klarge_partial_kernel");
    return FVS_OK;
  };
  int r;
  if (b.n_dev > 0 && (r = launch(b.dev, 0, b.n_dev))) return r;
  for (int c = 0, t = b.n_dev; t < b.t_total; ++c, t += b.chunk_frames)
    if ((r = launch(b.chunks[c], t, std::min(b.chunk_frames, b.t_total - t)))) return r;
  return FVS_OK;
}

// sweep kMode: one launch over every job's whole bank, or the range launches of `tiers` (a one-job group with host rows)
template <int kJobs, bool kBF16, int kMode>
int kl_sweep(KlLaunch<kJobs>& L, const KlargeBank* tiers, size_t smem, cudaStream_t stream, const char* name) {
  if (tiers) return klarge_tier_sweep<kBF16, kMode>(L.job[0], *tiers, stream);
  return kl_launch<kJobs, kBF16, kKlSweep0 + kMode>(L, 256, smem, stream, name);
}

template <int kJobs, bool kBF16>
int kl_group(KlLaunch<kJobs>& L, int metric, const KlargeBank* tiers, cudaStream_t stream) {
  int max_k = 1, r;
  for (int j = 0; j < L.n; ++j) max_k = std::max(max_k, L.job[j].k);
  const size_t smem = size_t(max_k) * SLICE * 2;
  if (metric == FVS_KLARGE_EUCLIDEAN) {
    if ((r = kl_sweep<kJobs, kBF16, 0>(L, tiers, smem, stream, "klarge_multi_kernel<sweep>"))) return r;
    if ((r = kl_launch<kJobs, kBF16, kKlReduceAll>(L, 256, 0, stream, "klarge_multi_kernel<seq_reduce>"))) return r;
    return kl_launch<kJobs, kBF16, kKlTail>(L, 32, 0, stream, "klarge_multi_kernel<tail>");
  }
  // cosine: squared norms -> norms -> normalised dot products -> argmin of the similarity (the bank is swept twice)
  if ((r = kl_sweep<kJobs, kBF16, 1>(L, tiers, smem, stream, "klarge_multi_kernel<sweep norms>"))) return r;
  if ((r = kl_launch<kJobs, kBF16, kKlReduceNorms>(L, 256, 0, stream, "klarge_multi_kernel<seq_reduce>"))) return r;
  if ((r = kl_launch<kJobs, kBF16, kKlNorms>(L, 256, 0, stream, "klarge_multi_kernel<norms>"))) return r;
  if ((r = kl_sweep<kJobs, kBF16, 2>(L, tiers, smem, stream, "klarge_multi_kernel<sweep cos>"))) return r;
  if ((r = kl_launch<kJobs, kBF16, kKlReduceAb>(L, 256, 0, stream, "klarge_multi_kernel<seq_reduce>"))) return r;
  return kl_launch<kJobs, kBF16, kKlCosTail>(L, 32, 0, stream, "klarge_multi_kernel<cos tail>");
}

// one launch group of n <= kJobs retrieval jobs
template <int kJobs>
int kl_run(const KlJobDev* jobs, int n, bool bf, int metric, const KlargeBank* tiers, cudaStream_t stream) {
  KlLaunch<kJobs> L;
  L.n = n;
  for (int j = 0; j < n; ++j) L.job[j] = jobs[j];
  return bf ? kl_group<kJobs, true>(L, metric, tiers, stream) : kl_group<kJobs, false>(L, metric, tiers, stream);
}

// fvs_qwen_klarge_retrieve and its tiered form: the one-job table, with the tiers' range sweeps for a bank with host rows
int klarge_retrieve(const char* who, const void* tem_x, const int64_t* klarge_idx, const KlargeBank& b, int k, int PD, int dtype,
                    int metric, int64_t* idx_out, float* dist_out, void* workspace, size_t workspace_bytes,
                    fvs_stream_t stream) {
  const int r = check_klarge(who, tem_x, klarge_idx, b, k, PD, dtype, metric, idx_out, workspace, workspace_bytes);
  if (r) return r;
  const KlJobDev J = kl_job_dev(tem_x, klarge_idx, b.dev, k, b.t_total, PD, idx_out, dist_out, workspace);
  return kl_run<1>(&J, 1, dtype == FVS_BF16, metric, b.n_dev < b.t_total ? &b : nullptr, (cudaStream_t)stream);
}
}  // namespace

extern "C" {

int fvs_qwen_temporal_pool(const void* x, void* out, int t, int h, int w, int dtype, fvs_stream_t stream) {
  FVS_REQUIRE(x && out, "fvs_qwen_temporal_pool: null pointer");
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "fvs_qwen_temporal_pool: dtype must be f16 or bf16");
  FVS_REQUIRE(t > 0 && h > 0 && w > 0 && h % 2 == 0 && w % 2 == 0, "fvs_qwen_temporal_pool: h, w must be even");
  // the reference raises NotImplementedError when (h/2) or (w/2) is odd (vstream_qwen2vl_model.py:130-133)
  if ((h / 2) % 2 || (w / 2) % 2) return set_error(FVS_ENOTIMPL, "Performing temporal pool, pad > 0 (h/2=%d, w/2=%d)", h / 2, w / 2);
  const size_t rows = size_t(t) * (h / 2) * (w / 2);          // one block per output row
  FVS_REQUIRE(rows < (size_t(1) << 31), "fvs_qwen_temporal_pool: clip too large");
  const size_t max_blocks = size_t(device_sm_count()) * 64;
  const int blocks = int(rows < max_blocks ? rows : max_blocks);
  if (dtype == FVS_BF16)
    temporal_pool_kernel<true><<<blocks, 196, 0, (cudaStream_t)stream>>>((const uint16_t*)x, (uint16_t*)out, t, h, w);
  else
    temporal_pool_kernel<false><<<blocks, 196, 0, (cudaStream_t)stream>>>((const uint16_t*)x, (uint16_t*)out, t, h, w);
  FVS_CHECK_LAUNCH("temporal_pool_kernel");
  return FVS_OK;
}

size_t fvs_qwen_unique_workspace_bytes(int T) { return T > 0 ? al(size_t(T) * T) : 0; }

int fvs_qwen_unique_rows(const void* X, int T, int PD, int dtype, int32_t* uniq_idx_out, int32_t* n_unique_out,
                         void* workspace, size_t workspace_bytes, fvs_stream_t stream) {
  MemJobDev J{};
  J.X = X; J.T = T; J.PD = PD; J.dt = dtype;
  J.uniq_idx = uniq_idx_out; J.n_unique = n_unique_out; J.uniq_ws = workspace;
  return mem_single("fvs_qwen_unique_rows", J, workspace_bytes, kCallUnique, stream);
}

size_t fvs_qwen_kmeans_workspace_bytes(int T, int K, int PD) {
  if (T <= 0 || K <= 0 || PD <= 0) return 0;
  const size_t S = size_t(PD) / SLICE, TK = size_t(T) * K + K;
  return al(32) + 2 * al(size_t(K) * PD * 4) + al(TK * S * 4) + al(TK * 4) + al(size_t(T) * S * 4) + al(size_t(T) * 4) +
         al(size_t(K) * S * 4) + 2 * al(size_t(K) * 4) + al(size_t(T) * 4) + 4 * al((size_t(K) + 1) * 4);
}

int fvs_qwen_kmeans(const void* X, int x_dtype, const float* w, const int32_t* uniq_idx, const int32_t* init_idx,
                    const int32_t* refill_idx, int T, int K, int PD, int max_iter, float tol, float* C_out, float* wsum_out,
                    int32_t* labels_out, int32_t* info_out, void* workspace, size_t workspace_bytes, fvs_stream_t stream) {
  MemJobDev J{};
  J.X = X; J.dt = x_dtype; J.w = w; J.uniq_idx = const_cast<int32_t*>(uniq_idx); J.init_idx = init_idx;
  J.refill_idx = refill_idx; J.T = T; J.K = K; J.PD = PD; J.max_iter = max_iter; J.tol = tol;
  J.C = C_out; J.wsum = wsum_out; J.labels = labels_out; J.info = info_out; J.km_ws = workspace;
  return mem_single("fvs_qwen_kmeans", J, workspace_bytes, kCallKmeans, stream);
}

int fvs_qwen_kmeans_finalize(const int32_t* labels, const float* wsum, int T, int K, const int64_t* order_in,
                             int64_t* sorted_idx_out, float* ts_out, float* w_out, int32_t* flags_out, fvs_stream_t stream) {
  MemJobDev J{};
  J.labels = const_cast<int32_t*>(labels); J.wsum = const_cast<float*>(wsum); J.T = T; J.K = K;
  J.order_in = (const long long*)order_in; J.sorted_idx = (long long*)sorted_idx_out; J.ts = ts_out; J.w_sorted = w_out;
  J.flags = flags_out;
  return mem_single("fvs_qwen_kmeans_finalize", J, 0, kCallFinalize, stream);
}

int fvs_gather_rows_cast(const float* src, const int64_t* idx, void* out, int n, int64_t row_elems, int out_dtype,
                         fvs_stream_t stream) {
  MemJobDev J{};
  J.C = const_cast<float*>(src); J.sorted_idx = (long long*)const_cast<int64_t*>(idx); J.out = out; J.K = n;
  J.row_elems = row_elems; J.out_dt = out_dtype;
  return mem_single("fvs_gather_rows_cast", J, 0, kCallGather, stream);
}

size_t fvs_qwen_klarge_workspace_bytes(int k, int t_total, int PD) {
  if (k <= 0 || t_total <= 0 || PD <= 0) return 0;
  const size_t units = size_t(t_total) * k + t_total + k;
  return al(units * (size_t(PD) / SLICE) * 4) + al(units * 4);
}

int fvs_qwen_klarge_retrieve(const void* tem_x, const int64_t* klarge_idx, const void* bank, int k, int t_total, int PD,
                             int dtype, int metric, int64_t* idx_out, float* dist_out, void* workspace,
                             size_t workspace_bytes, fvs_stream_t stream) {
  if (!bank) return set_error(FVS_EINVAL, "fvs_qwen_klarge_retrieve: null pointer");
  const KlargeBank b{bank, t_total, nullptr, 0, t_total};
  return klarge_retrieve("fvs_qwen_klarge_retrieve", tem_x, klarge_idx, b, k, PD, dtype, metric, idx_out, dist_out, workspace,
                         workspace_bytes, stream);
}

int fvs_qwen_klarge_retrieve_tiered(const void* tem_x, const int64_t* klarge_idx, const void* dev_bank, int n_dev,
                                    const void* const* host_chunks, int chunk_frames, int k, int t_total, int PD, int dtype,
                                    int metric, int64_t* idx_out, float* dist_out, void* workspace, size_t workspace_bytes,
                                    fvs_stream_t stream) {
  const KlargeBank b{dev_bank, n_dev, host_chunks, chunk_frames, t_total};
  return klarge_retrieve("fvs_qwen_klarge_retrieve_tiered", tem_x, klarge_idx, b, k, PD, dtype, metric, idx_out, dist_out,
                         workspace, workspace_bytes, stream);
}

int fvs_qwen_mem_plan(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, int32_t* blocks_h, int32_t* groups_h) {
  const char* api = "fvs_qwen_mem_plan";
  FVS_REQUIRE(jobs_h && n_jobs > 0 && budget >= 0 && blocks_h && groups_h, "%s: need jobs, n_jobs > 0, budget >= 0, outputs",
              api);
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_mem_job& j = jobs_h[i];
    FVS_REQUIRE(j.T > 0 && j.T <= 4096 && j.K > 0 && j.K <= j.T && j.PD > 0 && j.PD % SLICE == 0,
                "%s: job %d: bad shape T=%d K=%d PD=%d", api, i, j.T, j.K, j.PD);
  }
  return mem_groups(jobs_h, n_jobs, budget, blocks_h, groups_h);
}

int fvs_qwen_unique_rows_multi(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, fvs_stream_t stream) {
  return mem_table("fvs_qwen_unique_rows_multi", jobs_h, n_jobs, budget, stream, kCallUnique);
}
int fvs_qwen_kmeans_multi(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, fvs_stream_t stream) {
  return mem_table("fvs_qwen_kmeans_multi", jobs_h, n_jobs, budget, stream, kCallKmeans);
}
int fvs_qwen_kmeans_finalize_multi(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, fvs_stream_t stream) {
  return mem_table("fvs_qwen_kmeans_finalize_multi", jobs_h, n_jobs, budget, stream, kCallFinalize);
}
int fvs_gather_rows_cast_multi(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, fvs_stream_t stream) {
  return mem_table("fvs_gather_rows_cast_multi", jobs_h, n_jobs, budget, stream, kCallGather);
}

int fvs_qwen_klarge_retrieve_multi(const fvs_qwen_retrieve_job* jobs_h, int n_jobs, int dtype, int metric,
                                   fvs_stream_t stream) {
  const char* api = "fvs_qwen_klarge_retrieve_multi";
  FVS_REQUIRE(jobs_h && n_jobs > 0, "%s: need a job table and n_jobs > 0", api);
  std::vector<KlJobDev> dev(n_jobs);
  JobOutputs out;
  int r;
  for (int i = 0; i < n_jobs; ++i) {
    const fvs_qwen_retrieve_job& j = jobs_h[i];
    char who[96];
    snprintf(who, sizeof who, "%s: job %d", api, i);
    FVS_REQUIRE(j.n_dev == j.t_total, "%s: %d of its %d bank rows are in host memory: step it through "
                "fvs_qwen_klarge_retrieve_tiered", who, j.t_total - j.n_dev, j.t_total);
    const KlargeBank b{j.bank, j.n_dev, nullptr, 0, j.t_total};
    if ((r = check_klarge(who, j.tem_x, j.klarge_idx, b, j.k, j.PD, dtype, metric, j.idx_out, j.workspace, j.workspace_bytes)))
      return r;
    dev[i] = kl_job_dev(j.tem_x, j.klarge_idx, j.bank, j.k, j.t_total, j.PD, j.idx_out, j.dist_out, j.workspace);
    out.add(j.idx_out, size_t(j.k) * 8, i);
    out.add(j.workspace, fvs_qwen_klarge_workspace_bytes(j.k, j.t_total, j.PD), i);
    if (j.dist_out) out.add(j.dist_out, size_t(j.k) * j.t_total * 4, i);
  }
  if ((r = out.check(api))) return r;
  for (int i0 = 0; i0 < n_jobs; i0 += kMemJobs) {
    const int n = std::min(kMemJobs, n_jobs - i0);
    const bool bf = dtype == FVS_BF16;
    r = n == 1 ? kl_run<1>(dev.data() + i0, 1, bf, metric, nullptr, (cudaStream_t)stream)
               : kl_run<kMemJobs>(dev.data() + i0, n, bf, metric, nullptr, (cudaStream_t)stream);
    if (r) return r;
  }
  return FVS_OK;
}

int fvs_qwen_am_rope(const int64_t* spa_positions, int spa_t, int spa_h, int spa_w, const int64_t* tem_positions, int tem_t,
                     int tem_h, int tem_w, int64_t visual_start_id, int64_t* out, fvs_stream_t stream) {
  FVS_REQUIRE(out && spa_t >= 0 && tem_t >= 0 && spa_h >= 0 && spa_w >= 0 && tem_h >= 0 && tem_w >= 0, "fvs_qwen_am_rope: bad argument");
  FVS_REQUIRE((spa_t == 0 || spa_positions) && (tem_t == 0 || tem_positions), "fvs_qwen_am_rope: null positions");
  const int total = spa_t * spa_h * spa_w + tem_t * tem_h * tem_w;
  if (total == 0) return FVS_OK;
  am_rope_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>((const long long*)spa_positions, spa_t, spa_h, spa_w,
                                                                        (const long long*)tem_positions, tem_t, tem_h, tem_w,
                                                                        (long long)visual_start_id, (long long*)out, total);
  FVS_CHECK_LAUNCH("am_rope_kernel");
  return FVS_OK;
}

}  // extern "C"
