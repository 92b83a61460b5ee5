// memory_kernels.cu — Flash-Memory consolidation kernels (HBM/ALU-bound f16 work, no tensor cores):
// hierarchical spatial pooling, reference-exact weighted k-means, abstract-memory update, key-frame retrieval.
//
// "Reference-exact" means: every place where the reference's f16 PyTorch path rounds to binary16 we round too
// (element-wise sub/mul, reduction results, sqrt, division), reductions accumulate in fp32, argmin takes the first
// minimal index and lets NaN win. The ONE thing PyTorch leaves unspecified is the order of fp32 accumulation
// inside a reduction; we fix a canonical order (documented at `slice_sqdiff` in mem_device.cuh) and oracle/fvs_oracle.py
// mirrors it operation for operation, so kernel and oracle agree bit-for-bit.
//
// The k-means, abstract-memory, argsort and retrieval kernels here are the op-by-op form of the streaming step: each is a
// launch shape around one per-unit function of mem_device.cuh, the same functions the fused consolidate_kernel
// (stream_kernels.cu) calls, so the two paths compute the same bits.
//
// Reference anchors: compress_spatial_features vstream_arch.py:193-212; weighted_kmeans_feature
// compress_functions.py:130-169; attention / get_weight vstream_arch.py:174-183,47-52; key retrieval
// vstream_arch.py:261-268, 681-688.
#include "fvs_common.h"
#include "fvs_kernels.h"
#include "fvs_ptx.cuh"
#include "mem_device.cuh"

namespace fvs {
namespace mem {

// ------------------------------------------------------------------------------------------------ pooling
// feat [T, g*g, D] -> out [T, c*c, D]; fp32 window sum in (ky, kx) order, one division, one rounding.
__global__ void pool_kernel(const uint16_t* __restrict__ feat, uint16_t* __restrict__ out, int T, int g, int c, int D) {
  const int k = g / c;
  const int vecs = D / 8;
  const size_t total = size_t(T) * c * c * vecs;
  const float div = float(k * k);
  for (size_t idx = blockIdx.x * size_t(blockDim.x) + threadIdx.x; idx < total; idx += size_t(gridDim.x) * blockDim.x) {
    const int v = int(idx % vecs);
    const int cell = int((idx / vecs) % (c * c));
    const int t = int(idx / (size_t(vecs) * c * c));
    const int oy = cell / c, ox = cell % c;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int ky = 0; ky < k; ++ky)
      for (int kx = 0; kx < k; ++kx) {
        const int tok = (oy * k + ky) * g + ox * k + kx;
        const uint4 w = *reinterpret_cast<const uint4*>(feat + (size_t(t) * g * g + tok) * D + v * 8);
        const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&ww[p]));
          acc[2 * p] += f.x;
          acc[2 * p + 1] += f.y;
        }
      }
    uint32_t o[4];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      __half2 h = __floats2half2_rn(acc[2 * p] / div, acc[2 * p + 1] / div);
      o[p] = *reinterpret_cast<uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(out + (size_t(t) * c * c + cell) * D + v * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// Fused three-level pooling: one block per (frame, 64-channel slab).  Level a is pooled from the input, rounded to
// f16 into smem, and levels b (avg pool of the rounded level a) and c (mean over all a*a cells) are pooled from that
// rounded copy exactly as the reference pools its own rounded tensor (vstream_arch.py:649, 659-662).
// kResidual: the input is the ViT encoder's fp32 residual stream x [T, g*g+1, D] plus the last fc2 delta (f16, same
// shape) instead of the finished feature map: token (1 + p) of frame t contributes f16(x + delta) — exactly the value
// drop_cls_kernel would have written to hidden_states[-2][:, 1:] (clip_encoder.py:35,50-51) — so the [T,576,D] feature
// map is never materialised on the streaming path (SURVEY.md §8d: 4.17 -> 2.99 MB/frame).
// Frame t of the launch belongs to destination j = the last with dst.first[j] <= t; its rows go to that destination's own
// outputs (one stream's frame buffer / long / Turing working-set rows), so one launch pools the clips of many streams.
template <int kMaxCells, bool kResidual>
__global__ void __launch_bounds__(512) pool3_kernel(const void* __restrict__ feat_, const uint16_t* __restrict__ delta,
                                                    const __grid_constant__ Pool3Table dst, int g, int a, int b, int D) {
  __shared__ __half lvl_a[kMaxCells][64];
  const int t = blockIdx.x, slab = blockIdx.y;
  int j = 0;
  while (j + 1 < dst.n && t >= dst.first[j + 1]) ++j;
  const int tl = t - dst.first[j];
  uint16_t* __restrict__ out_a = dst.a[j];
  uint16_t* __restrict__ out_b = dst.b[j];
  uint16_t* __restrict__ out_c = dst.c[j];
  const int ka = g / a;
  const int ncell = a * a;
  const int v = threadIdx.x & 7;  // 8 vectors of 8 channels = 64 channels
  const float diva = float(ka * ka);
  for (int cell = threadIdx.x >> 3; cell < ncell; cell += blockDim.x >> 3) {
    const int oy = cell / a, ox = cell % a;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int ky = 0; ky < ka; ++ky)
      for (int kx = 0; kx < ka; ++kx) {
        const int tok = (oy * ka + ky) * g + ox * ka + kx;
        if (kResidual) {
          const size_t e0 = (size_t(t) * (g * g + 1) + 1 + tok) * D + slab * 64 + v * 8;
          const float4* xr = reinterpret_cast<const float4*>(static_cast<const float*>(feat_) + e0);
          const float4 x0 = xr[0], x1 = xr[1];
          float f[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
          if (delta != nullptr) {
            const uint4 w = *reinterpret_cast<const uint4*>(delta + e0);
            const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              const float2 d = __half22float2(*reinterpret_cast<const __half2*>(&ww[p]));
              f[2 * p] += d.x;
              f[2 * p + 1] += d.y;
            }
          }
#pragma unroll
          for (int p = 0; p < 4; ++p) {   // one rounding to the tower dtype, as the encoder output would carry
            const float2 r = __half22float2(__floats2half2_rn(f[2 * p], f[2 * p + 1]));
            acc[2 * p] += r.x;
            acc[2 * p + 1] += r.y;
          }
        } else {
          const uint4 w = *reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(feat_) + (size_t(t) * g * g + tok) * D + slab * 64 + v * 8);
          const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&ww[p]));
            acc[2 * p] += f.x;
            acc[2 * p + 1] += f.y;
          }
        }
      }
    uint32_t o[4];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      __half2 h = __floats2half2_rn(acc[2 * p] / diva, acc[2 * p + 1] / diva);
      o[p] = *reinterpret_cast<uint32_t*>(&h);
      lvl_a[cell][v * 8 + 2 * p] = __low2half(h);
      lvl_a[cell][v * 8 + 2 * p + 1] = __high2half(h);
    }
    *reinterpret_cast<uint4*>(out_a + (size_t(tl) * ncell + cell) * D + slab * 64 + v * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
  __syncthreads();
  const int ch = threadIdx.x & 63;
  if (out_b) {
    const int kb = a / b;
    const float divb = float(kb * kb);
    for (int cell = threadIdx.x >> 6; cell < b * b; cell += blockDim.x >> 6) {
      const int oy = cell / b, ox = cell % b;
      float acc = 0.f;
      for (int ky = 0; ky < kb; ++ky)
        for (int kx = 0; kx < kb; ++kx) acc += __half2float(lvl_a[(oy * kb + ky) * a + ox * kb + kx][ch]);
      out_b[(size_t(tl) * b * b + cell) * D + slab * 64 + ch] = f2h(acc / divb);
    }
  }
  if (out_c && threadIdx.x < 64) {
    float acc = 0.f;
    for (int cell = 0; cell < ncell; ++cell) acc += __half2float(lvl_a[cell][ch]);
    out_c[size_t(tl) * D + slab * 64 + ch] = f2h(acc / float(ncell));
  }
}

// ------------------------------------------------------------------------------------------------ k-means
struct KMState {
  int done;        // 1 once diff < tol (or max_iter reached)
  int cur;         // which of the two centroid buffers holds the current centroids
  int iter;        // index i of the last executed Lloyd iteration
  int refill_pos;  // cursor into refill_idx
  int converged;   // 1 if the loop broke on tol
  int pad[3];
};

struct KMBuffers {
  KMState* st;
  uint16_t* C[2];    // [K, PD] each
  float* part;       // [T, K, S] distance partials
  float* normpart;   // [K, S]
  uint16_t* wsum;    // [K] f16
  int* labels;       // [T]
};

__global__ void km_init_kernel(KMBuffers B, const uint16_t* __restrict__ X, const int* __restrict__ init_idx, int K,
                               int PD) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    B.st->done = 0; B.st->cur = 0; B.st->iter = 0; B.st->refill_pos = 0; B.st->converged = 0;
  }
  const int vecs = PD / 8;
  for (size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x; i < size_t(K) * vecs; i += size_t(gridDim.x) * blockDim.x) {
    const int k = int(i / vecs), v = int(i % vecs);
    reinterpret_cast<uint4*>(B.C[0])[i] = reinterpret_cast<const uint4*>(X + size_t(init_idx[k]) * PD)[v];
  }
}

// block = 8 warps = 8 consecutive rows t of one slice s (so the centroid slice stays hot in L1 for the block);
// each warp keeps its x slice in registers and sweeps all K centroids.
__global__ void __launch_bounds__(256) km_partial_kernel(KMBuffers B, const uint16_t* __restrict__ X, int T, int K,
                                                         int PD, int iter) {
  if (B.st->done) return;
  const int S = PD / SLICE;
  const int s = blockIdx.x % S;
  const int t = (blockIdx.x / S) * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const uint16_t* C = B.C[B.st->cur];
  uint4 x[4];
  load_slice(x, X + size_t(t) * PD + s * SLICE, lane);
  for (int k = 0; k < K; ++k) {
    const float p = slice_sqdiff(x, C + size_t(k) * PD + s * SLICE, lane);
    if (lane == 0) B.part[(size_t(t) * K + k) * S + s] = p;
  }
}

// one warp per row t: dist = f16(sqrt(f16(sum_s part))) ; first-index / NaN-wins argmin over k
__global__ void __launch_bounds__(256) km_assign_kernel(KMBuffers B, int T, int K, int PD) {
  if (B.st->done) return;
  const int S = PD / SLICE;
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const int label = km_row_label(B.part + size_t(t) * K * S, K, S, lane);
  if (lane == 0) B.labels[t] = label;
}

// one warp per (cluster j, slice s): weighted mean of the members (sequential in t), empty-cluster refill, and the
// partial of ||c_old - c_new||^2 for the convergence test.
__global__ void __launch_bounds__(256) km_update_kernel(KMBuffers B, const uint16_t* __restrict__ X,
                                                        const uint16_t* __restrict__ w, const int* __restrict__ refill_idx,
                                                        int T, int K, int PD) {
  if (B.st->done) return;
  const int S = PD / SLICE;
  const int unit = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (unit >= K * S) return;
  const int j = unit / S, s = unit % S;
  const int cur = B.st->cur;
  km_cluster_slice_update(X, w, B.labels, refill_idx + B.st->refill_pos, T, PD, S, j, s,
                          B.C[cur] + size_t(j) * PD + s * SLICE, B.C[cur ^ 1] + size_t(j) * PD + s * SLICE, B.normpart,
                          B.wsum, lane);
}

// single block: diff = f16(sum_k f16(sqrt(sum_s normpart))) ; break test; bookkeeping
__global__ void km_converge_kernel(KMBuffers B, int K, int PD, int iter, int max_iter, uint16_t tol_h) {
  if (B.st->done) return;
  if (threadIdx.x != 0) return;
  const int S = PD / SLICE;
  float diff = 0.f;
  int n_empty = 0;
  for (int k = 0; k < K; ++k) {
    diff = diff + centroid_shift(B.normpart, k, S);
    if (!(h2f(B.wsum[k]) > 0.f)) n_empty++;
  }
  const float diff_h = round_h(diff);
  B.st->iter = iter;
  B.st->refill_pos += n_empty;
  if (diff_h < h2f(tol_h)) {   // `if diff < tol: break` — centroids stay the OLD ones
    B.st->done = 1;
    B.st->converged = 1;
  } else {
    B.st->cur ^= 1;            // centroids = new_centroids
    if (iter == max_iter - 1) B.st->done = 1;
  }
}

__global__ void km_finish_kernel(KMBuffers B, uint16_t* __restrict__ C_out, uint16_t* __restrict__ wsum_out,
                                 int* __restrict__ labels_out, int* __restrict__ info_out, int T, int K, int PD) {
  const uint4* src = reinterpret_cast<const uint4*>(B.C[B.st->cur]);
  const size_t nvec = size_t(K) * PD / 8;
  for (size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x; i < nvec; i += size_t(gridDim.x) * blockDim.x)
    reinterpret_cast<uint4*>(C_out)[i] = src[i];
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < K; i += blockDim.x) wsum_out[i] = B.wsum[i];
    for (int i = threadIdx.x; i < T; i += blockDim.x) labels_out[i] = B.labels[i];
    if (threadIdx.x == 0) {
      info_out[0] = B.st->iter; info_out[1] = B.st->refill_pos; info_out[2] = B.st->converged; info_out[3] = 0;
    }
  }
}

// ------------------------------------------------------------------------------------------------ abstract memory
// Three small kernels (projections: one block per row; softmax: one block; apply: grid over T1 x D) instead of one serial
// block; the arithmetic is abs_proj_dot / abs_softmax_row / abs_apply_elem of mem_device.cuh.
struct AbsScratch {
  float* q;      // [T1, H]  (f16-rounded values)
  float* k;      // [T2, H]
  float* wgt;    // [T1, T2] softmax * ratio (f16-rounded)
  float* decay;  // [T1]
};

__global__ void __launch_bounds__(256) abs_proj_kernel(const uint16_t* __restrict__ M, const uint16_t* __restrict__ F,
                                                       const uint16_t* __restrict__ Wq, const uint16_t* __restrict__ bq,
                                                       const uint16_t* __restrict__ Wk, const uint16_t* __restrict__ bk,
                                                       AbsScratch S, int T1, int T2, int D, int H) {
  const int r = blockIdx.x;  // 0..T1-1 -> q rows, T1..T1+T2-1 -> k rows
  const bool isq = r < T1;
  const uint16_t* x = isq ? M + size_t(r) * D : F + size_t(r - T1) * D;
  const uint16_t* W = isq ? Wq : Wk;
  const uint16_t* b = isq ? bq : bk;
  float* out = isq ? S.q + size_t(r) * H : S.k + size_t(r - T1) * H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int h = warp; h < H; h += nwarps) {
    const float v = abs_proj_dot(x, W + size_t(h) * D, b + h, D, lane);
    if (lane == 0) out[h] = v;
  }
}

__global__ void __launch_bounds__(256) abs_softmax_kernel(AbsScratch S, int T1, int T2, int H, float ratio) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const float sqrtH = sqrtf(float(H));
  for (int i = warp; i < T1; i += nwarps) {  // one warp per memory row
    const float decay = abs_softmax_row(S.q, S.k, i, S.wgt + i * T2, T2, H, sqrtH, ratio, lane);
    if (lane == 0) S.decay[i] = decay;
  }
}

// M' = f16( f16(M * f16(1 - decay)) + f16(W @ F) ); one thread per (row i, channel d)
__global__ void __launch_bounds__(256) abs_apply_kernel(const uint16_t* __restrict__ M, const uint16_t* __restrict__ F,
                                                        uint16_t* __restrict__ Mout, AbsScratch S, int T1, int T2, int D) {
  const int i = blockIdx.y;
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  Mout[size_t(i) * D + d] = abs_apply_elem(S.wgt + i * T2, F, T2, D, d, M[size_t(i) * D + d], S.decay[i]);
}

// ------------------------------------------------------------------------------------------------ argsort / retrieval
// stable descending rank sort, NaN largest (torch.sort convention); single block, K <= 1024
__global__ void argsort_desc_kernel(const void* __restrict__ w, int K, long long* __restrict__ order, int dt) {
  extern __shared__ float sv[];
  for (int i = threadIdx.x; i < K; i += blockDim.x)
    sv[i] = dt == FVS_F32 ? static_cast<const float*>(w)[i]
          : dt == FVS_BF16 ? __uint_as_float(uint32_t(static_cast<const uint16_t*>(w)[i]) << 16)
                           : h2f(static_cast<const uint16_t*>(w)[i]);
  __syncthreads();
  for (int i = threadIdx.x; i < K; i += blockDim.x) order[stable_desc_rank(i, K, [&](int j) { return sv[j]; })] = i;
}

// one warp per (l, k): key_distance of working-set row l and key candidate order[k]
__global__ void __launch_bounds__(256) key_dist_kernel(const uint16_t* __restrict__ lm, const long long* __restrict__ order,
                                                       float* __restrict__ dist, int L, int P, int D, int key_len) {
  const int unit = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (unit >= L * key_len) return;
  const int l = unit / key_len, k = unit % key_len;
  const float d = key_distance(lm + size_t(l) * P * D, lm + size_t(order[k]) * P * D, P, D, lane);
  if (lane == 0) dist[unit] = d;
}

__global__ void key_argmin_kernel(const float* __restrict__ dist, long long* __restrict__ idx_out, int L, int key_len) {
  const int k = blockIdx.x;
  const int lane = threadIdx.x;  // one warp
  const int best = warp_argmin_of(L, [&](int l) { return dist[l * key_len + k]; }, lane);
  if (lane == 0) idx_out[k] = best;
}

__global__ void gather_rows_kernel(const uint4* __restrict__ src, const long long* __restrict__ idx, uint4* __restrict__ out,
                                   int n, size_t row_vecs) {
  for (size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x; i < size_t(n) * row_vecs; i += size_t(gridDim.x) * blockDim.x) {
    const size_t r = i / row_vecs, c = i % row_vecs;
    out[i] = src[size_t(idx[r]) * row_vecs + c];
  }
}

inline size_t al(size_t v) { return (v + 255) & ~size_t(255); }

}  // namespace mem
}  // namespace fvs

namespace fvs {
int pool3_launch(const void* in, bool residual, const Pool3Dst* dst, int n_dst, int f0, int n, int g, int a, int b, int D,
                 cudaStream_t stream) {
  using namespace mem;
  if (!(in && dst && n_dst > 0 && f0 >= 0 && n > 0)) return set_error(FVS_EINVAL, "pool3: null pointer or empty range");
  if (!(g % a == 0 && D % 64 == 0 && a * a <= 64)) return set_error(FVS_EINVAL, "pool3: bad pooling sizes g=%d a=%d b=%d D=%d", g, a, b, D);
  long long total = 0;
  for (int i = 0; i < n_dst; ++i) {
    if (!(dst[i].a && dst[i].frames > 0 && (dst[i].b == nullptr || (b > 0 && a % b == 0))))
      return set_error(FVS_EINVAL, "pool3: destination %d: null output, no frames or bad b=%d", i, b);
    total += dst[i].frames;
  }
  if (f0 + (long long)n > total) return set_error(FVS_EINVAL, "pool3: frames [%d, %d) beyond the %lld destination frames", f0, f0 + n, total);
  const size_t ca = size_t(a) * a * D, cb = size_t(b) * b * D;
  const size_t in_frame = residual ? size_t(g * g + 1) * D * 4 : size_t(g) * g * D * 2;   // bytes of one input frame
  int i = 0, base = 0;                           // destination i starts at frame `base` of the concatenation
  while (base + dst[i].frames <= f0) base += dst[i++].frames;
  for (int done = 0; done < n;) {               // one launch per kPoolDst destinations (one launch when the range spans fewer)
    Pool3Table tab = {};
    int lf = 0;
    while (tab.n < kPoolDst && done + lf < n) {
      const int skip = f0 + done + lf - base;    // frames of destination i written by an earlier range
      const int take = dst[i].frames - skip < n - done - lf ? dst[i].frames - skip : n - done - lf;
      auto at = [&](void* p, size_t row) { return p ? static_cast<uint16_t*>(p) + size_t(skip) * row : nullptr; };
      tab.first[tab.n] = lf;
      tab.a[tab.n] = at(dst[i].a, ca); tab.b[tab.n] = at(dst[i].b, cb); tab.c[tab.n] = at(dst[i].c, size_t(D));
      ++tab.n;
      lf += take;
      if (skip + take == dst[i].frames) base += dst[i++].frames;
    }
    tab.first[tab.n] = lf;
    const void* src = static_cast<const uint8_t*>(in) + size_t(done) * in_frame;
    if (residual) {
      pool3_kernel<64, true><<<dim3(lf, D / 64), 512, 0, stream>>>(src, nullptr, tab, g, a, b, D);
      FVS_CHECK_LAUNCH("pool3_kernel<residual>");
    } else {
      pool3_kernel<64, false><<<dim3(lf, D / 64), 512, 0, stream>>>(src, nullptr, tab, g, a, b, D);
      FVS_CHECK_LAUNCH("pool3_kernel");
    }
    done += lf;
  }
  return FVS_OK;
}
}  // namespace fvs

using namespace fvs;
using namespace fvs::mem;

extern "C" {

int fvs_spatial_pool(const void* feat, void* out, int T, int grid, int target, int D, int dtype, fvs_stream_t stream) {
  FVS_REQUIRE(feat && out, "fvs_spatial_pool: null pointer");
  FVS_REQUIRE(dtype == FVS_F16, "fvs_spatial_pool: only f16 is implemented (the reference casts to float16, vstream_arch.py:649)");
  FVS_REQUIRE(T > 0 && grid > 0 && target > 0 && grid % target == 0, "fvs_spatial_pool: grid %d not divisible by target %d", grid, target);
  FVS_REQUIRE(D % 8 == 0, "fvs_spatial_pool: D must be a multiple of 8");
  const size_t total = size_t(T) * target * target * (D / 8);
  int blocks = int((total + 255) / 256);
  if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  pool_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)feat, (uint16_t*)out, T, grid, target, D);
  FVS_CHECK_LAUNCH("pool_kernel");
  return FVS_OK;
}

int fvs_spatial_pool3(const void* feat, void* out_a, void* out_b, void* out_c, int T, int g, int a, int b, int D,
                      int dtype, fvs_stream_t stream) {
  FVS_REQUIRE(feat && out_a, "fvs_spatial_pool3: null pointer");
  FVS_REQUIRE(dtype == FVS_F16, "fvs_spatial_pool3: only f16 is implemented");
  FVS_REQUIRE(T > 0 && g % a == 0 && (out_b == nullptr || (b > 0 && a % b == 0)), "fvs_spatial_pool3: bad pooling sizes g=%d a=%d b=%d", g, a, b);
  FVS_REQUIRE(D % 64 == 0 && a * a <= 64, "fvs_spatial_pool3: D %% 64 and a*a <= 64 required");
  const Pool3Dst dst = {out_a, out_b, out_c, T};
  return pool3_launch(feat, false, &dst, 1, 0, T, g, a, b, D, (cudaStream_t)stream);
}

size_t fvs_kmeans_workspace_bytes(int T, int K, int PD) {
  if (T <= 0 || K <= 0 || PD <= 0) return 0;
  const size_t S = size_t(PD) / SLICE;
  return al(sizeof(KMState)) + 2 * al(size_t(K) * PD * 2) + al(size_t(T) * K * S * 4) + al(size_t(K) * S * 4) +
         al(size_t(K) * 2) + al(size_t(T) * 4);
}

int fvs_weighted_kmeans(const void* X, const void* w, const int32_t* init_idx, const int32_t* refill_idx, int T, int K,
                        int PD, int max_iter, float tol, void* C_out, void* wsum_out, int32_t* labels_out,
                        int32_t* info_out, void* workspace, size_t workspace_bytes, int dtype, fvs_stream_t stream_) {
  FVS_REQUIRE(X && init_idx && refill_idx && C_out && wsum_out && labels_out && info_out && workspace,
              "fvs_weighted_kmeans: null pointer");
  FVS_REQUIRE(dtype == FVS_F16, "fvs_weighted_kmeans: only f16 is implemented");
  FVS_REQUIRE(T > 0 && K > 0 && K <= T, "fvs_weighted_kmeans: need 0 < K <= T (T=%d K=%d); T <= K is the shim's pass-through", T, K);
  FVS_REQUIRE(PD % SLICE == 0, "fvs_weighted_kmeans: PD (%d) must be a multiple of %d", PD, SLICE);
  FVS_REQUIRE(max_iter > 0 && max_iter <= 1000, "fvs_weighted_kmeans: bad max_iter");
  FVS_REQUIRE(workspace_bytes >= fvs_kmeans_workspace_bytes(T, K, PD), "fvs_weighted_kmeans: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  const int S = PD / SLICE;
  uint8_t* p = (uint8_t*)workspace;
  KMBuffers B;
  B.st = (KMState*)p; p += al(sizeof(KMState));
  B.C[0] = (uint16_t*)p; p += al(size_t(K) * PD * 2);
  B.C[1] = (uint16_t*)p; p += al(size_t(K) * PD * 2);
  B.part = (float*)p; p += al(size_t(T) * K * S * 4);
  B.normpart = (float*)p; p += al(size_t(K) * S * 4);
  B.wsum = (uint16_t*)p; p += al(size_t(K) * 2);
  B.labels = (int*)p;
  const uint16_t tol_h = __half_as_ushort(__float2half_rn(tol));  // `diff < tol` is evaluated in the tensor dtype
  km_init_kernel<<<64, 256, 0, stream>>>(B, (const uint16_t*)X, init_idx, K, PD);
  FVS_CHECK_LAUNCH("km_init_kernel");
  for (int it = 0; it < max_iter; ++it) {
    km_partial_kernel<<<((T + 7) / 8) * S, 256, 0, stream>>>(B, (const uint16_t*)X, T, K, PD, it);
    FVS_CHECK_LAUNCH("km_partial_kernel");
    km_assign_kernel<<<(T + 7) / 8, 256, 0, stream>>>(B, T, K, PD);
    FVS_CHECK_LAUNCH("km_assign_kernel");
    km_update_kernel<<<(K * S + 7) / 8, 256, 0, stream>>>(B, (const uint16_t*)X, (const uint16_t*)w, refill_idx, T, K, PD);
    FVS_CHECK_LAUNCH("km_update_kernel");
    km_converge_kernel<<<1, 32, 0, stream>>>(B, K, PD, it, max_iter, tol_h);
    FVS_CHECK_LAUNCH("km_converge_kernel");
  }
  km_finish_kernel<<<64, 256, 0, stream>>>(B, (uint16_t*)C_out, (uint16_t*)wsum_out, labels_out, info_out, T, K, PD);
  FVS_CHECK_LAUNCH("km_finish_kernel");
  return FVS_OK;
}

int fvs_abstract_update(const void* M, const void* F, const void* Wq, const void* bq, const void* Wk, const void* bk,
                        void* M_out, int T1, int T2, int D, int H, float ratio, int dtype, fvs_stream_t stream_) {
  FVS_REQUIRE(M && F && Wq && bq && Wk && bk && M_out, "fvs_abstract_update: null pointer");
  FVS_REQUIRE(dtype == FVS_F16, "fvs_abstract_update: only f16 is implemented");
  FVS_REQUIRE(T1 > 0 && T2 > 0 && D > 0 && H > 0 && T1 <= 65535, "fvs_abstract_update: bad shape");
  cudaStream_t stream = (cudaStream_t)stream_;
  const size_t nfl = size_t(T1) * H + size_t(T2) * H + size_t(T1) * T2 + T1;
  float* scratch = nullptr;
  FVS_CUDA_OK(cudaMallocAsync(&scratch, nfl * sizeof(float), stream));
  AbsScratch S;
  S.q = scratch;
  S.k = S.q + size_t(T1) * H;
  S.wgt = S.k + size_t(T2) * H;
  S.decay = S.wgt + size_t(T1) * T2;
  abs_proj_kernel<<<T1 + T2, 256, 0, stream>>>((const uint16_t*)M, (const uint16_t*)F, (const uint16_t*)Wq, (const uint16_t*)bq,
                                               (const uint16_t*)Wk, (const uint16_t*)bk, S, T1, T2, D, H);
  FVS_CHECK_LAUNCH("abs_proj_kernel");
  abs_softmax_kernel<<<1, 256, 0, stream>>>(S, T1, T2, H, ratio);
  FVS_CHECK_LAUNCH("abs_softmax_kernel");
  abs_apply_kernel<<<dim3((D + 255) / 256, T1), 256, 0, stream>>>((const uint16_t*)M, (const uint16_t*)F, (uint16_t*)M_out, S, T1, T2, D);
  FVS_CHECK_LAUNCH("abs_apply_kernel");
  FVS_CUDA_OK(cudaFreeAsync(scratch, stream));
  return FVS_OK;
}

int fvs_argsort_desc(const void* w, int K, int64_t* order_out, int dtype, fvs_stream_t stream) {
  FVS_REQUIRE(w && order_out, "fvs_argsort_desc: null pointer");
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16 || dtype == FVS_F32, "fvs_argsort_desc: bad dtype");
  FVS_REQUIRE(K > 0 && K <= 1024, "fvs_argsort_desc: K must be in [1, 1024]");
  argsort_desc_kernel<<<1, 256, K * sizeof(float), (cudaStream_t)stream>>>(w, K, (long long*)order_out, dtype);
  FVS_CHECK_LAUNCH("argsort_desc_kernel");
  return FVS_OK;
}

int fvs_key_retrieve(const void* long_mem, const int64_t* order, int L, int P, int D, int key_len, int64_t* idx_out,
                     int dtype, fvs_stream_t stream_) {
  FVS_REQUIRE(long_mem && order && idx_out, "fvs_key_retrieve: null pointer");
  FVS_REQUIRE(dtype == FVS_F16, "fvs_key_retrieve: only f16 is implemented");
  FVS_REQUIRE(L > 0 && P > 0 && key_len > 0 && key_len <= L, "fvs_key_retrieve: bad shape L=%d P=%d key_len=%d", L, P, key_len);
  FVS_REQUIRE(D % 256 == 0, "fvs_key_retrieve: D (%d) must be a multiple of 256", D);
  cudaStream_t stream = (cudaStream_t)stream_;
  // distance scratch lives in a small stream-ordered allocation
  float* dist = nullptr;
  FVS_CUDA_OK(cudaMallocAsync(&dist, size_t(L) * key_len * sizeof(float), stream));
  key_dist_kernel<<<(L * key_len + 7) / 8, 256, 0, stream>>>((const uint16_t*)long_mem, (const long long*)order, dist, L, P, D, key_len);
  FVS_CHECK_LAUNCH("key_dist_kernel");
  key_argmin_kernel<<<key_len, 32, 0, stream>>>(dist, (long long*)idx_out, L, key_len);
  FVS_CHECK_LAUNCH("key_argmin_kernel");
  FVS_CUDA_OK(cudaFreeAsync(dist, stream));
  return FVS_OK;
}

int fvs_gather_rows(const void* src, const int64_t* idx, void* out, int n, int64_t row_elems, int dtype, fvs_stream_t stream) {
  FVS_REQUIRE(src && idx && out, "fvs_gather_rows: null pointer");
  FVS_REQUIRE(n > 0 && row_elems > 0, "fvs_gather_rows: bad shape");
  const int eb = dtype == FVS_F32 ? 4 : 2;
  FVS_REQUIRE((row_elems * eb) % 16 == 0, "fvs_gather_rows: row size must be a multiple of 16 bytes");
  const size_t row_vecs = size_t(row_elems) * eb / 16;
  size_t total = size_t(n) * row_vecs;
  int blocks = int((total + 255) / 256);
  if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  gather_rows_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const uint4*)src, (const long long*)idx, (uint4*)out, n, row_vecs);
  FVS_CHECK_LAUNCH("gather_rows_kernel");
  return FVS_OK;
}

}  // extern "C"
