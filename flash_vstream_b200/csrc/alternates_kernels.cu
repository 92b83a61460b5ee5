// alternates_kernels.cu — the alternate temporal compressors selectable through `video_sample_type`
// (Flash-VStream-LLaVA/flash_vstream/model/vstream_arch.py:222-236, 626-637):
//   drop_feature :19   merge_feature :57   kmeans_feature :91   k_drop_feature :170   k_merge_feature :213
// of flash_vstream/model/compress_functions.py.  The reference runs them as Python loops over the incoming frames with a
// host decision (argmax, coin flip) per frame; here each sequential compressor is ONE launch of a single persistent block
// that keeps the candidate set as slot indices, so a whole video is consolidated without a host round trip.  Work per
// frame is a handful of length-P*D reductions (HBM/L2-bound, no tensor-core shape).
// f16 arithmetic contract (oracle/alternates_oracle.py): one rounding per PyTorch op; fp32 sums in the canonical slice order
// (lane l of a warp owns elements i*256 + l*8 + e of a 1024-slice, sequential adds, xor butterfly; slices added in order).
#include <cuda_fp16.h>

#include "fvs_common.h"
#include "mem_device.cuh"

namespace fvs {
namespace alt {

using mem::SLICE;
using mem::butterfly_sum;
constexpr float NEG = -100.0f;

__device__ __forceinline__ float h2f(__half v) { return __half2float(v); }
__device__ __forceinline__ float rh(float v) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ bool better_max(float va, int ia, float vb, int ib) {  // NaN is maximal, then value, then first index
  const bool na = va != va, nb = vb != vb;
  if (na || nb) return (na && !nb) || (na && nb && ia < ib);
  return va > vb || (va == vb && ia < ib);
}

// canonical partial of one 1024-slice by one warp; term(e) gives element e of the slice
template <class F>
__device__ __forceinline__ float slice_partial(F term, int lane) {
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc = __fadd_rn(acc, term(i * 256 + lane * 8 + e));
  return butterfly_sum(acc);
}
// whole-row canonical sum by ONE warp (slices in order); every lane returns the total
template <class F>
__device__ __forceinline__ float warp_row_sum(F term, int PD, int lane) {
  float tot = 0.f;
  for (int s = 0; s < PD / SLICE; ++s) tot = __fadd_rn(tot, slice_partial([&](int e) { return term(s * SLICE + e); }, lane));
  return tot;
}
// whole-row canonical sum by the whole block (warp w takes slices w, w+nwarps, ...); every thread returns the total.
// sp: shared scratch of PD / 1024 floats.
template <class F>
__device__ __forceinline__ float block_row_sum(F term, int PD, float* sp) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5, S = PD / SLICE;
  __syncthreads();
  for (int s = warp; s < S; s += nw) {
    const float p = slice_partial([&](int e) { return term(s * SLICE + e); }, lane);
    if (lane == 0) sp[s] = p;
  }
  __syncthreads();
  float tot = 0.f;
  for (int s = 0; s < S; ++s) tot = __fadd_rn(tot, sp[s]);
  return tot;
}

__device__ __forceinline__ float norm_term(const __half* a, int e) { const float v = h2f(a[e]); return __fmul_rn(v, v); }
// F.cosine_similarity term: f16( f16(a/na) * f16(b/nb) )
__device__ __forceinline__ float cos_term(const __half* a, float na, const __half* b, float nb, int e) {
  return rh(__fmul_rn(rh(__fdiv_rn(h2f(a[e]), na)), rh(__fdiv_rn(h2f(b[e]), nb))));
}

struct SeqShared {
  float scratch[1024];   // slice partials (PD <= 1M elements)
  int decision[4];
};

// The global workspaces below (norms, frame slots, similarity matrix) are written by some threads of the block and read
// by others after a __syncthreads(), so their pointers are deliberately NOT __restrict__: with the qualifier the compiler
// may treat a read by another thread as unaffected by the barrier and hoist it above it (sm_90 code did exactly that for
// the norms, so every similarity against a new frame used that frame's stale norm).

// ------------------------------------------------------------------------------------------------ drop_feature
// nrm [T] workspace.  kept_out [T0] frame ids, sim_out [T0-1] f16, pos_out [T-T0] the row dropped at every step.
__global__ void __launch_bounds__(1024) drop_kernel(const __half* __restrict__ X, int T, int T0, int PD,
                                                    const __half* __restrict__ sim_in, const int* __restrict__ coins,
                                                    float* nrm, int* __restrict__ kept_out,
                                                    __half* __restrict__ sim_out, int* __restrict__ pos_out) {
  __shared__ SeqShared sh;
  extern __shared__ int dyn[];             // kept [T0+1] ints, then sim [T0+1] floats
  int* kept = dyn;
  float* sim = reinterpret_cast<float*>(dyn + T0 + 1);
  auto row = [&](int f) { return X + size_t(f) * PD; };
  auto norm_of = [&](int f) {
    const __half* a = row(f);
    return rh(sqrtf(block_row_sum([&](int e) { return norm_term(a, e); }, PD, sh.scratch)));
  };
  auto cosine = [&](int fa, int fb) {
    const __half *a = row(fa), *b = row(fb);
    const float na = nrm[fa], nb = nrm[fb];
    return rh(block_row_sum([&](int e) { return cos_term(a, na, b, nb, e); }, PD, sh.scratch));
  };
  for (int f = 0; f < T0; ++f) {
    const float v = norm_of(f);
    if (threadIdx.x == 0) { nrm[f] = v; kept[f] = f; }
  }
  __syncthreads();
  for (int j = 0; j < T0 - 1; ++j) {
    const float v = sim_in ? h2f(sim_in[j]) : cosine(j, j + 1);
    if (threadIdx.x == 0) sim[j] = v;
  }
  __syncthreads();
  for (int n = 0; n < T - T0; ++n) {
    const int i = T0 + n;
    const float nv = norm_of(i);
    if (threadIdx.x == 0) nrm[i] = nv;
    __syncthreads();
    const float new_sim = cosine(kept[T0 - 1], i);
    if (threadIdx.x == 0) {
      sim[T0 - 1] = new_sim;
      kept[T0] = i;
      float best = sim[0];
      int idx = 0;
      for (int j = 1; j < T0; ++j)
        if (better_max(sim[j], j, best, idx)) { best = sim[j]; idx = j; }
      if (coins[n] > 0) idx += 1;
      sh.decision[0] = idx;
      pos_out[n] = idx;
    }
    __syncthreads();
    const int idx = sh.decision[0];
    // the neighbours of the dropped row before the list is compacted
    const int left = idx > 0 ? kept[idx - 1] : -1, right = idx < T0 ? kept[idx + 1] : -1;
    float bridged = 0.f;
    if (idx > 0 && idx < T0) bridged = cosine(left, right);       // cur_sim[idx-1] = cos(all[idx-1], all[idx+1])
    __syncthreads();
    if (threadIdx.x == 0) {
      // all_sim has T0 entries (pairs j, j+1 of the T0+1 rows); dropping row idx removes pair idx-1 or idx
      if (idx == T0) {
        // keep all_sim[:T0-1]
      } else if (idx == 0) {
        for (int j = 0; j < T0 - 1; ++j) sim[j] = sim[j + 1];
      } else {
        for (int j = idx; j < T0 - 1; ++j) sim[j] = sim[j + 1];
        sim[idx - 1] = bridged;
      }
      for (int j = idx; j < T0; ++j) kept[j] = kept[j + 1];
    }
    __syncthreads();
  }
  for (int j = threadIdx.x; j < T0; j += blockDim.x) kept_out[j] = kept[j];
  for (int j = threadIdx.x; j < T0 - 1; j += blockDim.x) sim_out[j] = __float2half_rn(sim[j]);
}

// ------------------------------------------------------------------------------------------------ merge_feature
// W [T0+1, PD] f16 workspace of frame slots, nrm [T0+1].  out [T0, PD], sim_out [T0-1], pos_out [T-T0].
__global__ void __launch_bounds__(1024) merge_kernel(const __half* __restrict__ X, int T, int T0, int PD,
                                                     const __half* __restrict__ sim_in, __half* W,
                                                     float* nrm, __half* __restrict__ out,
                                                     __half* __restrict__ sim_out, int* __restrict__ pos_out) {
  __shared__ SeqShared sh;
  extern __shared__ int dyn[];             // order [T0+1] slots, then sim [T0+1] floats
  int* order = dyn;
  float* sim = reinterpret_cast<float*>(dyn + T0 + 1);
  auto slot = [&](int s) { return W + size_t(s) * PD; };
  auto renorm = [&](int s) {
    const __half* a = slot(s);
    const float v = rh(sqrtf(block_row_sum([&](int e) { return norm_term(a, e); }, PD, sh.scratch)));
    if (threadIdx.x == 0) nrm[s] = v;
    __syncthreads();
  };
  auto cosine = [&](int sa, int sb) {
    const __half *a = slot(sa), *b = slot(sb);
    const float na = nrm[sa], nb = nrm[sb];
    return rh(block_row_sum([&](int e) { return cos_term(a, na, b, nb, e); }, PD, sh.scratch));
  };
  for (size_t e = threadIdx.x; e < size_t(T0) * PD; e += blockDim.x) W[e] = X[e];
  if (threadIdx.x <= T0) order[threadIdx.x] = threadIdx.x;
  __syncthreads();
  for (int s = 0; s < T0; ++s) renorm(s);
  for (int j = 0; j < T0 - 1; ++j) {
    const float v = sim_in ? h2f(sim_in[j]) : cosine(j, j + 1);
    if (threadIdx.x == 0) sim[j] = v;
  }
  __syncthreads();
  for (int n = 0; n < T - T0; ++n) {
    const int fresh = order[T0];                                   // the free slot receives the new frame
    for (int e = threadIdx.x; e < PD; e += blockDim.x) slot(fresh)[e] = X[size_t(T0 + n) * PD + e];
    __syncthreads();
    renorm(fresh);
    const float new_sim = cosine(order[T0 - 1], fresh);
    if (threadIdx.x == 0) {
      sim[T0 - 1] = new_sim;
      float best = sim[0];
      int idx = 0;
      for (int j = 1; j < T0; ++j)
        if (better_max(sim[j], j, best, idx)) { best = sim[j]; idx = j; }
      sh.decision[0] = idx;
      pos_out[n] = idx;
    }
    __syncthreads();
    const int idx = sh.decision[0];
    const int sa = order[idx], sb = order[idx + 1];
    for (int e = threadIdx.x; e < PD; e += blockDim.x)             // all[idx+1] = (all[idx] + all[idx+1]) / 2
      slot(sb)[e] = __float2half_rn(__fdiv_rn(rh(__fadd_rn(h2f(slot(sa)[e]), h2f(slot(sb)[e]))), 2.0f));
    __syncthreads();
    renorm(sb);
    float s_left = 0.f, s_right = 0.f;
    if (idx > 0) s_left = cosine(order[idx - 1], sb);              // cur_sim[idx-1]
    if (idx + 1 < T0) s_right = cosine(sb, order[idx + 2]);        // cur_sim[idx]
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int j = idx; j < T0 - 1; ++j) sim[j] = sim[j + 1];      // remove pair idx
      for (int j = idx; j < T0; ++j) order[j] = order[j + 1];      // remove row idx
      order[T0] = sa;                                              // its slot is free again
      if (idx > 0) sim[idx - 1] = s_left;
      if (idx + 1 < T0) sim[idx] = s_right;
    }
    __syncthreads();
  }
  for (int r = 0; r < T0; ++r)
    for (int e = threadIdx.x; e < PD; e += blockDim.x) out[size_t(r) * PD + e] = slot(order[r])[e];
  for (int j = threadIdx.x; j < T0 - 1; j += blockDim.x) sim_out[j] = __float2half_rn(sim[j]);
}

// ------------------------------------------------------------------------------------------------ k_drop / k_merge
// all-pairs similarity over normalised rows.  NW [T0+1, PD] f16 normalised slots, W [T0+1, PD] feature slots (k_merge only),
// SM [(T0+1)^2] fp32 similarity matrix indexed by SLOT.  kMerge selects the variant.
template <bool kMerge>
__global__ void __launch_bounds__(1024) kpair_kernel(const __half* __restrict__ X, int T, int T0, int PD,
                                                     const int* __restrict__ coins, __half* W,
                                                     __half* NW, float* SM,
                                                     int* __restrict__ kept_out, __half* __restrict__ out,
                                                     __half* __restrict__ sim_out, int* __restrict__ pos_out) {
  __shared__ SeqShared sh;
  __shared__ float red_v[32];
  __shared__ int red_i[32];
  extern __shared__ int dyn[];             // order [T0+1] slots, frame [T0+1] frame id of every slot
  int* order = dyn;
  int* frame = dyn + T0 + 1;
  const int n1 = T0 + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  auto feat = [&](int s) -> const __half* { return kMerge ? W + size_t(s) * PD : X + size_t(frame[s]) * PD; };
  auto nslot = [&](int s) { return NW + size_t(s) * PD; };
  auto normalize = [&](int s) {                                    // NW[s] = f16(f / ||f||)
    const __half* a = feat(s);
    const float nv = rh(sqrtf(block_row_sum([&](int e) { return norm_term(a, e); }, PD, sh.scratch)));
    for (int e = threadIdx.x; e < PD; e += blockDim.x) nslot(s)[e] = __float2half_rn(__fdiv_rn(h2f(a[e]), nv));
    __syncthreads();
  };
  // sims of slot s against every slot in order[0..count): warp per partner row, written symmetrically
  auto sims_of = [&](int s, int count) {
    for (int p = warp; p < count; p += nw) {
      const int o = order[p];
      if (o == s) continue;
      const __half *a = nslot(o), *b = nslot(s);
      const float v = rh(warp_row_sum([&](int e) { return __fmul_rn(h2f(a[e]), h2f(b[e])); }, PD, lane));
      if (lane == 0) { SM[o * n1 + s] = v; SM[s * n1 + o] = v; }
    }
    if (threadIdx.x == 0) SM[s * n1 + s] = NEG;
    __syncthreads();
  };
  if (threadIdx.x <= T0) { order[threadIdx.x] = threadIdx.x; frame[threadIdx.x] = threadIdx.x; }
  if (kMerge)
    for (size_t e = threadIdx.x; e < size_t(T0) * PD; e += blockDim.x) W[e] = X[e];
  __syncthreads();
  for (int s = 0; s < T0; ++s) normalize(s);
  for (int s = 0; s < T0; ++s) sims_of(s, T0);
  for (int n = 0; n < T - T0; ++n) {
    const int fresh = order[T0];
    if (threadIdx.x == 0) frame[fresh] = T0 + n;
    if (kMerge)
      for (int e = threadIdx.x; e < PD; e += blockDim.x) W[size_t(fresh) * PD + e] = X[size_t(T0 + n) * PD + e];
    __syncthreads();
    normalize(fresh);
    sims_of(fresh, T0);                                            // new_sim column / last row; SM[fresh][fresh] = -100
    // argmax over the (T0+1)^2 matrix in logical (row-major over `order`) order
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int q = threadIdx.x; q < n1 * n1; q += blockDim.x) {
      const float v = SM[order[q / n1] * n1 + order[q % n1]];
      if (bi == 0x7fffffff || better_max(v, q, bv, bi)) { bv = v; bi = q; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi != 0x7fffffff && (bi == 0x7fffffff || better_max(ov, oi, bv, bi))) { bv = ov; bi = oi; }
    }
    if (lane == 0) { red_v[warp] = bv; red_i[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w2 = 1; w2 < nw; ++w2)
        if (red_i[w2] != 0x7fffffff && (bi == 0x7fffffff || better_max(red_v[w2], red_i[w2], bv, bi))) { bv = red_v[w2]; bi = red_i[w2]; }
      const int left = bi / n1, right = bi % n1;
      sh.decision[0] = left;
      sh.decision[1] = right;
      sh.decision[2] = kMerge ? left : (coins[n] > 0 ? left : right);   // the row that leaves
      pos_out[n] = kMerge ? bi : sh.decision[2];   // k_merge: the flat argmax left*(T0+1)+right; k_drop: the dropped row
    }
    __syncthreads();
    const int left = sh.decision[0], right = sh.decision[1], gone = sh.decision[2];
    if (kMerge) {
      const int sl = order[left], sr = order[right];
      for (int e = threadIdx.x; e < PD; e += blockDim.x)           // all[right] = (all[left] + all[right]) / 2
        W[size_t(sr) * PD + e] = __float2half_rn(__fdiv_rn(rh(__fadd_rn(h2f(W[size_t(sl) * PD + e]), h2f(W[size_t(sr) * PD + e]))), 2.0f));
      __syncthreads();
      normalize(sr);
      sims_of(sr, n1);                                             // row / column `right` against all T0+1 rows
    }
    if (threadIdx.x == 0) {
      const int freed = order[gone];
      for (int j = gone; j < T0; ++j) order[j] = order[j + 1];
      order[T0] = freed;
    }
    __syncthreads();
  }
  for (int j = threadIdx.x; j < T0; j += blockDim.x) kept_out[j] = frame[order[j]];
  if (kMerge) {
    for (int r = 0; r < T0; ++r)
      for (int e = threadIdx.x; e < PD; e += blockDim.x) out[size_t(r) * PD + e] = W[size_t(order[r]) * PD + e];
    for (int q = threadIdx.x; q < T0 * T0; q += blockDim.x)
      sim_out[q] = __float2half_rn(SM[order[q / T0] * n1 + order[q % T0]]);
  }
}

// ------------------------------------------------------------------------------------------------ kmeans_feature
struct KM {
  int* state;        // [0] done [1] cur [2] iter [3] refill_pos [4] converged
  __half* C[2];      // [K, PD]
  float* xn;         // [T]  f16(|x|^2) values
  float* cn;         // [K]
  float* dist;       // [T, K]
  float* nrm;        // [K]
  int* labels;       // [T]
  int* count;        // [K]
};
__device__ __forceinline__ float sq16_term(const __half* a, int e) { const float v = h2f(a[e]); return rh(__fmul_rn(v, v)); }

__global__ void kmf_init_kernel(KM B, const __half* __restrict__ X, const int* __restrict__ init_idx, int K, int PD) {
  if (blockIdx.x == 0 && threadIdx.x == 0) { B.state[0] = 0; B.state[1] = 0; B.state[2] = 0; B.state[3] = 0; B.state[4] = 0; }
  const int k = blockIdx.x;
  for (int e = threadIdx.x; e < PD; e += blockDim.x) B.C[0][size_t(k) * PD + e] = X[size_t(init_idx[k]) * PD + e];
}
// row |v|^2 = f16(sum_f32(f16(v^2))): warp per row; which = 0: X rows -> xn, 1: current centroids -> cn
__global__ void __launch_bounds__(256) kmf_rownorm_kernel(KM B, const __half* __restrict__ X, int rows, int PD, int which) {
  if (which && B.state[0]) return;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const __half* a = (which ? (B.state[1] ? B.C[1] : B.C[0]) : X) + size_t(r) * PD;
  const float v = rh(warp_row_sum([&](int e) { return sq16_term(a, e); }, PD, lane));
  if (lane == 0) (which ? B.cn : B.xn)[r] = v;
}
// dist[t,k] = f16(sqrt(max(f16(((-2x).c + |x|^2) + |c|^2), 0))): warp per (t, k)
__global__ void __launch_bounds__(256) kmf_dist_kernel(KM B, const __half* __restrict__ X, int T, int K, int PD) {
  if (B.state[0]) return;
  const int u = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (u >= T * K) return;
  const int t = u / K, k = u % K;
  const __half* x = X + size_t(t) * PD;
  const __half* c = (B.state[1] ? B.C[1] : B.C[0]) + size_t(k) * PD;
  const float ab = warp_row_sum([&](int e) { return __fmul_rn(__fmul_rn(-2.0f, h2f(x[e])), h2f(c[e])); }, PD, lane);
  const float tot = rh(__fadd_rn(__fadd_rn(ab, B.xn[t]), B.cn[k]));
  // clamp_min(0) keeps a NaN (-inf + inf once |x|^2 saturates); fmaxf(NaN, 0) would return 0, the nearest distance
  if (lane == 0) B.dist[u] = rh(sqrtf(tot < 0.0f ? 0.0f : tot));
}
__global__ void __launch_bounds__(256) kmf_assign_kernel(KM B, int T, int K) {
  if (B.state[0]) return;
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= T) return;
  float best = INFINITY;
  int bi = 0x7fffffff;
  for (int k = lane; k < K; k += 32) {
    const float d = B.dist[size_t(t) * K + k];
    const bool nd = d != d, nb = best != best;
    const bool take = bi == 0x7fffffff || (nd && !nb) || (nd == nb && (d < best || (d == best && k < bi))) || (nd && nb && k < bi);
    if (take) { best = d; bi = k; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi == 0x7fffffff) continue;
    const bool no = ov != ov, nb = best != best;
    const bool take = bi == 0x7fffffff || (no && !nb) || (no && nb && oi < bi) || (!no && !nb && (ov < best || (ov == best && oi < bi)));
    if (take) { best = ov; bi = oi; }
  }
  if (lane == 0) B.labels[t] = bi;
}
// new centroid slices: warp per (k, slice): mean of members (fp32, t ascending, / n, one rounding) or a refill row
__global__ void __launch_bounds__(256) kmf_update_kernel(KM B, const __half* __restrict__ X, const int* __restrict__ refill_idx,
                                                         int T, int K, int PD) {
  if (B.state[0]) return;
  const int S = PD / SLICE;
  const int u = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (u >= K * S) return;
  const int j = u / S, s = u % S;
  int n_j = 0, empties_before = 0;
  for (int c = lane; c <= j; c += 32) {
    int cnt = 0;
    for (int t = 0; t < T; ++t) cnt += B.labels[t] == c;
    if (c == j) n_j = cnt;
    else if (cnt == 0) empties_before++;
  }
  n_j = __reduce_add_sync(0xffffffffu, n_j);
  empties_before = __reduce_add_sync(0xffffffffu, empties_before);
  __half* dst = (B.state[1] ? B.C[0] : B.C[1]) + size_t(j) * PD + size_t(s) * SLICE;
  if (n_j > 0) {
    float acc[32];
#pragma unroll
    for (int q = 0; q < 32; ++q) acc[q] = 0.f;
    for (int t = 0; t < T; ++t) {
      if (B.labels[t] != j) continue;
      const __half* x = X + size_t(t) * PD + size_t(s) * SLICE;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[i * 8 + e] = __fadd_rn(acc[i * 8 + e], h2f(x[i * 256 + lane * 8 + e]));
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int e = 0; e < 8; ++e) dst[i * 256 + lane * 8 + e] = __float2half_rn(__fdiv_rn(acc[i * 8 + e], float(n_j)));
  } else {
    const __half* x = X + size_t(refill_idx[B.state[3] + empties_before]) * PD + size_t(s) * SLICE;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int e = 0; e < 8; ++e) dst[i * 256 + lane * 8 + e] = x[i * 256 + lane * 8 + e];
  }
  if (lane == 0 && s == 0) B.count[j] = n_j;
}
// nrm[k] = f16(||f16(c - c')||): warp per k
__global__ void __launch_bounds__(256) kmf_diff_kernel(KM B, int K, int PD) {
  if (B.state[0]) return;
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= K) return;
  const __half* a = (B.state[1] ? B.C[1] : B.C[0]) + size_t(k) * PD;
  const __half* b = (B.state[1] ? B.C[0] : B.C[1]) + size_t(k) * PD;
  const float v = warp_row_sum([&](int e) { const float d = rh(__fsub_rn(h2f(a[e]), h2f(b[e]))); return __fmul_rn(d, d); }, PD, lane);
  if (lane == 0) B.nrm[k] = rh(sqrtf(v));
}
__global__ void kmf_converge_kernel(KM B, int K, int iter, int max_iter, float tol_h) {
  if (B.state[0] || threadIdx.x != 0) return;
  float diff = 0.f;
  int n_empty = 0;
  for (int k = 0; k < K; ++k) {
    diff = __fadd_rn(diff, B.nrm[k]);
    n_empty += B.count[k] == 0;
  }
  diff = rh(diff);
  B.state[2] = iter;
  B.state[3] += n_empty;
  if (diff < tol_h) { B.state[0] = 1; B.state[4] = 1; }      // break: the OLD centroids stay
  else { B.state[1] ^= 1; if (iter == max_iter - 1) B.state[0] = 1; }
}
__global__ void kmf_finish_kernel(KM B, __half* __restrict__ C_out, int* __restrict__ labels_out, int* __restrict__ info_out,
                                  int T, int K, int PD) {
  const __half* src = B.state[1] ? B.C[1] : B.C[0];
  for (size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x; i < size_t(K) * PD; i += size_t(gridDim.x) * blockDim.x) C_out[i] = src[i];
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < T; i += blockDim.x) labels_out[i] = B.labels[i];
    if (threadIdx.x == 0) { info_out[0] = B.state[2]; info_out[1] = B.state[3]; info_out[2] = B.state[4]; info_out[3] = 0; }
  }
}

inline size_t al(size_t v) { return (v + 255) & ~size_t(255); }

}  // namespace alt
}  // namespace fvs

using namespace fvs;
using namespace fvs::alt;

extern "C" {

size_t fvs_alt_workspace_bytes(int method, int T, int T0, int PD) {
  if (T <= 0 || T0 <= 0 || PD <= 0) return 0;
  const size_t slots = size_t(T0) + 1;
  switch (method) {
    case FVS_ALT_DROP: return al(size_t(T) * 4);
    case FVS_ALT_MERGE: return al(slots * PD * 2) + al(slots * 4);
    case FVS_ALT_KDROP: return al(slots * PD * 2) + al(slots * slots * 4);
    case FVS_ALT_KMERGE: return 2 * al(slots * PD * 2) + al(slots * slots * 4);
    case FVS_ALT_KMEANS:
      return al(32) + 2 * al(size_t(T0) * PD * 2) + al(size_t(T) * 4) + 2 * al(size_t(T0) * 4) + al(size_t(T) * T0 * 4) +
             al(size_t(T) * 4) + al(size_t(T0) * 4);
    default: return 0;
  }
}

int fvs_alt_sequential(int method, const void* X, int T, int T0, int PD, const void* sim_in, const int32_t* coins,
                       int32_t* kept_out, void* feat_out, void* sim_out, int32_t* pos_out, void* workspace,
                       size_t workspace_bytes, int dtype, fvs_stream_t stream_) {
  FVS_REQUIRE(X && pos_out && workspace, "fvs_alt_sequential: null pointer");
  FVS_REQUIRE(dtype == FVS_F16, "fvs_alt_sequential: only f16 is implemented (the reference consolidates float16 features)");
  FVS_REQUIRE(method == FVS_ALT_DROP || method == FVS_ALT_MERGE || method == FVS_ALT_KDROP || method == FVS_ALT_KMERGE,
              "fvs_alt_sequential: unknown method %d", method);
  FVS_REQUIRE(T > T0 && T0 >= 2, "fvs_alt_sequential: need T > T0 >= 2 (T=%d T0=%d); T <= T0 is a pass-through handled by the caller", T, T0);
  FVS_REQUIRE(PD % SLICE == 0 && PD <= 1024 * SLICE, "fvs_alt_sequential: PD (%d) must be a multiple of 1024, at most 1048576", PD);
  FVS_REQUIRE(T0 <= 1023, "fvs_alt_sequential: T0 must be <= 1023");
  FVS_REQUIRE(workspace_bytes >= fvs_alt_workspace_bytes(method, T, T0, PD), "fvs_alt_sequential: workspace too small");
  FVS_REQUIRE((method != FVS_ALT_DROP && method != FVS_ALT_KDROP) || (coins && kept_out), "fvs_alt_sequential: drop variants need coins and kept_out");
  FVS_REQUIRE((method != FVS_ALT_MERGE && method != FVS_ALT_KMERGE) || feat_out, "fvs_alt_sequential: merge variants need feat_out");
  FVS_REQUIRE(method == FVS_ALT_KDROP || sim_out, "fvs_alt_sequential: sim_out required");
  cudaStream_t stream = (cudaStream_t)stream_;
  const size_t slots = size_t(T0) + 1;
  uint8_t* p = (uint8_t*)workspace;
  const size_t dyn = slots * 8;
  if (method == FVS_ALT_DROP) {
    drop_kernel<<<1, 1024, dyn, stream>>>((const __half*)X, T, T0, PD, (const __half*)sim_in, coins, (float*)p, kept_out,
                                          (__half*)sim_out, pos_out);
    FVS_CHECK_LAUNCH("drop_kernel");
  } else if (method == FVS_ALT_MERGE) {
    __half* W = (__half*)p; p += al(slots * PD * 2);
    merge_kernel<<<1, 1024, dyn, stream>>>((const __half*)X, T, T0, PD, (const __half*)sim_in, W, (float*)p, (__half*)feat_out,
                                           (__half*)sim_out, pos_out);
    FVS_CHECK_LAUNCH("merge_kernel");
  } else if (method == FVS_ALT_KDROP) {
    __half* NW = (__half*)p; p += al(slots * PD * 2);
    kpair_kernel<false><<<1, 1024, dyn, stream>>>((const __half*)X, T, T0, PD, coins, nullptr, NW, (float*)p, kept_out, nullptr,
                                                  nullptr, pos_out);
    FVS_CHECK_LAUNCH("kpair_kernel");
  } else {
    __half* W = (__half*)p; p += al(slots * PD * 2);
    __half* NW = (__half*)p; p += al(slots * PD * 2);
    FVS_REQUIRE(kept_out != nullptr, "fvs_alt_sequential: kept_out required");
    kpair_kernel<true><<<1, 1024, dyn, stream>>>((const __half*)X, T, T0, PD, nullptr, W, NW, (float*)p, kept_out,
                                                 (__half*)feat_out, (__half*)sim_out, pos_out);
    FVS_CHECK_LAUNCH("kpair_kernel");
  }
  return FVS_OK;
}

int fvs_alt_kmeans(const void* X, const int32_t* init_idx, const int32_t* refill_idx, int T, int K, int PD, int max_iter,
                   float tol, void* C_out, int32_t* labels_out, int32_t* info_out, void* workspace, size_t workspace_bytes,
                   int dtype, fvs_stream_t stream_) {
  FVS_REQUIRE(X && init_idx && refill_idx && C_out && labels_out && info_out && workspace, "fvs_alt_kmeans: null pointer");
  FVS_REQUIRE(dtype == FVS_F16, "fvs_alt_kmeans: only f16 is implemented");
  FVS_REQUIRE(T > 0 && K > 0 && K <= T && PD % SLICE == 0, "fvs_alt_kmeans: bad shape T=%d K=%d PD=%d", T, K, PD);
  FVS_REQUIRE(max_iter > 0 && max_iter <= 1000, "fvs_alt_kmeans: bad max_iter");
  FVS_REQUIRE(workspace_bytes >= fvs_alt_workspace_bytes(FVS_ALT_KMEANS, T, K, PD), "fvs_alt_kmeans: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  uint8_t* p = (uint8_t*)workspace;
  KM B;
  B.state = (int*)p; p += al(32);
  B.C[0] = (__half*)p; p += al(size_t(K) * PD * 2);
  B.C[1] = (__half*)p; p += al(size_t(K) * PD * 2);
  B.xn = (float*)p; p += al(size_t(T) * 4);
  B.cn = (float*)p; p += al(size_t(K) * 4);
  B.nrm = (float*)p; p += al(size_t(K) * 4);
  B.dist = (float*)p; p += al(size_t(T) * K * 4);
  B.labels = (int*)p; p += al(size_t(T) * 4);
  B.count = (int*)p;
  const __half* Xh = (const __half*)X;
  const int S = PD / SLICE;
  const float tol_h = __half2float(__float2half_rn(tol));   // `diff < tol` is evaluated in f16
  kmf_init_kernel<<<K, 256, 0, stream>>>(B, Xh, init_idx, K, PD);
  FVS_CHECK_LAUNCH("kmf_init_kernel");
  kmf_rownorm_kernel<<<(T + 7) / 8, 256, 0, stream>>>(B, Xh, T, PD, 0);
  FVS_CHECK_LAUNCH("kmf_rownorm_kernel");
  for (int it = 0; it < max_iter; ++it) {
    kmf_rownorm_kernel<<<(K + 7) / 8, 256, 0, stream>>>(B, Xh, K, PD, 1);
    FVS_CHECK_LAUNCH("kmf_rownorm_kernel");
    kmf_dist_kernel<<<(T * K + 7) / 8, 256, 0, stream>>>(B, Xh, T, K, PD);
    FVS_CHECK_LAUNCH("kmf_dist_kernel");
    kmf_assign_kernel<<<(T + 7) / 8, 256, 0, stream>>>(B, T, K);
    FVS_CHECK_LAUNCH("kmf_assign_kernel");
    kmf_update_kernel<<<(K * S + 7) / 8, 256, 0, stream>>>(B, Xh, refill_idx, T, K, PD);
    FVS_CHECK_LAUNCH("kmf_update_kernel");
    kmf_diff_kernel<<<(K + 7) / 8, 256, 0, stream>>>(B, K, PD);
    FVS_CHECK_LAUNCH("kmf_diff_kernel");
    kmf_converge_kernel<<<1, 32, 0, stream>>>(B, K, it, max_iter, tol_h);
    FVS_CHECK_LAUNCH("kmf_converge_kernel");
  }
  kmf_finish_kernel<<<device_sm_count(), 256, 0, stream>>>(B, (__half*)C_out, labels_out, info_out, T, K, PD);
  FVS_CHECK_LAUNCH("kmf_finish_kernel");
  return FVS_OK;
}

}  // extern "C"
