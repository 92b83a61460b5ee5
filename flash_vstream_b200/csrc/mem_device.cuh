// mem_device.cuh — the reference-exact f16 arithmetic of the Flash-Memory consolidation, written once.
//   * canonical-order primitives (SLICE, butterfly_sum, argmin_better, warp_argmin): the canonical slice reduction and the
//     torch.argmin ordering that make "index selections bit-exact" testable (DESIGN.md §1 "canonical summation order").
//     Used by every reduction kernel: memory_kernels.cu, stream_kernels.cu, qwen_kernels.cu, alternates_kernels.cu.
//   * per-unit bodies of the STAR consolidation (k-means update / label / convergence term, stable argsort rank, key-frame
//     distance, abstract-memory projection / softmax / apply). Each is the work of ONE warp or ONE thread and takes
//     pointers and strides, so the op-by-op kernels (memory_kernels.cu) and the fused step kernel (consolidate_kernel in
//     stream_kernels.cu) run the same code with their own launch geometry, barriers and bookkeeping.
// oracle/fvs_oracle.py mirrors all of it operation for operation.
#pragma once
#include <cuda_fp16.h>
#include <cstdint>

namespace fvs {
namespace mem {

constexpr int SLICE = 1024;  // elements per canonical reduction slice (32 lanes x 4 iterations x 8 elements)

__device__ __forceinline__ float h2f(uint16_t v) { return __half2float(__ushort_as_half(v)); }
__device__ __forceinline__ uint16_t f2h(float v) { return __half_as_ushort(__float2half_rn(v)); }
__device__ __forceinline__ float round_h(float v) { return __half2float(__float2half_rn(v)); }

__device__ __forceinline__ float butterfly_sum(float v) {
  // xor-butterfly: every lane ends with the same value; order 16, 8, 4, 2, 1 is part of the canonical order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Canonical slice reduction.  For a 1024-element slice, lane l owns elements {i*256 + l*8 + e : i<4, e<8};
// it adds its 32 terms sequentially in (i, e) order starting from 0.0f, then the 32 lane sums are combined
// with the xor-butterfly above.  Terms are f16(f16(a-b)^2) widened to fp32 (so no FMA contraction is possible).
__device__ __forceinline__ float slice_sqdiff(const uint4 (&a)[4], const uint16_t* __restrict__ b, int lane) {
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint4 bv = *reinterpret_cast<const uint4*>(b + i * 256 + lane * 8);
    const uint32_t aw[4] = {a[i].x, a[i].y, a[i].z, a[i].w};
    const uint32_t bw[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const __half2 d = __hsub2(*reinterpret_cast<const __half2*>(&aw[p]), *reinterpret_cast<const __half2*>(&bw[p]));
      const __half2 s = __hmul2(d, d);
      acc = acc + __low2float(s);
      acc = acc + __high2float(s);
    }
  }
  return butterfly_sum(acc);
}

__device__ __forceinline__ void load_slice(uint4 (&a)[4], const uint16_t* __restrict__ src, int lane) {
#pragma unroll
  for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const uint4*>(src + i * 256 + lane * 8);
}

// NaN-wins, first-index argmin ordering (torch.argmin semantics): true if (va, ia) beats (vb, ib)
__device__ __forceinline__ bool argmin_better(float va, int ia, float vb, int ib) {
  const bool na = va != va, nb = vb != vb;
  if (na || nb) return (na && !nb) || (na && nb && ia < ib);
  return va < vb || (va == vb && ia < ib);
}
__device__ __forceinline__ void warp_argmin(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (argmin_better(ov, oi, v, i)) { v = ov; i = oi; }
  }
}

// First-index / NaN-wins argmin of value_of(0 .. n-1) by one warp (lane-strided, then warp_argmin); every lane returns it.
template <class V>
__device__ __forceinline__ int warp_argmin_of(int n, V value_of, int lane) {
  float best = INFINITY;
  int besti = 0x7fffffff;
  for (int i = lane; i < n; i += 32) {
    const float d = value_of(i);
    if (besti == 0x7fffffff || argmin_better(d, i, best, besti)) { best = d; besti = i; }
  }
  warp_argmin(best, besti);
  return besti;
}

// ------------------------------------------------------------------------------------------------ weighted k-means
// Label of one row (one warp): argmin over k of f16(sqrt(f16(sum_s part[k*S + s]))), part = the row's [K, S] slice partials.
__device__ __forceinline__ int km_row_label(const float* part, int K, int S, int lane) {
  return warp_argmin_of(K, [&](int k) {
    float tot = 0.f;
    for (int s = 0; s < S; ++s) tot = tot + part[k * S + s];
    return round_h(sqrtf(round_h(tot)));
  }, lane);
}

// Lloyd update of cluster j, 1024-slice s, by one warp (compress_functions.py:144-153).  weights_sum[j] = f16 of the member
// weights summed in t order; c_new = f16(f16(sum_t f16(w_t x_t)) / weights_sum[j]), or, for an empty cluster, the slice of
// row refill[e] where e = number of empty clusters before j (refills are consumed in j order).  Then the partial of
// ||c_old - c_new||^2 for the convergence test.  X: [T, PD] rows; w: [T] f16 weights, nullptr for unit weights;
// Cold / Cnew: slice s of the old / new centroid j.  Lane 0 writes normpart[j*S + s] and, from slice 0, wsum[j].
__device__ __forceinline__ void km_cluster_slice_update(const uint16_t* X, const uint16_t* w, const int* labels,
                                                        const int* refill, int T, int PD, int S, int j, int s,
                                                        const uint16_t* Cold, uint16_t* Cnew, float* normpart,
                                                        uint16_t* wsum, int lane) {
  // Every warp recomputes the per-cluster sums it needs from the labels: T is small (<= a few thousand).
  // Lane-parallel over clusters 0..j to count empties (sum order inside a cluster: sequential in t).
  float wsum_j = 0.f;
  int empties_before = 0;
  for (int c = lane; c <= j; c += 32) {
    float ws = 0.f;
    for (int t = 0; t < T; ++t)
      if (labels[t] == c) ws = ws + (w ? h2f(w[t]) : 1.0f);
    const float wsh = round_h(ws);
    if (c == j) wsum_j = wsh;
    else if (!(wsh > 0.f)) empties_before++;
  }
  wsum_j = butterfly_sum(wsum_j);  // exactly one lane holds a non-zero value (or all zero)
  empties_before = __reduce_add_sync(0xffffffffu, empties_before);

  uint32_t outw[4][4];
  if (wsum_j > 0.f) {
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[i][e] = 0.f;
    for (int t = 0; t < T; ++t) {
      if (labels[t] != j) continue;
      const __half2 wt2 = __half2half2(w ? __ushort_as_half(w[t]) : __float2half_rn(1.0f));
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint4 xv = *reinterpret_cast<const uint4*>(X + size_t(t) * PD + s * SLICE + i * 256 + lane * 8);
        const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const __half2 pr = __hmul2(wt2, *reinterpret_cast<const __half2*>(&xw[p]));  // f16(w * x)
          acc[i][2 * p] = acc[i][2 * p] + __low2float(pr);
          acc[i][2 * p + 1] = acc[i][2 * p + 1] + __high2float(pr);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        // f16(f16(weighted_sum) / f16(weights_sum))
        const float a = round_h(acc[i][2 * p]) / wsum_j, b = round_h(acc[i][2 * p + 1]) / wsum_j;
        __half2 h = __floats2half2_rn(a, b);
        outw[i][p] = *reinterpret_cast<uint32_t*>(&h);
      }
  } else {
    const int src = refill[empties_before];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint4 xv = *reinterpret_cast<const uint4*>(X + size_t(src) * PD + s * SLICE + i * 256 + lane * 8);
      outw[i][0] = xv.x; outw[i][1] = xv.y; outw[i][2] = xv.z; outw[i][3] = xv.w;
    }
  }
  // convergence partial: sum of float(f16(c_old - c_new))^2 in canonical slice order (squares NOT rounded: torch.norm)
  float nacc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint4 ov = *reinterpret_cast<const uint4*>(Cold + i * 256 + lane * 8);
    const uint32_t ow[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const __half2 d = __hsub2(*reinterpret_cast<const __half2*>(&ow[p]), *reinterpret_cast<const __half2*>(&outw[i][p]));
      const float dl = __low2float(d), dh = __high2float(d);
      nacc = nacc + __fmul_rn(dl, dl);
      nacc = nacc + __fmul_rn(dh, dh);
    }
    *reinterpret_cast<uint4*>(Cnew + i * 256 + lane * 8) = make_uint4(outw[i][0], outw[i][1], outw[i][2], outw[i][3]);
  }
  nacc = butterfly_sum(nacc);
  if (lane == 0) {
    normpart[j * S + s] = nacc;
    if (s == 0) wsum[j] = f2h(wsum_j);
  }
}

// Cluster k's term of the convergence test diff = f16(sum_k f16(sqrt(sum_s normpart[k*S + s]))) < tol; the caller adds
// the terms in k order and rounds once.
__device__ __forceinline__ float centroid_shift(const float* normpart, int k, int S) {
  float tot = 0.f;
  for (int s = 0; s < S; ++s) tot = tot + normpart[k * S + s];
  return round_h(sqrtf(tot));
}

// ------------------------------------------------------------------------------------------------ argsort / retrieval
// Position of element i in the stable descending order of value_of(0 .. K-1), NaN largest (torch.sort convention).
template <class V>
__device__ __forceinline__ int stable_desc_rank(int i, int K, V value_of) {
  const float vi = value_of(i);
  const bool ni = vi != vi;
  int rank = 0;
  for (int j = 0; j < K; ++j) {
    const float vj = value_of(j);
    const bool nj = vj != vj;
    bool before;  // does j come before i in descending stable order?
    if (ni || nj) before = (nj && !ni) || (nj && ni && j < i);
    else before = vj > vi || (vj == vi && j < i);
    rank += before ? 1 : 0;
  }
  return rank;
}

// Key-frame distance of rows a, b of P patches x D channels (D % 256 == 0), one warp; every lane returns
// f16(sqrt(f16(sum_p f16(sum_d f16(f16(a-b)^2))))).  The per-patch sum over D is ONE warp pass: lane l owns elements
// i*256 + l*8 + e, sequential in (i, e), then the butterfly (oracle: _lane_sum).
__device__ __forceinline__ float key_distance(const uint16_t* a, const uint16_t* b, int P, int D, int lane) {
  float tot = 0.f;
  for (int p = 0; p < P; ++p) {
    float acc = 0.f;
    for (int i = 0; i < D / 256; ++i) {
      const uint4 av = *reinterpret_cast<const uint4*>(a + size_t(p) * D + i * 256 + lane * 8);
      const uint4 bv = *reinterpret_cast<const uint4*>(b + size_t(p) * D + i * 256 + lane * 8);
      const uint32_t aw[4] = {av.x, av.y, av.z, av.w};
      const uint32_t bw[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const __half2 d = __hsub2(*reinterpret_cast<const __half2*>(&aw[q]), *reinterpret_cast<const __half2*>(&bw[q]));
        const __half2 sq = __hmul2(d, d);
        acc = acc + __low2float(sq);
        acc = acc + __high2float(sq);
      }
    }
    tot = tot + round_h(butterfly_sum(acc));
  }
  return round_h(sqrtf(round_h(tot)));
}

// ------------------------------------------------------------------------------------------------ abstract memory
// Rounding points follow the f16 PyTorch expression tree of attention / get_weight (vstream_arch.py:174-183, :47-52).

// One projection output, one warp: f16(x . wrow + bias), one rounding after the bias (addmm epilogue); every lane returns it.
__device__ __forceinline__ float abs_proj_dot(const uint16_t* x, const uint16_t* wrow, const uint16_t* bias, int D, int lane) {
  float acc = 0.f;
  for (int d = lane; d < D; d += 32) acc = fmaf(h2f(x[d]), h2f(wrow[d]), acc);
  return round_h(butterfly_sum(acc) + h2f(*bias));
}

// One memory row i, one warp: wrow[j] = f16(f16(softmax_j(f16(f16(q_i k_j^T) / sqrt(H)))) * ratio) for the T2 rows of k
// (q, k: [.., H]); returns the row's decay f16(sum_j wrow[j]) on every lane.
__device__ __forceinline__ float abs_softmax_row(const float* q, const float* k, int i, float* wrow, int T2, int H,
                                                 float sqrtH, float ratio, int lane) {
  float mx = -INFINITY;
  for (int j = lane; j < T2; j += 32) {
    float acc = 0.f;
    for (int h = 0; h < H; ++h) acc = fmaf(q[i * H + h], k[j * H + h], acc);
    const float sc = round_h(round_h(acc) / sqrtH);
    wrow[j] = sc;
    mx = fmaxf(mx, sc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < T2; j += 32) {
    const float e = expf(wrow[j] - mx);
    wrow[j] = e;
    sum += e;
  }
  sum = butterfly_sum(sum);
  float dsum = 0.f;
  for (int j = lane; j < T2; j += 32) {
    const float wv = round_h(round_h(wrow[j] / sum) * ratio);
    wrow[j] = wv;
    dsum += wv;
  }
  return round_h(butterfly_sum(dsum));
}

// One element (row of wrow, channel d) of the updated memory, one thread:
// f16( f16(m * f16(1 - decay)) + f16(sum_j wrow[j] * F[j, d]) ), F: [T2, D].
__device__ __forceinline__ uint16_t abs_apply_elem(const float* wrow, const uint16_t* F, int T2, int D, int d, uint16_t m,
                                                   float decay) {
  float acc = 0.f;
  for (int j = 0; j < T2; ++j) acc = fmaf(wrow[j], h2f(F[size_t(j) * D + d]), acc);
  const float keep = round_h(h2f(m) * round_h(1.0f - decay));
  return f2h(keep + round_h(acc));
}

}  // namespace mem
}  // namespace fvs
