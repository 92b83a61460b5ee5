// vit_misc.cu — the HBM-bound glue kernels of the ViT encoder: LayerNorm, im2col for the patch-embed GEMM,
// CLS-drop copy. (SURVEY.md §2.2 K1/K2: CLIPVisionEmbeddings / pre_layrnorm / layer_norm1/2.)
#include "fvs_common.h"
#include "fvs_ptx.cuh"

namespace fvs {

template <bool kBF16>
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (kBF16) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
    } else {
      const __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
      const float2 t = __half22float2(h);
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
  }
}
template <bool kBF16>
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (kBF16) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    } else {
      __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One warp per row; the row (dim = kChunks * 256 elements) lives in registers between the two passes.
// x may be 16-bit (kBF16 selects f16/bf16) or fp32 (the ViT residual stream); y likewise. gamma/beta are 16-bit.
// If `delta` is non-null (only with fp32 x): x += delta first and the updated x is written back — the residual add of the
// ViT encoder fused into the LayerNorm that follows it (the GEMM before it emits the 16-bit delta).
template <int kChunks, bool kBF16, bool kXF32, bool kYF32>
__global__ void __launch_bounds__(256) layernorm_kernel(const void* __restrict__ x_, const uint4* __restrict__ gamma,
                                                        const uint4* __restrict__ beta, void* __restrict__ y_,
                                                        int rows, float eps, const uint4* __restrict__ delta) {
  pdl_trigger();  // PDL: let the GEMM that follows start its prologue; wait for the kernel that produced x / delta
  pdl_wait();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  constexpr int kDim = kChunks * 256;
  float v[kChunks][8];
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < kChunks; ++c) {
    if (kXF32) {
      float4* xr = reinterpret_cast<float4*>(const_cast<float*>(static_cast<const float*>(x_)) + size_t(row) * kDim + c * 256 + lane * 8);
      const float4 a = xr[0], b = xr[1];
      v[c][0] = a.x; v[c][1] = a.y; v[c][2] = a.z; v[c][3] = a.w;
      v[c][4] = b.x; v[c][5] = b.y; v[c][6] = b.z; v[c][7] = b.w;
      if (delta != nullptr) {
        float d[8];
        unpack8<kBF16>(delta[size_t(row) * (kDim / 8) + c * 32 + lane], d);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[c][e] += d[e];
        xr[0] = make_float4(v[c][0], v[c][1], v[c][2], v[c][3]);
        xr[1] = make_float4(v[c][4], v[c][5], v[c][6], v[c][7]);
      }
    } else {
      unpack8<kBF16>(reinterpret_cast<const uint4*>(x_)[size_t(row) * (kDim / 8) + c * 32 + lane], v[c]);
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) s += v[c][e];
  }
  const float mean = warp_sum(s) * (1.0f / kDim);
  float q = 0.f;
#pragma unroll
  for (int c = 0; c < kChunks; ++c)
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float d = v[c][e] - mean;
      q = fmaf(d, d, q);
    }
  const float var = warp_sum(q) * (1.0f / kDim);
  const float rstd = 1.0f / sqrtf(var + eps);
#pragma unroll
  for (int c = 0; c < kChunks; ++c) {
    float g[8], b[8], o[8];
    unpack8<kBF16>(gamma[c * 32 + lane], g);
    unpack8<kBF16>(beta[c * 32 + lane], b);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = fmaf((v[c][e] - mean) * rstd, g[e], b[e]);
    if (kYF32) {
      float4* yr = reinterpret_cast<float4*>(static_cast<float*>(y_) + size_t(row) * kDim + c * 256 + lane * 8);
      yr[0] = make_float4(o[0], o[1], o[2], o[3]);
      yr[1] = make_float4(o[4], o[5], o[6], o[7]);
    } else {
      reinterpret_cast<uint4*>(y_)[size_t(row) * (kDim / 8) + c * 32 + lane] = pack8<kBF16>(o);
    }
  }
}

// pixels [B,3,S,S] -> patches [B*(G*G+1), Kpad]; row 0 of every frame (the CLS slot) and columns >= 3*P*P are 0.
// Column order c*P*P + ky*P + kx matches Conv2d weight.view(hidden, -1).
__global__ void im2col_kernel(const uint16_t* __restrict__ pix, uint16_t* __restrict__ out, int B, int S, int P, int G,
                              int Kpad) {
  const int tok = blockIdx.x;  // 0 .. G*G
  const int b = blockIdx.y;
  uint16_t* orow = out + (size_t(b) * (G * G + 1) + tok) * Kpad;
  const int kreal = 3 * P * P;
  if (tok == 0) {
    for (int k = threadIdx.x; k < Kpad; k += blockDim.x) orow[k] = 0;
    return;
  }
  const int p = tok - 1, py = p / G, px = p % G;
  for (int k = threadIdx.x; k < Kpad; k += blockDim.x) {
    uint16_t v = 0;
    if (k < kreal) {
      const int c = k / (P * P), r = k % (P * P), ky = r / P, kx = r % P;
      v = pix[((size_t(b) * 3 + c) * S + (py * P + ky)) * S + (px * P + kx)];
    }
    orow[k] = v;
  }
}

// x fp32 [B, tokens, D] (residual stream) [+ 16-bit delta of the last GEMM] -> out 16-bit [B, tokens-1, D]
// (drop token 0, round once), 8 elements per thread
template <bool kBF16>
__global__ void drop_cls_kernel(const float* __restrict__ x, const uint4* __restrict__ delta, uint4* __restrict__ out,
                                int tokens, int first, int vec_per_row, size_t total_vec) {
  const size_t per_frame = size_t(tokens - first) * vec_per_row;   // first = 1: drop the CLS row ('patch'), 0: keep it
  for (size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x; i < total_vec; i += size_t(gridDim.x) * blockDim.x) {
    const size_t b = i / per_frame, r = i % per_frame;
    const size_t sv = (b * tokens + first) * vec_per_row + r;
    const float4* src = reinterpret_cast<const float4*>(x + sv * 8);
    const float4 a = src[0], c = src[1];
    float f[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
    if (delta != nullptr) {
      float d[8];
      unpack8<kBF16>(delta[sv], d);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] += d[e];
    }
    out[i] = pack8<kBF16>(f);
  }
}

int layernorm_launch(const void* x, const void* gamma, const void* beta, void* y, int rows, int dim, float eps,
                     int dtype, bool x_f32, bool y_f32, const void* delta, cudaStream_t stream, bool pdl) {
  if (delta != nullptr && !x_f32) return set_error(FVS_EINVAL, "layernorm: a residual delta needs an fp32 x");
  if (dim % 256 != 0 || dim > 2048) return set_error(FVS_EINVAL, "layernorm: dim %d must be a multiple of 256, <= 2048", dim);
  const int chunks = dim / 256;
  const dim3 grid((rows + 7) / 8), block(256);
  const bool bf = dtype == FVS_BF16;
  const uint4* g = (const uint4*)gamma;
  const uint4* b = (const uint4*)beta;
#define FVS_LN_LAUNCH(C, BF, XF, YF)                                                                                  \
  FVS_CUDA_OK(launch_ex(layernorm_kernel<C, BF, XF, YF>, grid, block, 0, stream, 1, pdl, x, g, b, y, rows, eps,          \
                        (const uint4*)delta))
#define FVS_LN_CASE(C)                                             \
  case C:                                                          \
    if (bf) {                                                      \
      if (x_f32 && y_f32) FVS_LN_LAUNCH(C, true, true, true);      \
      else if (x_f32) FVS_LN_LAUNCH(C, true, true, false);         \
      else if (y_f32) FVS_LN_LAUNCH(C, true, false, true);         \
      else FVS_LN_LAUNCH(C, true, false, false);                   \
    } else {                                                       \
      if (x_f32 && y_f32) FVS_LN_LAUNCH(C, false, true, true);     \
      else if (x_f32) FVS_LN_LAUNCH(C, false, true, false);        \
      else if (y_f32) FVS_LN_LAUNCH(C, false, false, true);        \
      else FVS_LN_LAUNCH(C, false, false, false);                  \
    }                                                              \
    break;
  switch (chunks) {
    FVS_LN_CASE(1) FVS_LN_CASE(2) FVS_LN_CASE(3) FVS_LN_CASE(4) FVS_LN_CASE(5) FVS_LN_CASE(6) FVS_LN_CASE(7) FVS_LN_CASE(8)
  }
#undef FVS_LN_CASE
#undef FVS_LN_LAUNCH
  FVS_CHECK_LAUNCH("layernorm_kernel");
  return FVS_OK;
}

int im2col_launch(const void* pixels, void* patches, int B, int S, int P, int Kpad, cudaStream_t stream) {
  const int G = S / P;
  im2col_kernel<<<dim3(G * G + 1, B), 128, 0, stream>>>((const uint16_t*)pixels, (uint16_t*)patches, B, S, P, G, Kpad);
  FVS_CHECK_LAUNCH("im2col_kernel");
  return FVS_OK;
}

int drop_cls_launch(const void* x, const void* delta, void* out, int B, int tokens, int D, int dtype, cudaStream_t stream,
                    bool keep_cls) {
  const int vec_per_row = D / 8;
  const int first = keep_cls ? 0 : 1;
  const size_t total = size_t(B) * (tokens - first) * vec_per_row;
  int blocks = int((total + 255) / 256);
  if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  if (dtype == FVS_BF16)
    drop_cls_kernel<true><<<blocks, 256, 0, stream>>>((const float*)x, (const uint4*)delta, (uint4*)out, tokens, first, vec_per_row, total);
  else
    drop_cls_kernel<false><<<blocks, 256, 0, stream>>>((const float*)x, (const uint4*)delta, (uint4*)out, tokens, first, vec_per_row, total);
  FVS_CHECK_LAUNCH("drop_cls_kernel");
  return FVS_OK;
}

}  // namespace fvs

extern "C" int fvs_layernorm(const void* x, const void* gamma, const void* beta, void* y, int rows, int dim, float eps,
                             int dtype, int x_dtype, int y_dtype, fvs_stream_t stream) {
  using namespace fvs;
  FVS_REQUIRE(x && gamma && beta && y, "fvs_layernorm: null pointer");
  FVS_REQUIRE(rows > 0, "fvs_layernorm: rows must be > 0");
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "fvs_layernorm: dtype must be f16 or bf16");
  FVS_REQUIRE((x_dtype == dtype || x_dtype == FVS_F32) && (y_dtype == dtype || y_dtype == FVS_F32),
              "fvs_layernorm: x/y dtype must be the parameter dtype or f32");
  return layernorm_launch(x, gamma, beta, y, rows, dim, eps, dtype, x_dtype == FVS_F32, y_dtype == FVS_F32, nullptr,
                          static_cast<cudaStream_t>(stream), /*pdl=*/true);
}

extern "C" int fvs_add_layernorm(void* x, const void* delta, const void* gamma, const void* beta, void* y, int rows,
                                 int dim, float eps, int dtype, fvs_stream_t stream) {
  using namespace fvs;
  FVS_REQUIRE(x && delta && gamma && beta && y, "fvs_add_layernorm: null pointer");
  FVS_REQUIRE(rows > 0, "fvs_add_layernorm: rows must be > 0");
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "fvs_add_layernorm: dtype must be f16 or bf16");
  return layernorm_launch(x, gamma, beta, y, rows, dim, eps, dtype, true, false, delta, static_cast<cudaStream_t>(stream),
                          /*pdl=*/true);
}
