// gemm_sm90.cu — fvs_linear: out = epilogue(A @ W^T) on Hopper tensor cores (wgmma, sm_90a).
//
// Persistent, warp-specialised kernel, one CTA per SM, 128 x kBN output tiles (kBN = 256, or 128 for grids that would
// leave SMs idle), 64-wide K blocks through a TMA / mbarrier ring.  Roles (384 threads = 3 warpgroups):
//   warpgroup 0 : TMA producer (one elected thread of warp 0; SWIZZLE_128B boxes of A and W, "full" / "empty" barriers)
//   warpgroups 1, 2 : consumers, 64 rows of the tile each: m64n{kBN}k16 wgmma straight from the swizzled stages into
//                 register accumulators, then the epilogue (bias / quick_gelu / gelu / residual / row table -> 16-bit ->
//                 swizzled smem -> TMA store; the fp32-residual form hands acc + bias to the L2 as a TMA reduce-add, so the
//                 residual stream is updated in place without entering the SM).  The producer runs ahead into the next
//                 tile while the consumers drain the current one.
// A [M,K] and W [N,K] are both K-major, so no transposes are needed for nn.Linear weights.
// Replaces the cuBLAS GEMMs behind HF CLIPEncoderLayer that the reference reaches from
// multimodal_encoder/clip_encoder.py:50 (SURVEY.md §2.2 K1/K2).
#include <cstdlib>

#include "fvs_common.h"
#include "fvs_ptx.cuh"

namespace fvs {
namespace gemm {

constexpr int BM = 128;  // tile rows (two consumer warpgroups of 64)
constexpr int BK = 64;   // 64 x 16-bit = 128 B = one swizzle row
constexpr int kEpiChunk = 64;     // columns per TMA-store box for 16-bit outputs (128 B)
constexpr int kEpiChunkF32 = 32;  // columns per TMA-store box for fp32 outputs (128 B)
constexpr int kThreads = 384;
constexpr int kWgRows = 64;
constexpr int A_TILE_BYTES = BM * BK * 2;              // 16 KB
constexpr int OUT_BUF_BYTES = kWgRows * 128;           // 8 KB: 64 rows x 128 B
constexpr int SMEM_BARRIERS = 256;

template <int kBN>
struct Cfg {
  static constexpr int kStages = kBN == 256 ? 4 : 6;
  static constexpr int B_TILE_BYTES = kBN * BK * 2;      // 32 KB / 16 KB
  static constexpr int STAGE_BYTES = A_TILE_BYTES + B_TILE_BYTES;
  static constexpr int SMEM_TILES = kStages * STAGE_BYTES + 2 * 2 * OUT_BUF_BYTES;   // + [consumer][2] store buffers
  static constexpr int SMEM_BYTES = SMEM_TILES + SMEM_BARRIERS + 1024;  // + manual 1024-alignment slack
};

template <bool kBF16>
struct Cvt;
template <>
struct Cvt<false> {
  static __device__ __forceinline__ float lo(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v & 0xFFFF))); }
  static __device__ __forceinline__ float hi(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v >> 16))); }
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};
template <>
struct Cvt<true> {
  static __device__ __forceinline__ float lo(uint32_t v) { return __uint_as_float(v << 16); }
  static __device__ __forceinline__ float hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};

template <int kEpi, bool kBF16, int kBN>
__global__ void __launch_bounds__(kThreads, 1)
linear_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
              const __grid_constant__ CUtensorMap tmap_out, const uint16_t* __restrict__ bias,
              const uint16_t* aux, int M, int N, int K, int ld_aux, int aux_period) {
  using C = Cfg<kBN>;
  constexpr int kStages = C::kStages;
  constexpr int BN = kBN;
  // SWIZZLE_128B operands need 1024-byte aligned tiles.  The alignment is declared (not rounded up by hand through an
  // integer cast) so the pointer keeps its shared address space: STS/LDS with 32-bit addresses instead of generic ST/LD.
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* smem_a = smem;                                  // [kStages][16 KB]
  uint8_t* smem_b = smem + kStages * A_TILE_BYTES;         // [kStages][B_TILE_BYTES]
  uint8_t* smem_out = smem + kStages * C::STAGE_BYTES;     // [consumer][2][8 KB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::SMEM_TILES);
  uint64_t* full_bar = bars;                 // [kStages]
  uint64_t* empty_bar = bars + kStages;      // [kStages] one arrival per consumer warpgroup

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  const int num_m = (M + BM - 1) / BM;
  const int num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (K + BK - 1) / BK;   // a K tail is zero-filled by the TMA (both operands), so it adds nothing

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  // PDL: the setup above overlapped the previous kernel's tail; from here on we touch global memory it may have produced.
  pdl_trigger();
  pdl_wait();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    reg_dealloc<40>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / num_n, n_blk = tile % num_n;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          tma_load_2d(smem_a + stage * A_TILE_BYTES, &tmap_a, &full_bar[stage], kb * BK, m_blk * BM);
          tma_load_2d(smem_b + stage * C::B_TILE_BYTES, &tmap_b, &full_bar[stage], kb * BK, n_blk * BN);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: 64 rows each
  reg_alloc<232>();
  const int cw = wg - 1;                       // consumer index
  const int t = threadIdx.x & 127;
  const int w = t >> 5;
  const int r_a = 16 * w + (lane >> 2);        // rows of this thread inside the 64-row slice: r_a, r_a + 8
  const int cq = 2 * (lane & 3);               // column pair inside each 8-column block
  const bool epi_leader = t == 0;
  uint8_t* const obuf0 = smem_out + cw * 2 * OUT_BUF_BYTES;
  const uint32_t a_base = smem_u32(smem_a) + cw * kWgRows * 128;
  const uint32_t b_base = smem_u32(smem_b);
  int stage = 0;
  uint32_t phase = 0;
  int out_buf = 0;
  float acc[BN / 2];

  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m_blk = tile / num_n, n_blk = tile % num_n;
    const int row0 = m_blk * BM + cw * kWgRows;

    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)   // a K step of 16 is 32 bytes inside the 128 B swizzle row
        Wgmma<BN, kBF16, 0>::ss(acc, wgmma_desc(a_base + stage * A_TILE_BYTES + 32 * k, 1024, kSw128),
                                wgmma_desc(b_base + stage * C::B_TILE_BYTES + 32 * k, 1024, kSw128),
                                (kb | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();                           // the previous K block's MMAs have read their stage
      if (prev_stage >= 0 && t == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_pin(acc);
    if (t == 0) mbar_arrive(&empty_bar[prev_stage]);

    if constexpr (kEpi == FVS_EPI_BIAS_RESIDUAL_F32) {
      // out_f32 += acc + bias, 32-column (128 B) chunks handed to the L2 as TMA reduce-add stores: the residual never
      // enters the SM and every element gets exactly one fp32 add per launch, so the result does not depend on any ordering.
      const int n_left = N - n_blk * BN;
      const int nchunks = (n_left < BN ? n_left : BN) / kEpiChunkF32;
#pragma unroll
      for (int c = 0; c < BN / kEpiChunkF32; ++c) {
        if (c < nchunks) {
          const int col0 = n_blk * BN + c * kEpiChunkF32;
          uint8_t* obuf = obuf0 + out_buf * OUT_BUF_BYTES;
          if (epi_leader) tma_store_wait_read<1>();   // the store issued two chunks ago has read this buffer
          named_bar_sync(1 + cw, 128);
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {            // 4 x (8 columns); this thread holds columns 8jj + cq, +1
            const uint32_t bv = *reinterpret_cast<const uint32_t*>(bias + col0 + 8 * jj + cq);
            const float b0 = Cvt<kBF16>::lo(bv), b1 = Cvt<kBF16>::hi(bv);
            const int j = c * 4 + jj;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = r_a + 8 * h;
              const int unit = 2 * jj + (cq >> 2);
              *reinterpret_cast<float2*>(obuf + r * 128 + ((unit ^ (r & 7)) << 4) + (cq & 3) * 4) =
                  make_float2(acc[4 * j + 2 * h] + b0, acc[4 * j + 2 * h + 1] + b1);
            }
          }
          fence_proxy_async_smem();
          named_bar_sync(1 + cw, 128);
          if (epi_leader) {
            tma_reduce_add_2d(&tmap_out, obuf, col0, row0);  // rows >= M are clipped by the map
            tma_store_commit();
          }
          out_buf ^= 1;
        }
      }
    } else {
#pragma unroll
      for (int c = 0; c < BN / kEpiChunk; ++c) {
        const int col0 = n_blk * BN + c * kEpiChunk;
        const bool col_ok = col0 < N;  // N is a multiple of 64, so a chunk is all-in or all-out
        if (col_ok) {
          uint8_t* obuf = obuf0 + out_buf * OUT_BUF_BYTES;
          // the TMA store that last read this buffer (two chunks ago) must have finished reading smem
          if (epi_leader) tma_store_wait_read<1>();
          named_bar_sync(1 + cw, 128);
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {   // 8 x (8 columns = 16 bytes); this thread holds columns 8jj + cq, +1
            const int j = c * 8 + jj;
            const int col = col0 + 8 * jj + cq;
            float b0 = 0.f, b1 = 0.f;
            if (kEpi != FVS_EPI_ROWTABLE) {
              const uint32_t bv = *reinterpret_cast<const uint32_t*>(bias + col);
              b0 = Cvt<kBF16>::lo(bv);
              b1 = Cvt<kBF16>::hi(bv);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = r_a + 8 * h;
              float x0 = acc[4 * j + 2 * h] + b0, x1 = acc[4 * j + 2 * h + 1] + b1;
              if (kEpi == FVS_EPI_BIAS_QUICKGELU) {  // x * sigmoid(1.702 x) = 0.5 x (1 + tanh(0.851 x)): one MUFU op instead of two
                const float h0 = 0.5f * x0, h1 = 0.5f * x1;
                x0 = fmaf(h0, tanh_approx(0.851f * x0), h0);
                x1 = fmaf(h1, tanh_approx(0.851f * x1), h1);
              }
              if (kEpi == FVS_EPI_BIAS_GELU) {    // exact GELU
                x0 = 0.5f * x0 * (1.0f + erff(x0 * 0.70710678118654752f));
                x1 = 0.5f * x1 * (1.0f + erff(x1 * 0.70710678118654752f));
              }
              if (kEpi == FVS_EPI_BIAS_RESIDUAL || kEpi == FVS_EPI_ROWTABLE) {
                const int row = row0 + r;
                uint32_t rv = 0;
                if (row < M) {
                  const size_t arow = (kEpi == FVS_EPI_ROWTABLE) ? size_t(row % aux_period) : size_t(row);
                  rv = *reinterpret_cast<const uint32_t*>(aux + arow * size_t(ld_aux) + col);
                }
                x0 += Cvt<kBF16>::lo(rv);
                x1 += Cvt<kBF16>::hi(rv);
              }
              // SWIZZLE_128B: 16-byte chunk jj of row r lives at chunk (jj ^ (r & 7))
              *reinterpret_cast<uint32_t*>(obuf + r * 128 + ((jj ^ (r & 7)) << 4) + cq * 2) = Cvt<kBF16>::pack(x0, x1);
            }
          }
          fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the TMA (async proxy)
          named_bar_sync(1 + cw, 128);
          if (epi_leader) {
            tma_store_2d(&tmap_out, obuf, col0, row0);  // rows >= M are clipped by the map
            tma_store_commit();
          }
          out_buf ^= 1;
        }
      }
    }
  }
  if (epi_leader) tma_store_wait_read<0>();   // smem has been read; completion of the global writes is ordered by the grid end
}

template <int kEpi, bool kBF16, int kBN>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const void* bias,
                  const void* aux, int M, int N, int K, int ld_aux, int aux_period, cudaStream_t stream, bool pdl) {
  auto kern = linear_kernel<kEpi, kBF16, kBN>;
  constexpr int smem = Cfg<kBN>::SMEM_BYTES;
  static bool attr_done = false;  // per instantiation
  if (!attr_done) {
    FVS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_done = true;
  }
  const int num_tiles = ((M + BM - 1) / BM) * ((N + kBN - 1) / kBN);
  int grid = device_sm_count();
  if (grid > num_tiles) grid = num_tiles;
  const int prof = prof_begin(FVS_PROF_LINEAR, 2.0 * M * double(N) * K, stream);
  cudaError_t e = launch_ex(kern, dim3(grid), dim3(kThreads), smem, stream, 1, pdl, ta, tb, to,
                            reinterpret_cast<const uint16_t*>(bias), reinterpret_cast<const uint16_t*>(aux), M, N, K,
                            ld_aux, aux_period);
  prof_end(prof, stream);
  if (e != cudaSuccess) return set_error(FVS_ECUDA, "launch linear_kernel: %s", cudaGetErrorString(e));
  FVS_CHECK_LAUNCH("linear_kernel");
  return FVS_OK;
}

template <int kEpi, int kBN>
static int launch_dt(bool bf, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const void* bias,
                     const void* aux, int M, int N, int K, int ld_aux, int aux_period, cudaStream_t stream, bool pdl) {
  return bf ? launch<kEpi, true, kBN>(ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl)
            : launch<kEpi, false, kBN>(ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl);
}
template <int kEpi>
static int launch_epi(bool bf, int bn, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to,
                      const void* bias, const void* aux, int M, int N, int K, int ld_aux, int aux_period,
                      cudaStream_t stream, bool pdl) {
  return bn == 128 ? launch_dt<kEpi, 128>(bf, ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl)
                   : launch_dt<kEpi, 256>(bf, ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl);
}

}  // namespace gemm

// Output-tile width.  256 normally; 128 when the 256-wide tiling fills at most half of the SMs (small M: single
// frames, 1-2-patch Qwen clips) so that twice as many SMs share the K loop.  The per-element K accumulation order does not
// depend on the tile shape, so results are bitwise identical either way.  FVS_GEMM_BN=128|256 forces it (tests).
int linear_tile_n(int M, int N) {
  static int forced = -1;
  if (forced < 0) {
    const char* e = getenv("FVS_GEMM_BN");
    forced = e ? atoi(e) : 0;
    if (forced != 128 && forced != 256) forced = 0;
  }
  if (forced) return forced;
  const int tiles256 = ((M + gemm::BM - 1) / gemm::BM) * ((N + 255) / 256);
  return 2 * tiles256 <= device_sm_count() ? 128 : 256;
}

// Internal entry used by the ViT engine as well (tensor maps can be cached by the caller).
int linear_launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const void* bias,
                  const void* aux, int M, int N, int K, int ld_aux, int epilogue, int aux_period, int dtype,
                  cudaStream_t stream, bool pdl) {
  using namespace gemm;
  const bool bf = dtype == FVS_BF16;
  const int bn = linear_tile_n(M, N);
  switch (epilogue) {
    case FVS_EPI_BIAS: return launch_epi<FVS_EPI_BIAS>(bf, bn, ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl);
    case FVS_EPI_BIAS_QUICKGELU:
      return launch_epi<FVS_EPI_BIAS_QUICKGELU>(bf, bn, ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl);
    case FVS_EPI_BIAS_RESIDUAL:
      return launch_epi<FVS_EPI_BIAS_RESIDUAL>(bf, bn, ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl);
    case FVS_EPI_ROWTABLE: return launch_epi<FVS_EPI_ROWTABLE>(bf, bn, ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl);
    case FVS_EPI_BIAS_RESIDUAL_F32:
      return launch_epi<FVS_EPI_BIAS_RESIDUAL_F32>(bf, bn, ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl);
    case FVS_EPI_BIAS_GELU:
      return launch_epi<FVS_EPI_BIAS_GELU>(bf, bn, ta, tb, to, bias, aux, M, N, K, ld_aux, aux_period, stream, pdl);
  }
  return set_error(FVS_EINVAL, "fvs_linear: unknown epilogue %d", epilogue);
}

// The W box holds one tile's rows; the output box one consumer warpgroup's 64 rows (must match linear_launch: same policy).
int linear_make_maps(CUtensorMap* ta, CUtensorMap* tb, CUtensorMap* to, const void* A, const void* W, void* out,
                     int M, int N, int K, int lda, int ldo, bool out_f32) {
  using namespace gemm;
  int r;
  if ((r = make_tmap_2d(ta, A, M, K, lda, BM, BK, true))) return r;
  if ((r = make_tmap_2d(tb, W, N, K, K, linear_tile_n(M, N), BK, true))) return r;
  if (out_f32) {
    if ((r = make_tmap_2d(to, out, M, N, ldo, kWgRows, kEpiChunkF32, true, 4))) return r;
  } else {
    if ((r = make_tmap_2d(to, out, M, N, ldo, kWgRows, kEpiChunk, true))) return r;
  }
  return FVS_OK;
}

}  // namespace fvs

extern "C" int fvs_linear(const void* A, const void* W, const void* bias, const void* aux, void* out, int M, int N,
                          int K, int lda, int ldo, int epilogue, int aux_period, int dtype, fvs_stream_t stream) {
  using namespace fvs;
  FVS_REQUIRE(A && W && out, "fvs_linear: null pointer");
  FVS_REQUIRE(M > 0 && N > 0 && K > 0, "fvs_linear: bad shape M=%d N=%d K=%d", M, N, K);
  FVS_REQUIRE(K % 8 == 0 && N % 64 == 0, "fvs_linear: K (%d) must be a multiple of 8 and N (%d) a multiple of 64", K, N);
  FVS_REQUIRE(lda % 8 == 0 && ldo % 8 == 0 && lda >= K && ldo >= N, "fvs_linear: bad pitches lda=%d ldo=%d", lda, ldo);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "fvs_linear: dtype must be f16 or bf16");
  FVS_REQUIRE(epilogue == FVS_EPI_ROWTABLE || bias != nullptr, "fvs_linear: bias required");
  FVS_REQUIRE((epilogue != FVS_EPI_BIAS_RESIDUAL && epilogue != FVS_EPI_ROWTABLE && epilogue != FVS_EPI_BIAS_RESIDUAL_F32) ||
                  aux != nullptr,
              "fvs_linear: aux required for this epilogue");
  FVS_REQUIRE(epilogue != FVS_EPI_ROWTABLE || aux_period > 0, "fvs_linear: aux_period must be > 0");
  CUtensorMap ta, tb, to;
  int r = linear_make_maps(&ta, &tb, &to, A, W, out, M, N, K, lda, ldo, epilogue == FVS_EPI_BIAS_RESIDUAL_F32);
  if (r) return r;
  const int ld_aux = (epilogue == FVS_EPI_ROWTABLE) ? N : ldo;
  if (epilogue == FVS_EPI_BIAS_RESIDUAL_F32 && aux != out)   // the epilogue ADDS into `out`: seed it with the residual first
    FVS_CUDA_OK(cudaMemcpy2DAsync(out, size_t(ldo) * 4, aux, size_t(ldo) * 4, size_t(N) * 4, size_t(M), cudaMemcpyDeviceToDevice,
                                  static_cast<cudaStream_t>(stream)));
  return linear_launch(ta, tb, to, bias, aux, M, N, K, ld_aux, epilogue, aux_period, dtype,
                       static_cast<cudaStream_t>(stream), /*pdl=*/true);
}
