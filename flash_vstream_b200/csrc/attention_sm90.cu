// attention_sm90.cu — fvs_attention / fvs_attention80: per-frame multi-head self-attention on Hopper tensor cores (wgmma),
// head_dim 64, or head_dim 80 = 64 "main" + 16 "extra" dims (kX variant, the Qwen2-VL vision tower): the extra dims travel
// as 16-column SWIZZLE_32B tiles next to the 64-column SWIZZLE_128B ones, cost one more K = 16 MMA per S tile and one
// N = 16 MMA per P V step, and live in their own column block of the activation ([main | extra] layout, see
// include/fvs_b200.h).
//
// Persistent: one CTA per SM (min(SMs, tiles) CTAs) walks the (128-query block, head, frame) tiles with a grid stride, the
// query block varying fastest so that the CTAs in flight at one time read the same frame's K / V from L2.
//   warpgroup 2    : producer (24 registers).  One thread issues the TMA loads: each tile's Q into one of two buffers,
//                    then 64-row (K, V) tile pairs through a 6-stage ring (SWIZZLE_128B boxes cut from the packed
//                    [frames, tokens, 3*H*64] QKV activation by 3-D tensor maps; rows past `tokens` are zero-filled by
//                    the TMA, so frames never bleed into each other).  It runs ahead into the next tile while the
//                    consumers finish the current one.
//   warpgroups 0, 1 : consumers (240 registers), 64 query rows each.  S = Q K^T (m64n64k16 wgmma, both operands from the
//                    swizzled stages) into registers, online softmax in registers (4 threads per row pair, quad shuffles),
//                    P rounded to 16 bits and fed back as the register A operand of O += P V (V MN-major straight from
//                    its TMA tile).  Row sums add up the rounded P, so O / L is the softmax of exactly the P that was
//                    multiplied.
// Schedule: inside a warpgroup, S_{j+1} = Q K_{j+1}^T and O += P_j V_j are issued together, and the softmax of S_{j+1}
// runs while P_j V_j is still on the tensor cores; O is rescaled by factor_{j+1} once P_j V_j has landed, so every
// element still computes o = o * f_j + P_j V_j in the same order.  Between the two warpgroups, two named barriers hand
// the tensor cores back and forth (ping-pong): one warpgroup's softmax runs while the other's MMAs run.
// A last KV tile with 1..16 valid keys (ViT-L/14-336: 577 = 9 * 64 + 1; the Qwen2-VL 144-token grid: 16) takes S as
// m64n16, 8 exponentials per thread instead of 32 and a single K = 16 step of P V: the columns it leaves out would be -inf
// in S, 0 in P and meet zero-filled V rows, so the result is bit for bit the full-width one.  The O rescale is skipped
// when every row of a warp has factor 1 (o * 1 == o).
// Replaces HF CLIPAttention reached from multimodal_encoder/clip_encoder.py:50 (SURVEY.md §2.2 K2).
#include "fvs_common.h"
#include "fvs_kernels.h"
#include "fvs_ptx.cuh"

namespace fvs {
namespace attn {

constexpr int HD = 64;          // head dim
constexpr int BQ = 128;         // query rows per tile
constexpr int WQ = 64;          // query rows per consumer warpgroup
constexpr int BKV = 64;         // kv rows per tile
constexpr int kNarrow = 16;     // a last KV tile with at most this many valid keys runs at N = 16
constexpr int kStages = 6;
constexpr int kThreads = 384;   // 2 consumer warpgroups + 1 producer warpgroup
constexpr int kProducerRegs = 24, kConsumerRegs = 240;   // 128 x 24 + 256 x 240 <= 64 K registers
constexpr int Q_BYTES = BQ * HD * 2;      // 16 KB
constexpr int KV_BYTES = BKV * HD * 2;    // 8 KB: [64 rows][64 x 16-bit], 128 B per row
constexpr int XD = 16;                    // extra head dims of the head_dim-80 variant
constexpr int QX_BYTES = BQ * XD * 2;     // 4 KB: [128 rows][16 x 16-bit], 32 B per row (SWIZZLE_32B)
constexpr int KVX_BYTES = BKV * XD * 2;   // 2 KB
// named barriers (0 is __syncthreads): consumer c waits on kSchedBar + c for its turn on the tensor cores; kEpiBar + c
// orders consumer c's output staging against its TMA store
constexpr uint32_t kSchedBar = 1, kEpiBar = 3;
template <bool kX> struct Lay {
  static constexpr int Q_TOTAL = Q_BYTES + (kX ? QX_BYTES : 0);  // one Q buffer [main | extra]: 16 KB | 20 KB
  static constexpr int TILE = KV_BYTES + (kX ? KVX_BYTES : 0);     // one K or V tile: 8 KB | 10 KB, multiples of 1024
  static constexpr int STAGE = 2 * TILE;                           // [K | V]
  static constexpr int OUT = 2 * Q_TOTAL;                          // output staging, laid out like a Q buffer
  static constexpr int KV = 3 * Q_TOTAL;
  static constexpr int TILES = KV + kStages * STAGE;               // 144 KB | 180 KB
  static constexpr int BYTES = TILES + 256 + 1024;
};

template <bool kBF16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if (kBF16) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  } else {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
}
template <bool kBF16>
__device__ __forceinline__ float2 unpack2(uint32_t v) {
  if (kBF16) return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xFFFF0000u));
  const __half2 h = *reinterpret_cast<const __half2*>(&v);
  return __half22float2(h);
}

// S = Q K^T of one KV tile: 64 columns, or (kN, narrow) the first 16; s[4j + 2h + c] is column 8j + cq + c either way
template <bool kN> using STile = float[kN ? kNarrow / 2 : BKV / 2];
template <bool kBF16, bool kX, bool kN>
__device__ __forceinline__ void issue_s(STile<kN>& s, uint32_t q_addr, uint32_t qx_addr, uint32_t k_addr) {
  constexpr int N = kN ? kNarrow : BKV;
#pragma unroll
  for (int k = 0; k < HD / 16; ++k)
    Wgmma<N, kBF16, 0>::ss(s, wgmma_desc(q_addr + 32 * k, 1024, kSw128), wgmma_desc(k_addr + 32 * k, 1024, kSw128),
                           k != 0 ? 1u : 0u);
  if constexpr (kX)   // dims 64..79: one more K = 16 step from the SWIZZLE_32B tiles
    Wgmma<N, kBF16, 0>::ss(s, wgmma_desc(qx_addr, 256, kSw32), wgmma_desc(k_addr + KV_BYTES, 256, kSw32), 1u);
  wgmma_commit();
}

// O += P V: B = V[16k..16k+16, 0..64) MN-major, 16 kv rows = 2048 B per K step; narrow: the first K step only
template <bool kBF16, bool kX, bool kN>
__device__ __forceinline__ void issue_pv(float (&o)[HD / 2], float (&ox)[kX ? XD / 2 : 1], const uint32_t (&p)[BKV / 16][4],
                                         uint32_t v_addr) {
#pragma unroll
  for (int k = 0; k < (kN ? 1 : BKV / 16); ++k) {
    Wgmma<HD, kBF16, 1>::rs(o, p[k], wgmma_desc(v_addr + 2048 * k, 1024, kSw128), 1u);
    if constexpr (kX)   // O[:, 64..80) += P V_extra: SWIZZLE_32B, 16 kv rows = 512 B per K step
      Wgmma<XD, kBF16, 1>::rs(ox, p[k], wgmma_desc(v_addr + KV_BYTES + 512 * k, 256, kSw32), 1u);
  }
  wgmma_commit();
}

// Online softmax over one S tile (64 keys, or kN: the first 16).  Columns past the sequence end (zero-filled keys) are
// forced to -inf.  Updates the running max and sum, returns the O rescale factor per row half and leaves
// exp2((S - m) * scale*log2e) in s; the row sum adds those values rounded to 16 bits, exactly as pack_p hands them to P V.
template <bool kBF16, bool kN>
__device__ __forceinline__ void softmax_tile(STile<kN>& s, int valid, int cq, float scale_log2e, float (&m_run)[2],
                                             float (&l_run)[2], float (&factor)[2]) {
  constexpr int NJ = (kN ? kNarrow : BKV) / 8;
  if (valid < BKV) {
#pragma unroll
    for (int i = 0; i < 4 * NJ; ++i)
      if ((i >> 2) * 8 + cq + (i & 1) >= valid) s[i] = -INFINITY;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float tmax = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < NJ; ++jj) tmax = fmaxf(tmax, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
    tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
    tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
    const float m_new = fmaxf(m_run[h], tmax);
    factor[h] = ex2_approx((m_run[h] - m_new) * scale_log2e);   // 0 on the first tile (m_run = -inf)
    m_run[h] = m_new;
  }
  float lsum[2] = {0.f, 0.f};
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float nm = -m_run[h] * scale_log2e;
      s[4 * jj + 2 * h] = ex2_approx(fmaf(s[4 * jj + 2 * h], scale_log2e, nm));
      s[4 * jj + 2 * h + 1] = ex2_approx(fmaf(s[4 * jj + 2 * h + 1], scale_log2e, nm));
      const float2 f = unpack2<kBF16>(pack2<kBF16>(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
      lsum[h] += f.x + f.y;
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    lsum[h] += __shfl_xor_sync(0xffffffffu, lsum[h], 1);
    lsum[h] += __shfl_xor_sync(0xffffffffu, lsum[h], 2);
    l_run[h] = l_run[h] * factor[h] + lsum[h];
  }
}

// P rounded to 16 bits: fragment kk holds the A operand of K step kk of P V.  Written only once the previous P V has
// completed: registers that an in-flight wgmma reads are not rewritten, so ptxas keeps the MMAs asynchronous.
template <bool kBF16, bool kN>
__device__ __forceinline__ void pack_p(const STile<kN>& s, uint32_t (&p)[BKV / 16][4]) {
#pragma unroll
  for (int jj = 0; jj < (kN ? kNarrow : BKV) / 8; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h) p[jj >> 1][(jj & 1) * 2 + h] = pack2<kBF16>(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]);
}

template <bool B> struct Bool { static constexpr bool value = B; };

struct TileCoord {
  int q0, head, frame;
};
__device__ __forceinline__ TileCoord tile_coord(int tile, int nq, int heads) {
  const int rest = tile / nq;
  return {(tile - rest * nq) * BQ, rest % heads, rest / heads};
}

template <bool kBF16, bool kX>
__global__ void __launch_bounds__(kThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv,
                 const __grid_constant__ CUtensorMap tmap_ctx, const __grid_constant__ CUtensorMap tmap_qx,
                 const __grid_constant__ CUtensorMap tmap_kvx, const __grid_constant__ CUtensorMap tmap_ctxx, int tokens,
                 int heads, int tiles, float scale_log2e) {
  using L_ = Lay<kX>;
  // SWIZZLE_128B tiles need 1024-byte alignment.  The alignment is declared (not rounded up by hand through an integer
  // cast): the pointer keeps its shared address space, so the compiler emits 32-bit STS/LDS instead of generic ST/LD.
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* smem_out = smem + L_::OUT;          // [128][128 B] output staging, then [128][32 B] of the extra dims (kX)
  uint8_t* smem_kv = smem + L_::KV;            // [kStages][K main | K extra | V main | V extra]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L_::TILES);
  uint64_t* q_full = bars;                     // [2]
  uint64_t* q_empty = bars + 2;                // [2] one arrival per consumer warpgroup
  uint64_t* kv_full = bars + 4;                // [kStages]
  uint64_t* kv_empty = bars + 4 + kStages;     // [kStages] one arrival per consumer warpgroup

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // broadcast from lane 0 so that ptxas sees a warp-uniform value: wgmmas issued under a branch on it are not serialized
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
  const int nq = (tokens + BQ - 1) / BQ;
  const int nkv = (tokens + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_kv);
    tma_prefetch_desc(&tmap_ctx);
    for (int b = 0; b < 2; ++b) {
      mbar_init(&q_full[b], 1);
      mbar_init(&q_empty[b], 2);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  pdl_trigger();  // PDL: the setup above overlapped the QKV GEMM's tail; its output is read from here on
  pdl_wait();

  if (wg == 2) {
    // ------------------------------------------------------------------ TMA producer
    reg_dealloc<kProducerRegs>();
    if (warp == 8 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      int it = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
        const TileCoord tc = tile_coord(tile, nq, heads);
        const int k_col = heads * HD + tc.head * HD, v_col = 2 * heads * HD + tc.head * HD;
        // extra-dim column blocks follow the three main blocks: [q main | k main | v main | q extra | k extra | v extra]
        const int xq_col = 3 * heads * HD + tc.head * XD;
        const int xk_col = xq_col + heads * XD, xv_col = xk_col + heads * XD;
        const int qb = it & 1;
        uint8_t* sq = smem + qb * L_::Q_TOTAL;
        mbar_wait(&q_empty[qb], ((it >> 1) & 1) ^ 1);
        mbar_arrive_expect_tx(&q_full[qb], L_::Q_TOTAL);
        tma_load_3d(sq, &tmap_q, &q_full[qb], tc.head * HD, tc.q0, tc.frame);
        if (kX) tma_load_3d(sq + Q_BYTES, &tmap_qx, &q_full[qb], xq_col, tc.q0, tc.frame);
        for (int j = 0; j < nkv; ++j) {
          mbar_wait(&kv_empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&kv_full[stage], L_::STAGE);
          uint8_t* st = smem_kv + stage * L_::STAGE;
          tma_load_3d(st, &tmap_kv, &kv_full[stage], k_col, j * BKV, tc.frame);
          tma_load_3d(st + L_::TILE, &tmap_kv, &kv_full[stage], v_col, j * BKV, tc.frame);
          if (kX) {
            tma_load_3d(st + KV_BYTES, &tmap_kvx, &kv_full[stage], xk_col, j * BKV, tc.frame);
            tma_load_3d(st + L_::TILE + KV_BYTES, &tmap_kvx, &kv_full[stage], xv_col, j * BKV, tc.frame);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: 64 query rows per warpgroup
  reg_alloc<kConsumerRegs>();
  const int t = threadIdx.x & 127;
  const int r_a = 16 * (warp & 3) + (lane >> 2);   // rows of this thread inside the warpgroup's 64: r_a, r_a + 8
  const int cq = 2 * (lane & 3);                   // column pair inside each 8-column block
  const uint32_t kv_addr = smem_u32(smem_kv);
  uint8_t* stg = smem_out + wg * WQ * 128;
  uint8_t* stgx = smem_out + Q_BYTES + wg * WQ * 32;
  // the tensor cores go to consumer 0 first; afterwards each consumer hands them over when its MMAs are issued
  if (wg == 1) named_bar_arrive(kSchedBar + 0, 256);

  int stage = 0;
  uint32_t phase = 0;
  int it = 0;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
    const TileCoord tc = tile_coord(tile, nq, heads);
    const int qb = it & 1;
    const uint32_t q_addr = smem_u32(smem) + qb * L_::Q_TOTAL + wg * WQ * 128;
    const uint32_t qx_addr = smem_u32(smem) + qb * L_::Q_TOTAL + Q_BYTES + wg * WQ * 32;
    const bool narrow_last = tokens - (nkv - 1) * BKV <= kNarrow;

    float o[HD / 2];            // O[64 x 64] accumulators
    float ox[kX ? XD / 2 : 1];  // O[64 x 16] extra dims
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (kX ? XD / 2 : 1); ++i) ox[i] = 0.f;
    uint32_t p[BKV / 16][4];

    // One KV step: take the tensor cores, issue S_j = Q K_j^T and (after the first tile) O += P_{j-1} V_{j-1} from stage
    // `prev`, hand the tensor cores over, run the softmax of S_j while P_{j-1} V_{j-1} is still in flight, then rescale O
    // by factor_j and release stage `prev`.  kFirst: O is still 0 and needs no rescale.
    auto step = [&](auto first_c, auto narrow_c, int j, int prev) {
      constexpr bool kFirst = decltype(first_c)::value, kN = decltype(narrow_c)::value;
      STile<kN> s;
      float factor[2];
      mbar_wait(&kv_full[stage], phase);
      named_bar_sync(kSchedBar + wg, 256);
      wgmma_fence();
      issue_s<kBF16, kX, kN>(s, q_addr, qx_addr, kv_addr + stage * L_::STAGE);
      if constexpr (!kFirst) issue_pv<kBF16, kX, false>(o, ox, p, kv_addr + prev * L_::STAGE + L_::TILE);
      named_bar_arrive(kSchedBar + (wg ^ 1), 256);
      wgmma_wait<kFirst ? 0 : 1>();
      wgmma_pin(s);
      softmax_tile<kBF16, kN>(s, tokens - j * BKV, cq, scale_log2e, m_run, l_run, factor);
      if constexpr (!kFirst) {
        // The wait for P V sits inside the branch on purpose.  Within one basic block ptxas hoists WARPGROUP.DEPBAR above
        // independent ALU work, which put every exponential of this step after the wait; the block boundary keeps the
        // softmax between the two waits (tests/test_attention_sass.py checks the SASS).
        if (__any_sync(0xffffffffu, factor[0] != 1.f || factor[1] != 1.f)) {
          wgmma_wait<0>();
          wgmma_pin(o);
          if constexpr (kX) wgmma_pin(ox);
#pragma unroll
          for (int i = 0; i < HD / 2; ++i) o[i] *= factor[(i >> 1) & 1];
          if constexpr (kX) {
#pragma unroll
            for (int i = 0; i < XD / 2; ++i) ox[i] *= factor[(i >> 1) & 1];
          }
        } else {
          wgmma_wait<0>();
          wgmma_pin(o);
          if constexpr (kX) wgmma_pin(ox);
        }
        if (t == 0) mbar_arrive(&kv_empty[prev]);
      }
      pack_p<kBF16, kN>(s, p);
    };

    mbar_wait(&q_full[qb], (it >> 1) & 1);
    if (nkv == 1 && narrow_last) step(Bool<true>{}, Bool<true>{}, 0, 0);
    else step(Bool<true>{}, Bool<false>{}, 0, 0);
    for (int j = 1; j < nkv; ++j) {
      const int prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
      if (j == nkv - 1 && narrow_last) step(Bool<false>{}, Bool<true>{}, j, prev);
      else step(Bool<false>{}, Bool<false>{}, j, prev);
    }

    // ---- O += P_last V_last
    wgmma_fence();
    if (narrow_last) issue_pv<kBF16, kX, true>(o, ox, p, kv_addr + stage * L_::STAGE + L_::TILE);
    else issue_pv<kBF16, kX, false>(o, ox, p, kv_addr + stage * L_::STAGE + L_::TILE);
    wgmma_wait<0>();
    wgmma_pin(o);
    if constexpr (kX) wgmma_pin(ox);
    if (t == 0) {
      mbar_arrive(&kv_empty[stage]);
      mbar_arrive(&q_empty[qb]);
    }
    if (++stage == kStages) { stage = 0; phase ^= 1; }

    // ---- epilogue: O / L -> 16-bit -> swizzled staging -> TMA store (once the previous tile's store has read it)
    const float inv[2] = {1.0f / l_run[0], 1.0f / l_run[1]};
    if (t == 0) tma_store_wait_read<0>();
    named_bar_sync(kEpiBar + wg, 128);
#pragma unroll
    for (int jj = 0; jj < HD / 8; ++jj) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_a + 8 * h;
        *reinterpret_cast<uint32_t*>(stg + r * 128 + ((jj ^ (r & 7)) << 4) + cq * 2) =
            pack2<kBF16>(o[4 * jj + 2 * h] * inv[h], o[4 * jj + 2 * h + 1] * inv[h]);
      }
    }
    if constexpr (kX) {   // the 16 extra dims: SWIZZLE_32B staging
#pragma unroll
      for (int jj = 0; jj < XD / 8; ++jj) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r_a + 8 * h;
          *reinterpret_cast<uint32_t*>(stgx + r * 32 + ((jj ^ ((r >> 2) & 1)) << 4) + cq * 2) =
              pack2<kBF16>(ox[4 * jj + 2 * h] * inv[h], ox[4 * jj + 2 * h + 1] * inv[h]);
        }
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(kEpiBar + wg, 128);
    if (t == 0) {
      tma_store_3d(&tmap_ctx, stg, tc.head * HD, tc.q0 + wg * WQ, tc.frame);  // rows >= tokens are clipped by the map
      if (kX) tma_store_3d(&tmap_ctxx, stgx, heads * HD + tc.head * XD, tc.q0 + wg * WQ, tc.frame);
      tma_store_commit();
    }
  }
  if (wg == 0) named_bar_sync(kSchedBar + 0, 256);   // consumer 1's last hand-over: every arrival meets a wait
  if (t == 0) tma_store_wait_all<0>();
}

}  // namespace attn

template <bool kBF16, bool kX>
static int attention_launch_t(const AttnMaps& m, int tokens, int heads, int tiles, float scale_log2e, cudaStream_t stream,
                              bool pdl) {
  using namespace attn;
  static bool done = false;
  if (!done) {
    FVS_CUDA_OK(cudaFuncSetAttribute(attention_kernel<kBF16, kX>, cudaFuncAttributeMaxDynamicSharedMemorySize, Lay<kX>::BYTES));
    done = true;
  }
  const int grid = tiles < device_sm_count() ? tiles : device_sm_count();
  FVS_CUDA_OK(launch_ex(attention_kernel<kBF16, kX>, dim3(grid), dim3(kThreads), Lay<kX>::BYTES, stream, 1, pdl, m.q,
                        m.kv, m.ctx, m.qx, m.kvx, m.ctxx, tokens, heads, tiles, scale_log2e));
  return FVS_OK;
}

int attention_launch(const AttnMaps& m, int frames, int tokens, int heads, float scale, int dtype, cudaStream_t stream,
                     int head_dim, bool pdl) {
  using namespace attn;
  const float scale_log2e = scale * 1.4426950408889634f;
  const long long tiles_ll = (long long)((tokens + BQ - 1) / BQ) * heads * frames;
  FVS_REQUIRE(tiles_ll <= 0x7fffffffLL, "attention: %lld tiles exceed the int range", tiles_ll);
  const int tiles = int(tiles_ll);
  const bool bf = dtype == FVS_BF16, x80 = head_dim == 80;
  const int prof = prof_begin(FVS_PROF_ATTENTION, 4.0 * frames * double(heads) * tokens * double(tokens) * head_dim, stream);
  const int r = x80 ? (bf ? attention_launch_t<true, true>(m, tokens, heads, tiles, scale_log2e, stream, pdl)
                          : attention_launch_t<false, true>(m, tokens, heads, tiles, scale_log2e, stream, pdl))
                    : (bf ? attention_launch_t<true, false>(m, tokens, heads, tiles, scale_log2e, stream, pdl)
                          : attention_launch_t<false, false>(m, tokens, heads, tiles, scale_log2e, stream, pdl));
  if (r) return r;
  prof_end(prof, stream);
  FVS_CHECK_LAUNCH("attention_kernel");
  return FVS_OK;
}

// head_dim 64: qkv [frames*tokens, 3*H*64], ctx [.., H*64].  head_dim 80: qkv [.., 3*H*80] laid out as
// [q main H*64 | k main | v main | q extra H*16 | k extra | v extra], ctx [.., H*80] as [main H*64 | extra H*16].
// The ctx boxes hold one consumer warpgroup's 64 rows.
int attention_make_maps(AttnMaps* m, const void* qkv, void* ctx, int frames, int tokens, int heads, int head_dim) {
  using namespace attn;
  const uint64_t wq = uint64_t(3) * heads * head_dim, wc = uint64_t(heads) * head_dim;
  int r;
  if ((r = make_tmap_3d(&m->q, qkv, frames, tokens, wq, wq, uint64_t(tokens) * wq, BQ, HD, 1))) return r;
  if ((r = make_tmap_3d(&m->kv, qkv, frames, tokens, wq, wq, uint64_t(tokens) * wq, BKV, HD, 1))) return r;
  if ((r = make_tmap_3d(&m->ctx, ctx, frames, tokens, wc, wc, uint64_t(tokens) * wc, WQ, HD, 1))) return r;
  if (head_dim == 80) {
    if ((r = make_tmap_3d(&m->qx, qkv, frames, tokens, wq, wq, uint64_t(tokens) * wq, BQ, XD, 2))) return r;
    if ((r = make_tmap_3d(&m->kvx, qkv, frames, tokens, wq, wq, uint64_t(tokens) * wq, BKV, XD, 2))) return r;
    if ((r = make_tmap_3d(&m->ctxx, ctx, frames, tokens, wc, wc, uint64_t(tokens) * wc, WQ, XD, 2))) return r;
  } else {
    m->qx = m->q; m->kvx = m->kv; m->ctxx = m->ctx;
  }
  return FVS_OK;
}

}  // namespace fvs

static int attention_entry(const void* qkv, void* ctx, int frames, int tokens, int heads, float scale, int dtype,
                           fvs_stream_t stream, int head_dim, const char* who) {
  using namespace fvs;
  FVS_REQUIRE(qkv && ctx, "%s: null pointer", who);
  FVS_REQUIRE(frames > 0 && tokens > 0 && heads > 0, "%s: bad shape", who);
  FVS_REQUIRE(frames <= 65535 && heads <= 65535, "%s: grid too large", who);
  FVS_REQUIRE(dtype == FVS_F16 || dtype == FVS_BF16, "%s: dtype must be f16 or bf16", who);
  FVS_REQUIRE(scale > 0.f, "%s: scale must be positive", who);
  AttnMaps m;
  int r = attention_make_maps(&m, qkv, ctx, frames, tokens, heads, head_dim);
  if (r) return r;
  return attention_launch(m, frames, tokens, heads, scale, dtype, static_cast<cudaStream_t>(stream), head_dim);
}

extern "C" int fvs_attention(const void* qkv, void* ctx, int frames, int tokens, int heads, float scale, int dtype,
                             fvs_stream_t stream) {
  return attention_entry(qkv, ctx, frames, tokens, heads, scale, dtype, stream, 64, "fvs_attention");
}

extern "C" int fvs_attention80(const void* qkv, void* ctx, int frames, int tokens, int heads, float scale, int dtype,
                               fvs_stream_t stream) {
  return attention_entry(qkv, ctx, frames, tokens, heads, scale, dtype, stream, 80, "fvs_attention80");
}
