// fvs_kernels.h — launchers shared between translation units of libfvs_b200.so (internal, not part of the C ABI).
#pragma once
#include "fvs_common.h"

namespace fvs {

// The ViT launchers take `pdl`: launch with the programmatic-dependent-launch attribute (the kernels trigger their
// dependents on entry, so a dependent's CTAs take SMs as soon as any free up).

// gemm_sm90.cu
int linear_make_maps(CUtensorMap* ta, CUtensorMap* tb, CUtensorMap* to, const void* A, const void* W, void* out,
                     int M, int N, int K, int lda, int ldo, bool out_f32);
int linear_launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const void* bias,
                  const void* aux, int M, int N, int K, int ld_aux, int epilogue, int aux_period, int dtype,
                  cudaStream_t stream, bool pdl = true);

// attention_sm90.cu
struct AttnMaps {
  CUtensorMap q, kv, ctx;
  CUtensorMap qx, kvx, ctxx;   // head_dim-80 variant only (otherwise copies of the main maps, never dereferenced)
};
int attention_make_maps(AttnMaps* m, const void* qkv, void* ctx, int frames, int tokens, int heads, int head_dim = 64);
int attention_launch(const AttnMaps& m, int frames, int tokens, int heads, float scale, int dtype, cudaStream_t stream,
                     int head_dim = 64, bool pdl = true);

// vit_misc.cu
int layernorm_launch(const void* x, const void* gamma, const void* beta, void* y, int rows, int dim, float eps,
                     int dtype, bool x_f32, bool y_f32, const void* delta, cudaStream_t stream, bool pdl = true);
int im2col_launch(const void* pixels, void* patches, int B, int S, int P, int Kpad, cudaStream_t stream);
int drop_cls_launch(const void* x, const void* delta, void* out, int B, int tokens, int D, int dtype, cudaStream_t stream,
                    bool keep_cls = false);

// memory_kernels.cu: the three pooled STAR levels (pool3_kernel) of consecutive frames into per-destination outputs.
// Destination i takes the next dst[i].frames frames of the concatenation: its frame f goes to rows a + f*a*a*D,
// b + f*b*b*D and c + f*D (b / c may be null).  pool3_launch pools frames [f0, f0 + n) of the concatenation from `in`
// (whose frame 0 is frame f0): the ViT encoder's fp32 residual stream [.., g*g+1, D] (residual) or f16 features
// [.., g*g, D].  One launch per kPoolDst destinations the range touches.
struct Pool3Dst {
  void *a, *b, *c;
  int frames;
};
constexpr int kPoolDst = 32;
struct Pool3Table {   // kernel-parameter form of up to kPoolDst destinations; first[j] = first frame of the launch for j
  int n;
  int first[kPoolDst + 1];
  uint16_t *a[kPoolDst], *b[kPoolDst], *c[kPoolDst];
};
int pool3_launch(const void* in, bool residual, const Pool3Dst* dst, int n_dst, int f0, int n, int g, int a, int b, int D,
                 cudaStream_t stream);

// vit_engine.cu: fvs_vit_encode_pool3 with the pooled levels going to n_dst destinations (frames of dst[0], then dst[1], ...)
int vit_encode_pool3(fvs_vit_t h, const void* pixels, const Pool3Dst* dst, int n_dst, int a, int b, void* workspace,
                     size_t workspace_bytes, cudaStream_t stream);

}  // namespace fvs
