/* fvs_b200.h — C ABI of libfvs_b200.so: the H100-native (sm_90a) implementation of Flash-VStream's
 * streaming hot path (ViT-L/14 frame encoding + Flash-Memory consolidation).
 *
 * The reference (IVGSZ/Flash-VStream) is pure Python and defines NO FFI; its seam is Python attribute
 * lookup (SURVEY.md §8b). Each entry point below therefore cites the reference Python callable whose
 * arithmetic it replaces; INTEGRATION.md shows the ctypes stub a reference maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name ends in _h (host);
 *   - tensors are dense row-major; "f16" = IEEE binary16;
 *   - every call enqueues on `stream` (a cudaStream_t passed as void*) and returns immediately;
 *     nothing synchronises, nothing allocates except fvs_vit_create (small prepared-weight buffers
 *     owned by the handle);
 *   - return value: FVS_OK (0) or a negative FVS_E* code; fvs_last_error() gives a thread-local message;
 *   - threading: re-entrant across handles/streams; a single handle must not be used concurrently
 *     (the reference has one memory-manager writer per stream, cli_video_stream.py:253).
 */
#ifndef FVS_B200_H
#define FVS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FVS_OK 0
#define FVS_EINVAL (-1)   /* bad argument / shape: Python shim raises ValueError / AssertionError */
#define FVS_ECUDA (-2)    /* CUDA runtime/driver error: RuntimeError */
#define FVS_ENOTIMPL (-3) /* unsupported option: NotImplementedError (cf. vstream_arch.py:235) */

#define FVS_F16 0
#define FVS_BF16 1
#define FVS_F32 2

typedef void* fvs_stream_t; /* cudaStream_t */

int fvs_version(void);
const char* fvs_last_error(void);
/* number of kernels this library has launched in the calling process (for bench.py's gpu_launches) */
uint64_t fvs_launch_count(void);

/* Optional in-library CUDA-event timing of the tensor-core launches (used by bench.py for the live roofline):
 * fvs_prof_enable(n) allocates n event pairs (n = 0 disables); afterwards every fvs_linear / fvs_attention launch
 * (also those issued inside fvs_vit_encode) is bracketed by two events on its stream until the pool is full.
 * After the caller has synchronised, fvs_prof_collect copies (kind, milliseconds, algorithmic FLOPs) per launch to
 * HOST arrays, returns the record count and resets the pool. */
#define FVS_PROF_LINEAR 1
#define FVS_PROF_ATTENTION 2
int fvs_prof_enable(int max_records);
int fvs_prof_collect(int32_t* kind_h, float* ms_h, double* work_h, int max_records);
/* fvs_prof_pause(1) suspends the event bracketing without freeing the pool (bench.py samples every 4th step so the
 * events perturb the timed region by ~1 % instead of ~5 %); fvs_prof_pause(0) resumes. */
int fvs_prof_pause(int paused);

/* ------------------------------------------------------------------------------------------------
 * Linear layer on tensor cores (wgmma m64nNk16, register accumulators, TMA-fed, fused epilogue).
 *   out[M,N] = epilogue( A[M,K] @ W[N,K]^T )          (W in torch.nn.Linear layout)
 * Replaces the cuBLAS calls behind HF CLIPEncoderLayer / CLIPVisionEmbeddings that
 * clip_encoder.py:50 reaches (SURVEY §2.2 K1,K2).
 *   FVS_EPI_BIAS            out = acc + bias[n]
 *   FVS_EPI_BIAS_QUICKGELU  out = g(acc + bias[n]),  g(x) = x * sigmoid(1.702 x)
 *   FVS_EPI_BIAS_RESIDUAL   out = acc + bias[n] + aux[m, n]        (aux row pitch = ldo; may alias out)
 *   FVS_EPI_ROWTABLE        out = acc + aux[(m % aux_period), n]   (aux is [aux_period, N], pitch N)
 *   FVS_EPI_BIAS_GELU       out = gelu(acc + bias[n]), exact erf GELU (torch.nn.GELU(), the mm_projector's activation,
 *                           multimodal_projector/builder.py:44)
 *   FVS_EPI_BIAS_RESIDUAL_F32  out_f32 = aux_f32[m, n] + (acc + bias[n])  (aux and out are fp32, pitch ldo; A, W, bias stay
 *                           16-bit).  aux == out is the fast path — the fp32 residual stream of the ViT encoder updated in
 *                           place, the addition performed by the L2 (TMA reduce-add); otherwise aux is copied to out first.
 * K must be a multiple of 8 (a tail below the 64-wide k-block is zero-filled by the TMA: Qwen2-VL's PatchEmbed has
 * K = 1176), N a multiple of 64; lda/ldo are row pitches in elements (multiples of 8).
 * dtype: FVS_F16 or FVS_BF16 (A, W, bias, aux, out all share it; accumulation is fp32).
 */
#define FVS_EPI_BIAS 0
#define FVS_EPI_BIAS_QUICKGELU 1
#define FVS_EPI_BIAS_RESIDUAL 2
#define FVS_EPI_ROWTABLE 3
#define FVS_EPI_BIAS_RESIDUAL_F32 4
#define FVS_EPI_BIAS_GELU 5
int fvs_linear(const void* A, const void* W, const void* bias, const void* aux, void* out, int M, int N, int K,
               int lda, int ldo, int epilogue, int aux_period, int dtype, fvs_stream_t stream);

/* Multi-head self-attention over packed QKV, one sequence per frame (no mask, softmax scale given):
 *   qkv [frames*tokens, 3*heads*64]  (q | k | v, each heads*64 wide)  ->  ctx [frames*tokens, heads*64]
 * head_dim is fixed at 64 (CLIP ViT-L/14: 16 x 64). Replaces HF CLIPAttention (SURVEY K2). */
int fvs_attention(const void* qkv, void* ctx, int frames, int tokens, int heads, float scale, int dtype,
                  fvs_stream_t stream);

/* Same with head_dim 80 (Qwen2-VL vision tower: 16 x 80), held as 64 "main" + 16 "extra" dims per head in separate column
 * blocks so that every tile is a whole swizzle atom:
 *   qkv [frames*tokens, 3*heads*80] = [ q main (heads*64) | k main | v main | q extra (heads*16) | k extra | v extra ]
 *   ctx [frames*tokens, heads*80]   = [ main (heads*64) | extra (heads*16) ]
 * where main holds dims 0..63 and extra dims 64..79 of every head.  The layout is produced for free by permuting the
 * rows of the QKV weight (and the columns of the output projection) once at load time. */
int fvs_attention80(const void* qkv, void* ctx, int frames, int tokens, int heads, float scale, int dtype,
                    fvs_stream_t stream);

/* Row LayerNorm: y = (x - mean)/sqrt(var + eps) * gamma + beta, fp32 statistics. x,y [rows, dim].
 * gamma/beta have `dtype` (f16|bf16); x_dtype / y_dtype are `dtype` or FVS_F32 (the encoder keeps its residual
 * stream in fp32 and feeds the GEMMs 16-bit normalised activations). dim % 256 == 0, dim <= 2048. */
int fvs_layernorm(const void* x, const void* gamma, const void* beta, void* y, int rows, int dim, float eps,
                  int dtype, int x_dtype, int y_dtype, fvs_stream_t stream);
/* Residual add fused with the LayerNorm that follows it: x_f32[rows,dim] += delta (16-bit, `dtype`), x is written back,
 * y (`dtype`) = LayerNorm(x). This is how the encoder applies the out-proj / fc2 residuals. */
int fvs_add_layernorm(void* x, const void* delta, const void* gamma, const void* beta, void* y, int rows, int dim,
                      float eps, int dtype, fvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * ViT-L/14 frame encoder = CLIPVisionTower.forward + feature_select
 * (multimodal_encoder/clip_encoder.py:31-53 -> transformers CLIPVisionModel, hidden_states[select_layer][:,1:]).
 */
typedef struct fvs_vit_layer_weights {
  const void* ln1_w; const void* ln1_b;   /* [hidden] */
  const void* qkv_w; const void* qkv_b;   /* [3*hidden, hidden], [3*hidden]  (q;k;v stacked) */
  const void* o_w;   const void* o_b;     /* [hidden, hidden], [hidden] */
  const void* ln2_w; const void* ln2_b;   /* [hidden] */
  const void* fc1_w; const void* fc1_b;   /* [mlp, hidden], [mlp] */
  const void* fc2_w; const void* fc2_b;   /* [hidden, mlp], [hidden] */
} fvs_vit_layer_weights;

typedef struct fvs_vit_config {
  int image_size;   /* 336 */
  int patch_size;   /* 14 */
  int hidden;       /* 1024 */
  int heads;        /* 16 (head_dim must be 64) */
  int mlp;          /* 4096 */
  int layers_run;   /* encoder layers actually executed: select_layer=-2 on 24 layers -> 23 */
  float ln_eps;     /* 1e-5 */
  int dtype;        /* FVS_F16 | FVS_BF16 */
  int keep_cls;     /* 0: output drops the CLS row (select_feature 'patch', clip_encoder.py:35); 1: keeps it ('cls_patch', :37) */
} fvs_vit_config;

typedef struct fvs_vit_weights {
  const void* patch_w;   /* [hidden, 3*patch*patch] conv weight, no bias */
  const void* class_emb; /* [hidden] */
  const void* pos_emb;   /* [tokens, hidden], tokens = (image/patch)^2 + 1 */
  const void* pre_ln_w; const void* pre_ln_b; /* [hidden] */
  const fvs_vit_layer_weights* layers_h;       /* host array, layers_run entries (device pointers inside) */
} fvs_vit_weights;

typedef struct fvs_vit* fvs_vit_t;

int fvs_vit_create(fvs_vit_t* out, const fvs_vit_config* cfg_h, const fvs_vit_weights* w_h, fvs_stream_t stream);
int fvs_vit_destroy(fvs_vit_t h);
/* bytes of caller-owned workspace needed to encode up to max_frames per call */
size_t fvs_vit_workspace_bytes(fvs_vit_t h, int max_frames);
/* pixels [frames,3,image,image] -> out [frames, (image/patch)^2 (+1 with cfg.keep_cls), hidden], both `dtype`.
 * Internally the residual stream is fp32 (DESIGN.md "precision"); frames are processed in micro-batches sized by
 * the workspace. */
int fvs_vit_encode(fvs_vit_t h, const void* pixels, void* out, int frames, void* workspace, size_t workspace_bytes,
                   fvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Flash-Memory consolidation (f16 only: the reference forces .to(torch.float16), vstream_arch.py:649).
 */

/* compress_spatial_features, compress_type='mean' (vstream_arch.py:193-212):
 * feat [T, grid*grid, D] -> out [T, target*target, D]; avg_pool2d kernel=stride=grid/target, or global mean
 * when target==1. fp32 window sum, one division, one rounding. */
int fvs_spatial_pool(const void* feat, void* out, int T, int grid, int target, int D, int dtype, fvs_stream_t stream);

/* The three STAR levels in one pass over the ViT output (vstream_arch.py:644,659-662):
 * feat [T, g*g, D] -> out_a [T, a*a, D] (rounded), then from the ROUNDED out_a: out_b [T, b*b, D] and
 * out_c [T, 1, D]. Defaults g=24,a=8,b=4. Any of out_b/out_c may be NULL. */
int fvs_spatial_pool3(const void* feat, void* out_a, void* out_b, void* out_c, int T, int g, int a, int b, int D,
                      int dtype, fvs_stream_t stream);

/* weighted_kmeans_feature's inner Lloyd loop (compress_functions.py:130-157), reference-exact rounding:
 *   dist[t,k] = f16(sqrt(f16(sum_f32(f16(f16(x-c)^2)))));  labels = first-index argmin (NaN wins);
 *   centroid = f16(f16(sum_f32(f16(w*x))) / f16(sum_f32(w)));  empty cluster <- X[refill_idx[next]];
 *   stop when f16(sum_k f16(norm2(c_old-c_new))) < f16(tol); on stop the OLD centroids are returned (:155).
 * X [T, PD]; w [T] or NULL (ones); init_idx [K] (the randperm draw, :134); refill_idx [max_iter*K]
 * (random.randint draws, :152, consumed in order). Outputs: C_out [K,PD], wsum_out [K] (f16),
 * labels_out [T] (int32), info_out [4] int32 = {exit_step i, refills consumed, converged(0/1), 0}.
 * PD must be a multiple of 1024. workspace: fvs_kmeans_workspace_bytes(T,K,PD). */
size_t fvs_kmeans_workspace_bytes(int T, int K, int PD);
int fvs_weighted_kmeans(const void* X, const void* w, const int32_t* init_idx, const int32_t* refill_idx, int T,
                        int K, int PD, int max_iter, float tol, void* C_out, void* wsum_out, int32_t* labels_out,
                        int32_t* info_out, void* workspace, size_t workspace_bytes, int dtype, fvs_stream_t stream);

/* VStreamMetaForCausalLM.attention + NeuralTuringMachine.get_weight (vstream_arch.py:174-183, :47-52):
 *   W = softmax((M Wq^T + bq)(F Wk^T + bk)^T / sqrt(H)) * ratio ;  M <- M*(1 - rowsum(W)) + W F
 * M [T1,D] (updated in place into M_out, may alias M), F [T2,D], Wq/Wk [H,D], bq/bk [H]. */
int fvs_abstract_update(const void* M, const void* F, const void* Wq, const void* bq, const void* Wk, const void* bk,
                        void* M_out, int T1, int T2, int D, int H, float ratio, int dtype, fvs_stream_t stream);

/* Stable descending argsort of K (<=1024) weights -> order_out [K] int64 (ties: lower index first).
 * The reference calls torch.argsort(weight, descending=True) (vstream_arch.py:261,681), which is unstable;
 * see DESIGN.md "tie contract". */
int fvs_argsort_desc(const void* w, int K, int64_t* order_out, int dtype, fvs_stream_t stream);

/* Key-frame retrieval (vstream_arch.py:261-268 / :681-688):
 *   keyc = long_mem[order[:key_len]];  d[l,k] = f16(sqrt(f16(sum_p f16(sum_d f16(f16(a-b)^2)))));
 *   idx_out[k] = first-index argmin_l d[l,k].    long_mem [L,P,D]; order int64 [>=key_len]. */
int fvs_key_retrieve(const void* long_mem, const int64_t* order, int L, int P, int D, int key_len, int64_t* idx_out,
                     int dtype, fvs_stream_t stream);

/* out[i, :] = src[idx[i], :] for i < n (rows of row_elems elements); idx int64 device. */
int fvs_gather_rows(const void* src, const int64_t* idx, void* out, int n, int64_t row_elems, int dtype,
                    fvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Streaming step on a persistent bank = embed_video_streaming (vstream_arch.py:611-697; SURVEY.md §8b, Appendix B).
 *
 * One stream = one fvs_bank: caller-owned device buffers plus host-side row counters that fvs_stream_step advances
 * (every shape of a step is host-known; only WHICH rows win is data-dependent and stays on the device).
 *   prefix     [prefix_rows, D] f16 — always holds the published state packed in the reader's order
 *              [Turing (n_tur x 1) | long (n_long x long_size^2) | key + current (n_cur x cur_size^2)]   (vstream_arch.py:483),
 *              i.e. the LLM's visual prefix is prefix[:rows] — a view, no concatenation copy;
 *   long_work  [long_work_rows, long_size^2 * D] — rows [0, n_long) = the long memory, then the incoming clip's rows
 *              (the k-means working set of vstream_arch.py:677-678 is built in place);
 *   tur_work   [tur_work_rows, D] — same for the abstract (Turing) memory (:690);
 *   frames     [frames_cap, cur_size^2 * D] — img_feature_buffer (:650,:676), appended in place; the caller grows it.
 *              With a device window (frames_window = N > 0) it holds only frames [0, N) plus a slot of chunk_cap rows
 *              [N, N + chunk_cap) that receives the current clip's frames at or past N, in order, so frames_cap must be at
 *              least N + chunk_cap and never grows.  A step reads only frames below N (key frames: frames[i] for a row i of
 *              the long working set, so N must be >= fvs_bank_rows' long_work_rows) and the current clip's own frames, so
 *              the caller may copy the slot's rows elsewhere (host memory) after the step and before the next one;
 *   header     8 x uint64 {seq, n_tur, n_long, n_cur, n_frames, step, 0, 0}: seq is odd while a step is writing the
 *              prefix, even otherwise — readers in other processes / on other GPUs (CUDA IPC) use fvs_bank_snapshot.
 * fvs_bank_rows gives the row capacities for a given maximum clip length (chunk_cap frames per call).
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct fvs_star_config {   /* the reference's STAR knobs (scripts/train_and_eval.sh:7-14) */
  int D;          /* 1024 */
  int grid;       /* 24: ViT patch grid */
  int cur_size;   /* compress_size 8 */
  int long_size;  /* compress_long_memory_size 4 (compress_Turing_memory_size must be 1) */
  int long_len;   /* video_long_memory_length 25 */
  int tur_len;    /* video_Turing_memory_length 25 */
  int cur_len;    /* video_current_memory_length 1 */
  int key_len;    /* 3 (hard-coded at vstream_arch.py:683) */
  int ntm_dim;    /* NeuralTuringMachine output_dim 32 */
  float ratio;    /* compress_Turing_update_ratio 0.2 */
} fvs_star_config;

typedef struct fvs_ntm_weights {   /* NeuralTuringMachine.q_proj / k_proj (vstream_arch.py:38-39), f16 */
  const void* q_w; const void* q_b;   /* [ntm_dim, D], [ntm_dim] */
  const void* k_w; const void* k_b;
} fvs_ntm_weights;

typedef struct fvs_bank {
  void* prefix; void* long_work; void* tur_work; void* frames; void* header;   /* device, caller-owned */
  int64_t frames_cap;    /* rows of `frames` */
  int32_t chunk_cap;     /* maximum frames per fvs_stream_step call the buffers were sized for */
  int32_t n_long, n_tur, n_cur;   /* host counters, maintained by the library */
  int64_t n_frames;
  uint64_t step;
  int64_t frames_window; /* 0: `frames` holds every frame; N > 0: only frames [0, N) stay there, a clip's frames at or past
                            N land in the slot [N, N + chunk_cap) (see `frames` above) */
} fvs_bank;

#define FVS_INPUT_PIXELS 0     /* input = [frames, 3, image, image] pixels; encoded with `vit`, pooled in the encoder's tail */
#define FVS_INPUT_FEATURES 1   /* input = [frames, grid*grid, D] f16 finished ViT features */

size_t fvs_stream_workspace_bytes(const fvs_star_config* cfg_h, int chunk_cap);
int fvs_bank_rows(const fvs_star_config* cfg_h, int chunk_cap, int64_t* long_work_rows_h, int64_t* tur_work_rows_h,
                  int64_t* prefix_rows_h);
int fvs_bank_reset(fvs_bank* bank_h, fvs_stream_t stream);
/* Restore a stream's state into `bank` (same STAR config; any chunk_cap whose capacities hold it), e.g. a checkpoint taken
 * on another device or in another process.  Sources are device pointers on the bank's device or pinned host pointers (UVA);
 * counts are the saved bank's host counters:
 *   prefix_src [rows, D] packed [Turing | long | key + current] with rows = n_tur + n_long*long_size^2 + n_cur*cur_size^2;
 *   long_src [n_long, long_size^2*D]; tur_src [n_tur, D]; frames_src [n_frames, cur_size^2*D].
 * Saving needs no entry point: between two steps, on the writer's stream, prefix[:rows], long_work[:n_long],
 * tur_work[:n_tur] and frames[:n_frames] are a consistent state.
 * The working sets and the frame buffer are copied with cudaMemcpyAsync; the prefix and header words 1-5 by one cooperative
 * kernel under the writer side of the seqlock (seq odd, copy, fence + grid barrier, counters, seq even), so a reader that
 * has the bank mapped sees the old prefix or the restored one, never a mix, and seq keeps growing.
 * Limits: n_long <= max(long_len, chunk_cap), n_tur <= max(tur_len, chunk_cap) (a first clip longer than a memory leaves
 * that many rows), n_cur <= key_len + cur_len, the prefix rows within fvs_bank_rows' capacity, n_frames <= frames_cap
 * (with a device window N: any n_frames; only frames_src's first min(n_frames, N) rows are copied, the caller keeps the
 * rest), step == 0 exactly when n_frames == 0 (and then no memory rows), sources non-null where their count is non-zero.
 * Validated before anything is enqueued; on FVS_EINVAL nothing was launched and no counter or header changed.
 * The next fvs_stream_step needs the bank's workspace arrival counters at zero: a workspace that completed a step, or
 * a zeroed one. */
int fvs_bank_restore(const fvs_star_config* cfg_h, fvs_bank* bank_h, int32_t n_tur, int32_t n_long, int32_t n_cur,
                     int64_t n_frames, uint64_t step, const void* prefix_src, const void* long_src, const void* tur_src,
                     const void* frames_src, fvs_stream_t stream);
/* prefix pointer (= bank->prefix) and its current row count; pure host arithmetic */
int fvs_bank_prefix(const fvs_star_config* cfg_h, const fvs_bank* bank_h, void** prefix_out_h, int64_t* rows_out_h);
/* One clip of `frames` frames into the bank: pooling (encoder tail or pool3) + ONE cooperative kernel doing the weighted
 * k-means (device-side early exit), key-frame retrieval, abstract-memory update and the write-back.
 * init_idx [long_len] / refill_idx [10*long_len]: the torch.randperm / random.randint draws of weighted_kmeans_feature
 * (compress_functions.py:134,152) for a working set of n_long + frames rows; only read when that exceeds long_len.
 * vit / vit_workspace: only for FVS_INPUT_PIXELS.  workspace: fvs_stream_workspace_bytes(cfg, bank->chunk_cap). */
int fvs_stream_step(const fvs_star_config* cfg_h, fvs_bank* bank_h, const fvs_ntm_weights* ntm_h, fvs_vit_t vit,
                    const void* input, int input_kind, int frames, const int32_t* init_idx, const int32_t* refill_idx,
                    void* vit_workspace, size_t vit_workspace_bytes, void* workspace, size_t workspace_bytes,
                    fvs_stream_t stream);
/* Many streams in one call.  Job i steps bank i with a clip of `frames` frames; the clips lie back to back in `input`
 * (job 0's frames, then job 1's, ...; pixels or features as for fvs_stream_step, one input_kind for all).  The call is
 * bit-identical to calling fvs_stream_step for job 0, then job 1, ... with the same draws: every bank array, prefix,
 * header and fvs_stream_step_info diagnostic — whatever point of its stream each bank is at (first step, warm-up,
 * steady state) and whatever the clip lengths.  The ViT is invariant to batch composition, so all clips are encoded
 * together in the engine's micro-batches, and each frame's pooled levels go straight into its own bank.  The
 * consolidation runs as few cooperative launches ("waves") as the co-residency limit allows: each job owns a contiguous
 * range of blocks and its own barriers, and its bits do not depend on how many blocks it gets.
 * Every job is validated before anything is enqueued (a bank or workspace in two jobs, frames > chunk_cap, a full frame
 * buffer, draws missing where the k-means runs, a workspace too small, ...): on FVS_EINVAL nothing was launched and no
 * bank counter or header changed.  Jobs may share one fvs_ntm_weights.  max_blocks caps the blocks of one launch
 * (0 = the device's co-residency limit); per-job tables travel as kernel parameters (no allocation, no host sync). */
typedef struct fvs_stream_job {
  fvs_bank* bank;                     /* host struct; its counters advance only when the call succeeds */
  const fvs_ntm_weights* ntm;
  int frames;                         /* 1 <= frames <= bank->chunk_cap */
  const int32_t* init_idx;            /* device draws, as for fvs_stream_step */
  const int32_t* refill_idx;
  void* workspace;                    /* this bank's own fvs_stream_workspace_bytes(cfg, bank->chunk_cap) bytes */
  size_t workspace_bytes;
} fvs_stream_job;
int fvs_stream_step_multi(const fvs_star_config* cfg_h, fvs_stream_job* jobs_h, int n_jobs, fvs_vit_t vit, const void* input,
                          int input_kind, void* vit_workspace, size_t vit_workspace_bytes, int max_blocks,
                          fvs_stream_t stream);
/* The launch plan fvs_stream_step_multi uses for a budget of `budget` blocks per launch (pure host arithmetic, validates
 * like the step, no CUDA call): job i gets blocks_h[2i] Lloyd-loop blocks and blocks_h[2i+1] abstract-memory blocks in
 * launch waves_h[i].  Returns the number of launches (>= 1) or a negative error code. */
int fvs_stream_plan(const fvs_star_config* cfg_h, const fvs_stream_job* jobs_h, int n_jobs, int budget, int32_t* blocks_h,
                    int32_t* waves_h);
/* device pointers (inside `workspace`) to the last step's diagnostics: labels int32 [T], info int32 [4] = {exit step,
 * refills consumed, converged, k-means ran}, key_idx int64 [key_len], wsum f16 [long_len] */
int fvs_stream_step_info(const fvs_star_config* cfg_h, const fvs_bank* bank_h, void* workspace, int32_t** labels_out_h,
                         int32_t** info_out_h, int64_t** key_idx_out_h, void** wsum_out_h);
/* Consistent copy of a (possibly remote: CUDA-IPC-mapped, other GPU over NVLink) bank prefix: out [max_rows, D] <- prefix.
 * status (device uint64[7]) = {seq before, seq after, n_tur, n_long, n_cur, n_frames, step}; the snapshot is valid iff
 * status[0] == status[1] and even — otherwise a step was writing, call again. */
int fvs_bank_snapshot(const void* prefix, const void* header, void* out, int64_t max_rows, int D, int cur_size,
                      int long_size, uint64_t* status, fvs_stream_t stream);

/* ViT encoder with the pooled tail of the streaming path: pixels [frames,3,image,image] -> the three STAR levels
 * out_a [frames, a*a, hidden] (f16-rounded 24->a pooling of hidden_states[select_layer][:,1:]), out_b [frames, b*b, hidden]
 * and out_c [frames, 1, hidden] pooled from the rounded out_a (vstream_arch.py:644,649,659-662); out_b / out_c may be NULL.
 * The [frames, 576, hidden] feature map is never written.  f16 towers with select_feature 'patch' only. */
int fvs_vit_encode_pool3(fvs_vit_t h, const void* pixels, void* out_a, void* out_b, void* out_c, int frames, int a, int b,
                         void* workspace, size_t workspace_bytes, fvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Qwen2-VL vision tower blocks = what forward_simple_not_merge runs between temporal_pool and the Flash Memory
 * (Flash-VStream-Qwen/models/vstream_qwen2vl_realtime.py:392-426, vstream_qwen2vl_model.py:388-428 over transformers'
 * PatchEmbed, VisionRotaryEmbedding, Qwen2VLVisionBlock): PatchEmbed GEMM, then `depth` x [LayerNorm -> QKV -> 2-D rotary
 * -> attention within every (temporal patch, grid) segment -> proj -> residual -> LayerNorm -> fc1 quick-GELU -> fc2 ->
 * residual].  Layer weights use fvs_vit_layer_weights (qkv_w [3*embed, embed] with q;k;v stacked and heads of 80 dims in
 * natural order — the handle keeps permuted copies for fvs_attention80); patch_w [embed, patch_dim] is the flattened
 * Conv3d weight (no bias); inv_freq_h[20] = VisionRotaryEmbedding(head_dim/2).inv_freq (host).
 * encode: patches [rows, patch_dim] with rows = sum_i t_i*h_i*w_i over the n_grids (t, h, w) entries of grid_thw_h (host
 * int32 [n_grids, 3]; rows of a grid ordered (t, h/2, w/2, 2, 2)); out [rows, embed], same dtype.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct fvs_qwen_vit_config {
  int embed_dim;   /* 1280 */
  int heads;       /* 16 (head_dim must be 80) */
  int mlp_dim;     /* 5120 */
  int depth;       /* 32 */
  int patch_dim;   /* 3*2*14*14 = 1176 */
  float ln_eps;    /* 1e-6 */
  int dtype;       /* FVS_F16 | FVS_BF16 */
} fvs_qwen_vit_config;
typedef struct fvs_qwen_vit* fvs_qwen_vit_t;
int fvs_qwen_vit_create(fvs_qwen_vit_t* out, const fvs_qwen_vit_config* cfg_h, const void* patch_w,
                        const fvs_vit_layer_weights* layers_h, const float* inv_freq_h, fvs_stream_t stream);
int fvs_qwen_vit_destroy(fvs_qwen_vit_t h);
size_t fvs_qwen_vit_workspace_bytes(fvs_qwen_vit_t h, int64_t rows);
int fvs_qwen_vit_encode(fvs_qwen_vit_t h, const void* patches, void* out, const int32_t* grid_thw_h, int n_grids,
                        void* workspace, size_t workspace_bytes, fvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Alternate temporal compressors selectable through `video_sample_type` (vstream_arch.py:222-236, 626-637):
 * drop_feature / merge_feature / k_drop_feature / k_merge_feature / kmeans_feature of
 * flash_vstream/model/compress_functions.py (:19, :57, :170, :213, :91).  X [T, PD] f16, reduced to T0 rows; T > T0 >= 2
 * (T <= T0 is the callers' pass-through), PD % 1024 == 0.
 *
 * fvs_alt_sequential runs the whole frame-by-frame loop of one of the four sequential compressors in ONE launch:
 *   coins    [T-T0] int32: the random.randint(0, 1) draws of the drop variants (NULL for merge variants)
 *   sim_in   optional [T0-1] f16 adjacent similarities carried over by the caller (drop / merge; NULL = compute)
 *   kept_out [T0] int32: frame index of every surviving row (drop variants: the result is X[kept_out])
 *   feat_out [T0, PD] f16: the merged rows (merge variants)
 *   sim_out  drop / merge: [T0-1] f16 adjacent cosine similarities; k_merge: [T0, T0] f16 similarity matrix; k_drop: unused
 *   pos_out  [T-T0] int32: the row that left the candidate list at every step (k_merge: the flat argmax
 *            left*(T0+1)+right, row `left` leaves after being merged into `right`); the caller rebuilds the reference's
 *            per-step member lists from it
 * ------------------------------------------------------------------------------------------------------------------ */
#define FVS_ALT_DROP 0
#define FVS_ALT_MERGE 1
#define FVS_ALT_KDROP 2
#define FVS_ALT_KMERGE 3
#define FVS_ALT_KMEANS 4
size_t fvs_alt_workspace_bytes(int method, int T, int T0, int PD);
int fvs_alt_sequential(int method, const void* X, int T, int T0, int PD, const void* sim_in, const int32_t* coins,
                       int32_t* kept_out, void* feat_out, void* sim_out, int32_t* pos_out, void* workspace,
                       size_t workspace_bytes, int dtype, fvs_stream_t stream);
/* kmeans_feature's Lloyd loop (compress_functions.py:92-113): torch.cdist in ATen's matmul form on f16, unweighted means,
 * random refills, `diff < tol` in f16, OLD centroids kept on the tolerance break.  init_idx [K] = torch.randperm(T)[:K],
 * refill_idx [max_iter*K] = the random.randint(0, T-1) draws.  info_out[4] = {last iteration, refills used, converged, 0}. */
int fvs_alt_kmeans(const void* X, const int32_t* init_idx, const int32_t* refill_idx, int T, int K, int PD, int max_iter,
                   float tol, void* C_out, int32_t* labels_out, int32_t* info_out, void* workspace, size_t workspace_bytes,
                   int dtype, fvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Qwen2-VL variant of the Flash Memory (Flash-VStream-Qwen/models/vstream_qwen2vl_model.py class FlashMemory and
 * Flash-VStream-Qwen/models/compress_functions.py).  Rows are flattened visual tokens: one "frame" is P*D elements.
 * ------------------------------------------------------------------------------------------------------------------ */

/* FlashMemory.temporal_pool (vstream_qwen2vl_model.py:113-142): x [t*h*w, 1176] patchified pixels, rows ordered
 * (t, h/2, w/2, 2, 2), columns (3, 2, 14, 14); out [t*(h/2)*(w/2), 1176] = 2x2 pixel average re-patchified with rows
 * ordered (t, h/4, w/4, 2, 2).  16-bit dtype (f16/bf16), fp32 accumulate, one rounding.  Returns FVS_ENOTIMPL when h/2
 * or w/2 is odd (the reference raises NotImplementedError there). */
int fvs_qwen_temporal_pool(const void* x, void* out, int t, int h, int w, int dtype, fvs_stream_t stream);

/* torch.unique(X, dim=0) of weighted_kmeans_ordered_feature (compress_functions.py:197): uniq_idx_out[r] = index of the
 * first row of the r-th duplicate class in ascending lexicographic order, n_unique_out[0] = number of classes.
 * X [T, PD] in `dtype` (f16/bf16/f32), T <= 4096. */
size_t fvs_qwen_unique_workspace_bytes(int T);
int fvs_qwen_unique_rows(const void* X, int T, int PD, int dtype, int32_t* uniq_idx_out, int32_t* n_unique_out,
                         void* workspace, size_t workspace_bytes, fvs_stream_t stream);

/* The fp32 Lloyd loop of weighted_kmeans_ordered_feature (compress_functions.py:199-263).  X [T, PD] (x_dtype, widened to
 * fp32 on load like the reference's X.float()), w [T] fp32 frame weights.  Initial centroid k = X[uniq_idx[init_idx[k]]]
 * (uniq_idx NULL: X[init_idx[k]]); init_idx is the caller's torch.randperm draw, refill_idx[max_iter*K] the
 * torch.randint draws consumed (in order) by empty clusters.  Distances in GEMM form sqrt((|x|^2+|c|^2) - 2 x.c), argmin
 * first-index; update = weighted mean; stop when sum_k ||c_k - c'_k|| < tol (the OLD centroids are the result then, as in
 * the reference's `break` before `centroids = new_centroids`) or after max_iter.  max_iter == 0 runs the degenerate branch (compress_functions.py:200-213): one assignment against
 * the initial centroids, no update.  Outputs: C_out [K, PD] fp32, wsum_out [K], labels_out [T],
 * info_out[4] = {last iteration, refills consumed, converged, 0}.  PD % 1024 == 0. */
size_t fvs_qwen_kmeans_workspace_bytes(int T, int K, int PD);
int fvs_qwen_kmeans(const void* X, int x_dtype, const float* w, const int32_t* uniq_idx, const int32_t* init_idx,
                    const int32_t* refill_idx, int T, int K, int PD, int max_iter, float tol, float* C_out, float* wsum_out,
                    int32_t* labels_out, int32_t* info_out, void* workspace, size_t workspace_bytes, fvs_stream_t stream);

/* The bookkeeping after the Lloyd loop (compress_functions.py:274-290) without a host round trip: cluster timestamp =
 * mean member row index (Python int / int, then fp32), clusters ordered by timestamp (stable; or order_in [K] int64 = the
 * permutation to replay), sorted_idx_out [K] int64 = that order (feed it to fvs_gather_rows_cast), ts_out / w_out [K] the
 * permuted timestamps / cluster weights, flags_out[0] = number of empty clusters (ZeroDivisionError in the reference).
 * labels [T] and wsum [K] are fvs_qwen_kmeans outputs.  K <= 1024. */
int fvs_qwen_kmeans_finalize(const int32_t* labels, const float* wsum, int T, int K, const int64_t* order_in,
                             int64_t* sorted_idx_out, float* ts_out, float* w_out, int32_t* flags_out, fvs_stream_t stream);

/* out[i, :] = cast<out_dtype>(src[idx[i], :]): the `reduced_feature[sorted_indices] ... .to(dtype)` of
 * compress_functions.py:283,297 in one pass.  src fp32, idx int64, 0 < n <= 65535, row_elems % 4 == 0. */
int fvs_gather_rows_cast(const float* src, const int64_t* idx, void* out, int n, int64_t row_elems, int out_dtype,
                         fvs_stream_t stream);

/* ---- the CSM chain of many Qwen2-VL streams in one launch per kernel (DESIGN.md §3.17) -------------------------------
 * One fvs_qwen_mem_job per stream: its candidates X [T, PD] (x_dtype), draws and outputs, all device pointers.  Each
 * single-stream call above runs as a table of one job, so each *_multi call below gives job i exactly the bits the
 * single-stream call gives it, whatever the other jobs are: a job always gets the blocks of its one-job launch, laid end
 * to end with the other jobs' blocks in one flat grid (a block finds its job in a block-offset table passed as a kernel
 * parameter), so no reduction of a job depends on its neighbours or on the budget.  Jobs go into launches in order, at most FVS_QWEN_MEM_JOBS_PER_LAUNCH per launch and, when
 * budget > 0, at most `budget` Lloyd-sweep blocks per launch (a larger job goes alone); every kernel of a call is then
 * launched once per launch group.  Every job gets the checks of its single call plus the table's own (the shapes of
 * fvs_qwen_mem_plan, known dtype codes, no output range shared by two jobs) before anything is enqueued: on FVS_EINVAL
 * nothing was launched.  No allocation, no host sync.
 *   fvs_qwen_unique_rows_multi:     fvs_qwen_unique_rows(X, T, PD, x_dtype, uniq_idx, n_unique, uniq_workspace, ...)
 *   fvs_qwen_kmeans_multi:          fvs_qwen_kmeans(X, x_dtype, w, uniq_idx, init_idx, refill_idx, T, K, PD, max_iter, tol,
 *                                                   C, wsum, labels, info, km_workspace, ...); each job keeps its own
 *                                   max_iter and tolerance exit (a job that has stopped skips the remaining iterations)
 *   fvs_qwen_kmeans_finalize_multi: fvs_qwen_kmeans_finalize(labels, wsum, T, K, order_in, sorted_idx, ts, w_sorted, flags)
 *   fvs_gather_rows_cast_multi:     fvs_gather_rows_cast(C, sorted_idx, out, K, PD, out_dtype)
 * Fields a call does not read may be anything. */
#define FVS_QWEN_MEM_JOBS_PER_LAUNCH 16
typedef struct fvs_qwen_mem_job {
  const void* X;                   /* [T, PD] candidate rows */
  int T, K, PD, x_dtype;           /* T <= 4096, 0 < K <= min(T, 1024), PD % 1024 == 0 */
  const float* w;                  /* [T] fp32 weights */
  const int32_t* init_idx;         /* [K] */
  const int32_t* refill_idx;       /* [max(1, max_iter * K)] */
  int max_iter;
  float tol;
  int32_t* uniq_idx;               /* [T]: written by unique_rows, read by kmeans (NULL there: X[init_idx[k]]) */
  int32_t* n_unique;               /* [1] */
  void* uniq_workspace;            /* fvs_qwen_unique_workspace_bytes(T) */
  size_t uniq_workspace_bytes;
  float* C;                        /* [K, PD] fp32 centroids */
  float* wsum;                     /* [K] */
  int32_t* labels;                 /* [T] */
  int32_t* info;                   /* [4] */
  void* km_workspace;              /* fvs_qwen_kmeans_workspace_bytes(T, K, PD) */
  size_t km_workspace_bytes;
  const int64_t* order_in;         /* [K] permutation to replay, or NULL (stable order) */
  int64_t* sorted_idx;             /* [K] */
  float* ts;                       /* [K] */
  float* w_sorted;                 /* [K] */
  int32_t* flags;                  /* [1] */
  void* out;                       /* [K, PD] out_dtype: the ordered, cast centroids */
  int out_dtype;
} fvs_qwen_mem_job;
/* The launch plan of the *_multi calls for `budget` (pure host arithmetic, no CUDA call): job i gets blocks_h[i] Lloyd-
 * sweep blocks ((T+7)/8 * PD/1024, the widest grid of its chain) in launch group groups_h[i].  Returns the number of
 * launch groups (>= 1) or a negative error code. */
int fvs_qwen_mem_plan(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, int32_t* blocks_h, int32_t* groups_h);
int fvs_qwen_unique_rows_multi(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, fvs_stream_t stream);
int fvs_qwen_kmeans_multi(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, fvs_stream_t stream);
int fvs_qwen_kmeans_finalize_multi(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, fvs_stream_t stream);
int fvs_gather_rows_cast_multi(const fvs_qwen_mem_job* jobs_h, int n_jobs, int budget, fvs_stream_t stream);

/* spatial_enhance with spatial_method='klarge_retrieve' (vstream_qwen2vl_model.py:197-207, 229-238): for the k centroids
 * c_i = tem_x[klarge_idx[i]] (tem_x [st, PD], klarge_idx int64 [k] = the k heaviest clusters) and the bank [t_total, PD] of
 * half-resolution frames, idx_out[i] = argmin_t sqrt((|c_i|^2 + |b_t|^2) - 2 c_i.b_t) with every op rounded to the 16-bit
 * `dtype` exactly like efficient_euclidean_distance on 16-bit tensors (|v|^2 = dt(sum_f32(dt(v^2))), c.b = dt(sum_f32(c*b)));
 * a NaN from a negative radicand wins the argmin, as in torch.  dist_out (optional, may be NULL): fp32 [k, t_total] holding
 * the rounded distances.  k <= 64, PD % 1024 == 0.
 * metric FVS_KLARGE_COSINE = spatial_method 'klarge_retrieve_cos' (:208-215): idx_out[i] = argmin_t cos(c_i, b_t) — the
 * reference takes the ARGMIN of the similarity (the least similar frame); mirrored as is — with |v| = dt(sqrt(sum_f32(v^2)))
 * (Tensor.norm), vn = dt(v / |v|), cos = dt(sum_f32(cn * bn)); a zero row gives NaN, which wins.  dist_out then holds the
 * rounded similarities. */
#define FVS_KLARGE_EUCLIDEAN 0
#define FVS_KLARGE_COSINE 1
size_t fvs_qwen_klarge_workspace_bytes(int k, int t_total, int PD);
int fvs_qwen_klarge_retrieve(const void* tem_x, const int64_t* klarge_idx, const void* bank, int k, int t_total, int PD,
                             int dtype, int metric, int64_t* idx_out, float* dist_out, void* workspace,
                             size_t workspace_bytes, fvs_stream_t stream);
/* The same retrieval over a two-tier bank (DESIGN.md §3.13): rows [0, n_dev) are contiguous device rows dev_bank (may be
 * NULL when n_dev == 0); row n_dev + c*chunk_frames + r is row r of pinned host chunk c, read in place through its mapped
 * device pointer host_chunks[c] (a HOST array of ceil((t_total - n_dev) / chunk_frames) pointers, fvs_host_device_ptr).
 * One sweep launch covers the device rows and one each host chunk; the reductions and the tail run once over all t_total
 * rows, so the results are bit-identical to fvs_qwen_klarge_retrieve on the same rows.  Each step reads the host rows
 * over PCIe once (Euclidean) or twice (cosine).  With n_dev == t_total it launches exactly what fvs_qwen_klarge_retrieve
 * launches.  FVS_EINVAL with nothing launched on a bad argument (n_dev outside [0, t_total], a NULL chunk table or chunk
 * pointer, or chunk_frames <= 0 while host rows exist). */
int fvs_qwen_klarge_retrieve_tiered(const void* tem_x, const int64_t* klarge_idx, const void* dev_bank, int n_dev,
                                    const void* const* host_chunks, int chunk_frames, int k, int t_total, int PD, int dtype,
                                    int metric, int64_t* idx_out, float* dist_out, void* workspace, size_t workspace_bytes,
                                    fvs_stream_t stream);

/* The klarge retrieval of many streams in one launch per kernel (DESIGN.md §3.17): job i gets exactly the bits of
 * fvs_qwen_klarge_retrieve(tem_x, klarge_idx, bank, k, t_total, PD, dtype, metric, idx_out, dist_out, workspace, ...)
 * whatever the other jobs are (the single call is the one-job table): its sweep keeps the split-K partition (PD/1024
 * slices x ceil(t_total/32) row splits), laid end to end with the other jobs' blocks.  dtype and metric are the call's; k, t_total, PD, the bank
 * and klarge_idx are each job's.  The bank must be wholly in HBM: a job with n_dev != t_total (host rows, which the
 * tiered sweep reads through fvs_qwen_klarge_retrieve_tiered) is refused.  At most FVS_QWEN_MEM_JOBS_PER_LAUNCH jobs per
 * launch; FVS_EINVAL with nothing launched on a bad job or an output shared by two jobs. */
typedef struct fvs_qwen_retrieve_job {
  const void* tem_x;               /* [st, PD] centroids */
  const int64_t* klarge_idx;       /* [k] */
  const void* bank;                /* [t_total, PD] half-resolution frames, device rows */
  int k, t_total, n_dev, PD;       /* 0 < k <= 64; n_dev must equal t_total */
  int64_t* idx_out;                /* [k] */
  float* dist_out;                 /* [k, t_total] or NULL */
  void* workspace;                 /* fvs_qwen_klarge_workspace_bytes(k, t_total, PD) */
  size_t workspace_bytes;
} fvs_qwen_retrieve_job;
int fvs_qwen_klarge_retrieve_multi(const fvs_qwen_retrieve_job* jobs_h, int n_jobs, int dtype, int metric,
                                   fvs_stream_t stream);

/* FlashMemory.calc_am_rope (vstream_qwen2vl_model.py:254-277): out [3, n] int64 position ids of the n = spa_t*spa_h*spa_w
 * + tem_t*tem_h*tem_w memory tokens (DAM rows first, then CSM rows offset by the DAM size), plus visual_start_id. */
int fvs_qwen_am_rope(const int64_t* spa_positions, int spa_t, int spa_h, int spa_w, const int64_t* tem_positions, int tem_t,
                     int tem_h, int tem_w, int64_t visual_start_id, int64_t* out, fvs_stream_t stream);

/* ---- feature bank of the Qwen2-VL streaming state (DESIGN.md §3.13, §3.18-§3.20) ------------------------------------------
 * Frames [0, n_dev) of the full-resolution bank (x, x_frame_elems 16-bit elements per frame) and of the PatchMerger bank
 * (merged, merged_frame_elems per frame) are contiguous device rows dev_x / dev_merged.  Later frames live in pinned host
 * chunks: chunk c holds frames n_dev + c*chunk_frames + [0, chunk_frames) as [chunk_frames x rows | chunk_frames merged
 * rows]; host_chunks is a DEVICE table of the chunks' mapped device pointers (fvs_host_device_ptr).
 * Every call below is a job table (one stream = the one-job table): every job is checked before anything is enqueued
 * (FVS_EINVAL naming the job otherwise), at most FVS_QWEN_MEM_JOBS_PER_LAUNCH jobs go into one launch, and no two jobs
 * may share an output.
 *
 * fvs_qwen_dam_gather_multi: per job, for every pick i (picks: device int64 [n], e.g. fvs_qwen_klarge_retrieve's
 * output), spa_x_out[i] = x[picks[i]] and merged_out[i] = merged[picks[i]] (either output may be NULL; not both), each
 * read from the first source that holds the frame:
 *   1. the previous step's DAM: prev_picks [m], prev_x [m, x_frame_elems], prev_merged [m, merged_frame_elems];
 *   2. this step's fresh rows: fresh_frames [n_fresh], fresh_x [n_fresh, x_frame_elems], fresh_merged [n_fresh,
 *      merged_frame_elems] (a stream without a full-resolution bank: the tower and PatchMerger output of its planned
 *      frames, in plan order; n_fresh is a host integer);
 *   3. the device tier, frames [0, n_dev);
 *   4. the host chunks, frames [n_dev, n_base), as zero-copy 16-byte loads; *host_fetches (device, optional) grows by
 *      the number of picks read there.
 * A pick outside [0, n_frames), or in no source, yields zero rows.  A stream with a bank passes n_fresh = 0 and
 * n_base = n_frames.  The outputs must not alias any source.  Row tensors 16-byte aligned, frame sizes multiples of
 * 16 bytes, n, m, n_fresh <= 65535.  dtype is the call's. */
typedef struct fvs_qwen_gather_job {
  const int64_t* picks;
  int n;
  int64_t n_frames;
  const void* dev_x;
  const void* dev_merged;
  int64_t n_dev;
  const void* const* host_chunks;  /* DEVICE table */
  int chunk_frames;
  const int64_t* prev_picks;
  int m;
  const void* prev_x;
  const void* prev_merged;
  int64_t x_frame_elems, merged_frame_elems;
  void* spa_x_out;
  void* merged_out;
  uint64_t* host_fetches;
  const int64_t* fresh_frames;
  int n_fresh;
  const void* fresh_x;
  const void* fresh_merged;
  int64_t n_base;
} fvs_qwen_gather_job;
int fvs_qwen_dam_gather_multi(const fvs_qwen_gather_job* jobs_h, int n_jobs, int dtype, fvs_stream_t stream);

/* Lazy full-resolution bank (DESIGN.md §3.18): a stream keeps each frame's full-resolution pixel rows in pinned host
 * chunks and encodes a frame the first time the DAM picks it.  Without a full-resolution bank (§3.19) it stores no x or
 * merged row of the frames it encodes and re-encodes a pick the previous DAM does not hold; a stream restored from a
 * checkpoint may then still hold a frozen base bank of stored rows (frames [0, n_base) of fvs_qwen_dam_gather_multi).
 *
 * fvs_qwen_pick_plan_multi: per job, walks picks (device int64 [n]; NULL = frames 0..n-1, the DAM while it is the whole
 * bank) in order and writes to plan (device int64 [n]) every pick p that is in [0, n_frames), that no earlier pick
 * names, that is not in prev_picks (device int64 [m], the previous step's DAM; NULL when m = 0) and whose byte in
 * `frames` (device uint8 [n_frames]) is below `stored`: a byte >= stored means the frame's rows are held.  A stream with
 * a bank passes stored = 1 and m = 0 (byte 0: not yet encoded); a stream without one passes stored = 2 (2: the frame's
 * rows are in the base bank) and its previous DAM, so it keeps no mask that a redone clip would have to roll back.  A
 * planned frame whose byte is 1 (encoded before) adds 1 to *re_encodes (device uint64, optional); every planned frame's
 * byte is then set to 1.  The plan's length goes to *count (int32; device memory or the mapped address of pinned host
 * memory, e.g. a slot of the stream's read-back row). */
typedef struct fvs_qwen_pick_plan_job {
  const int64_t* picks;
  int n;
  int64_t n_frames;
  uint8_t* frames;
  int64_t* plan;
  int32_t* count;
  const int64_t* prev_picks;
  int m;
  uint64_t* re_encodes;
  uint8_t stored;
} fvs_qwen_pick_plan_job;
int fvs_qwen_pick_plan_multi(const fvs_qwen_pick_plan_job* jobs, int n_jobs, fvs_stream_t stream);
/* fvs_qwen_pixel_gather_multi: per job, out[i] = the pixel rows of frame plan[i] (i < n), out [n, frame_elems] of
 * `dtype`: frame f >= base is frame f - base of the pinned pixel chunks, chunk c holding chunk_frames frames, read in
 * place through host_chunks (a DEVICE table of the chunks' mapped device pointers); a frame outside [base, n_frames)
 * yields zeros.  table NULL: the chunks hold frame_elems 16-bit elements per frame, gathered as fvs_qwen_dam_gather_multi
 * reads its host tier.  table non-null: the chunks hold frame_elems uint8 codes per frame (whole rows: frame_elems % 1176
 * == 0), decoded through `table` (device float32 [3, 256]) in the same pass as fvs_qwen_pixel_decode decodes them.
 * One call takes jobs of one kind: a table in every job or in none. */
typedef struct fvs_qwen_pixel_job {
  const int64_t* plan;
  int n;
  int64_t n_frames;
  int64_t base;
  const void* const* host_chunks;
  int chunk_frames;
  int64_t frame_elems;
  void* out;
  const float* table;
} fvs_qwen_pixel_job;
int fvs_qwen_pixel_gather_multi(const fvs_qwen_pixel_job* jobs, int n_jobs, int dtype, fvs_stream_t stream);
/* fvs_qwen_bank_scatter_multi: per job, the reverse of fvs_qwen_dam_gather_multi's bank tiers: x[plan[i]] = x_rows[i]
 * and, when merged_rows is given, merged[plan[i]] = merged_rows[i], into the two-tier bank (device tier frames [0, n_dev),
 * host chunks laid out as above).  A plan entry outside [0, n_frames) writes nothing. */
typedef struct fvs_qwen_scatter_job {
  const int64_t* plan;
  int n;
  int64_t n_frames;
  const void* x_rows;
  const void* merged_rows;
  void* dev_x;
  void* dev_merged;
  int64_t n_dev;
  void* const* host_chunks;  /* DEVICE table */
  int chunk_frames;
  int64_t x_frame_elems;
  int64_t merged_frame_elems;
} fvs_qwen_scatter_job;
int fvs_qwen_bank_scatter_multi(const fvs_qwen_scatter_job* jobs, int n_jobs, int dtype, fvs_stream_t stream);

/* 8-bit pixel codes (DESIGN.md §3.20): a stream fed uint8 frames keeps each full-resolution pixel row as the bytes u of
 * FVS_PRE_QWEN_CODES, which the tower's input row dtype(table[c][u]) is a function of (c = column / 392, table the
 * pre-processor's float32 [3, 256]).  Decode rounds to nearest even, as torch's fp32 -> bf16 / f16 cast does, so a
 * decoded row equals the cast of the FVS_PRE_QWEN row bit for bit.
 *
 * fvs_qwen_pixel_decode: out[r, k] = dtype(table[k / 392][codes[r, k]]) for codes uint8 [rows, 1176] (8-byte aligned),
 * table device float32 [3, 256], out f16 / bf16 [rows, 1176] (16-byte aligned).  One launch, no synchronisation. */
int fvs_qwen_pixel_decode(const uint8_t* codes, int64_t rows, const float* table, int dtype, void* out,
                          fvs_stream_t stream);
/* *dev_out = the device address of pinned host memory `host` (cudaHostGetDevicePointer); FVS_EINVAL if it is not pinned */
int fvs_host_device_ptr(const void* host, void** dev_out);

/* ---- publication of the Qwen2-VL streaming memory for readers in other processes / on other GPUs ----------------------
 * One device allocation (so one CUDA IPC handle) of fvs_qwen_pub_layout(...) bytes:
 *   header        8 x uint64 {seq, epoch, clips, n_frames, n_tem, n_spa, rows, grid}: seq is odd while a publish is writing
 *                 and only ever grows; grid packs (h, w, hs, ws) as 16-bit fields, h in the low bits;
 *   tem_timestamp fp32 [tem_len] at layout[1];
 *   spa_positions int64 [spa_len] at layout[2];
 *   video_embeds  16-bit [rows_cap, dim] at layout[3]: DAM rows (n_spa * h * w / 4) then CSM rows (n_tem * hs * ws / 4).
 * rows_cap = spa_len * h * w / 4 + tem_len * hs * ws / 4 (the memory at its fullest for this grid). */
/* layout_out int64[5] = {rows_cap, tem_timestamp offset, spa_positions offset, video_embeds offset, total bytes} */
int fvs_qwen_pub_layout(int tem_len, int spa_len, int h, int w, int hs, int ws, int dim, int64_t* layout_out);
/* One launch on `stream`: seq odd, copy the clip's n_tem timestamps, n_spa positions and `rows` embedding rows into the
 * publication, a grid-wide barrier, the counters, seq even.  rows must equal n_spa * h * w / 4 + n_tem * hs * ws / 4. */
int fvs_qwen_publish(void* pub, size_t pub_bytes, int tem_len, int spa_len, int64_t rows_cap, int dim,
                     const void* video_embeds, int64_t rows, const float* tem_timestamp, int n_tem,
                     const int64_t* spa_positions, int n_spa, int h, int w, int hs, int ws, uint64_t epoch, uint64_t clips,
                     int64_t n_frames, fvs_stream_t stream);
/* Consistent copy of a (possibly IPC-mapped or peer) publication into the caller's buffers on the current device:
 * embeds_out [out_rows >= rows_cap, dim], ts_out fp32 [ts_cap >= tem_len], pos_out int64 [pos_cap >= spa_len].
 * status (device uint64[9]) = {seq before, seq after, epoch, clips, n_frames, n_tem, n_spa, rows, grid}; the copy is valid
 * iff status[0] == status[1] and even.  Counts read from a torn header are clamped to the capacities, so nothing outside
 * the publication or the outputs is touched.  A publication on another device needs peer access: it is enabled once per
 * device pair; a pair that cannot peer is refused (FVS_EINVAL). */
int fvs_qwen_snapshot(const void* pub, size_t pub_bytes, int tem_len, int spa_len, int64_t rows_cap, int dim,
                      void* embeds_out, int64_t out_rows, float* ts_out, int64_t ts_cap, int64_t* pos_out, int64_t pos_cap,
                      uint64_t* status, fvs_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Frame pre-processing: decoded uint8 RGB frames [T, H, W, 3] -> the pixels the vision towers take, bit-identical to
 * the reference's CPU processors: LLaVA's CLIPImageProcessor.preprocess(clip)['pixel_values'].half()
 * (Flash-VStream-LLaVA/flash_vstream/serve/cli_video_stream.py:186) and Qwen2-VL's
 * FlashVStreamQwen2VLImageProcessor._preprocess (Flash-VStream-Qwen/models/vstream_qwen2vl_processor.py:38-157, called
 * from cli_server_2gpu.py:214-219).  The resize is Pillow's fixed-point BICUBIC resample (transformers'
 * image_transforms.resize); rescale + normalize come in as a float32 [3, 256] table, one value per channel and byte.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct fvs_resample_axis {
  int in_size, out_size;        /* source length -> resized length */
  int first, count;             /* the window of the resized axis that is produced: [first, first + count) */
  int taps;                     /* coefficients per output: 2 * ceil(2 * max(in_size / out_size, 1)) + 1 */
  int span_first, span_count;   /* the source indices the window reads */
  const int32_t* bounds;        /* device int32 [count, 2] = {first source index, taps used}, 8-byte aligned */
  const int32_t* coeffs;        /* device int32 [count, taps], 22 fractional bits */
} fvs_resample_axis;
enum { FVS_PRE_CLIP = 0, FVS_PRE_QWEN = 1, FVS_PRE_QWEN_CODES = 2, FVS_PRE_RGB8 = 3 };

/* Host: PIL's per-axis plan (precompute_coeffs + normalize_coeffs_8bpc, in double, in PIL's order, no FMA contraction)
 * for the window [first, first + count) of in_size -> out_size.  Fills every field of *axis_h but bounds / coeffs, which
 * are left as they were (the caller points them at its device copies).  bounds_h [count, 2] and coeffs_h [count, taps]
 * are filled when given (both or neither): call once without them to learn `taps`. */
int fvs_resample_plan(int in_size, int out_size, int first, int count, fvs_resample_axis* axis_h, int32_t* bounds_h,
                      int32_t* coeffs_h);
/* uint8 workspace fvs_preprocess needs for `frames` frames: frames * 3 * y.span_count * x.count (0 on bad arguments) */
size_t fvs_preprocess_workspace_bytes(const fvs_resample_axis* x_h, const fvs_resample_axis* y_h, int frames);
/* Two launches on `stream`, no allocation, no synchronisation.  frames: device uint8 [T, H, W, C = 3]; x_h / y_h: host
 * structs of fvs_resample_plan with device tables; table: device float32 [3, 256].
 *   FVS_PRE_CLIP: out f16 [T, 3, y.count, x.count] (the resize with the center crop folded into the windows);
 *   FVS_PRE_QWEN: out fp32 pixel_values_videos [max(T, 2) / 2 * gh * gw, 1176] with gh = y.out_size / 14,
 *                 gw = x.out_size / 14 — the patchify of vstream_qwen2vl_processor.py:141-155; a one-frame clip fills both
 *                 temporal slots (:136-137).  The windows must be whole, T 1 or even, and both sizes multiples of 28 * pool.
 *   FVS_PRE_QWEN_CODES: out uint8 [max(T, 2) / 2 * gh * gw, 1176], FVS_PRE_QWEN's rows and columns holding the resampled
 *                 byte u itself instead of table[c][u], c = column / 392 (DESIGN.md §3.20); the same rules, the same plan.
 *   FVS_PRE_RGB8: out uint8 [T, y.count, x.count, 3], the resized 8-bit image itself (np.asarray of the PIL image that
 *                 Image.resize returns); the table is not read.
 * FVS_EINVAL, with nothing launched, on null pointers, C != 3, an empty input, a plan that does not match the frames or
 * fvs_resample_plan, a window outside the resized image, a workspace below fvs_preprocess_workspace_bytes, or a Qwen2-VL
 * call breaking the rules above. */
int fvs_preprocess(const uint8_t* frames, int T, int H, int W, int C, const fvs_resample_axis* x_h,
                   const fvs_resample_axis* y_h, const float* table, int layout, int pool, void* out, void* workspace,
                   size_t workspace_bytes, fvs_stream_t stream);
/* Many clips, one configuration (table, layout, pool), one contiguous output.  Job i is clip i with its own frames, size
 * and axis plans (host structs of fvs_resample_plan with device tables).  Each job writes at its own offset: the outputs
 * of the jobs lie back to back in job order (CLIP: f16 [sum T, 3, y.count, x.count] when every job has the same window;
 * Qwen2-VL: fp32 rows [sum t * gh * gw, 1176]), and each takes its own slice of one workspace.  Every job's bits equal
 * fvs_preprocess on that clip alone (it is the one-job case of the same code).  One launch pair per 32 jobs: a flat grid
 * whose blocks find their job in a block-offset table passed as a kernel parameter.  Every job is checked as
 * fvs_preprocess checks its clip before anything is launched; FVS_EINVAL names the first bad job.
 * A job whose x2 / y2 are set (out_size != 0) has two stages, the chain of Qwen2-VL's evaluation drivers
 * (qwen_vl_utils fetch_image's Pillow resize, then the image processor's, DESIGN.md §3.11): x / y resize the frames to
 * an 8-bit RGB image [T, y.count, x.count, 3] kept in the job's workspace, exactly the bytes FVS_PRE_RGB8 writes, and
 * x2 / y2 (planned for x.count -> x2.out_size, y.count -> y2.out_size) resize that image into `layout`.  A group of 32
 * jobs holding a two-stage job takes a second launch pair, ahead of its own, for the first stages.  With x2 / y2 zeroed
 * a job is the single-stage job it always was. */
typedef struct fvs_preprocess_job {
  const uint8_t* frames;        /* device uint8 [T, H, W, C = 3] */
  int T, H, W, C;
  fvs_resample_axis x, y;
  fvs_resample_axis x2, y2;     /* second stage, or all zero */
} fvs_preprocess_job;
/* Host plan of a job table (pure host arithmetic, validates like fvs_preprocess_multi, no CUDA call): plan_h [n_jobs, 4] =
 * {first block of the job in its rows launch, in its cols launch, output elements before it, workspace bytes before it};
 * an element is 2 bytes (CLIP), 4 (Qwen2-VL) or 1 (Qwen2-VL codes, RGB8), and the codes layout plans as FVS_PRE_QWEN
 * does; the block offsets are those of the job's last stage.  totals_h [2] = {output elements, workspace bytes}; a
 * two-stage job's workspace holds its first-stage image after the scratch of its passes.  Returns the number of groups
 * of up to 32 jobs (>= 1) or a negative error. */
int fvs_preprocess_plan(const fvs_preprocess_job* jobs_h, int n_jobs, int layout, int pool, int64_t* plan_h,
                        int64_t* totals_h);
/* workspace: at least totals_h[1] bytes of fvs_preprocess_plan; out: totals_h[0] elements. */
int fvs_preprocess_multi(const fvs_preprocess_job* jobs_h, int n_jobs, const float* table, int layout, int pool, void* out,
                         void* workspace, size_t workspace_bytes, fvs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* FVS_B200_H */
