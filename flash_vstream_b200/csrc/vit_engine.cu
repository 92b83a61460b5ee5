// vit_engine.cu — fvs_vit_*: ViT-L/14 frame encoder (CLIP vision tower) assembled from the sm_90a kernels.
//
// Behavioural spec = CLIPVisionTower.forward + feature_select
// (Flash-VStream-LLaVA/flash_vstream/model/multimodal_encoder/clip_encoder.py:31-53) over HF CLIPVisionModel:
//   patch conv (no bias) -> [CLS | patches] + position embedding -> pre_layrnorm ->
//   layers_run x { LN -> QKV(+bias) -> MHA(16x64, scale 1/8) -> out-proj(+bias) + residual ->
//                  LN -> fc1(+bias) -> quick_gelu -> fc2(+bias) + residual }
//   -> hidden_states[select_layer][:, 1:]            (select_layer = -2 => layers_run = 23 of 24; the
//      reference executes and discards the 24th layer and post_layernorm — we do not run them).
// Precision: weights/activations 16-bit, fp32 accumulation, and an FP32 RESIDUAL STREAM (x) — with an f16 stream the
// output sits 1.3e-3 (rel. Frobenius) from the fp32 evaluation of the same weights, with fp32 it sits at 4.7e-4
// (measured with oracle.vit_forward(round_dtype=f16), see DESIGN.md).
// Launch plan per micro-batch (M = frames * tokens rows):
//   im2col -> linear(ROWTABLE: + pos/cls table) -> layernorm(pre) ->
//   23 x [layernorm, linear(BIAS) qkv, attention, linear(BIAS_RESIDUAL_F32: x += out-proj),
//         layernorm, linear(BIAS_QUICKGELU), linear(BIAS_RESIDUAL_F32: x += fc2)] -> drop_cls / pooled tail (x rounded once)
// with everything between im2col and the tail run as two concurrent half-batches from kSplitMinRows rows on (stack_launches).
// The residual adds live in the out-proj / fc2 epilogue as TMA reduce-add stores (the L2 performs x += acc + bias), so
// the fp32 stream never enters an SM on that side and a LayerNorm only reads x and writes y: 6 B/element per LayerNorm
// instead of 12.  Round 1's row-per-thread version of the epilogue (uncoalesced fp32 loads and stores) made out-proj
// run at 20 % tensor-pipe utilisation and was replaced by a 16-bit delta + add-LayerNorm; a TMA-staged in-place ring
// (residual chunk loaded into the staging buffer, updated, stored back) worked but put 25 % more inbound bytes on
// out-proj's L2->SM path (measured 41 us vs 40 us for out-proj and 102 us vs 95 us for fc2 with the reduce form;
// DESIGN.md §3.1).  Keeping x in the persisting part of the L2 (access-policy window, micro-batches of 16 or 32 frames)
// changed nothing measurable.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdlib>
#include <vector>

#include "fvs_common.h"
#include "fvs_kernels.h"

namespace fvs {
// patch weight [hidden, kreal] -> [hidden, kpad] zero padded; table[t] = pos[t] + (t == 0 ? cls : 0)
__global__ void vit_prepare_kernel(const uint16_t* __restrict__ patch_w, const uint16_t* __restrict__ cls,
                                   const uint16_t* __restrict__ pos, uint16_t* __restrict__ patch_w_pad,
                                   uint16_t* __restrict__ table, int hidden, int kreal, int kpad, int tokens, int bf16) {
  const size_t n1 = size_t(hidden) * kpad, n2 = size_t(tokens) * hidden;
  for (size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x; i < n1 + n2; i += size_t(gridDim.x) * blockDim.x) {
    if (i < n1) {
      const int r = int(i / kpad), c = int(i % kpad);
      patch_w_pad[i] = c < kreal ? patch_w[size_t(r) * kreal + c] : uint16_t(0);
    } else {
      const size_t j = i - n1;
      const int t = int(j / hidden), d = int(j % hidden);
      if (t != 0) {
        table[j] = pos[j];
      } else if (bf16) {
        const float a = __uint_as_float(uint32_t(pos[j]) << 16), b = __uint_as_float(uint32_t(cls[d]) << 16);
        const __nv_bfloat16 h = __float2bfloat16_rn(a + b);
        table[j] = *reinterpret_cast<const uint16_t*>(&h);
      } else {
        const float a = __half2float(__ushort_as_half(pos[j])), b = __half2float(__ushort_as_half(cls[d]));
        table[j] = __half_as_ushort(__float2half_rn(a + b));
      }
    }
  }
}

}  // namespace fvs

// Execution plan of one micro-batch shape on one workspace: every tensor map of the layer stack is encoded ONCE (279
// cuTensorMapEncodeTiled calls per micro-batch otherwise), and from the second use on the whole layer stack — patch GEMM to
// the last fc2, 209 launches for 23 layers, twice that as two half-batch branches — replays as ONE CUDA graph (captured from
// the very launches it replaces, PDL edges and the branches' fork and join included).  Only im2col (reads the caller's
// pixels) and the tail (writes the caller's output) stay outside, so the graph depends on nothing but the workspace and
// the weights.  What this buys is host independence: a step is 3 driver
// calls instead of ~500, which is what keeps 8 ranks on one host from starving their GPUs (SCALE_r01: 0.51 at N=8).
struct VitPlan {
  const void* ws_base = nullptr;
  int nf = 0;
  std::vector<CUtensorMap> maps;      // in consumption order (see MapCursor)
  fvs::AttnMaps attn[2];              // one per half-batch (only [0] without the split)
  bool maps_ready = false;
  cudaGraphExec_t exec = nullptr;
  cudaGraphExec_t exec_prof = nullptr;   // same launches with an external event-record node before and after every tensor-core kernel
  fvs::ProfGraphRecs* prof_recs = nullptr;   // (heap: the profiler keeps a pointer to it)
  int kernels = 0;                    // kernel launches one replay stands for (fvs_launch_count bookkeeping)
  int uses = 0;
  uint64_t stamp = 0;                 // LRU
};

struct fvs_vit {
  fvs_vit_config cfg;
  fvs_vit_weights w;
  std::vector<fvs_vit_layer_weights> layers;
  int grid = 0, tokens = 0, kreal = 0, kpad = 0;
  void* patch_w_pad = nullptr;  // [hidden, kpad]
  void* table = nullptr;        // [tokens, hidden]
  std::vector<VitPlan> plans;
  uint64_t clock = 0;
  cudaStream_t cap_stream = nullptr;   // capture happens here: the caller's stream may be the legacy default stream, which cannot capture
  cudaStream_t side = nullptr;         // the second half-batch's stream (see stack_launches)
  cudaEvent_t fork = nullptr, join = nullptr;
};

namespace {
size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

struct Workspace {
  uint8_t *patches, *x, *y, *qkv, *ctx, *act;
  size_t total;
};
Workspace carve(const fvs_vit* h, int frames, void* base) {
  const size_t M = size_t(frames) * h->tokens, H = h->cfg.hidden;
  Workspace ws;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? static_cast<uint8_t*>(base) + off : nullptr;
    off += align256(bytes);
    return p;
  };
  ws.patches = take(M * h->kpad * 2);
  ws.x = take(M * H * 4);  // fp32 residual stream
  ws.y = take(M * H * 2);
  ws.qkv = take(M * 3 * H * 2);
  ws.ctx = take(M * H * 2);
  ws.act = take(M * size_t(h->cfg.mlp) * 2);
  ws.total = off;
  return ws;
}

// FVS_VIT_GRAPH=0 disables the graph replay (A/B switch; the launches are identical either way)
bool graph_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("FVS_VIT_GRAPH");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}

void drop_plan(VitPlan& p) {
  if (p.exec) cudaGraphExecDestroy(p.exec);
  if (p.exec_prof) cudaGraphExecDestroy(p.exec_prof);
  if (p.prof_recs) { fvs::prof_graph_forget(p.prof_recs); delete p.prof_recs; }
  p.exec = p.exec_prof = nullptr;
  p.prof_recs = nullptr;
}

VitPlan& find_plan(fvs_vit* h, const void* ws_base, int nf) {
  ++h->clock;
  for (auto& p : h->plans)
    if (p.ws_base == ws_base && p.nf == nf) { p.stamp = h->clock; return p; }
  if (h->plans.size() >= 8) {   // evict the least recently used plan
    size_t lru = 0;
    for (size_t i = 1; i < h->plans.size(); ++i)
      if (h->plans[i].stamp < h->plans[lru].stamp) lru = i;
    drop_plan(h->plans[lru]);
    h->plans.erase(h->plans.begin() + lru);
  }
  h->plans.emplace_back();
  VitPlan& p = h->plans.back();
  p.ws_base = ws_base;
  p.nf = nf;
  p.stamp = h->clock;
  return p;
}

// hands out the plan's tensor maps in consumption order; the first pass encodes them, later passes reuse them
struct MapCursor {
  VitPlan& p;
  size_t i = 0;
  int linear(const CUtensorMap*& ta, const CUtensorMap*& tb, const CUtensorMap*& to, const void* A, const void* W, void* out,
             int M, int N, int K, bool out_f32 = false) {
    if (!p.maps_ready) {
      p.maps.resize(p.maps.size() + 3);
      int r = fvs::linear_make_maps(&p.maps[i], &p.maps[i + 1], &p.maps[i + 2], A, W, out, M, N, K, K, N, out_f32);
      if (r) return r;
    }
    ta = &p.maps[i]; tb = &p.maps[i + 1]; to = &p.maps[i + 2];
    i += 3;
    return FVS_OK;
  }
};

// Rows per micro-batch (frames x tokens) from which the layer stack runs as two concurrent half-batches
// (stack_launches).  On an H100 the split is faster at every ViT-L/14-336 micro-batch measured, from 2 frames (2 x 577
// rows) to 32 (DESIGN.md §4); smaller micro-batches (small towers) were not measured and stay whole.
constexpr int kSplitMinRows = 2 * 577;

// frames [f0, ..) of a micro-batch's workspace: the same buffers from the frame's first row on
Workspace frames_from(const fvs_vit* h, const Workspace& ws, int f0) {
  const size_t rows = size_t(f0) * h->tokens, H = h->cfg.hidden;
  Workspace s = ws;
  s.patches += rows * h->kpad * 2;
  s.x += rows * H * 4;
  s.y += rows * H * 2;
  s.qkv += rows * 3 * H * 2;
  s.ctx += rows * H * 2;
  s.act += rows * size_t(h->cfg.mlp) * 2;
  return s;
}

// one half-batch of the layer stack: its frames' rows of the workspace, its stream, its attention maps
struct Branch {
  Workspace ws;
  int nf;
  fvs::AttnMaps* attn;
  cudaStream_t stream;
};

// stage -1: patch GEMM (+pos/CLS table) -> pre_layrnorm; stage l >= 0: layer l
int stage_launches(fvs_vit* h, VitPlan& p, MapCursor& mc, const Branch& b, int l, bool pdl) {
  using namespace fvs;
  const fvs_vit_config& c = h->cfg;
  const int H = c.hidden, T = h->tokens, dt = c.dtype, M = b.nf * T;
  const Workspace& ws = b.ws;
  cudaStream_t stream = b.stream;
  const CUtensorMap *ta, *tb, *to;
  int r;
  if (l < 0) {
    if ((r = mc.linear(ta, tb, to, ws.patches, h->patch_w_pad, ws.y, M, H, h->kpad))) return r;
    if ((r = linear_launch(*ta, *tb, *to, nullptr, h->table, M, H, h->kpad, H, FVS_EPI_ROWTABLE, T, dt, stream, pdl))) return r;
    if ((r = layernorm_launch(ws.y, h->w.pre_ln_w, h->w.pre_ln_b, ws.x, M, H, c.ln_eps, dt, false, true, nullptr, stream, pdl)))
      return r;
    if (!p.maps_ready && (r = attention_make_maps(b.attn, ws.qkv, ws.ctx, b.nf, T, c.heads))) return r;
    return FVS_OK;
  }
  const float scale = 0.125f;  // head_dim^-0.5
  const fvs_vit_layer_weights& L = h->layers[l];
  if ((r = layernorm_launch(ws.x, L.ln1_w, L.ln1_b, ws.y, M, H, c.ln_eps, dt, true, false, nullptr, stream, pdl))) return r;
  if ((r = mc.linear(ta, tb, to, ws.y, L.qkv_w, ws.qkv, M, 3 * H, H))) return r;
  if ((r = linear_launch(*ta, *tb, *to, L.qkv_b, nullptr, M, 3 * H, H, 3 * H, FVS_EPI_BIAS, 0, dt, stream, pdl))) return r;
  if ((r = attention_launch(*b.attn, b.nf, T, c.heads, scale, dt, stream, 64, pdl))) return r;
  // out-proj and fc2 add straight into the fp32 residual stream (TMA-staged in the GEMM epilogue), so a LayerNorm
  // only reads x and writes y
  if ((r = mc.linear(ta, tb, to, ws.ctx, L.o_w, ws.x, M, H, H, true))) return r;
  if ((r = linear_launch(*ta, *tb, *to, L.o_b, ws.x, M, H, H, H, FVS_EPI_BIAS_RESIDUAL_F32, 0, dt, stream, pdl))) return r;
  if ((r = layernorm_launch(ws.x, L.ln2_w, L.ln2_b, ws.y, M, H, c.ln_eps, dt, true, false, nullptr, stream, pdl))) return r;
  if ((r = mc.linear(ta, tb, to, ws.y, L.fc1_w, ws.act, M, c.mlp, H))) return r;
  if ((r = linear_launch(*ta, *tb, *to, L.fc1_b, nullptr, M, c.mlp, H, c.mlp, FVS_EPI_BIAS_QUICKGELU, 0, dt, stream, pdl)))
    return r;
  if ((r = mc.linear(ta, tb, to, ws.act, L.fc2_w, ws.x, M, H, c.mlp, true))) return r;
  if ((r = linear_launch(*ta, *tb, *to, L.fc2_b, ws.x, M, H, c.mlp, H, FVS_EPI_BIAS_RESIDUAL_F32, 0, dt, stream, pdl))) return r;
  return FVS_OK;
}

// the layer stack of one micro-batch: patch GEMM (+pos/CLS table) -> pre_layrnorm -> layers_run x [...] (everything
// between im2col and the tail); reads ws.patches, leaves the residual stream (fp32) in ws.x.
// From kSplitMinRows rows on, frames [0, nf/2) and [nf/2, nf) run the whole stack as two independent chains, the second on
// h->side, forked from and joined back into `stream` by events (captured, the graph has two parallel branches).  While
// one half's GEMM drains its last wave or runs a LayerNorm, the other half's kernels take the idle SMs.  Every kernel is
// row-wise or frame-wise and each output element's K sum runs in the same order whatever M is, so the split leaves every
// bit as it was; the halves meet at a frame boundary, so the ROWTABLE row % tokens still holds, and each half's tensor
// maps end at its last row, so neither half reads or writes the other's rows.
int stack_launches(fvs_vit* h, VitPlan& p, const Workspace& ws, int nf, cudaStream_t stream) {
  const bool split = nf >= 2 && nf * h->tokens >= kSplitMinRows;
  const int n0 = split ? nf / 2 : nf;
  Branch br[2] = {{ws, n0, &p.attn[0], stream}, {frames_from(h, ws, n0), nf - n0, &p.attn[1], h->side}};
  const int nb = split ? 2 : 1;
  // Split, the launches go without PDL: every kernel triggers its dependents on entry, so a same-half dependent would
  // park its CTAs on exactly the SMs the other half should fill (measured slower at every micro-batch, DESIGN.md §4).
  const bool pdl = !split;
  if (split) {
    FVS_CUDA_OK(cudaEventRecord(h->fork, stream));
    FVS_CUDA_OK(cudaStreamWaitEvent(h->side, h->fork, 0));
  }
  MapCursor mc{p};
  int r = FVS_OK;
  for (int l = -1; l < h->cfg.layers_run && !r; ++l)   // issued layer by layer, alternating halves (matters eagerly only)
    for (int b = 0; b < nb && !r; ++b) r = stage_launches(h, p, mc, br[b], l, pdl);
  if (split) {   // joined even after a failed launch, so no work is left unordered behind the caller's stream
    FVS_CUDA_OK(cudaEventRecord(h->join, h->side));
    FVS_CUDA_OK(cudaStreamWaitEvent(stream, h->join, 0));
  }
  if (r) return r;
  p.maps_ready = true;
  return FVS_OK;
}

int run_stack(fvs_vit* h, VitPlan& p, const Workspace& ws, int nf, cudaStream_t stream) {
  using namespace fvs;
  const bool prof = prof_active();   // bracket the tensor-core launches with events: a second graph with event-record nodes
  bool graph = graph_enabled() && p.uses > 0;
  if (graph) {   // inside somebody else's capture our launches simply become part of their graph
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(stream, &st) != cudaSuccess || st != cudaStreamCaptureStatusNone) graph = false;
  }
  ++p.uses;
  if (!graph) return stack_launches(h, p, ws, nf, stream);
  cudaGraphExec_t& exec = prof ? p.exec_prof : p.exec;
  if (!exec) {
    if (!h->cap_stream) FVS_CUDA_OK(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
    if (prof && !p.prof_recs) p.prof_recs = new ProfGraphRecs();
    const uint64_t before = g_launches.load();
    FVS_CUDA_OK(cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal));
    prof_capture_sink(prof ? p.prof_recs : nullptr);
    const int r = stack_launches(h, p, ws, nf, h->cap_stream);
    prof_capture_sink(nullptr);
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(h->cap_stream, &g);
    p.kernels = int(g_launches.load() - before);
    g_launches.fetch_sub(uint64_t(p.kernels));      // counted while capturing, not launched
    if (r) { if (g) cudaGraphDestroy(g); return r; }
    if (e != cudaSuccess || !g) return set_error(FVS_ECUDA, "fvs_vit: stream capture failed: %s", cudaGetErrorString(e));
    const cudaError_t ei = cudaGraphInstantiate(&exec, g, 0);
    cudaGraphDestroy(g);
    if (ei != cudaSuccess) { exec = nullptr; return set_error(FVS_ECUDA, "fvs_vit: cudaGraphInstantiate: %s", cudaGetErrorString(ei)); }
  }
  FVS_CUDA_OK(cudaGraphLaunch(exec, stream));
  if (prof) prof_graph_replayed(p.prof_recs);
  g_launches.fetch_add(uint64_t(p.kernels));
  return FVS_OK;
}
}  // namespace

extern "C" {

int fvs_vit_create(fvs_vit_t* out, const fvs_vit_config* cfg, const fvs_vit_weights* w, fvs_stream_t stream_) {
  using namespace fvs;
  FVS_REQUIRE(out && cfg && w && w->layers_h, "fvs_vit_create: null argument");
  FVS_REQUIRE(cfg->patch_size > 0 && cfg->image_size % cfg->patch_size == 0, "fvs_vit_create: image %d / patch %d",
              cfg->image_size, cfg->patch_size);
  FVS_REQUIRE(cfg->heads > 0 && cfg->hidden == cfg->heads * 64, "fvs_vit_create: head_dim must be 64 (hidden %d, heads %d)",
              cfg->hidden, cfg->heads);
  FVS_REQUIRE(cfg->hidden % 256 == 0 && cfg->mlp % 64 == 0, "fvs_vit_create: hidden %% 256 and mlp %% 64 required");
  FVS_REQUIRE(cfg->layers_run >= 0 && cfg->layers_run <= 256, "fvs_vit_create: bad layers_run");
  FVS_REQUIRE(cfg->dtype == FVS_F16 || cfg->dtype == FVS_BF16, "fvs_vit_create: dtype must be f16 or bf16");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  fvs_vit* h = new fvs_vit();
  h->cfg = *cfg;
  h->w = *w;
  h->layers.assign(w->layers_h, w->layers_h + cfg->layers_run);
  h->w.layers_h = nullptr;
  h->grid = cfg->image_size / cfg->patch_size;
  h->tokens = h->grid * h->grid + 1;
  h->kreal = 3 * cfg->patch_size * cfg->patch_size;
  h->kpad = (h->kreal + 63) / 64 * 64;
  cudaError_t e = cudaMalloc(&h->patch_w_pad, size_t(cfg->hidden) * h->kpad * 2);
  if (e == cudaSuccess) e = cudaMalloc(&h->table, size_t(h->tokens) * cfg->hidden * 2);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->join, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    fvs_vit_destroy(h);
    return set_error(FVS_ECUDA, "fvs_vit_create: %s", cudaGetErrorString(e));
  }
  vit_prepare_kernel<<<256, 256, 0, stream>>>((const uint16_t*)w->patch_w, (const uint16_t*)w->class_emb,
                                              (const uint16_t*)w->pos_emb, (uint16_t*)h->patch_w_pad,
                                              (uint16_t*)h->table, cfg->hidden, h->kreal, h->kpad, h->tokens,
                                              cfg->dtype == FVS_BF16);
  FVS_COUNT_LAUNCH();
  e = cudaGetLastError();
  if (e != cudaSuccess) {
    fvs_vit_destroy(h);
    return set_error(FVS_ECUDA, "fvs_vit_create: prepare kernel: %s", cudaGetErrorString(e));
  }
  *out = h;
  return FVS_OK;
}

int fvs_vit_destroy(fvs_vit_t h) {
  if (!h) return FVS_OK;
  if (h->patch_w_pad) cudaFree(h->patch_w_pad);
  if (h->table) cudaFree(h->table);
  for (auto& p : h->plans) drop_plan(p);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  if (h->side) cudaStreamDestroy(h->side);
  if (h->fork) cudaEventDestroy(h->fork);
  if (h->join) cudaEventDestroy(h->join);
  delete h;
  return FVS_OK;
}

size_t fvs_vit_workspace_bytes(fvs_vit_t h, int max_frames) {
  if (!h || max_frames <= 0) return 0;
  return carve(h, max_frames, nullptr).total;
}

// tail selector of encode_impl
struct VitTail {
  void* out = nullptr;                                   // full feature map [frames, tokens(-1), hidden] ...
  const fvs::Pool3Dst* pool = nullptr;                   // ... or the three pooled STAR levels of every frame
  int n_pool = 0, a = 0, b = 0;
};

static int encode_impl(fvs_vit_t h, const void* pixels, const VitTail& tail, int frames, void* workspace,
                       size_t workspace_bytes, cudaStream_t stream, const char* who) {
  using namespace fvs;
  const fvs_vit_config& c = h->cfg;
  const int H = c.hidden, T = h->tokens;
  // largest micro-batch the caller's workspace can hold
  int mb = frames;
  while (mb > 1 && carve(h, mb, nullptr).total > workspace_bytes) mb = (mb + 1) / 2;
  FVS_REQUIRE(carve(h, mb, nullptr).total <= workspace_bytes,
              "%s: workspace of %zu bytes cannot hold even one frame (%zu needed)", who, workspace_bytes,
              carve(h, 1, nullptr).total);
  const size_t pix_per_frame = size_t(3) * c.image_size * c.image_size;
  const size_t out_per_frame = size_t(T - (c.keep_cls ? 0 : 1)) * H;

  for (int f0 = 0; f0 < frames; f0 += mb) {
    const int nf = (frames - f0 < mb) ? frames - f0 : mb;
    Workspace ws = carve(h, nf, workspace);
    int r;
    if ((r = im2col_launch(static_cast<const uint16_t*>(pixels) + f0 * pix_per_frame, ws.patches, nf, c.image_size,
                           c.patch_size, h->kpad, stream)))
      return r;
    if ((r = run_stack(h, find_plan(h, workspace, nf), ws, nf, stream))) return r;
    if (tail.out) {
      if ((r = drop_cls_launch(ws.x, nullptr, static_cast<uint16_t*>(tail.out) + f0 * out_per_frame,
                               nf, T, H, c.dtype, stream, c.keep_cls != 0)))
        return r;
    } else {
      if ((r = pool3_launch(ws.x, true, tail.pool, tail.n_pool, f0, nf, h->grid, tail.a, tail.b, H, stream))) return r;
    }
  }
  return FVS_OK;
}

}  // extern "C"

namespace fvs {
int vit_encode_pool3(fvs_vit_t h, const void* pixels, const Pool3Dst* dst, int n_dst, int a, int b, void* workspace,
                     size_t workspace_bytes, cudaStream_t stream) {
  FVS_REQUIRE(h && pixels && dst && n_dst > 0 && workspace, "fvs_vit_encode_pool3: null argument");
  FVS_REQUIRE(h->cfg.dtype == FVS_F16 && !h->cfg.keep_cls,
              "fvs_vit_encode_pool3: needs an f16 tower with select_feature 'patch' (the reference casts to float16 before pooling, vstream_arch.py:649)");
  int frames = 0;
  for (int i = 0; i < n_dst; ++i) {
    FVS_REQUIRE(dst[i].a && dst[i].frames > 0, "fvs_vit_encode_pool3: destination %d has no output or no frames", i);
    FVS_REQUIRE(a > 0 && h->grid % a == 0 && a * a <= 64 && (dst[i].b == nullptr || (b > 0 && a % b == 0)),
                "fvs_vit_encode_pool3: bad pooling sizes grid=%d a=%d b=%d", h->grid, a, b);
    frames += dst[i].frames;
  }
  VitTail tail;
  tail.pool = dst; tail.n_pool = n_dst;
  tail.a = a; tail.b = b;
  return encode_impl(h, pixels, tail, frames, workspace, workspace_bytes, stream, "fvs_vit_encode_pool3");
}
}  // namespace fvs

extern "C" {

int fvs_vit_encode(fvs_vit_t h, const void* pixels, void* out, int frames, void* workspace, size_t workspace_bytes,
                   fvs_stream_t stream_) {
  using namespace fvs;
  FVS_REQUIRE(h && pixels && out && workspace, "fvs_vit_encode: null argument");
  FVS_REQUIRE(frames > 0, "fvs_vit_encode: frames must be > 0");
  VitTail tail;
  tail.out = out;
  return encode_impl(h, pixels, tail, frames, workspace, workspace_bytes, static_cast<cudaStream_t>(stream_), "fvs_vit_encode");
}

int fvs_vit_encode_pool3(fvs_vit_t h, const void* pixels, void* out_a, void* out_b, void* out_c, int frames, int a, int b,
                         void* workspace, size_t workspace_bytes, fvs_stream_t stream_) {
  using namespace fvs;
  FVS_REQUIRE(out_a && frames > 0, "fvs_vit_encode_pool3: null output or frames <= 0");
  const Pool3Dst dst = {out_a, out_b, out_c, frames};
  return vit_encode_pool3(h, pixels, &dst, 1, a, b, workspace, workspace_bytes, static_cast<cudaStream_t>(stream_));
}

}  // extern "C"
