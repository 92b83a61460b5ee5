"""GPU: every stage of one Qwen2-VL and one CLIP vision block bounded element by element, read back from the tower's own
workspace.  fvs_qwen_vit_encode / fvs_vit_encode take a caller-owned workspace with a fixed layout (qcarve in
qwen_vit_engine.cu, carve in vit_engine.cu); after a depth-1 encode it still holds pos, the post-rotary qkv, the attention
ctx, the LN2 output y, the quick-GELU act, the patch embedding delta and the final fp32 x.  The two stage inputs the call
overwrites come from companion towers with the same weights and one knob neutralised, so that every stage before the knob
produces the same bits:
  inv_freq = 0         every angle is 0, cos = 1 and sin = 0: fl(fl(x * 1) + fl(-y * 0)) = x, so the companion's qkv is
                       the pre-rotary qkv;
  fc2_w = fc2_b = 0    the fc2 reduce-add adds +0, so the companion's final x is x after the attention half (x1).
Both are exact up to the sign of a zero.  Where the premise is observable (pos, delta and, for the fc2 companion, qkv,
ctx, y and act) the companion's bits are asserted equal to the main tower's.  The workspace is filled with 0xFF bytes
before every encode (NaN in f16 / bf16 / fp32, -1 as an int32 pos), so an element no kernel wrote fails its check.
Every reference is fp64 from the kernel's own inputs and every bound is the one test_kernel_bounds_gpu.py derives for
the kernel; each check prints its largest err / bound.  Each bound is also shown to reject a deliberately wrong
reference computed on the same GPU outputs: a localised mistake that a tower-level Frobenius norm does not see."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import qwen_vit_inputs as VI
from tests.test_kernel_bounds_gpu import DTYPES, U32, attention_bound, check, half_ulp, layernorm_bound, linear_bound
from tests.test_qwen_vit_gpu_parity import TOL, rel
from tests.test_qwen_vit_grids_host import REAL_GRIDS, ROPE_MUTATIONS, grid_positions, rope_apply, vit_forward

pytestmark = pytest.mark.gpu

HD, HALF, NFREQ = 80, 40, 20
E, HEADS, MLP, PATCH_DIM = 1280, 16, 5120, 1176
QWEN_EPS = float(np.float32(1e-6))
INV_FREQ = 1.0 / (10000.0 ** (torch.arange(0, HALF, 2, dtype=torch.float) / HALF))      # fp32, as the model computes it
COSF_ULP = 2                                      # CUDA Math API: cosf and sinf have a maximum error of 2 ulp


@pytest.fixture(scope="module")
def L():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    return _lib


# ----------------------------------------------------------------------------------------------- workspace layouts
def al256(n):
    return (n + 255) // 256 * 256


def carve(ws, rows, spec):
    """the workspace restated: `spec` lists (name, dtype, columns) in carve order, every piece 256-byte aligned; returns
    {name: [rows, columns] view of ws} (ws None: no views) and the total bytes"""
    off, views = 0, {}
    for name, dt, cols in spec:
        n = rows * cols * dt.itemsize
        if ws is not None:
            views[name] = ws[off:off + n].view(dt).view(rows, cols)
        off += al256(n)
    return views, off


def qwen_spec(dtype):          # qcarve, qwen_vit_engine.cu
    return [("x", torch.float32, E), ("y", dtype, E), ("qkv", dtype, 3 * E), ("ctx", dtype, E), ("act", dtype, MLP),
            ("delta", dtype, E), ("pos", torch.int32, 1)]


CLIP_IMAGE, CLIP_PATCH, CLIP_H, CLIP_MLP = 336, 14, 1024, 4096
CLIP_GRID = CLIP_IMAGE // CLIP_PATCH
CLIP_TOKENS, KREAL = CLIP_GRID ** 2 + 1, 3 * CLIP_PATCH ** 2
KPAD = (KREAL + 63) // 64 * 64
CLIP_EPS = float(np.float32(1e-5))


def clip_spec(dtype):          # carve, vit_engine.cu
    return [("patches", dtype, KPAD), ("x", torch.float32, CLIP_H), ("y", dtype, CLIP_H), ("qkv", dtype, 3 * CLIP_H),
            ("ctx", dtype, CLIP_H), ("act", dtype, CLIP_MLP)]


def filled(nbytes):
    return torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")


def bits(t):
    return t.view({1: torch.int8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def assert_bits(name, got, want):
    assert got.dtype == want.dtype and torch.equal(bits(got), bits(want)), f"{name}: not bit-identical"


# ---------------------------------------------------------------------------------- the permuted qkv / ctx columns
def perm_cols(heads, sections):
    """perm_col of qwen_vit_engine.cu as an index map: perm[n] is the permuted column that holds natural column
    n = sec * heads * 80 + head * 80 + d.  Each head's 80 dims are split into 64 "main" and 16 "extra" columns in two
    separate blocks (every section's main block first, then every section's extra block):
      main[i] = dim i, main[32 + i] = dim 40 + i (i < 32);  extra[i] = dim 32 + i, extra[8 + i] = dim 72 + i (i < 8)"""
    n = torch.arange(sections * heads * HD)
    sec, head, d = n // (heads * HD), (n // HD) % heads, n % HD
    lo, hi = d % HALF, d // HALF
    main = sec * heads * 64 + head * 64 + hi * 32 + lo
    extra = sections * heads * 64 + sec * heads * 16 + head * 16 + hi * 8 + (lo - 32)
    return torch.where(lo < 32, main, extra)


def to_natural(t, heads, sections):
    return t[:, perm_cols(heads, sections).to(t.device)]


def to_permuted(t, heads, sections):
    out = torch.empty_like(t)
    out[:, perm_cols(heads, sections).to(t.device)] = t
    return out


# ------------------------------------------------------------------------------------------------------ the rotary
# qwen_rope_kernel: a = fl(p * inv_freq[j]) (p = hpos for j < 20, wpos for the next 20), c = cosf(a), s = sinf(a), then
# r = fl(fl(x * c) + fl(-x' * s)) with __fmul_rn / __fadd_rn (no FMA) and one rounding to the 16-bit output.  The angle is
# computed exactly as the reference's fp32 outer product computes it, so the reference takes cos and sin of the same fp32 a
# in fp64.  Per element, with e_c = 2 ulp(cos a) <= 2^-22 |cos a| (and e_s likewise):
#   e1 = |x| e_c + u32 |x| (|cos a| + e_c)        fl(x * c)
#   e2 = |x'| e_s + u32 |x'| (|sin a| + e_s)      fl(x' * s)
#   e  = e1 + e2 + u32 (|ref| + e1 + e2)          the fp32 add, then half an ulp of the 16-bit output
def rope_bound(pre, pos, inv_freq, out, rope_mutation=None):
    """pre: the natural pre-rotary q and k [rows, 2, heads, 80] (16-bit), pos [rows] packed (hpos << 16 | wpos), out: the
    rotated q and k in the same layout.  Returns the fp64 reference (with `rope_mutation`, a wrong one: see
    ROPE_MUTATIONS), the element-wise bound of the kernel's arithmetic and its output-rounding part."""
    rows = pre.shape[0]
    p = torch.stack([pos.flatten() >> 16, pos.flatten() & 0xFFFF], -1).float()
    ang = (p[:, :, None] * inv_freq.float().to(p.device)[None, None, :]).reshape(rows, HALF)       # fp32 products
    a = torch.cat([ang, ang], -1).double()[:, None, :]
    cos, sin = a.cos(), a.sin()
    x = pre.double()
    ref_true = torch.stack([rope_apply(x[:, i], cos, sin) for i in range(2)], 1)
    ref = ref_true if rope_mutation is None else \
        torch.stack([rope_apply(x[:, i], cos, sin, rope_mutation) for i in range(2)], 1)
    xa = x.abs()
    pa = torch.cat([xa[..., HALF:], xa[..., :HALF]], -1)                                          # |partner|
    cos, sin = cos[:, None].abs(), sin[:, None].abs()
    e_c = COSF_ULP * 2.0 ** -23 * cos * (1 + 2.0 ** -20) + 2.0 ** -148
    e_s = COSF_ULP * 2.0 ** -23 * sin * (1 + 2.0 ** -20) + 2.0 ** -148
    e1 = xa * e_c + U32 * xa * (cos + e_c)
    e2 = pa * e_s + U32 * pa * (sin + e_s)
    e = e1 + e2 + U32 * (ref_true.abs() + e1 + e2)
    rounding = half_ulp(out)
    return ref, e + rounding, rounding


def packed_positions(grids):
    """pos as qwen_pos_kernel packs it, from grid_positions (pinned to transformers' rot_pos_emb)"""
    hw = torch.cat([grid_positions(h, w).repeat(t, 1) for t, h, w in grids])
    return ((hw[:, 0] << 16) | hw[:, 1]).to(torch.int32)


# --------------------------------------------------------------------------------------------------- Qwen2-VL tower
class QwenTower:
    """a fvs_qwen_vit handle over its own device weights; `encode` fills a fresh workspace with 0xFF, encodes and returns
    (out, {workspace piece: view})"""

    def __init__(self, L, sd, dtype, depth, inv_freq, zero_fc2=False):
        self.L, self.lib, self.dtype = L, L.load(), dtype
        dev = lambda t: t.to(device="cuda", dtype=dtype).contiguous()
        self.keep = [dev(sd["patch_embed.proj.weight"].reshape(E, -1))]
        arr = (L.VitLayerWeights * max(depth, 1))()
        names = dict(ln1_w="norm1.weight", ln1_b="norm1.bias", qkv_w="attn.qkv.weight", qkv_b="attn.qkv.bias",
                     o_w="attn.proj.weight", o_b="attn.proj.bias", ln2_w="norm2.weight", ln2_b="norm2.bias",
                     fc1_w="mlp.fc1.weight", fc1_b="mlp.fc1.bias", fc2_w="mlp.fc2.weight", fc2_b="mlp.fc2.bias")
        for i in range(depth):
            for field, key in names.items():
                t = sd[f"blocks.{i}.{key}"]
                if zero_fc2 and field in ("fc2_w", "fc2_b"):
                    t = torch.zeros_like(t)
                self.keep.append(dev(t))
                setattr(arr[i], field, self.keep[-1].data_ptr())
        cfg = L.QwenVitConfig(E, HEADS, MLP, depth, PATCH_DIM, 1e-6, L.dtype_code(dtype))
        inv = (C.c_float * NFREQ)(*inv_freq.tolist())
        self.h = C.c_void_p()
        L.check(self.lib.fvs_qwen_vit_create(C.byref(self.h), C.byref(cfg), self.keep[0].data_ptr(), arr, inv,
                                             L.cur_stream()), "fvs_qwen_vit_create")
        torch.cuda.synchronize()

    def encode(self, patches, grids):
        rows = patches.shape[0]
        need = self.lib.fvs_qwen_vit_workspace_bytes(self.h, rows)
        assert carve(None, rows, qwen_spec(self.dtype))[1] == need, "qcarve changed: restate it here"
        ws = filled(need)
        out = filled(rows * E * 2).view(self.dtype).view(rows, E)
        flat = (C.c_int32 * (3 * len(grids)))(*[v for g in grids for v in g])
        self.L.check(self.lib.fvs_qwen_vit_encode(self.h, self.L.ptr(patches), self.L.ptr(out), flat, len(grids),
                                                  self.L.ptr(ws), need, self.L.cur_stream()), "fvs_qwen_vit_encode")
        torch.cuda.synchronize()
        return out, carve(ws, rows, qwen_spec(self.dtype))[0]

    def close(self):
        self.lib.fvs_qwen_vit_destroy(self.h)


@pytest.fixture(scope="module")
def qwen(L):
    """dt -> (state dict, {main, rope0 (inv_freq = 0), fc2zero, depth0}), built on first use"""
    made = {}

    def get(dt):
        if dt not in made:
            dtype = DTYPES[dt]
            sd = VI.state_dict(dict(depth=1, embed=E, heads=HEADS, seed=401), dt)
            made[dt] = sd, dict(main=QwenTower(L, sd, dtype, 1, INV_FREQ),
                                rope0=QwenTower(L, sd, dtype, 1, torch.zeros(NFREQ)),
                                fc2zero=QwenTower(L, sd, dtype, 1, INV_FREQ, zero_fc2=True),
                                depth0=QwenTower(L, sd, dtype, 0, INV_FREQ))
        return made[dt]
    yield get
    for _, towers in made.values():
        for t in towers.values():
            t.close()


# The real video grids (full resolution and pooled, test_qwen_vit_grids_host.REAL_GRIDS) plus two of one 2x2 block row.
GRIDS = sorted({g for r in REAL_GRIDS for g in r[4:]}) + [(1, 2, 2), (1, 2, 6)]
MIXED16 = [(2, 12, 18), (1, 2, 2), (2, 36, 24), (2, 6, 36), (1, 2, 6), (2, 24, 24), (2, 26, 46), (2, 12, 12),
           (2, 24, 40), (1, 2, 2), (2, 18, 12), (2, 12, 72), (1, 2, 6), (2, 12, 20), (2, 24, 36), (2, 24, 24)]
QWEN_CALLS = {"one_2x52x92": [(2, 52, 92)], "one_1x2x6": [(1, 2, 6)], "mixed16": MIXED16}
SEG_MOVE_GRID = 14                               # MIXED16[14] = (2, 24, 36): its temporal-patch boundary moves by one


def qwen_attention(nat, grids, heads, moved=None):
    """the fp64 attention reference and bound [rows, heads, 80] per (grid, temporal patch) segment; `moved`: the grid
    whose boundary between its two temporal patches moves one token later (a wrong segmentation)"""
    refs, bounds, rnds, r0 = [], [], [], 0
    scale = float(np.float32(80 ** -0.5))
    for gi, (t, h, w) in enumerate(grids):
        n = h * w
        segs = [n] * t if gi != moved else [n + 1, n - 1] + [n] * (t - 2)
        for s in segs:
            ref, bound, rnd = attention_bound(nat[r0:r0 + s], 1, s, heads, HD, scale)
            refs.append(ref[0]); bounds.append(bound[0]); rnds.append(rnd[0])
            r0 += s
    return torch.cat(refs), torch.cat(bounds), torch.cat(rnds)


@pytest.mark.parametrize("call", list(QWEN_CALLS))
@pytest.mark.parametrize("dt", list(DTYPES))
def test_qwen_block_stages(qwen, dt, call):
    dtype = DTYPES[dt]
    grids = QWEN_CALLS[call]
    sd, tw = qwen(dt)
    w = lambda k: sd[f"blocks.0.{k}"].to(device="cuda")
    rows = sum(t * h * w_ for t, h, w_ in grids)
    g = torch.Generator().manual_seed(17 + rows)
    patches = (torch.randn(rows, PATCH_DIM, generator=g) * 1.2).to(dtype).cuda()
    out, ws = tw["main"].encode(patches, grids)
    _, ws_r = tw["rope0"].encode(patches, grids)
    out_f, ws_f = tw["fc2zero"].encode(patches, grids)
    out_0, ws_0 = tw["depth0"].encode(patches, grids)
    tag = f"qwen {dt} {call}"

    # the companions' premise: every stage before the neutralised knob gives the main tower's bits
    for name, other in (("rope0", ws_r), ("fc2zero", ws_f), ("depth0", ws_0)):
        for k in ("pos", "delta"):
            assert_bits(f"{name} {k}", other[k], ws[k])
    for k in ("qkv", "ctx", "y", "act"):
        assert_bits(f"fc2zero {k}", ws_f[k], ws[k])

    # 1. pos
    assert torch.equal(ws["pos"].flatten().cpu(), packed_positions(grids)), "pos"

    # 2. rotary: q and k from the pre-rotary qkv, v untouched
    pre = to_natural(ws_r["qkv"], HEADS, 3).view(rows, 3, HEADS, HD)
    post = to_natural(ws["qkv"], HEADS, 3).view(rows, 3, HEADS, HD)
    assert_bits("v section", post[:, 2], pre[:, 2])
    rope = rope_bound(pre[:, :2], ws["pos"], INV_FREQ, post[:, :2])
    check(f"{tag} rotary", post[:, :2], *rope)

    # 3. attention per (grid, temporal patch) segment, on the observed post-rotary q, k, v
    nat = post.reshape(rows, 3 * E)
    ctx = to_natural(ws["ctx"], HEADS, 1).view(rows, HEADS, HD)
    check(f"{tag} attention", ctx, *qwen_attention(nat, grids, HEADS))

    # 4. out-proj + fp32 residual: x1 = float(delta) + ctx Wo^T + bo (x is +0 + float(delta) before it)
    x1 = ws_f["x"]
    ctx2 = ctx.reshape(rows, E)
    check(f"{tag} out-proj + residual", x1,
          *linear_bound(ctx2, w("attn.proj.weight"), w("attn.proj.bias"), "residual_f32", ws["delta"].float(), x1))

    # 5. LN2
    check(f"{tag} LN2", ws["y"], *layernorm_bound(x1, w("norm2.weight"), w("norm2.bias"), QWEN_EPS, ws["y"]))

    # 6. fc1 + quick-GELU
    check(f"{tag} fc1 + quick-GELU", ws["act"],
          *linear_bound(ws["y"], w("mlp.fc1.weight"), w("mlp.fc1.bias"), "quickgelu", None, ws["act"]))

    # 7. fc2 + fp32 residual
    check(f"{tag} fc2 + residual", ws["x"],
          *linear_bound(ws["act"], w("mlp.fc2.weight"), w("mlp.fc2.bias"), "residual_f32", x1, ws["x"]))

    # 8. the output: the fp32 x rounded once (add_cast_kernel adds a +0 delta)
    assert_bits("out", out, (ws["x"] + 0.0).to(dtype))
    assert_bits("fc2zero out", out_f, (x1 + 0.0).to(dtype))

    # 9. depth 0: x stays the +0 the encode sets, out is the patch embedding, which meets the bias GEMM bound (K = 1176)
    assert not bits(ws_0["x"]).any(), "depth 0: x"
    assert_bits("depth 0 out", out_0, (ws_0["x"] + ws_0["delta"].float()).to(dtype))
    assert_bits("depth 0 out == delta", out_0, ws_0["delta"])
    patch_w = sd["patch_embed.proj.weight"].reshape(E, -1).to(device="cuda")
    check(f"{tag} patch embedding", ws["delta"],
          *linear_bound(patches, patch_w, torch.zeros(E, dtype=dtype, device="cuda"), "bias", None, ws["delta"]))

    if call != "mixed16":
        return
    # discrimination: each bound rejects a deliberately wrong reference on the same outputs
    for m in ROPE_MUTATIONS:
        wrong = rope_bound(pre[:, :2], ws["pos"], INV_FREQ, post[:, :2], rope_mutation=m)
        with pytest.raises(AssertionError):
            check(f"{tag} rotary, wrong reference '{m}' (must fail)", post[:, :2], *wrong)
    r0 = sum(t * h * w_ for t, h, w_ in grids[:SEG_MOVE_GRID])
    t, h, w_ = grids[SEG_MOVE_GRID]
    seg_rows = slice(r0, r0 + t * h * w_)
    with pytest.raises(AssertionError):
        check(f"{tag} attention, a segment boundary one token late (must fail)", ctx[seg_rows],
              *qwen_attention(nat[seg_rows], [grids[SEG_MOVE_GRID]], HEADS, moved=0))

    # what the same mistakes do to the whole tower output, the number the parity tests' tolerances judge
    true = vit_forward(patches.cpu(), grids, sd, depth=1, heads=HEADS, device="cuda")
    for m in ROPE_MUTATIONS:
        d = rel(vit_forward(patches.cpu(), grids, sd, depth=1, heads=HEADS, device="cuda", rope_mutation=m), true)
        print(f"\n[{tag}] tower-level relative Frobenius error of rotary mistake '{m}': {d:.2e} "
              f"(parity tolerance f16 {TOL['f16']:.1e}, bf16 {TOL['bf16']:.1e})")


# ------------------------------------------------------------------------------------------------------- CLIP tower
class ClipTower:
    """a fvs_vit handle (336 px / 14, hidden 1024, 16 heads, mlp 4096) over its own device weights and a workspace that
    holds every frame in one micro-batch"""

    def __init__(self, L, wts, dtype, layers_run, keep_cls, frames, zero_fc2=False):
        self.L, self.lib, self.dtype, self.frames, self.keep_cls = L, L.load(), dtype, frames, keep_cls
        self.keep = []

        def dev(t):
            self.keep.append(t.to(device="cuda", dtype=dtype).contiguous())
            return self.keep[-1].data_ptr()
        arr = (L.VitLayerWeights * max(layers_run, 1))()
        for i in range(layers_run):
            p = dict(wts["layers"][i])
            p["qkv_w"] = torch.cat([p["q_w"], p["k_w"], p["v_w"]])
            p["qkv_b"] = torch.cat([p["q_b"], p["k_b"], p["v_b"]])
            if zero_fc2:
                p["fc2_w"], p["fc2_b"] = torch.zeros_like(p["fc2_w"]), torch.zeros_like(p["fc2_b"])
            for field, _ in L.VitLayerWeights._fields_:
                setattr(arr[i], field, dev(p[field]))
        cfg = L.VitConfig(CLIP_IMAGE, CLIP_PATCH, CLIP_H, 16, CLIP_MLP, layers_run, 1e-5, L.dtype_code(dtype), int(keep_cls))
        w = L.VitWeights(dev(wts["patch_w"].reshape(CLIP_H, -1)), dev(wts["class_emb"]), dev(wts["pos_emb"]),
                         dev(wts["pre_ln_w"]), dev(wts["pre_ln_b"]), arr)
        self.h = C.c_void_p()
        L.check(self.lib.fvs_vit_create(C.byref(self.h), C.byref(cfg), C.byref(w), L.cur_stream()), "fvs_vit_create")
        self.need = self.lib.fvs_vit_workspace_bytes(self.h, frames)
        assert carve(None, frames * CLIP_TOKENS, clip_spec(dtype))[1] == self.need, "carve changed: restate it here"
        self.ws = filled(self.need)
        torch.cuda.synchronize()

    def encode(self, pixels):
        """the first call runs the layer stack eagerly, later calls replay its CUDA graph"""
        self.ws.fill_(0xFF)
        n = self.frames * (CLIP_TOKENS - (0 if self.keep_cls else 1)) * CLIP_H
        out = filled(n * 2).view(self.dtype).view(self.frames, -1, CLIP_H)
        self.L.check(self.lib.fvs_vit_encode(self.h, self.L.ptr(pixels), self.L.ptr(out), self.frames, self.L.ptr(self.ws),
                                             self.need, self.L.cur_stream()), "fvs_vit_encode")
        torch.cuda.synchronize()
        return out, carve(self.ws, self.frames * CLIP_TOKENS, clip_spec(self.dtype))[0]

    def close(self):
        self.lib.fvs_vit_destroy(self.h)


def unfolded(pixels):
    """im2col's expected rows: per frame a zero CLS row, then the patches in (c, ky, kx) column order, zero-padded to
    KPAD columns"""
    B = pixels.shape[0]
    p = pixels.view(B, 3, CLIP_GRID, CLIP_PATCH, CLIP_GRID, CLIP_PATCH).permute(0, 2, 4, 1, 3, 5)
    want = torch.zeros(B, CLIP_TOKENS, KPAD, dtype=pixels.dtype, device=pixels.device)
    want[:, 1:, :KREAL] = p.reshape(B, CLIP_GRID ** 2, KREAL)
    return want.view(B * CLIP_TOKENS, KPAD)


def tail_check(name, out, x, first):
    """the tail rounds the fp32 x once, from row `first` of every frame on: 1 drops the CLS row ('patch'), 0 keeps it
    ('cls_patch')"""
    x = x.view(out.shape[0], CLIP_TOKENS, CLIP_H)[:, first:first + out.shape[1]]
    assert x.shape == out.shape and torch.equal(bits(out), bits(x.to(out.dtype))), f"{name}: tail"


@pytest.mark.parametrize("keep_cls", [0, 1])
@pytest.mark.parametrize("frames", [1, 3])
@pytest.mark.parametrize("layers_run", [0, 1])
@pytest.mark.parametrize("dt", list(DTYPES))
def test_clip_block_stages(L, dt, layers_run, frames, keep_cls):
    from oracle import fvs_oracle as O
    from tests import golden_inputs as GI
    dtype = DTYPES[dt]
    cfg = O.VitConfig(layers=1)
    wts = O.random_vit_weights(cfg, 501, n_layers=1)
    cast = lambda t: t.to(device="cuda", dtype=dtype)
    main = ClipTower(L, wts, dtype, layers_run, keep_cls, frames)
    towers = [main]
    if layers_run:
        emb = ClipTower(L, wts, dtype, 0, keep_cls, frames)                 # x after pre-LN (x0)
        fc2zero = ClipTower(L, wts, dtype, 1, keep_cls, frames, zero_fc2=True)
        towers += [emb, fc2zero]
    table = cast(wts["pos_emb"]).clone()
    table[0] = (cast(wts["pos_emb"])[0].float() + cast(wts["class_emb"]).float()).to(dtype)
    patch_w = cast(wts["patch_w"].reshape(CLIP_H, -1))
    lw = {k: cast(v) for k, v in wts["layers"][0].items()}
    try:
        for rnd in ("eager", "graph replay"):
            pixels = cast(GI.vit_pixels(cfg, frames, 600 + frames + (rnd != "eager")))
            tag = f"clip {dt} layers {layers_run} frames {frames} keep_cls {keep_cls} {rnd}"
            out, ws = main.encode(pixels)
            # 1. im2col
            assert_bits("patches", ws["patches"], unfolded(pixels))
            if layers_run:
                _, ws_e = emb.encode(pixels)
                out_f, ws_f = fc2zero.encode(pixels)
                assert_bits("embedding tower patches", ws_e["patches"], ws["patches"])
                for k in ("patches", "qkv", "ctx", "y", "act"):
                    assert_bits(f"fc2zero {k}", ws_f[k], ws[k])
            else:
                ws_e = ws
            # 2. patch GEMM + row table (period 577 across the frames), 3. pre-LayerNorm into the fp32 x
            pe = linear_bound(ws_e["patches"][:, :KREAL], patch_w, None, "rowtable", table, ws_e["y"])
            check(f"{tag} patch GEMM + row table", ws_e["y"], *pe)
            x0 = ws_e["x"]
            check(f"{tag} pre-LayerNorm", x0,
                  *layernorm_bound(ws_e["y"], cast(wts["pre_ln_w"]), cast(wts["pre_ln_b"]), CLIP_EPS, x0))
            # 4. tail
            tail_check(tag, out, ws["x"], 1 - keep_cls)
            if layers_run:
                # 5. attention on the observed qkv, then out-proj, LN2, fc1, fc2 via the fc2 companion
                check(f"{tag} attention", ws["ctx"].view(frames, CLIP_TOKENS, 16, 64),
                      *attention_bound(ws["qkv"], frames, CLIP_TOKENS, 16, 64, 0.125))
                x1 = ws_f["x"]
                check(f"{tag} out-proj + residual", x1,
                      *linear_bound(ws["ctx"], lw["o_w"], lw["o_b"], "residual_f32", x0, x1))
                check(f"{tag} LN2", ws["y"], *layernorm_bound(x1, lw["ln2_w"], lw["ln2_b"], CLIP_EPS, ws["y"]))
                check(f"{tag} fc1 + quick-GELU", ws["act"],
                      *linear_bound(ws["y"], lw["fc1_w"], lw["fc1_b"], "quickgelu", None, ws["act"]))
                check(f"{tag} fc2 + residual", ws["x"],
                      *linear_bound(ws["act"], lw["fc2_w"], lw["fc2_b"], "residual_f32", x1, ws["x"]))
                tail_check(f"{tag} fc2zero", out_f, x1, 1 - keep_cls)
            if rnd == "eager" and frames == 3 and not keep_cls:
                # discrimination: a row table of period 576, a tail that keeps the CLS row
                wrong = linear_bound(ws_e["patches"][:, :KREAL], patch_w, None, "rowtable", table[:576], ws_e["y"])
                with pytest.raises(AssertionError):
                    check(f"{tag} patch GEMM, row table of period 576 (must fail)", ws_e["y"], *wrong)
                with pytest.raises(AssertionError):
                    tail_check(f"{tag} tail without dropping CLS (must fail)", out, ws["x"], 0)
    finally:
        for t in towers:
            t.close()
