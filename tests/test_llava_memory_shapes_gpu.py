"""The LLaVA streaming memory at every STAR configuration the fused step admits, up to its limits (GPU half).

Every case of tests/test_llava_memory_shapes_host.py runs in each way that applies to it — the one-job fused kernel
(StreamBank), several streams of the case in one batched step (StreamPool, or stream_step_many for key_len 8, once with
max_blocks forcing several cooperative launches), the op-by-op mirror (fvs_fused_stream = False) and a bank whose frame
buffer is capped at ops.min_device_frames — and is compared with the oracle after every step, exactly: current and long
rows, the prefix, the frame count, and for the banks key_idx, labels, info (exit step, refills, converged, k-means ran)
and the cluster weights.  The Turing rows are held to tests.llava_abstract: bit for bit where the kernel's expf (<= 2
ulp) cannot move an f16 rounding, else equal to one of the values the chain gives when each such rounding is taken either
way.  The number of elements decided by that second rule is printed at the end of the module."""
import time

import numpy as np
import pytest
import torch

from oracle import fvs_oracle as O
from tests import golden_inputs as GI
from tests import llava_abstract as LA
from tests.test_gpu_parity import bits, cu, fvs  # noqa: F401  (fvs is a fixture)
from tests.test_llava_memory_shapes_host import (CASES, RATIO, case_draws, case_features, case_ntm, oracle_run, plan,
                                                 star_dict)

pytestmark = pytest.mark.gpu

RULE = {"elements": 0, "rows": 0, "weights": 0, "steps": 0}


@pytest.fixture(scope="module", autouse=True)
def report():
    t0 = time.time()
    yield
    print(f"\nTuring elements decided by the expf rule: {RULE['elements']} (in {RULE['rows']} rows with undetermined "
          f"weights; {RULE['weights']} undetermined weights over {RULE['steps']} checked steps); module {time.time() - t0:.0f} s")


def np16(t):
    return t.detach().cpu().contiguous().numpy()


def turing_candidates(name, s, prev_tur, tur_new):
    """candidate Turing rows after step s, from the device's Turing rows before it (prev_tur [n, D] f16)"""
    c = CASES[name]
    if s == 0:
        Tm = tur_new
    else:
        Tm = np.concatenate([prev_tur, tur_new])
    T1 = c["tur_len"]
    if s == 0 or Tm.shape[0] <= T1:
        return [Tm[i][None] for i in range(Tm.shape[0])], 0
    chunks = [Tm[i:i + T1] for i in range(T1, Tm.shape[0], T1)]
    ntm = [x.numpy() for x in case_ntm(name)]
    return LA.update_candidates(Tm[:T1], chunks, *ntm, RATIO)


def check_step(name, s, way, cur, lng, tur, prefix, n_frames, prev_tur, info=None):
    """one step of one way against the oracle; returns the device's Turing rows [n, D] for the next step"""
    r = oracle_run(name)[s]
    where = (name, way, s)
    assert np.array_equal(bits(cur), r["cur"].view(np.int16)), (where, "cur")
    assert np.array_equal(bits(lng), r["long"].view(np.int16)), (where, "long")
    assert n_frames == r["n_frames"], (where, "frames", n_frames)
    D = tur.shape[-1]
    got_tur = np16(tur).reshape(-1, D)
    cands, n_undet = turing_candidates(name, s, prev_tur, r["tur_new"].reshape(-1, D))
    assert got_tur.shape[0] == len(cands), (where, "Turing rows", got_tur.shape[0], len(cands))
    n_rule = LA.check_rows(got_tur, cands)
    RULE["elements"] += n_rule
    RULE["rows"] += sum(1 for cnd in cands if len(cnd) > 1)
    RULE["weights"] += n_undet
    RULE["steps"] += 1
    want_prefix = np.concatenate([got_tur, r["long"].reshape(-1, D), r["cur"].reshape(-1, D)])
    assert np.array_equal(bits(prefix), want_prefix.view(np.int16)), (where, "prefix")
    if info is not None:
        lab, inf, key, wsum = info
        p = plan(CASES[name])[s]
        inf = inf.cpu().numpy()
        assert int(inf[3]) == int(p["kmeans"]), (where, "kmeans ran")
        kl = len(r["key_idx"])
        assert kl == p["kl"], (where, "kl")
        assert np.array_equal(key.cpu().numpy()[:kl], r["key_idx"]), (where, "key_idx")
        if p["kmeans"]:
            conv = int(r["trace"]["iters"][-1]["stop"])
            assert (int(inf[0]), int(inf[1]), int(inf[2])) == (r["exit_step"], r["refills"], conv), (where, "info", inf)
            assert np.array_equal(lab.cpu().numpy(), r["labels"]), (where, "labels")
            assert np.array_equal(bits(wsum), r["wsum"].view(np.int16)), (where, "wsum")
    return got_tur


def ntm_cuda(name):
    return tuple(x.cuda() for x in case_ntm(name))


def step_draws(name, s, T):
    c = CASES[name]
    if s == 0 or not 0 < c["long_len"] < T:
        return None
    return tuple(cu(d) for d in case_draws(name, s, T, c["long_len"]))


def run_banks(name, ops, n_banks=1, device_frames=None, max_blocks=0):
    c = CASES[name]
    cfg = star_dict(c)
    cap = max(c["chunks"])
    df = ops.min_device_frames(cfg, cap) if device_frames == "min" else None
    banks = [ops.StreamBank(cfg, ntm_cuda(name), chunk_cap=cap, device_frames=df) for _ in range(n_banks)]
    feats = case_features(name)
    way = f"{n_banks} bank(s)" + (f", device_frames {df}" if df else "") + (f", max_blocks {max_blocks}" if max_blocks else "")
    prev = [None] * n_banks
    pos = 0
    for s, t in enumerate(c["chunks"]):
        clip = feats[pos:pos + t].cuda()
        pos += t
        T = banks[0].working_rows(t)
        d = step_draws(name, s, T)
        assert banks[0].needs_draws(t) == (d is not None)
        if n_banks == 1:
            banks[0].step(clip, draws=d)
        else:
            ops.stream_step_many(banks, [clip] * n_banks, draws=[d] * n_banks, max_blocks=max_blocks)
        for i, bank in enumerate(banks):
            cur, lng, tur, _ = bank.state()
            prev[i] = check_step(name, s, f"{way} #{i}", cur, lng, tur, bank.prefix(), bank.bank.n_frames, prev[i],
                                 info=bank.info())
    if df:
        assert banks[0].n_host() > 0 or sum(c["chunks"]) <= df


def make_case_model(name, pkg):
    from flash_vstream_b200.vstream_arch import FlashVStreamB200, NeuralTuringMachine
    c = CASES[name]
    ntm = NeuralTuringMachine(c["D"], c["ntm_dim"])
    qw, qb, kw, kb = case_ntm(name)
    with torch.no_grad():
        ntm.q_proj.weight.copy_(qw); ntm.q_proj.bias.copy_(qb)
        ntm.k_proj.weight.copy_(kw); ntm.k_proj.bias.copy_(kb)
    return FlashVStreamB200(None, ntm.half().cuda(), compress_size=c["a"], compress_long_memory_size=c["b"],
                            video_long_memory_length=c["long_len"], video_Turing_memory_length=c["tur_len"],
                            video_current_memory_length=c["cur_len"], compress_Turing_update_ratio=RATIO)


def run_pool(name, pkg, ops):
    c = CASES[name]
    if c["key_len"] != 3:      # StreamPool takes its config from a model, whose key length is the reference's 3
        run_banks(name, ops, n_banks=2)
        return
    pool = pkg.StreamPool(make_case_model(name, pkg), chunk_cap=max(c["chunks"]))
    sids = [pool.open(seed=i) for i in range(3)]
    feats = case_features(name)
    prev = {sid: None for sid in sids}
    pos = 0
    for s, t in enumerate(c["chunks"]):
        clip = feats[pos:pos + t].cuda()
        pos += t
        d = step_draws(name, s, pool.bank(sids[0]).working_rows(t))
        pool.step({sid: clip for sid in sids}, draws={sid: d for sid in sids} if d is not None else None)
        for sid in sids:
            bank = pool.bank(sid)
            cur, lng, tur, _ = pool.state(sid)
            prev[sid] = check_step(name, s, f"pool #{sid}", cur, lng, tur, pool.prefix(sid), bank.bank.n_frames, prev[sid],
                                   info=bank.info())


def run_op_by_op(name, pkg):
    c = CASES[name]
    model = make_case_model(name, pkg)
    model.fvs_fused_stream = False
    feats = case_features(name)
    prev, pos, n_long = None, 0, 0
    for s, t in enumerate(c["chunks"]):
        d = step_draws(name, s, n_long + t)
        model.consolidate_streaming(feats[pos:pos + t].cuda(), draws=d)
        pos += t
        cur, lng, tur, buf = model.video_embedding_memory
        n_long = lng.shape[0]
        prev = check_step(name, s, "op-by-op", cur, lng, tur, model.memory_prefix(), buf.shape[0], prev)
    assert "_fvs_bank" not in model.__dict__


# (case, way) with the case outermost: the oracle of a case is computed once for all its ways.  "op" needs the model's
# key length (3); "waves": two streams with max_blocks 3 — each job needs a Lloyd block and an abstract-memory block, so
# they cannot share one launch.
WAYS = [(n, w) for n, c in CASES.items() for w in c["ways"] if w != "op" or c["key_len"] == 3]


@pytest.mark.parametrize("name,way", WAYS)
def test_case_vs_oracle(fvs, name, way):
    pkg, ops = fvs
    if way == "bank":
        run_banks(name, ops)
    elif way == "capped":
        run_banks(name, ops, device_frames="min")
    elif way == "pool":
        run_pool(name, pkg, ops)
    elif way == "waves":
        run_banks(name, ops, n_banks=2, max_blocks=3)
    else:
        run_op_by_op(name, pkg)


# ------------------------------------------------------------------------------------------------ pixels: the pooled tail
@pytest.fixture(scope="module")
def vit_l14(fvs):
    from flash_vstream_b200.clip_encoder import CLIPVisionTower
    cfg = O.VitConfig(layers=3)
    w = O.random_vit_weights(cfg, 23)
    return cfg, CLIPVisionTower.from_weights(w, image_size=336, patch_size=14, heads=16, select_layer=-2, max_batch=4)


@pytest.mark.parametrize("a,b", [(2, 1), (3, 1), (4, 2), (6, 3), (8, 4)])
def test_pooled_tail_equals_encode_then_pool(fvs, vit_l14, a, b):
    """pool3 from the fp32 residual stream (the encoder's tail) == encode_images, then oracle.spatial_pool to a, then b
    and 1 from the rounded level a — for every admitted compress_size, through 2 layers of a full-width ViT-L/14-336"""
    pkg, ops = fvs
    cfg, tower = vit_l14
    D = cfg.hidden
    pix = (GI.vit_pixels(cfg, 3, 40 + a) * 0.5).half().cuda()
    feats = tower(pix)
    la, lb, lc = O.spatial_pool3(feats.cpu().numpy(), a, b)
    star = dict(D=D, grid=24, cur_size=a, long_size=b, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                ratio=RATIO)
    w = GI.ntm_weights(D, 32, 5)
    bank = ops.StreamBank(star, tuple(w[k].cuda() for k in ("q_w", "q_b", "k_w", "k_b")), chunk_cap=3)
    bank.step(pix, vit=tower.engine)
    assert np.array_equal(bits(bank.frames[:3]), la.view(np.int16)), "level a"
    assert np.array_equal(bits(bank.long_work[:3]), lb.view(np.int16)), "level b"
    assert np.array_equal(bits(bank.tur_work[:3]), lc.view(np.int16)), "level 1"
    cur, lng, tur, _ = bank.state()
    assert np.array_equal(bits(cur), la[-1:].view(np.int16)) and np.array_equal(bits(lng), lb.view(np.int16))
