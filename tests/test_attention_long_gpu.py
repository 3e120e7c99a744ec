"""Attention beyond 384 tokens: sv_attention_fwd_long_bf16 (K / V streamed through a TMA ring) and
sv_attention_bwd_long_bf16, up to 2048 queries and keys.

* float64 bounds (the reference and bounds of tests/test_attention_fp64_gpu.py) on plain, gated and dropout attention
  above 384, masks whose live keys all lie past key 384, a scene with every key masked, one query row of 512 (the
  CLS-only caption layer) and a packed dq | dk | dv gradient;
* on the shapes the resident entries take too (<= 384), the long entries give the same bits as those;
* block skipping above 384 gives the bits of the full sweep;
* the modules and training / evaluation steps that reach these lengths (BERT on 512-token captions, the spatial encoder
  at 512 and 1024 objects, the joint text + object encoder at 50 + 400 tokens);
* argument validation without a GPU.
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from sceneverse_b200 import ops
from tests.test_attention_fp64_gpu import GATED, P_DROP, PLAIN, SCALE, SEED, check, inputs


# ---- the long entries -------------------------------------------------------------------------------------------------
def forward(x, q=None, k=None, v=None, long=True, seq_rows=None):
    from sceneverse_b200 import native
    sh = 0 if x.sw is None else x.sw.shape[-1] // 6
    return native.attention(x.q if q is None else q, x.k if k is None else k, x.v if v is None else v, x.H,
                            key_padding_mask=x.mask, spatial_w=x.sw, spatial_heads=sh, pairwise_locs=x.locs,
                            return_lse=True, dropout_p=P_DROP if x.keep is not None else 0.0, seed=SEED,
                            seq_rows=seq_rows, long=long)


def backward(x, out, lse, long=True):
    """The backward entry called directly, so that D (dvec) is returned too; outputs start as NaN."""
    from sceneverse_b200 import _lib, native
    B, Lq, E = x.q.shape
    Lk = x.k.shape[1]
    nan = dict(dtype=torch.bfloat16, device=x.q.device)
    dq, dk, dv = torch.full((B, Lq, E), math.nan, **nan), torch.full((B, Lk, E), math.nan, **nan), \
        torch.full((B, Lk, E), math.nan, **nan)
    dvec = torch.full((B, x.H, Lq), math.nan, device=x.q.device)
    dsw = torch.full_like(x.sw, math.nan) if x.sw is not None else None
    kpm = native._mask_bytes(x.mask)
    name = "sv_attention_bwd_long_bf16" if long else "sv_attention_bwd_rows_bf16"
    lib = _lib.gps()
    st = getattr(lib, name)(
        x.q.data_ptr(), x.q.stride(0), x.q.stride(1), x.k.data_ptr(), x.k.stride(0), x.k.stride(1), x.v.data_ptr(),
        x.v.stride(0), x.v.stride(1), out.data_ptr(), x.go.data_ptr(), _lib.ptr(kpm), _lib.ptr(x.sw), _lib.ptr(x.locs),
        lse.data_ptr(), B, x.H, Lq, Lk, SCALE, dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), E, _lib.ptr(dsw), dvec.data_ptr(),
        P_DROP if x.keep is not None else 0.0, SEED, Lq, torch.cuda.current_stream().cuda_stream)
    _lib.check(lib, st, name)
    got = dict(dq=dq, dk=dk, dv=dv, dvec=dvec)
    if dsw is not None:
        got["dsw"] = dsw
    return got


def run(x, with_backward=True, long=True):
    out, lse = forward(x, long=long)
    got = dict(out=out, lse=lse)
    if with_backward:
        got.update(backward(x, out, lse, long=long))
    return got


# ---- a. float64 bounds --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("Lq,Lk,H", [(385, 385, 12), (1, 2048, 12), (64, 513, 12), (512, 512, 12), (130, 1024, 12),
                                     (2048, 2048, 4)])
def test_plain_attention_within_fp64_bound(Lq, Lk, H):
    x = inputs(Lq, Lk, H)
    check(x, run(x), f"long plain Lq={Lq} Lk={Lk} H={H}")


@pytest.mark.gpu
@pytest.mark.parametrize("L,H", [(385, 12), (512, 12), (1024, 4)])
def test_gated_attention_within_fp64_bound(L, H):
    x = inputs(L, L, H, gate="per_head")
    got = run(x)
    check(x, got, f"long gated L={L} H={H}")


@pytest.mark.gpu
def test_gate_shared_across_heads_within_fp64_bound():
    """spatial_heads = 1 at 512 objects: the native forward within the bound, and ops.spatial_attention (native forward,
    recomputed backward) returns the same forward bits."""
    L, H = 512, 12
    x = inputs(L, L, H, gate="shared")
    got = run(x, with_backward=False)
    check(x, got, f"long shared gate L={L}")
    out, _ = ops.spatial_attention(x.q, x.k, x.v, x.sw, x.locs, H, 1, key_padding_mask=x.mask)
    assert torch.equal(out, got["out"])


@pytest.mark.gpu
def test_dropout_attention_within_fp64_bound():
    x = inputs(512, 512, 12, dropout=True)
    assert abs(x.keep.double().mean().item() - (1 - P_DROP)) < 0.01
    check(x, run(x), "long dropout Lq=Lk=512")


@pytest.mark.gpu
@pytest.mark.parametrize("gate", [None, "per_head"])
def test_scene_with_every_key_masked(gate):
    x = inputs(512, 512, 12, gate=gate)
    x.mask[1] = True
    got = run(x)
    for name, t in got.items():
        assert not torch.isnan(t).any(), f"{name}: NaN"
    assert not got["out"][1].any() and torch.equal(got["lse"][1], torch.full_like(got["lse"][1], math.inf))
    for name in ("dq", "dk", "dv", "dvec") + (("dsw",) if gate else ()):
        assert not got[name][1].any(), f"{name}: non-zero for the scene without a live key"
    check(x, got, f"long scene fully masked gate={gate}")


@pytest.mark.gpu
@pytest.mark.parametrize("gate", [None, "per_head"])
def test_live_keys_only_past_384(gate):
    """Every key block up to 384 masked: the visited blocks all lie past the resident limit."""
    x = inputs(512, 512, 12, gate=gate)
    x.mask[:] = True
    x.mask[0, 400:450] = False
    x.mask[1, 385] = False
    x.mask[1, 500:512] = False
    got = run(x)
    check(x, got, f"long keys past 384 gate={gate}")


@pytest.mark.gpu
@pytest.mark.parametrize("dropout", [False, True])
def test_one_query_row_of_512(dropout):
    """query_rows = 1 of a 512-row sequence (the CLS-only last layer of the caption encoder): within the bound without
    dropout, and with dropout the bits and masks of row 0 of the 512-query call; dq rows past the first are zero."""
    from sceneverse_b200 import native
    H, L = 12, 512
    if not dropout:
        x = inputs(1, L, H)
        check(x, run(x), "long one query of 512")
        return
    full = inputs(L, L, H, dropout=True)
    E = H * 64
    qkv = torch.cat([full.q, full.k, full.v], -1)
    out_full, lse_full = native.attention(full.q, full.k, full.v, H, key_padding_mask=full.mask, return_lse=True,
                                          dropout_p=P_DROP, seed=SEED)
    out1, lse1 = native.attention(qkv[:, :1, :E], qkv[..., E:2 * E], qkv[..., 2 * E:], H, key_padding_mask=full.mask,
                                  return_lse=True, dropout_p=P_DROP, seed=SEED, seq_rows=L)
    assert torch.equal(out1, out_full[:, :1]) and torch.equal(lse1, lse_full[..., :1])
    packed = torch.full((2, L, 3 * E), math.nan, dtype=torch.bfloat16, device="cuda")
    dq, dk, dv, _ = native.attention_backward(qkv[:, :1, :E], qkv[..., E:2 * E], qkv[..., 2 * E:], out1, full.go[:, :1],
                                              lse1, H, key_padding_mask=full.mask, dropout_p=P_DROP, seed=SEED,
                                              packed_grad=packed, seq_rows=L)
    assert not dq[:, 1:].any() and not torch.isnan(packed).any()
    # the same gradients as the 512-query backward with a zero output gradient on every row but the first
    go = torch.zeros_like(full.go)
    go[:, :1] = full.go[:, :1]
    ref = native.attention_backward(full.q, full.k, full.v, out_full, go, lse_full, H, key_padding_mask=full.mask,
                                    dropout_p=P_DROP, seed=SEED)
    assert torch.equal(dq[:, :1], ref[0][:, :1])
    for a, b in ((dk, ref[1]), (dv, ref[2])):
        assert (a.float() - b.float()).abs().max() <= 1e-2 * b.float().abs().max()


@pytest.mark.gpu
@pytest.mark.parametrize("gate", [None, "per_head"])
def test_packed_gradient_within_fp64_bound(gate):
    """q, k, v as column views of one packed (B, L, 3E) projection and dq | dk | dv written into one packed gradient
    (d_rs = 3E): the bits of the contiguous run, and within the bound."""
    from sceneverse_b200 import native
    L, H = 512, 12
    x = inputs(L, L, H, gate=gate)
    E = H * 64
    qkv = torch.cat([x.q, x.k, x.v], -1)
    qv, kv, vv = qkv[..., :E], qkv[..., E:2 * E], qkv[..., 2 * E:]
    got = run(x)
    out, lse = forward(x, qv, kv, vv)
    assert torch.equal(out, got["out"]) and torch.equal(lse, got["lse"])
    packed = torch.full((2, L, 3 * E), math.nan, dtype=torch.bfloat16, device="cuda")
    dq, dk, dv, dsw = native.attention_backward(qv, kv, vv, out, x.go, lse, H, key_padding_mask=x.mask, spatial_w=x.sw,
                                                pairwise_locs=x.locs, packed_grad=packed)
    for name, t in (("dq", dq), ("dk", dk), ("dv", dv)):
        assert torch.equal(t, got[name]), f"packed {name} differs from the contiguous run"
    check(x, dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv, **({"dsw": dsw} if gate else {})), f"long packed gate={gate}")


# ---- b. the same bits as the resident entries on shared ground -----------------------------------------------------------
def _same_bits(x, what):
    long, rows = run(x, long=True), run(x, long=False)
    for name in rows:
        if name == "dvec":
            continue
        assert torch.equal(long[name], rows[name]), f"{what} {name}: the long entry differs from the resident one"


@pytest.mark.gpu
@pytest.mark.parametrize("Lq,Lk", PLAIN)
def test_plain_same_bits_as_resident_entries(Lq, Lk):
    _same_bits(inputs(Lq, Lk, 12), f"plain Lq={Lq} Lk={Lk}")


@pytest.mark.gpu
@pytest.mark.parametrize("L", GATED)
def test_gated_same_bits_as_resident_entries(L):
    _same_bits(inputs(L, L, 12, gate="per_head"), f"gated L={L}")


@pytest.mark.gpu
@pytest.mark.parametrize("Lq,Lk", [(80, 50), (384, 384)])
def test_dropout_same_bits_as_resident_entries(Lq, Lk):
    _same_bits(inputs(Lq, Lk, 12, dropout=True), f"dropout Lq={Lq} Lk={Lk}")


# ---- c. block skipping above 384 ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("Lq,Lk,gate,dropout", [(512, 512, None, False), (130, 1024, None, True),
                                                (1024, 1024, "per_head", False), (2048, 2048, None, False)])
def test_block_skip_matches_full_sweep(Lq, Lk, gate, dropout):
    from sceneverse_b200 import native
    x = inputs(Lq, Lk, 4, gate=gate, dropout=dropout)
    x.mask[0, 64:200] = True            # two whole blocks masked in scene 0 too
    skip = run(x)
    native.attention_visit_all_blocks(1)
    try:
        full = run(x)
    finally:
        native.attention_visit_all_blocks(0)
    for name in skip:
        assert torch.equal(skip[name], full[name]), f"{name}: block skipping changed the result"


# ---- d. modules -------------------------------------------------------------------------------------------------------
def _rel(got, want, valid=None):
    d = (got.float() - want.float()).abs()
    w = want.float().abs()
    if valid is not None:
        d, w = d[valid], w[valid]
    return d.max().item() / w.max().item()


@pytest.mark.gpu
def test_bert_on_512_token_captions_matches_huggingface_bert():
    """The re-routed text encoder on 512-token batches (the longest caption BERT's positions allow), full and CLS-only,
    against the unpatched HuggingFace module with the same weights (the pattern of
    test_rerouted_bert_matches_huggingface_bert_gpu)."""
    from transformers import BertConfig, BertModel
    from sceneverse_b200 import model as M
    from sceneverse_b200.modules.layers import route_linears
    torch.manual_seed(0)
    enc = route_linears(M.BERTLanguageEncoder(None)).cuda().eval()
    ref = BertModel(BertConfig(hidden_size=768, num_hidden_layers=4, num_attention_heads=12, type_vocab_size=2)).cuda().eval()
    ref.load_state_dict(enc.model.state_dict())
    L = 512
    ids = torch.randint(1000, 30000, (8, L), device="cuda")
    lens = torch.tensor([512, 12, 385, 512, 8, 440, 129, 500], device="cuda")
    mask = (torch.arange(L, device="cuda")[None, :] < lens[:, None]).long()
    with torch.no_grad():
        want = ref(ids, mask).last_hidden_state
        with torch.autocast("cuda", dtype=torch.bfloat16):
            got = enc(ids, mask)
            cls = enc(ids, mask, cls_only=True)
    valid = mask.bool()
    err = _rel(got, want, valid)
    err_cls = _rel(cls, want[:, 0])
    print(f"BERT_512 relative error full {err:.3g}, CLS-only {err_cls:.3g}")
    assert err < 3e-2 and err_cls < 3e-2, (err, err_cls)
    # training mode, dropout off: the backward runs through the long entries and matches HF's gradients
    enc.train()
    ref.train()
    for m in list(enc.modules()) + list(ref.modules()):
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    proj = torch.randn(L, 768, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = enc(ids, mask)
    (out.float() * proj * valid[..., None]).sum().backward()
    (ref(ids, mask).last_hidden_state * proj * valid[..., None]).sum().backward()
    scale = max(q.grad.abs().max().item() for n, q in ref.named_parameters() if "pooler" not in n)
    for (n, p), (_, q) in zip(enc.model.named_parameters(), ref.named_parameters()):
        if "pooler" in n:
            continue
        rel = (p.grad.float() - q.grad).abs().max().item() / (q.grad.abs().max().item() + 2e-3 * scale)
        assert rel < 8e-2, (n, rel)


def _scene(B, O, seed, n_valid):
    g = torch.Generator().manual_seed(seed)
    locs = torch.cat([torch.randn(B, O, 3, generator=g) * 3.0, torch.rand(B, O, 3, generator=g) + 0.1], -1)
    masks = torch.arange(O)[None, :] < torch.tensor(n_valid)[:, None]
    return locs.cuda(), masks.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("O", [512, 1024])
def test_spatial_encoder_layers_match_fp32_formulation(O):
    """PointOpenVocabEncoder's spatial self-attention layers on O objects (bf16, native gated attention through the long
    entries) against the same module in fp32 (the torch formulation of the gate), from the same backbone features."""
    from sceneverse_b200 import weights
    from sceneverse_b200.modules import vision
    from tests.test_gps_modules import load
    torch.backends.cuda.matmul.allow_tf32 = False
    B = 2
    tf = weights.synthetic_tensor("text_features", (607, 768))
    enc = load(vision.PointOpenVocabEncoder(None, freeze=True, text_features=tf), 0).cuda().eval()
    feats = torch.randn(B * O, 768, generator=torch.Generator().manual_seed(2)).cuda()

    class Backbone(torch.nn.Module):          # fixed backbone features: the test is about the spatial layers
        def forward(self, x):
            return feats
    enc.point_feature_extractor = Backbone()
    locs, masks = _scene(B, O, 3, [O, O - 77])
    pcds = torch.zeros(B, O, 1, 6, device="cuda")
    with torch.no_grad():
        want, _, _ = enc(pcds, locs, masks, masks, None)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            got, _, _ = enc(pcds, locs, masks, masks, None)
    assert got.dtype == torch.bfloat16
    err = _rel(got, want, masks)
    print(f"SPATIAL_ENCODER O={O} relative error {err:.3g}")
    assert err < 3e-2, err


@pytest.mark.gpu
def test_unified_encoder_v2_at_50_text_and_400_objects():
    """UnifiedSpatialCrossEncoderV2's joint self-attention over T + O = 450 tokens: bf16 native against fp32 torch."""
    from sceneverse_b200.modules import grounding
    from tests.test_gps_modules import load
    torch.backends.cuda.matmul.allow_tf32 = False
    B, T, O = 2, 50, 400
    v2 = load(grounding.UnifiedSpatialCrossEncoderV2(None), 1).cuda().eval()
    g = torch.Generator().manual_seed(4)
    txt = (torch.randn(B, T, 768, generator=g) * 0.5).cuda()
    obj = (torch.randn(B, O, 768, generator=g) * 0.5).cuda()
    txt_masks = (torch.arange(T)[None, :] < torch.tensor([T, 17])[:, None]).cuda()
    locs, obj_masks = _scene(B, O, 5, [O, 333])
    with torch.no_grad():
        want_t, want_o = v2(txt, txt_masks, obj, locs, obj_masks)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            got_t, got_o = v2(txt, txt_masks, obj, locs, obj_masks)
    et, eo = _rel(got_t, want_t, txt_masks), _rel(got_o, want_o, obj_masks)
    print(f"UNIFIED_V2 T={T} O={O} relative error text {et:.3g}, objects {eo:.3g}")
    assert et < 3e-2 and eo < 3e-2, (et, eo)


# ---- e. steps ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_graph_step_matches_eager_step_at_400_objects_and_512_token_captions():
    """One GPS pre-training step through the captured path against the eager step (the parameter tolerance of
    test_graph_step_matches_eager_step_parameters), on scenes of 400 objects with 512-token scene captions."""
    from sceneverse_b200 import model as M, synthetic, train, weights
    tf = weights.synthetic_tensor("text_features", (607, 768))
    d = synthetic.scene_batch(9, B=8, O=400, P=1024, L=50, Ls=512, min_obj=300)
    batch = {k: torch.from_numpy(v).cuda() for k, v in d.items()}

    def make(graph):
        cfg = M.pretrain_config(1, text_features=tf)
        cfg["solver"]["sched"]["args"]["warmup_steps"] = 0
        ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=3, cuda_graph=graph)
        for m in ps.module.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
            if hasattr(m, "dropout") and isinstance(m.dropout, float):
                m.dropout = 0.0
        return ps
    eager, graph = make(False), make(True)
    graph.module.load_state_dict(eager.module.state_dict())
    p0 = {n: p.detach().clone() for n, p in eager.module.named_parameters()}
    eager._probe_unused(dict(batch))
    graph._probe_unused(dict(batch))
    eager.step(dict(batch))
    graph.static_batch = {k: v.clone() for k, v in batch.items()}
    graph._make_flat_state()
    graph._raw_step()
    ops.clear_shadows()
    checked = 0
    for (n, pe), (_, pg) in zip(eager.module.named_parameters(), graph.module.named_parameters()):
        if not pe.requires_grad or pe.grad is None:
            continue
        ge = pe.grad.float()
        big = ge.abs() > 0.2 * ge.abs().max()
        if big.sum() == 0 or ge.abs().max() == 0:
            continue
        de, dg = (pe.detach() - p0[n]).float(), (pg.detach() - p0[n]).float()
        agree = (torch.sign(de[big]) == torch.sign(dg[big])).float().mean().item()
        ratio = (dg[big].abs().mean() / (de[big].abs().mean() + 1e-20)).item()
        checked += 1
        assert agree > 0.98 and 0.9 < ratio < 1.1, (n, agree, ratio)
    assert checked > 100, checked


@pytest.mark.gpu
def test_scanrefer_eval_runner_at_512_objects():
    """ScanRefer evaluation on 512-object scenes: the counters of the graph-captured run equal the host restatement of
    the metrics on an eager forward of the same model."""
    from sceneverse_b200 import evaluate, model as M, synthetic, train, weights
    from tests.test_eval_gpu import host_counters
    tf = weights.synthetic_tensor("text_features", (607, 768))
    B, O = 4, 512
    ps = train.PretrainStep(M.scanrefer_config(text_features=tf), "cuda:0", seed=0)
    try:
        d = synthetic.scene_batch(5, B=B, O=O, P=1024, L=50, min_obj=400)
        rng = np.random.default_rng(1)
        d["tgt_object_id_iou25"] = (rng.random((B, O)) < 0.05).astype(np.int64)
        d["tgt_object_id_iou50"] = d["tgt_object_id_iou25"]
        d["is_multiple"] = rng.random(B) < 0.5
        d["tgt_object_label"] = rng.integers(0, 607, (B, 1))
        batch_ = {k: torch.from_numpy(np.asarray(v)).cuda() for k, v in d.items()}
        ev = evaluate.ScanReferEval()
        evaluate.EvalRunner(ps, [ev], batch_size=B).run([batch_])
        model = ps.module.model.eval()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(dict(batch_))
        model.train()
        cpu = {k: (v.float().cpu() if v.dtype == torch.bfloat16 else v.cpu()) for k, v in out.items() if torch.is_tensor(v)}
        want = torch.zeros(ev.size, dtype=torch.float64).tolist()
        host_counters("scanrefer", cpu, want)
        assert ev.counters.cpu().tolist() == want
    finally:
        ps.close()


# ---- f. without a GPU -------------------------------------------------------------------------------------------------
_VALIDATION = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from sceneverse_b200 import _lib
lib = _lib.gps()
a = 0x1000      # 16-byte aligned fake address


def fwd(Lq=4, Lk=64, sw=None, sh=0, locs=None, p=0.0):
    return lib.sv_attention_fwd_long_bf16(a, 8, 768, a, 8, 768, a, 8, 768, a, 8, 768, None, sw, sh, locs, 1, 12, Lq, Lk,
                                          0.125, None, p, 0, Lq, None)


def bwd(Lq=64, Lk=64, sw=None, locs=None, dsw=None, p=0.0):
    return lib.sv_attention_bwd_long_bf16(a, 8, 768, a, 8, 768, a, 8, 768, a, a, None, sw, locs, a, 1, 12, Lq, Lk, 0.125,
                                          a, a, a, 768, dsw, a, p, 0, Lq, None)


out = {"fwd Lq 2049": fwd(Lq=2049), "fwd Lk 2049": fwd(Lk=2049), "fwd gate with dropout": fwd(sw=a, locs=a, sh=12, p=0.1),
       "fwd spatial_heads 2": fwd(sw=a, locs=a, sh=2), "fwd gate without locs": fwd(sw=a, sh=12),
       "bwd Lq 2049": bwd(Lq=2049), "bwd Lk 2049": bwd(Lk=2049), "bwd gate with dropout": bwd(sw=a, locs=a, dsw=a, p=0.1),
       # accepted by the validation: they get as far as the device, which this process does not see
       "fwd Lq Lk 2048": fwd(Lq=2048, Lk=2048), "fwd Lk 385": fwd(Lk=385), "fwd gate 2048": fwd(Lq=2048, Lk=2048, sw=a, locs=a, sh=1),
       "bwd Lq Lk 2048": bwd(Lq=2048, Lk=2048), "bwd gate 2048": bwd(Lq=2048, Lk=2048, sw=a, locs=a, dsw=a)}
print(json.dumps(out))
"""


def test_long_entry_argument_validation_without_gpu():
    """The long entries reject more than 2048 queries or keys and a gate with dropout (1 = SV_ERR_INVALID_ARG) before
    touching the device, and accept 2048 (2: the call reached the device, which the process does not see)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", _VALIDATION, root], capture_output=True, text=True, timeout=120,
                         env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    accepted = ("fwd Lq Lk 2048", "fwd Lk 385", "fwd gate 2048", "bwd Lq Lk 2048", "bwd gate 2048")
    want = {k: 2 if k in accepted else 1 for k in got}
    assert len(got) == 13 and got == want, {k: v for k, v in got.items() if v != want[k]}


@pytest.mark.gpu
def test_ops_refuse_more_than_2048_tokens():
    """Above 2048 queries or keys the bf16 path still refuses, and the message names the limit."""
    assert ops.ATTENTION_MAX_LEN == 2048
    long = torch.zeros(1, 2049, 64, dtype=torch.bfloat16, device="cuda")
    short = torch.zeros(1, 16, 64, dtype=torch.bfloat16, device="cuda")
    for q, k in ((long, short), (short, long)):
        with pytest.raises(NotImplementedError, match="2048"):
            ops.attention(q, k, k, 1)
    with pytest.raises(NotImplementedError, match="2048"):
        ops.attention_packed(torch.zeros(1, 2049, 192, dtype=torch.bfloat16, device="cuda"), 1)
