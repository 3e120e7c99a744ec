"""ScanQA / SQA3D fine-tuning: QAHeadV1 wired into OpenVocab, `answer_loss`, the ScanQA form of TextObjWithinBatch, and the
native kernels of csrc/qa_ops.cu (sv_bce_logits_fwd_bwd, sv_attn_pool_fwd / _bwd).

* CPU: the fp32 stack (V2 + QAHeadV1 + answer_loss + ScanQA TextObjWithinBatch) against the unmodified reference
  (tests/golden/model_qa_grads.npz, oracle/make_golden_qa.py); the default within-batch loss is still the cross-entropy;
  configs, the synthetic QA batch, and argument validation of the new entry points in a process that sees no CUDA device.
* GPU: BCE and attention pool against float64 with bounds derived from fp32 / bf16 rounding; QAHeadV1 in bf16; the whole
  bf16 backward against the reference fixture; eager and CUDA-graph training steps of both configs."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sceneverse_b200 import synthetic, weights
from sceneverse_b200.modules import grounding, heads, losses

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
U32, UBF = 2.0 ** -24, 2.0 ** -8          # unit roundoff of fp32 and bf16


def gamma(n):
    return n * U32 / (1 - n * U32)


def load(m, seed):
    m.load_state_dict(weights.synthetic_state_dict(m, seed=seed))
    return m.eval()


def golden_inputs(G):
    """The batch and encoder input features of oracle/make_golden_qa.py::qa_inputs, from the seeds stored in the fixture."""
    B, O, L, A = (int(G[k]) for k in ("B", "O", "L", "num_answers"))
    d = synthetic.qa_batch(int(G["data_seed"]), "ScanQA", B=B, O=O, L=L, num_answers=A, min_obj=6, edge_rows=True)
    g = torch.Generator().manual_seed(int(G["feat_seed"]))
    txt = torch.randn(B, L, 768, generator=g) * 0.5
    obj = torch.randn(B, O, 768, generator=g) * 0.5
    return d, txt, obj


def qa_stack(G, device):
    return {"v2": load(grounding.UnifiedSpatialCrossEncoderV2(None), int(G["v2_seed"])).to(device),
            "qa": load(heads.QAHeadV1(None, num_answers=int(G["num_answers"])), int(G["head_seed"])).to(device),
            "l_within": losses.TextObjWithinBatch({"num_gpu": 1, "task": "ScanQA"}).to(device)}


def run_stack(mods, t, txt, obj):
    t2, o2 = mods["v2"](txt, t["txt_masks"], obj, t["obj_locs"], t["obj_masks"])
    scores = mods["qa"](o2, t["obj_masks"], t2, t["txt_masks"])
    dd = dict(t)
    dd.update(intra_obj_embeds=o2, intra_text_embed=t2[:, 0], answer_scores=scores)
    return scores, {"answer": losses.answer_loss(dd), "within": mods["l_within"](dd)}


def grad_norms(mods):
    return {f"{mn}.{n}": float(p.grad.double().norm()) for mn, m in mods.items() for n, p in m.named_parameters()
            if p.grad is not None}


# ---- CPU ------------------------------------------------------------------------------------------------------------------
def test_qa_stack_matches_reference_cpu_fp32():
    """Loss terms within 1e-4 relative, gradient norms of every trainable parameter within 2e-3 relative + 1e-6, five gradient
    slices within 1e-4 (of the slice's largest entry): the autograd structure of the head and both losses."""
    G = np.load(os.path.join(GOLDEN, "model_qa_grads.npz"))
    want_norms = json.load(open(os.path.join(GOLDEN, "model_qa_grad_norms.json")))
    d, txt, obj = golden_inputs(G)
    t = {k: torch.from_numpy(v) for k, v in d.items()}
    mods = qa_stack(G, "cpu")
    scores, parts = run_stack(mods, t, txt, obj)
    want_scores = G["answer_scores"]
    assert np.abs(scores.detach().numpy() - want_scores).max() <= 1e-4 * np.abs(want_scores).max()
    for k, v in parts.items():
        assert abs(float(v) - float(G["loss_" + k])) < 1e-4 * max(1.0, abs(float(G["loss_" + k]))), k
    total = sum(parts.values())
    assert abs(float(total) - float(G["total"])) < 1e-4 * abs(float(G["total"]))
    total.backward()
    got = grad_norms(mods)
    assert set(got) == set(want_norms), set(got) ^ set(want_norms)
    # the score layers' biases have a mathematically zero gradient (softmax over tokens is shift invariant): both sides are
    # fp32 rounding noise of the gradients behind them (norms up to 1.6e3), so they get a floor of 1e-8 of the largest norm
    zero = {k for k in want_norms if k.endswith("mlp.linear.bias")}
    scale = max(want_norms.values())
    assert all(got[k] <= 1e-8 * scale and want_norms[k] <= 1e-8 * scale for k in zero), {k: (got[k], want_norms[k]) for k in zero}
    bad = {k: (got[k], w) for k, w in want_norms.items() if k not in zero and abs(got[k] - w) > 2e-3 * abs(w) + 1e-6}
    assert not bad, bad
    for key in [k for k in G.files if k.startswith("slice:")]:
        mname, n = key[6:].split(".", 1)
        g = dict(mods[mname].named_parameters())[n].grad.reshape(-1)[:96].numpy()
        assert np.abs(g - G[key]).max() <= 1e-4 * (np.abs(G[key]).max() + 1e-8), key


def test_within_batch_default_task_is_cross_entropy_and_scanqa_needs_multi_hot():
    g = torch.Generator().manual_seed(3)
    o, t = torch.randn(3, 10, 64, generator=g), torch.randn(3, 64, generator=g)
    masks = torch.arange(10)[None] < torch.tensor([10, 6, 3])[:, None]
    dd = {"intra_obj_embeds": o, "intra_text_embed": t, "obj_masks": masks, "tgt_object_id": torch.tensor([[4], [5], [0]])}
    logits = torch.einsum("bod,bd->bo", F.normalize(o, dim=-1), F.normalize(t, dim=-1)).masked_fill(~masks, -float("inf"))
    want = F.cross_entropy(logits, dd["tgt_object_id"].squeeze(-1))
    for cfg_task in (None, "SQA3D", "Pretrain"):
        total, parts = losses.Loss(["TextObjWithinBatch"], task=cfg_task)(dict(dd))
        assert torch.equal(parts["TextObjWithinBatch"], want), cfg_task
    with pytest.raises(ValueError, match="multi-hot"):
        losses.Loss(["TextObjWithinBatch"], task="ScanQA")(dict(dd))
    multi = torch.zeros(3, 10, dtype=torch.int64)
    multi[0, 4] = multi[1, 2] = multi[1, 5] = multi[2, 3] = 1            # row 2: the masked placeholder slot only
    raw = torch.einsum("bod,bd->bo", F.normalize(o, dim=-1), F.normalize(t, dim=-1))
    want_bce = F.binary_cross_entropy_with_logits(raw, multi.float(), weight=masks.float(), reduction="sum") / 3
    _, parts = losses.Loss(["TextObjWithinBatch"], task="ScanQA")(dict(dd, tgt_object_id=multi))
    assert torch.allclose(parts["TextObjWithinBatch"], want_bce, rtol=1e-6, atol=0)


def test_qa_configs_and_batch():
    from sceneverse_b200 import model as M
    for fn, task, n_ans, ll in ((M.scanqa_config, "ScanQA", 8864, ["answer_loss", "TextObjWithinBatch"]),
                                (M.sqa3d_config, "SQA3D", 706, ["answer_loss"])):
        c = M.to_cfg(fn(2))
        assert c.task == task and c.num_gpu == 2 and c.model.loss_list == ll and c.model.vis_loss_list == ll
        assert c.solver.lr == 1e-4 and c.solver.grad_norm == 5.0 and list(c.solver.optim.args.betas) == [0.9, 0.98]
        assert c.solver.sched.args.warmup_steps == 5000
        assert (c.model.language.lr, c.model.vision.lr, c.model.grounding.lr) == (1e-5, 1e-4, 1e-4)
        assert c.model.vision.args.freeze and c.model.inter == "before" and not c.data.args.use_scene_cap
        assert c.model.heads.head_list == ["qa_head"] and c.model.heads.qa_head.name == "QAHeadV1"
        assert dict(c.model.heads.qa_head.args) == {"hidden_size": 768, "mlp_size": 256, "glimpse": 1, "flat_out_size": 512,
                                                    "num_answers": n_ans}
    # scene_batch is unchanged by the new max_obj argument; the QA targets come from their own stream
    a, b = synthetic.scene_batch(5, B=6, O=12, P=64, L=20, Ls=30), synthetic.qa_batch(5, "SQA3D", B=6, O=12, P=64, L=20, Ls=30,
                                                                                      num_answers=706)
    assert all(np.array_equal(a[k], b[k]) for k in a)
    d = synthetic.qa_batch(4, "ScanQA", B=64, O=20, P=32, L=20, Ls=30, num_answers=706)
    ans, tgt, m = d["answer_label"], d["tgt_object_id"], d["obj_masks"]
    assert ans.dtype == np.int64 and tgt.dtype == np.int64 and tgt.shape == (64, 20)
    assert set(np.unique(ans.sum(1))) <= {0, 1, 2, 3} and 0 < (ans.sum(1) == 0).sum() < 20
    n = m.sum(1)
    assert (n < 20).all() and (tgt.sum(1) >= 1).all()
    placeholder = tgt[np.arange(64), n] == 1
    assert placeholder.any() and (tgt[placeholder].sum(1) == 1).all()
    assert (tgt[~placeholder] * ~m[~placeholder]).sum() == 0        # real targets are valid objects


_VALIDATION = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from sceneverse_b200 import _lib
lib = _lib.gps()
a = 0x1000      # 16-byte aligned fake address


def bce(x=a, rs=712, bf=1, y=a, w=a, R=4, C=706, rows=a, out=a, cnt=a, g=a, gs=712):
    return lib.sv_bce_logits_fwd_bwd(x, rs, bf, y, w, R, C, rows, out, cnt, g, gs, None)


def fwd(s=a, srs=8, x=a, xbs=50 * 768, xrs=768, m=a, B=2, L=50, D=768, p=a, out=a):
    return lib.sv_attn_pool_fwd(s, srs, x, xbs, xrs, m, B, L, D, p, out, None)


def bwd(g=a, grs=768, p=a, x=a, xbs=50 * 768, xrs=768, m=a, B=2, L=50, D=768, dx=a, ds=a, srs=8):
    return lib.sv_attn_pool_bwd(g, grs, p, x, xbs, xrs, m, B, L, D, dx, ds, srs, None)


out = {"bce R 0": bce(R=0), "bce C 0": bce(C=0), "bce row stride < C": bce(rs=700), "bce grad stride < C": bce(gs=700),
       "bce NULL logits": bce(x=None), "bce NULL labels": bce(y=None), "bce NULL rows": bce(rows=None),
       "bce NULL out": bce(out=None), "bce NULL counter": bce(cnt=None), "bce misaligned labels": bce(y=a + 4),
       "bce misaligned bf16 logits": bce(x=a + 1), "bce misaligned f32 logits": bce(bf=0, x=a + 2),
       "bce misaligned grad": bce(g=a + 1), "bce misaligned counter": bce(cnt=a + 2)}
for name, f in (("fwd", fwd), ("bwd", bwd)):
    out.update({f"{name} B 0": f(B=0), f"{name} L 0": f(L=0), f"{name} L > 8192": f(L=8193, xbs=8193 * 768),
                f"{name} D % 8": f(D=764, xrs=764, xbs=50 * 764), f"{name} D 0": f(D=0),
                f"{name} x row stride < D": f(xrs=760), f"{name} x row stride % 8": f(xrs=772, xbs=50 * 772),
                f"{name} x batch stride small": f(xbs=768), f"{name} misaligned x": f(x=a + 8), f"{name} NULL x": f(x=None)})
out.update({"fwd NULL score": fwd(s=None), "fwd score stride 0": fwd(srs=0), "fwd NULL p": fwd(p=None),
            "fwd NULL pooled": fwd(out=None), "fwd misaligned pooled": fwd(out=a + 8), "fwd misaligned p": fwd(p=a + 2),
            "bwd NULL dscore": bwd(ds=None), "bwd NULL dpooled": bwd(g=None), "bwd misaligned dpooled": bwd(g=a + 8),
            "bwd dpooled stride < D": bwd(grs=760), "bwd NULL p": bwd(p=None), "bwd NULL dx": bwd(dx=None),
            "bwd misaligned dx": bwd(dx=a + 8)})
print(json.dumps(out))
"""


def test_qa_entry_points_validate_arguments_without_gpu():
    """sv_bce_logits_fwd_bwd and sv_attn_pool_fwd / _bwd reject malformed calls before any launch (1 = SV_ERR_INVALID_ARG).
    The calls run in a process that sees no CUDA device: a missing check would reach the launch and return 2 instead."""
    res = subprocess.run([sys.executable, "-c", _VALIDATION, ROOT], capture_output=True, text=True, timeout=120,
                         env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    bad = {k: v for k, v in got.items() if v != 1}
    assert len(got) == 14 + 2 * 10 + 13 and not bad, bad


# ---- GPU: BCE with logits -------------------------------------------------------------------------------------------------
def _bce_case(dtype, padded, seed=0, R=48, C=706):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    W = (C + 7) // 8 * 8 if padded else C
    x = torch.randn(R, W, device=dev, generator=g) * 4
    big = torch.rand(R, W, device=dev, generator=g) < 0.05
    x[big] = (torch.rand(int(big.sum()), device=dev, generator=g) * 200 - 100)      # |x| up to 100
    x[0, :4] = torch.tensor([100.0, -100.0, 0.0, -0.0])
    x[:, C:] = 0
    x = x.to(dtype)
    y = (torch.rand(R, C, device=dev, generator=g) < 0.01).long()
    y[0, :2] = 1                                                                       # saturated correct / wrong
    y[3] = 0                                                                           # all-zero label rows
    y[7] = 0
    w = torch.rand(R, C, device=dev, generator=g) < 0.8
    return x, y, w, C


def _bce_reference(x, y, w, C):
    xd, yd = x[:, :C].double(), y.double()
    wd = torch.ones_like(xd) if w is None else w.double()
    terms = wd * (xd.clamp(min=0) - xd * yd + torch.log1p(torch.exp(-xd.abs())))
    scale = wd * (xd.clamp(min=0) + (xd * yd).abs() + torch.log1p(torch.exp(-xd.abs())))
    return terms, scale, wd * (torch.sigmoid(xd) - yd)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_bce_kernel_vs_float64(dtype, padded, weighted):
    """Loss: each term costs a few fp32 roundings (exp, log1p, the products) relative to max(x,0) + |x y| + log1p(.), then a
    stripe sum over C / 256 + 8 warp terms per row and the same over the rows: bound (6 u32 + gamma(chain)) * sum of those
    magnitudes / R.  Gradient: sigmoid in fp32 (absolute error <= 4 u32), one rounding of the stored value to the logits
    dtype and one of the in-place scale by 1/R: bound |ref| (2 u + 4 u32) + 4 u32 / R.  Pad columns are exactly 0; two runs
    are bitwise equal."""
    from sceneverse_b200 import _lib, ops
    x, y, w, C = _bce_case(dtype, padded)
    w = w if weighted else None
    R, W = x.shape
    leaf = x.clone().requires_grad_(True)
    logits = leaf[:, :C] if padded else leaf
    if padded:
        logits._sv_padded = leaf
    n0 = _lib.launch_count()
    loss = ops.bce_with_logits_sum(logits, y, w)
    assert _lib.launch_count() == n0 + 1
    loss.backward()
    terms, mags, gref = _bce_reference(x, y, w, C)
    chain = math.ceil(C / 256) + 12 + math.ceil(R / 256) + 12 + 2     # stripe + warp (5) + block (7) adds, twice; scale
    tol = (6 * U32 + gamma(chain)) * float(mags.sum()) / R
    err = abs(float(loss) - float(terms.sum()) / R)
    assert err <= tol, (err, tol)
    u = UBF if dtype == torch.bfloat16 else U32
    gd = leaf.grad[:, :C].double()
    gtol = (gref / R).abs() * (2 * u + 4 * U32) + 4 * U32 / R
    gerr = (gd - gref / R).abs()
    assert (gerr <= gtol).all(), float((gerr / gtol).max())
    if padded:
        assert torch.count_nonzero(leaf.grad[:, C:]) == 0
    assert not torch.isnan(leaf.grad).any() and torch.isfinite(loss)
    leaf2 = x.clone().requires_grad_(True)
    logits2 = leaf2[:, :C] if padded else leaf2
    if padded:
        logits2._sv_padded = leaf2
    loss2 = ops.bce_with_logits_sum(logits2, y, w)
    loss2.backward()
    assert torch.equal(loss, loss2) and torch.equal(leaf.grad, leaf2.grad)
    print(f"BCE {dtype} padded={padded} weighted={weighted}: loss err / bound {err / tol:.3g}, "
          f"grad err / bound {float((gerr / gtol).max()):.3g}")


@pytest.mark.gpu
def test_bce_weight_mask_knockout():
    """The ScanQA within-batch form: dropping obj_masks from the loss moves it far outside the bound of the weighted loss."""
    from sceneverse_b200 import ops
    dev = torch.device("cuda", 0)
    d = synthetic.qa_batch(2, "ScanQA", B=32, O=80, P=16, L=20, Ls=20, num_answers=706)
    y, m = torch.from_numpy(d["tgt_object_id"]).to(dev), torch.from_numpy(d["obj_masks"]).to(dev)
    x = (torch.randn(32, 80, device=dev, generator=torch.Generator(device=dev).manual_seed(1))).to(torch.bfloat16)
    terms, mags, _ = _bce_reference(x, y, m, 80)
    tol = (6 * U32 + gamma(1 + 12 + 1 + 12 + 2)) * float(mags.sum()) / 32
    good = abs(float(ops.bce_with_logits_sum(x, y, m)) - float(terms.sum()) / 32)
    knocked = abs(float(ops.bce_with_logits_sum(x, y)) - float(terms.sum()) / 32)
    assert good <= tol and knocked > 1e3 * tol, (good, knocked, tol)


# ---- GPU: attention pool --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 37, 50, 80])
@pytest.mark.parametrize("masked", [False, True])
def test_attention_pool_vs_float64(L, masked):
    """Rows: no mask, a partial mask, a single valid token, everything masked (uniform weights 1/L, zero score gradient, no
    NaN).  x is a strided view (row stride 832).  Bounds: one bf16 rounding of each output plus fp32 accumulation,
    gamma(L + 16) (pooled) or gamma(D / 8 + 32 + L) (score gradient: dot products over D, then the sum over L), times the
    sums of absolute values; 8 u32 for exp / division in the softmax weights."""
    from sceneverse_b200 import _lib, ops
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(L)
    B, D = 4, 768
    base = torch.randn(B, L, 832, device=dev, generator=g).to(torch.bfloat16)
    xl = base.clone().requires_grad_(True)
    x = xl[:, :, 32:32 + D]
    sp = torch.zeros(B, L, 8, device=dev, dtype=torch.bfloat16)
    sp[..., 0] = (torch.randn(B, L, device=dev, generator=g) * 3).to(torch.bfloat16)
    sp = sp.requires_grad_(True)
    scores = sp[..., :1]
    scores._sv_padded = sp
    pad = None
    if masked:
        pad = torch.zeros(B, L, dtype=torch.bool, device=dev)
        pad[1, L // 2:] = True
        pad[2, 1:] = True
        pad[3, :] = True
    n0 = _lib.launch_count()
    pooled = ops.attention_pool(scores, x, pad)
    dp = torch.randn(B, D, device=dev, generator=g).to(torch.bfloat16)
    pooled.backward(dp)
    assert _lib.launch_count() == n0 + 2
    s = sp[..., 0].detach().double()
    if pad is not None:
        s = s.masked_fill(pad, -1e9)
    p = torch.softmax(s, dim=1)
    xd, dpd = x.detach().double(), dp.double()
    want = torch.einsum("bl,bld->bd", p, xd)
    absacc = torch.einsum("bl,bld->bd", p, xd.abs())
    tol = want.abs() * UBF + (gamma(L + 16) + 8 * U32) * absacc
    assert ((pooled.double() - want).abs() <= tol).all()
    dx_want = p[:, :, None] * dpd[:, None, :]
    dx_tol = dx_want.abs() * (UBF + 10 * U32)
    assert ((xl.grad[:, :, 32:32 + D].double() - dx_want).abs() <= dx_tol).all()
    assert torch.count_nonzero(xl.grad[:, :, :32]) == 0 and torch.count_nonzero(xl.grad[:, :, 32 + D:]) == 0
    dots = torch.einsum("bld,bd->bl", xd, dpd)
    mags = torch.einsum("bld,bd->bl", xd.abs(), dpd.abs())
    c = (p * dots).sum(1, keepdim=True)
    ds_want = p * (dots - c)
    if pad is not None:
        ds_want = ds_want.masked_fill(pad, 0.0)
    ds_tol = ds_want.abs() * UBF + (gamma(D // 8 + 32 + L) + 8 * U32) * p * (mags + (p * mags).sum(1, keepdim=True))
    ds = sp.grad[..., 0].double()
    assert ((ds - ds_want).abs() <= ds_tol).all(), float(((ds - ds_want).abs() / ds_tol).max())
    assert torch.count_nonzero(sp.grad[..., 1:]) == 0
    assert not torch.isnan(pooled).any() and not torch.isnan(xl.grad).any() and not torch.isnan(sp.grad).any()
    if masked:
        assert torch.equal(p[3], torch.full_like(p[3], 1.0 / L))     # the reference's -1e9: uniform weights, checked above
        assert torch.count_nonzero(sp.grad[3]) == 0                   # fully masked row: no score gradient
        assert torch.count_nonzero(sp.grad[2]) == 0                   # one valid token: p = 1, dscore = dot - dot = 0


# ---- GPU: QAHeadV1 in bf16 ------------------------------------------------------------------------------------------------
HEAD_OUT_TOL = 1e-2        # max |err| / max |ref|; measured 5.7e-3 on an H100 80GB HBM3 (700 W)
HEAD_GRAD_TOL = 2e-2       # relative Frobenius error of each parameter gradient; measured 1.18e-2 (same card)


@pytest.mark.gpu
def test_qa_head_bf16_gpu(monkeypatch):
    """The head under bf16 autocast on the native path (GEMMs, fused LayerNorm, attention pool) against the reference head's
    stored output, and its parameter gradients against fp32 CPU autograd of the same module.  The torch pooling may not run."""
    from sceneverse_b200 import ops

    def no_fallback(*a, **k):
        raise AssertionError("attention_pool fell back to torch")
    cpu = heads.QAHeadV1(None, num_answers=200).eval()
    cpu.load_state_dict(weights.synthetic_state_dict(cpu, seed=11))
    gpu = heads.QAHeadV1(None, num_answers=200).eval()
    gpu.load_state_dict(weights.synthetic_state_dict(gpu, seed=11))
    gpu = gpu.cuda()
    g = torch.Generator().manual_seed(0)
    obj, txt = torch.randn(3, 20, 768, generator=g), torch.randn(3, 12, 768, generator=g)
    om = torch.rand(3, 20, generator=g) > 0.3
    om[:, 0] = True
    tm = torch.arange(12)[None, :] < torch.tensor([12, 5, 9])[:, None]
    gout = torch.randn(3, 200, generator=torch.Generator().manual_seed(1))
    want = np.load(os.path.join(GOLDEN, "qa_head_v1.npz"))["out"]
    ref = cpu(obj, om, txt, tm)
    ref.backward(gout)
    monkeypatch.setattr(ops, "_attention_pool_torch", no_fallback)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = gpu(obj.cuda(), om.cuda(), txt.cuda(), tm.cuda())
    out.float().backward(gout.cuda())
    out_err = float(np.abs(out.float().cpu().detach().numpy() - want).max() / np.abs(want).max())
    grad_err = {}
    for (n, pc), (_, pg) in zip(cpu.named_parameters(), gpu.named_parameters()):
        if n.endswith("mlp.linear.bias"):
            continue        # mathematically zero (softmax is shift invariant): rounding noise in both
        grad_err[n] = float((pg.grad.cpu().double() - pc.grad.double()).norm() / pc.grad.double().norm())
    worst = max(grad_err.items(), key=lambda kv: kv[1])
    print("QA_HEAD_BF16 " + json.dumps({"out_err": out_err, "worst_grad": worst}))
    assert out_err < HEAD_OUT_TOL, out_err
    assert worst[1] < HEAD_GRAD_TOL, worst


# ---- GPU: whole bf16 backward against the reference fixture ----------------------------------------------------------------
# measured on an H100 80GB HBM3 (700 W): loss terms 1.2e-4 relative, worst gradient-norm deviation 4.4e-3
QA_LOSS_TOL, QA_NORM_TOL, QA_FLOOR = 3e-4, 7e-3, 1e-3


@pytest.mark.gpu
def test_qa_backward_matches_reference_gradients_gpu_bf16():
    G = np.load(os.path.join(GOLDEN, "model_qa_grads.npz"))
    want_norms = json.load(open(os.path.join(GOLDEN, "model_qa_grad_norms.json")))
    d, txt, obj = golden_inputs(G)
    t = {k: torch.from_numpy(v).cuda() for k, v in d.items()}
    mods = qa_stack(G, "cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, parts = run_stack(mods, t, txt.cuda(), obj.cuda())
        total = sum(parts.values())
    loss_err = {k: abs(float(v) - float(G["loss_" + k])) / max(1.0, abs(float(G["loss_" + k]))) for k, v in parts.items()}
    total.backward()
    got = grad_norms(mods)
    scale = max(want_norms.values())
    worst, bad = (0.0, None), {}
    for k, w in want_norms.items():
        gk = got.get(k, 0.0)
        if abs(w) > QA_FLOOR * scale:
            worst = max(worst, (abs(gk - w) / abs(w), k), key=lambda v: v[0])
        if abs(gk - w) > QA_NORM_TOL * abs(w) + QA_FLOOR * scale:
            bad[k] = (gk, w)
    res = {"loss_err": loss_err, "worst_grad_norm_dev": worst[0], "worst_param": worst[1], "params": len(want_norms)}
    print("QA_GRAD_PARITY_BF16 " + json.dumps(res))
    for k, e in loss_err.items():
        assert e < QA_LOSS_TOL, (k, e)
    assert not bad, bad


# ---- GPU: training steps --------------------------------------------------------------------------------------------------
def _qa_step(config, graph, no_dropout=True, seed=3):
    from sceneverse_b200 import model as M, train
    tf = weights.synthetic_tensor("text_features", (607, 768))
    cfg = getattr(M, config)(1, text_features=tf)
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 0      # lr factor 1 from the first step
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=seed, cuda_graph=graph)
    if no_dropout:
        for m in ps.module.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
            if hasattr(m, "dropout") and isinstance(m.dropout, float):
                m.dropout = 0.0
            if isinstance(m, heads._AttentionPool):
                m.pdrop = 0.0
    return ps


def _qa_batch(config, seed, B=4, O=24):
    task, A = ("ScanQA", 8864) if config == "scanqa_config" else ("SQA3D", 706)
    d = synthetic.qa_batch(seed, task, B=B, O=O, P=1024, L=50, Ls=300, num_answers=A, min_obj=6)
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["scanqa_config", "sqa3d_config"])
def test_qa_eager_steps_decrease_loss(config):
    ps = _qa_step(config, graph=False)
    batch = _qa_batch(config, 11)
    head0 = {n: p.detach().clone() for n, p in ps.module.model.qa_head.named_parameters()}
    got = [float(ps.step(dict(batch))) for _ in range(4)]
    print(config, "eager losses", got)
    assert all(math.isfinite(v) for v in got) and all(b < a for a, b in zip(got, got[1:])), got
    # the score layer's bias has a mathematically zero gradient (the softmax over tokens is shift invariant)
    expect = {n for n in head0 if not n.endswith("mlp.linear.bias")}
    moved = {n for n, p in ps.module.model.qa_head.named_parameters() if not torch.equal(p.detach(), head0[n])}
    assert expect <= moved, expect - moved
    ps.close()


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["scanqa_config", "sqa3d_config"])
def test_qa_graph_replay_reads_new_batch(config):
    """Graph mode: the loss a replay returns for a new batch is that batch's loss under the current parameters (an eager
    forward of the same dropout-free module), not the captured batch's."""
    from sceneverse_b200 import _lib
    ps = _qa_step(config, graph=True)
    a, b = _qa_batch(config, 21), _qa_batch(config, 22)
    la = float(ps.step(dict(a)))
    assert ps.native_launches_per_step > 0 and math.isfinite(la)
    ps.module.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        want_b = float(ps.module(dict(b))[0])
        want_a = float(ps.module(dict(a))[0])
    ps.module.train()
    n0 = _lib.launch_count()
    lb = float(ps.step(dict(b)))
    assert _lib.launch_count() == n0        # a replay: no eager native launch
    print(config, "graph replay", {"captured": want_a, "new batch": want_b, "replay": lb})
    assert abs(lb - want_b) < 0.1 * abs(want_b - want_a) and abs(lb - want_b) < 1e-3 * abs(want_b), (lb, want_b, want_a)
    ps.close()


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["scanqa_config", "sqa3d_config"])
def test_qa_graph_step_matches_eager_step_parameters(config):
    """One step through the captured path's flat state (what the graph records) moves every parameter like the eager step:
    same sign on the coordinates whose gradient is far above the bf16 noise, and the same mean step size."""
    from sceneverse_b200 import ops
    batch = _qa_batch(config, 9)
    eager, graph = _qa_step(config, False), _qa_step(config, True)
    graph.module.load_state_dict(eager.module.state_dict())
    p0 = {n: p.detach().clone() for n, p in eager.module.named_parameters()}
    eager._probe_unused(dict(batch))
    graph._probe_unused(dict(batch))
    eager.step(dict(batch))
    graph.static_batch = {k: v.clone() for k, v in batch.items()}
    graph._make_flat_state()
    graph._raw_step()
    ops.clear_shadows()
    worst, checked, qa = (1.0, None), 0, 0
    for (n, pe), (_, pg) in zip(eager.module.named_parameters(), graph.module.named_parameters()):
        if not pe.requires_grad or pe.grad is None:
            continue
        ge = pe.grad.float()
        big = ge.abs() > 0.2 * ge.abs().max()
        if big.sum() == 0 or ge.abs().max() == 0 or n.endswith("mlp.linear.bias"):
            continue
        de, dg = (pe.detach() - p0[n]).float(), (pg.detach() - p0[n]).float()
        agree = (torch.sign(de[big]) == torch.sign(dg[big])).float().mean().item()
        ratio = (dg[big].abs().mean() / (de[big].abs().mean() + 1e-20)).item()
        worst = min(worst, (agree, n), key=lambda v: v[0])
        checked += 1
        qa += n.startswith("model.qa_head.")
        assert agree > 0.98 and 0.9 < ratio < 1.1, (n, agree, ratio)
    assert checked > 100 and qa >= 14, (checked, qa)
    print(config, "GRAPH_VS_EAGER worst sign agreement", worst, "parameters checked", checked)
    eager.close()
    graph.close()
