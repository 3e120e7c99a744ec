"""The object-classification and multi-target grounding losses on the GPU: sv_masked_cross_entropy_fwd_bwd against float64
with per-element bounds, its reproducibility under launches and graph replays, a mask knockout, the ScanRefer and GPS
training steps with the new losses in their loss lists, and the two BCE losses against torch."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sceneverse_b200 import evaluate, model as M, synthetic, train, weights
from sceneverse_b200.modules import heads, losses
from tests.test_train_logs_gpu import Stash, check_entry, ref_scanrefer_metrics, scanrefer_batches

pytestmark = pytest.mark.gpu
U32, UBF = 2.0 ** -24, 2.0 ** -8
V = 607


def gamma(n):
    return n * U32 / (1 - n * U32)


def _case(dtype, padded, B=16, O=80, seed=0):
    """(B, O, V) logits (a 608-wide padded parent when `padded`), labels with -100 at the padded slots, obj / sem masks."""
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    W = 608 if padded else V
    x = torch.zeros(B, O, W, device=dev)
    x[..., :V] = torch.randn(B, O, V, device=dev, generator=g) * 3
    x = x.to(dtype)
    n = torch.randint(O // 4, O + 1, (B,), device=dev, generator=g)
    obj = torch.arange(O, device=dev)[None] < n[:, None]
    obj[0] = True                                                          # a scene without padding
    sem = obj & (torch.rand(B, O, device=dev, generator=g) > 0.25)
    y = torch.randint(0, V, (B, O), device=dev, generator=g).masked_fill(~obj, -100)
    return x, y, obj, sem


def _leaf(x, padded):
    leaf = x.clone().requires_grad_(True)
    view = leaf[..., :V] if padded else leaf
    if padded:
        view._sv_padded = leaf
    return leaf, view


def _weight(obj, sem, mode):
    return obj if mode == 0 else (obj & ~sem if mode == 1 else obj & sem)


def _reference(x, y, w):
    """float64: per-row CE, logsumexp, probabilities, and the gradient of sum(w CE) / sum(w)."""
    xd = x[..., :V].double()
    lse = torch.logsumexp(xd, dim=2)
    yc = y.clamp(min=0)
    xl = xd.gather(2, yc[..., None])[..., 0]
    live = w & (y >= 0)
    ce = torch.where(live, lse - xl, torch.zeros_like(lse))
    p = torch.softmax(xd, dim=2)
    onehot = F.one_hot(yc, V).double()
    n = float(w.sum())
    grad = (p - onehot) * live[..., None] / n
    return ce, lse, xl, p, grad, n


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_masked_ce_kernel_vs_float64(dtype, padded, mode):
    """Loss: each row costs the fp32 max / exp / log of its logsumexp (fast intrinsics: at most 64 u32 relative to
    |lse| + |x_label| + 1), then the fixed-order sums over 256 threads, 8 warps and the rows: bound
    sum_r w_r (64 u32 (|lse| + |x_label| + 1) + gamma(R / 256 + 24) CE_r) / sum_r w_r.  Gradient: the probability in fp32
    (error at most (48 + 1.2 |x - max|) u32 relative to p), one rounding of the stored value to the logits dtype and one of
    the in-place division: |ref| 2 u + p (48 + 1.2 |x - max|) u32 / sum w.  Pad columns and rows of weight 0 are exactly
    zero; one native launch in the forward."""
    from sceneverse_b200 import _lib, ops
    x, y, obj, sem = _case(dtype, padded, seed=mode)
    leaf, logits = _leaf(x, padded)
    n0 = _lib.launch_count()
    loss = ops.masked_cross_entropy(logits, y, obj, None if mode == 0 else sem, mode)
    assert _lib.launch_count() == n0 + 1
    loss.backward()
    w = _weight(obj, sem, mode)
    ce, lse, xl, p, gref, n = _reference(x, y, w)
    R = y.numel()
    want = float(ce.sum()) / n
    tol = float((64 * U32 * (lse.abs() + xl.abs() + 1) * w).sum() + gamma(R / 256 + 24) * ce.sum()) / n
    err = abs(float(loss) - want)
    assert err <= tol, (err, tol)
    u = UBF if dtype == torch.bfloat16 else U32
    xd = x[..., :V].double()
    spread = xd - xd.max(dim=2, keepdim=True).values
    gtol = gref.abs() * 2 * u + p * (48 + 1.2 * spread.abs()) * U32 / n * w[..., None]
    gd = leaf.grad[..., :V].double()
    gerr = (gd - gref).abs()
    assert (gerr <= gtol).all(), float((gerr / gtol.clamp(min=1e-30)).max())
    assert torch.count_nonzero(leaf.grad[~w]) == 0
    if padded:
        assert torch.count_nonzero(leaf.grad[..., V:]) == 0
    print(f"masked CE {dtype} padded={padded} mode={mode}: loss err / bound {err / tol:.3g}, "
          f"grad err / bound {float((gerr / gtol.clamp(min=1e-30)).max()):.3g}")


def test_zero_weight_sum_is_nan():
    """The `_mask` split of a batch whose valid objects are all semantically masked has no member: 0 / 0 = NaN, as torch."""
    from sceneverse_b200 import ops
    x, y, obj, _ = _case(torch.bfloat16, True)
    _, logits = _leaf(x, True)
    assert torch.isnan(ops.masked_cross_entropy(logits, y, obj, obj.clone(), mode=1))
    want = (F.cross_entropy(x[..., :V].float().permute(0, 2, 1), y, reduction="none") * obj * obj.logical_not()).sum() / \
        (obj * obj.logical_not()).sum()
    assert torch.isnan(want)


def test_no_gradient_buffer_for_detached_logits():
    """obj_cls_raw_logits (detached probabilities, f32): the loss alone, nothing to differentiate."""
    from sceneverse_b200 import ops
    x, y, obj, _ = _case(torch.float32, False)
    p = torch.softmax(x, dim=2)
    loss = ops.masked_cross_entropy(p, y, obj)
    assert not loss.requires_grad
    want = (F.cross_entropy(p.double().permute(0, 2, 1), y, reduction="none") * obj).sum() / obj.sum()
    assert abs(float(loss) - float(want)) <= 1e-5 * float(want)


def _raw_call(x, y, obj, sem, mode, counter):
    """The entry point directly: (loss_rows, sums, loss, unscaled gradient)."""
    from sceneverse_b200 import _lib
    R, W = y.numel(), x.shape[-1]
    rows = torch.empty(R, device=x.device)
    sums = torch.empty(2, device=x.device)
    out = torch.empty((), device=x.device)
    g = torch.empty((R, W), dtype=x.dtype, device=x.device)
    _lib.call(_lib.gps(), "sv_masked_cross_entropy_fwd_bwd", x.device, x.data_ptr(), W, 1 if x.dtype == torch.bfloat16 else 0,
              y.data_ptr(), obj.view(torch.uint8).data_ptr(), sem.view(torch.uint8).data_ptr(), mode, R, V, rows.data_ptr(),
              sums.data_ptr(), out.data_ptr(), counter.data_ptr(), g.data_ptr(), W)
    return rows, sums, out, g


def test_launches_and_graph_replays_are_bitwise_equal():
    x, y, obj, sem = _case(torch.bfloat16, True, seed=3)
    x, y, obj, sem = x.contiguous(), y.contiguous(), obj.contiguous(), sem.contiguous()
    counter = torch.zeros(1, dtype=torch.int32, device=x.device)
    a = _raw_call(x, y, obj, sem, 2, counter)
    b = _raw_call(x, y, obj, sem, 2, counter)
    assert all(torch.equal(s, t) for s, t in zip(a, b))
    assert int(counter) == 0
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _raw_call(x, y, obj, sem, 2, counter)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = _raw_call(x, y, obj, sem, 2, counter)
    for _ in range(3):
        for t in c:
            t.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(s_, t) for s_, t in zip(a, c))
    assert int(counter) == 0


def test_mask_knockout_changes_one_row_and_the_normaliser():
    """Clearing one obj_masks byte zeroes exactly that row's loss and unscaled gradient, lowers the weight sum by exactly 1
    and leaves every other row bitwise unchanged."""
    x, y, obj, sem = _case(torch.bfloat16, True, seed=4)
    counter = torch.zeros(1, dtype=torch.int32, device=x.device)
    rows, sums, _, g = _raw_call(x, y, obj, sem, 0, counter)
    b, o = 5, 2
    assert bool(obj[b, o]) and int(y[b, o]) >= 0
    obj2 = obj.clone()
    obj2[b, o] = False
    rows2, sums2, out2, g2 = _raw_call(x, y, obj2, sem, 0, counter)
    r = b * obj.shape[1] + o
    keep = torch.ones(rows.numel(), dtype=torch.bool, device=x.device)
    keep[r] = False
    assert torch.equal(rows[keep], rows2[keep]) and torch.equal(g[keep], g2[keep])
    assert float(rows[r]) > 0 and float(rows2[r]) == 0 and torch.count_nonzero(g2[r]) == 0 and torch.count_nonzero(g[r]) > 0
    assert float(sums[1]) - float(sums2[1]) == 1.0
    assert abs(float(sums2[0]) - (float(sums[0]) - float(rows[r]))) <= 1e-5 * float(sums[0])
    assert torch.equal(out2, sums2[0] / sums2[1])


# ---- training steps ---------------------------------------------------------------------------------------------------------
AUX = ["og3d_loss", "obj_cls_raw_loss", "obj_cls_pre_loss", "obj_cls_post_loss"]


def _tf():
    return weights.synthetic_tensor("text_features", (607, 768))


def _no_dropout(ps):
    for m in ps.module.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
        if hasattr(m, "dropout") and isinstance(m.dropout, float):
            m.dropout = 0.0


def _scanrefer_step(graph, loss_list=AUX, seed=3, detach=True, **kw):
    cfg = M.scanrefer_config(1, text_features=_tf())
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 0
    cfg["model"]["loss_list"] = cfg["model"]["vis_loss_list"] = list(loss_list)
    cfg["model"]["heads"]["ground_head"]["args"]["detach_all_aux_loss"] = detach
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=seed, cuda_graph=graph, **kw)
    _no_dropout(ps)
    return ps


def _batch(seed, B=4, O=24):
    d = synthetic.scene_batch(seed, B=B, O=O, P=1024, L=50, min_obj=6)
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def test_scanrefer_eager_steps_lower_the_aux_losses():
    """Four eager steps on one batch: obj_cls_pre_loss and obj_cls_post_loss fall at every step (their heads train);
    obj_cls_raw_loss reads the frozen encoder's detached class probabilities, so it stays where it is."""
    ps = _scanrefer_step(False)
    stash = Stash(ps)
    batch = _batch(11)
    seen = []
    for _ in range(4):
        ps.step(dict(batch))
        seen.append({k: float(v) for k, v in stash.losses.items()})
    print("eager aux losses", seen)
    for k in ("og3d_loss", "obj_cls_pre_loss", "obj_cls_post_loss", "total_loss"):
        vals = [s[k] for s in seen]
        assert all(math.isfinite(v) for v in vals) and all(b < a for a, b in zip(vals, vals[1:])), (k, vals)
    raw = [s["obj_cls_raw_loss"] for s in seen]
    assert math.isfinite(raw[0]) and max(raw) - min(raw) <= 1e-6 * raw[0], raw
    ps.close()


def test_aux_heads_train_and_the_encoders_get_no_gradient_from_them():
    """With only the aux losses in the list, the probe finds no gradient in any encoder (detach_all_aux_loss), and the two
    object heads are trainable; without the detach the encoders do receive it."""
    batch = _batch(5)
    ps = _scanrefer_step(False, loss_list=["obj_cls_pre_loss", "obj_cls_post_loss"])
    ps._probe_unused(dict(batch))
    unused = set(ps.unused_parameters)
    trainable = {n for n, p in ps.module.named_parameters() if p.requires_grad}
    enc = ("model.lang_encoder.", "model.unified_encoder.", "model.point_encoder.")
    assert not any(n.startswith(enc) for n in trainable), sorted(n for n in trainable if n.startswith(enc))[:5]
    heads_ = {n for n, _ in ps.module.named_parameters()
              if n.startswith(("model.ground_head.obj3d_clf_head.", "model.ground_head.obj3d_clf_pre_head."))}
    assert heads_ and heads_ <= trainable and not (heads_ & unused)
    ps.close()
    ps = _scanrefer_step(False, loss_list=["obj_cls_pre_loss", "obj_cls_post_loss"], detach=False)
    ps._probe_unused(dict(batch))
    trainable = {n for n, p in ps.module.named_parameters() if p.requires_grad}
    assert any(n.startswith("model.unified_encoder.") for n in trainable)
    ps.close()


def test_scanrefer_graph_step_matches_eager_step_parameters():
    """One step through the captured path's flat state moves every parameter like the eager step (the QA tests' criterion:
    sign agreement above 0.98 on the coordinates with large gradients and a mean step ratio within 10 %), the aux heads
    included."""
    from sceneverse_b200 import ops
    batch = _batch(9)
    eager, graph = _scanrefer_step(False), _scanrefer_step(True)
    graph.module.load_state_dict(eager.module.state_dict())
    p0 = {n: p.detach().clone() for n, p in eager.module.named_parameters()}
    eager._probe_unused(dict(batch))
    graph._probe_unused(dict(batch))
    eager.step(dict(batch))
    graph.static_batch = {k: v.clone() for k, v in batch.items()}
    graph._make_flat_state()
    graph._raw_step()
    ops.clear_shadows()
    checked, aux = 0, 0
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
        aux += n.startswith(("model.ground_head.obj3d_clf_head.", "model.ground_head.obj3d_clf_pre_head."))
        assert agree > 0.98 and 0.9 < ratio < 1.1, (n, agree, ratio)
    assert checked > 100 and aux >= 10, (checked, aux)
    eager.close()
    graph.close()


def test_scanrefer_graph_replay_reads_new_batch_and_logs_the_aux_losses():
    """Graph mode with ScanReferEval: each replay's TrainLog entry holds that replay's loss values (og3d and the three aux
    losses) and metrics; a replay's total for a new batch is that batch's loss under the current parameters; the
    checkpoint carries AdamW moments for the aux heads."""
    from sceneverse_b200 import _lib
    ps = _scanrefer_step(True, train_eval=evaluate.ScanReferEval(), log_every=4)
    stash = Stash(ps)
    batches = scanrefer_batches(2)
    ps.step(batches[0])
    ps.logs()
    for i in range(3):
        loss = ps.step(batches[i % 2])
        (entry,) = ps.logs()
        check_entry(ps, entry, stash, ref_scanrefer_metrics, i + 2, loss)
        assert all(f"train/{k}" in entry and math.isfinite(entry[f"train/{k}"]) for k in AUX)
    a, b = batches[0], _batch(22, O=16)
    for k in ("tgt_object_id_iou25", "tgt_object_id_iou50", "is_multiple", "tgt_object_label"):
        b[k] = a[k]
    ps.module.eval()
    log, ps.module.train_log = ps.module.train_log, None       # these forwards are not training steps
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        want_b = float(ps.module(dict(b))[0])
        want_a = float(ps.module(dict(a))[0])
    ps.module.train_log = log
    ps.module.train()
    n0 = _lib.launch_count()
    lb = float(ps.step(dict(b)))
    assert _lib.launch_count() == n0
    (entry,) = ps.logs()
    print("graph replay", {"captured": want_a, "new batch": want_b, "replay": lb})
    assert abs(lb - want_b) < 0.1 * abs(want_b - want_a) and abs(lb - want_b) < 1e-3 * abs(want_b), (lb, want_b, want_a)
    state = ps.state_dict()["optimizer"]["state"]
    index = {id(p): i for i, p in enumerate(p for g in ps.module.opt_order for p in g)}
    for n, p in ps.module.model.ground_head.named_parameters():
        if n.startswith(("obj3d_clf_head.", "obj3d_clf_pre_head.")) and n.endswith("weight"):
            assert index[id(p)] in state and float(state[index[id(p)]]["exp_avg_sq"].abs().max()) > 0, n
    ps.close()


def test_pretrain_step_trains_the_object_lm_head_with_the_mask_split_losses():
    """GPS pre-training with obj_cls_post_loss_mask / _unmask: the object LM head of OVPretrainHead is no longer frozen as
    unused, and a graph-mode step moves it."""
    cfg = M.pretrain_config(1, text_features=_tf())
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 0
    names = cfg["model"]["loss_list"] + ["obj_cls_post_loss_mask", "obj_cls_post_loss_unmask"]
    cfg["model"]["loss_list"] = cfg["model"]["vis_loss_list"] = names
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=0, cuda_graph=True)
    batch = _batch(13, O=16)
    head0 = {n: p.detach().clone() for n, p in ps.module.model.pretrain_head.obj_pred_head.named_parameters()}
    l0 = float(ps.step(dict(batch)))
    assert not any(".obj_pred_head." in n for n in ps.unused_parameters)
    l1 = float(ps.step(dict(batch)))
    assert math.isfinite(l0) and math.isfinite(l1)
    moved = {n for n, p in ps.module.model.pretrain_head.obj_pred_head.named_parameters() if not torch.equal(p.detach(), head0[n])}
    assert moved == set(head0), set(head0) - moved
    ps.close()


# ---- BCE losses --------------------------------------------------------------------------------------------------------------
def test_og3d_multi_loss_and_txt_cls_multi_loss_match_torch():
    """og3d_multi_loss on a qa-style multi-hot (B, O) target over the finite logits of a model without a ground head, and
    txt_cls_multi_loss on a 608-wide padded text head output: loss and gradient against torch's formulation in float64."""
    from sceneverse_b200 import _lib
    dev = torch.device("cuda", 0)
    d = synthetic.qa_batch(3, "ScanQA", B=32, O=40, P=16, L=20, Ls=20, num_answers=706)
    s = synthetic.scene_batch(3, B=32, O=40, P=16, L=20, Ls=20, multi_label=True)
    g = torch.Generator(device=dev).manual_seed(0)
    og = (torch.randn(32, 40, device=dev, generator=g) * 3).to(torch.bfloat16).requires_grad_(True)
    tp = torch.zeros(32, 608, device=dev)
    tp[:, :V] = torch.randn(32, V, device=dev, generator=g) * 3
    tp = tp.to(torch.bfloat16).requires_grad_(True)
    txt = tp[:, :V]
    txt._sv_padded = tp
    dd = {"og3d_logits": og, "tgt_object_id": torch.from_numpy(d["tgt_object_id"]).to(dev), "txt_cls_logits": txt,
          "tgt_object_label": torch.from_numpy(s["tgt_object_label"]).to(dev)}
    for name, leaf, x, y in (("og3d_multi_loss", og, og, dd["tgt_object_id"]),
                             ("txt_cls_multi_loss", tp, txt, dd["tgt_object_label"])):
        n0 = _lib.launch_count()
        loss = getattr(losses, name)(dd)
        assert _lib.launch_count() == n0 + 1, name
        loss.backward()
        xd = x.detach().double().requires_grad_(True)
        want = F.binary_cross_entropy_with_logits(xd, y.double(), reduction="sum") / 32
        want.backward()
        assert abs(float(loss) - float(want)) <= 1e-5 * abs(float(want)), (name, float(loss), float(want))
        got = leaf.grad[:, :x.shape[1]].double()
        assert ((got - xd.grad).abs() <= xd.grad.abs() * 2 * UBF + 1e-6 / 32).all(), name
        if leaf is tp:
            assert torch.count_nonzero(tp.grad[:, V:]) == 0


def test_og3d_multi_loss_on_the_ground_head_is_nan_with_zero_gradient_at_padded_objects():
    """GroundHeadV1's og3d_logits are -inf at padded objects: the loss is NaN and those entries get a zero gradient, as in
    torch; the valid entries' gradient is finite."""
    dev = torch.device("cuda", 0)
    gh = heads.GroundHeadV1(None, input_size=768, hidden_size=384, sem_cls_size=607).cuda()
    gh.load_state_dict(weights.synthetic_state_dict(gh, seed=4))
    g = torch.Generator(device=dev).manual_seed(1)
    obj = torch.randn(4, 16, 768, device=dev, generator=g).requires_grad_(True)
    txt = torch.randn(4, 10, 768, device=dev, generator=g)
    masks = torch.arange(16, device=dev)[None] < torch.tensor([16, 9, 12, 6], device=dev)[:, None]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, _, _, og = gh(txt, obj, obj, masks)
    tgt = torch.zeros(4, 16, dtype=torch.int64, device=dev)
    tgt[:, 0] = 1
    og.retain_grad()
    loss = losses.og3d_multi_loss({"og3d_logits": og, "tgt_object_id": tgt})
    loss.backward()
    assert torch.isnan(loss)
    assert torch.count_nonzero(og.grad[~masks]) == 0 and torch.isfinite(og.grad[masks]).all()
