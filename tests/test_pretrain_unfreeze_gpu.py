"""GPS pre-training with the object encoder unfrozen (model.pretrain_unfreeze_config, all_pretrain_unfreeze.yaml): PointNet++ trains
inside PretrainStep on the channels-last kernels of pn_train.py, its evaluation reads the current weights, and its checkpoints
move between the stages ObjCls -> unfrozen GPS -> frozen fine-tuning."""
import copy
import gc

import numpy as np
import pytest
import torch

from sceneverse_b200 import model as M, synthetic, train, weights
from tests import test_checkpoint_gpu as ck

pytestmark = pytest.mark.gpu

TF = weights.synthetic_tensor("text_features", (607, 768))
BACKBONE = "point_encoder.point_feature_extractor."


def unfrozen(seed, graph, warmup=2, no_dropout=False, total_steps=50):
    cfg = M.pretrain_unfreeze_config(1, text_features=TF)
    cfg["solver"]["sched"]["args"]["warmup_steps"] = warmup
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=seed, cuda_graph=graph, total_steps=total_steps)
    if no_dropout:
        for m in ps.module.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
            if hasattr(m, "dropout") and isinstance(m.dropout, float):
                m.dropout = 0.0
    return ps


def scene_batches(n, B, O, seed):
    out = []
    for i in range(n):
        d = synthetic.scene_batch(seed + i, B=B, O=O, P=1024, L=50, Ls=300)
        out.append({k: torch.from_numpy(v).cuda() for k, v in d.items()})
    return out


def backbone_of(ps):
    return ps.module.model.point_encoder.point_feature_extractor


def bn_buffers(net):
    return {n: b.detach().clone() for n, b in net.named_buffers()}


def test_step_trains_the_backbone_on_the_native_path_and_matches_the_fp32_operator_sequence():
    """One eager step at 2 scenes x 8 objects against the reference operator sequence in fp32 (forward_generic: torch Conv2d /
    BatchNorm2d / max_pool2d on the native point ops) on the same batch, with the bounds of DESIGN.md §4.8: the backbone's
    features, the loss, every backbone gradient by direction (tightly behind the last max), and the running statistics.  No
    ATen convolution or BatchNorm runs in the native step, and the unused-parameter probe finds the backbone used."""
    from torch.profiler import ProfilerActivity, profile
    ps = unfrozen(0, False, no_dropout=True)
    net = backbone_of(ps)
    ref = copy.deepcopy(net)
    (batch,) = scene_batches(1, 2, 8, 70)
    seen = []

    def keep(_m, _i, out):
        out.retain_grad()
        seen.append(out)
    h = net.register_forward_hook(keep)
    with profile(activities=[ProfilerActivity.CPU]) as prof:
        loss = float(ps.step(dict(batch)))          # the probing forward / backward, then the step
    h.remove()
    ops_run = {e.name for e in prof.events()}
    assert not any(n in ops_run for n in ("aten::convolution", "aten::cudnn_convolution", "aten::batch_norm",
                                          "aten::native_batch_norm", "aten::cudnn_batch_norm")), sorted(ops_run)
    assert np.isfinite(loss)
    named = dict(ps.module.model.named_parameters())
    assert not any(n.startswith("model." + BACKBONE) for n in ps.unused_parameters)
    assert all(p.requires_grad for n, p in named.items() if n.startswith(BACKBONE))
    assert not any(p.requires_grad for n, p in named.items()
                   if n.startswith(("point_encoder.sem_cls_embed_layer.", "point_encoder.sem_mask_embeddings.")))
    y, gy = seen[-1], seen[-1].grad
    x = batch["obj_fts"].float().reshape(-1, 1024, 6)
    ref.train()
    yr = ref.forward_generic(x)                     # the probe's forward: the running statistics advance twice
    yr = ref.forward_generic(x)
    err = (y.float() - yr).abs().max().item() / yr.abs().max().item()
    assert err < 4e-2, err
    yr.backward(gy.float())
    worst = {}
    for (n, p), (_, q) in zip(net.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, n
        e = (p.grad.float() - q.grad).abs().max().item() / (q.grad.abs().max().item() + 1e-8)
        cos = torch.nn.functional.cosine_similarity(p.grad.float().flatten(), q.grad.flatten(), dim=0).item()
        worst[n] = (e, cos)
    # p.grad is clipped to the norm 5.0 (one common factor): directions are compared, and the layers behind the last
    # neighbourhood max tightly after undoing that factor
    scale = net.fc.weight.grad.float().norm().item() / ref.fc.weight.grad.norm().item()
    for n in ("fc.weight", "fc.bias", "encoder.2.mlps.0.layer2.bn.bn.weight", "encoder.2.mlps.0.layer2.bn.bn.bias"):
        p, q = dict(net.named_parameters())[n], dict(ref.named_parameters())[n]
        e = (p.grad.float() / scale - q.grad).abs().max().item() / (q.grad.abs().max().item() + 1e-8)
        assert worst[n][1] > 0.999 and e < 0.1, (n, e, worst[n])
    for n, (e, cos) in worst.items():
        assert cos > 0.8, (n, e, cos)
    for (n, b1), (_, b2) in zip(net.named_buffers(), ref.named_buffers()):
        if "running" in n:
            assert (b1 - b2).abs().max().item() <= 3e-2 * (b2.abs().max().item() + 1e-3), n
        elif "num_batches_tracked" in n:
            assert int(b1) == int(b2) == 2, n
    # the loss with the fp32 reference backbone in place of the native one (same state, no dropout)
    ref2 = copy.deepcopy(net)

    def fp32_backbone(pc):
        with torch.autocast("cuda", enabled=False):
            return ref2.forward_generic(pc)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        got = float(ps.module(dict(batch))[0])
        net.forward = fp32_backbone
        try:
            want = float(ps.module(dict(batch))[0])
        finally:
            del net.forward
    assert abs(got - want) < 2e-2 * abs(want), (got, want)
    print("UNFROZEN parity: features", err, "loss", got, want, "grads", worst)
    ps.close()


def test_graph_steps_match_eager_steps_at_full_size():
    """64 scenes x 80 objects x 1024 points: the captured step (probe, three set-up steps and the replay on the first batch, then
    two replays) against the eager step on the same batches (four steps on the first), dropout-free, from the same weights:
    equal losses, equal BatchNorm buffers and equal backbone updates: the coordinates that moved most move the same way by
    about the same amount, by the criterion of test_graph_step_matches_eager_step_parameters behind the last neighbourhood
    max.  In front of a max over bf16 values, ties route the gradient by the last bits of the run (DESIGN.md §4.8), so over
    six steps a few such coordinates may part (measured on an H100: sign agreement >= 0.978, size ratio 0.918-1.006)."""
    bs = scene_batches(3, 64, 80, 500)
    plan = [0, 0, 0, 0, 1, 2]
    init = None
    res = {}
    for mode in ("graph", "eager"):
        ps = unfrozen(3, mode == "graph", warmup=0, no_dropout=True)
        if init is None:
            init = copy.deepcopy(ps.module.state_dict())
        else:
            ps.module.load_state_dict(init)
        if mode == "graph":
            losses = [float(ps.step(dict(bs[i]))) for i in (0, 1, 2)]
            assert ps.native_launches_per_step > 0
            res["launches"] = ps.native_launches_per_step
        else:
            losses = [float(ps.step(dict(bs[i]))) for i in plan][3:]
        res[mode] = (losses, {n: p.detach().float().clone() for n, p in backbone_of(ps).named_parameters()},
                     bn_buffers(backbone_of(ps)))
        ps.close()
        del ps
        gc.collect()
        torch.cuda.empty_cache()
    (lg, pg, bg), (le, pe, be) = res["graph"], res["eager"]
    assert np.allclose(lg, le, rtol=2e-3), (lg, le)
    p0 = {n: init["model." + BACKBONE + n].float() for n in pe}
    report = {}
    for n in pe:
        de, dg = pe[n] - p0[n], pg[n] - p0[n]
        big = de.abs() > 0.2 * de.abs().max()
        agree = (torch.sign(de[big]) == torch.sign(dg[big])).float().mean().item()
        ratio = (dg[big].abs().mean() / (de[big].abs().mean() + 1e-20)).item()
        report[n] = (round(agree, 4), round(ratio, 4))
    print("UNFROZEN graph vs eager: losses", lg, le, "launches", res["launches"], "backbone updates", report)
    for n, (agree, ratio) in report.items():
        if n.startswith(("fc.", "encoder.2.mlps.0.layer2.")):
            assert agree > 0.98 and 0.9 < ratio < 1.1, (n, agree, ratio)
        else:
            assert agree > 0.95 and 0.85 < ratio < 1.15, (n, agree, ratio)
    for n, b in be.items():
        if "num_batches_tracked" in n:
            assert int(bg[n]) == int(b) == 7, (n, int(bg[n]), int(b))      # probe + 6 steps, in both modes
        else:
            assert (bg[n] - b).abs().max().item() <= 2e-2 * (b.abs().max().item() + 1e-3), n


def test_evaluation_after_replayed_steps_reads_the_current_weights():
    """Evaluate (packs the eval-mode images, captures the runner's graph), train k = 3 more replayed steps, evaluate again:
    the eval-mode forward equals a fresh pack of a deep copy of the current weights and running statistics, and the images
    the runner's graph reads were refreshed in place."""
    from sceneverse_b200 import evaluate
    ps = unfrozen(0, True)
    bs = scene_batches(4, 2, 16, 80)
    ps.step(dict(bs[0]))
    runner = evaluate.EvalRunner(ps, [evaluate.PretrainEval()], batch_size=2)
    runner.run([bs[0]])
    net = backbone_of(ps)
    assert net._packed is not None and net.training
    sa1_ptr = net._packed["sa1"].data_ptr()
    before = net._packed["sa1"].clone()
    for b in bs[1:]:
        ps.step(dict(b))
    ps.module.model.eval()
    x = bs[0]["obj_fts"].float().reshape(-1, 1024, 6)
    fresh = copy.deepcopy(net)
    fresh._packed = fresh._packed_key = None
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        assert net.fused_available(x)
        got = net(x)
        want = fresh.forward_fused(x)
    assert not torch.equal(before, fresh._pack()["sa1"])        # the weights did move
    assert torch.equal(got, want)
    ps.module.model.train()
    runner.run([bs[0]])
    assert net._packed["sa1"].data_ptr() == sa1_ptr
    assert torch.equal(net._packed["sa1"], fresh._pack()["sa1"]) and torch.equal(net._packed["sa2"], fresh._pack()["sa2"])
    ps.close()


def test_resume_continues_bitwise(tmp_path):
    """3 unfrozen steps, save, steps 4-6; a fresh captured step loads the checkpoint (backbone weights, moments and BatchNorm
    buffers in place into the graph's buffers) and runs steps 4-6 on the same batches: step 4's loss is bitwise the
    original's, 5-6 and the parameters agree within the gradient-atomics tolerance."""
    bs = ck.batches(6)
    a = unfrozen(0, True)
    for b in bs[:3]:
        a.step(b)
    a.save_state(tmp_path)
    saved = ck.graph_buffers(a)
    want = [float(a.step(b)) for b in bs[3:]]
    want_p = ck.params_of(a)
    a.close()
    r = unfrozen(1, True)
    r.load_state(tmp_path)
    got = [float(r.step(b)) for b in bs[3:]]
    assert got[0] == want[0], (got, want)
    assert np.allclose(got[1:], want[1:], rtol=2e-3), (got, want)
    ck.close_params(ck.params_of(r), want_p)
    c = unfrozen(2, True)
    c.step(bs[0])                                   # captured on other weights, then loaded in place
    c.load_state(tmp_path)
    ck.assert_same_tensors(ck.graph_buffers(c), saved, "graph buffers")
    assert any(k.startswith("buffer:model." + BACKBONE) and "running_mean" in k for k in saved)
    r.close()
    c.close()


def test_stage_hand_off_objcls_unfrozen_gps_frozen_scanrefer(tmp_path):
    """ObjCls checkpoint -> unfrozen GPS through vision.args.path (and load_pretrain) -> frozen ScanRefer through load_pretrain,
    with no missing or unexpected backbone keys; ScanRefer's fused eval-mode path then packs the trained weights."""
    from sceneverse_b200.modules.pointnet import GPS_SPEC, PointNetPP
    o = ck.objcls(0, False)
    for b in ck.obj_batches(2):
        o.step(b)
    o.save_state(tmp_path / "objcls")
    pn_want = {k: v.clone() for k, v in o.model.point_feature_extractor.state_dict().items()}
    cfg = M.pretrain_unfreeze_config(1, text_features=TF)
    cfg["model"]["vision"]["args"]["path"] = str(tmp_path / "objcls")
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 2
    g = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=2, cuda_graph=True, total_steps=50)
    ck.assert_same_tensors(backbone_of(g).state_dict(), pn_want, "backbone from vision.args.path")
    g2 = unfrozen(5, False)
    missing, unexpected = g2.load_pretrain(tmp_path / "objcls")
    assert not any(k.startswith(BACKBONE) for k in missing) and not any(k.startswith(BACKBONE) for k in unexpected)
    ck.assert_same_tensors(backbone_of(g2).state_dict(), pn_want, "backbone from load_pretrain")
    g2.close()
    for b in ck.batches(2):
        g.step(b)
    g.save_state(tmp_path / "gps")
    trained = {k: v.detach().cpu().clone() for k, v in backbone_of(g).state_dict().items()}
    g.close()
    assert not torch.equal(trained["encoder.0.mlps.0.layer0.conv.weight"], pn_want["encoder.0.mlps.0.layer0.conv.weight"].cpu())
    f = ck.gps(3, True, cfg=M.scanrefer_config(1, text_features=TF))
    missing, unexpected = f.load_pretrain(tmp_path / "gps")
    assert not any(k.startswith(BACKBONE) for k in list(missing) + list(unexpected)), (missing, unexpected)
    ck.assert_same_tensors(backbone_of(f).state_dict(), trained, "backbone in ScanRefer")
    assert np.isfinite(float(f.step(ck.batches(1)[0])))
    ref = PointNetPP(**GPS_SPEC)
    ref.load_state_dict(trained)
    ref = ref.cuda().eval()
    got, want = backbone_of(f)._packed, ref._pack()
    assert got is not None and torch.equal(got["sa1"], want["sa1"]) and torch.equal(got["sa2"], want["sa2"])
    f.close()
