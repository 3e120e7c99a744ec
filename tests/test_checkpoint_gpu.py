"""Checkpoints of the training steps on the GPU: bitwise round trips of every buffer a captured step reads, resume =
continue (loaded before the first step and after the capture), and the stage hand-off ObjCls -> GPS -> fine-tuning."""
import os

import numpy as np
import pytest
import torch

from sceneverse_b200 import model as M, synthetic, train, weights

pytestmark = pytest.mark.gpu

TF = weights.synthetic_tensor("text_features", (607, 768))


def batches(n, B=2, seed=40):
    out = []
    for i in range(n):
        d = synthetic.scene_batch(seed + i, B=B, O=80, P=1024, L=50, Ls=300)
        out.append({k: torch.from_numpy(v).cuda() for k, v in d.items()})
    return out


def gps(seed, graph, cfg=None, no_dropout=False):
    cfg = cfg or M.pretrain_config(1, text_features=TF)
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 2
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=seed, cuda_graph=graph, total_steps=50)
    if no_dropout:
        for m in ps.module.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
            if hasattr(m, "dropout") and isinstance(m.dropout, float):
                m.dropout = 0.0
    return ps


def objcls(seed, graph):
    return train.ObjClsStep("cuda", TF, dtype=torch.bfloat16, seed=seed, cuda_graph=graph)


def obj_batches(n, seed=60):
    out = []
    for i in range(n):
        d = synthetic.scene_batch(seed + i, B=2, O=16, P=1024, L=50, Ls=300)
        out.append({k: torch.from_numpy(d[k]).cuda() for k in ("obj_fts", "obj_labels", "obj_masks")})
    return out


def assert_same_tensors(a, b, what):
    assert set(a) == set(b), (what, set(a) ^ set(b))
    for k in a:
        assert torch.equal(a[k].cpu(), b[k].cpu()), f"{what}: {k} differs"


def graph_buffers(ps):
    f = ps.flat_grads
    out = {n: getattr(f, n).clone() for n in ("flat_p", "exp_avg", "exp_avg_sq", "shadow", "step_t", "lr_factor")}
    out["dropout_counter"] = ps._step_counter.clone()
    out.update({"buffer:" + n: b.clone() for n, b in ps.module.named_buffers()})
    out.update({"loss:" + n: p.detach().clone() for n, p in ps.module.loss.named_parameters()})
    return out


def rng():
    return {"cpu": torch.get_rng_state(), "cuda": torch.cuda.get_rng_state()}


def test_graph_round_trip_bitwise(tmp_path):
    """GPS graph step after 3 steps -> save -> a fresh step built with another seed and captured on its own weights loads it:
    every buffer the graph reads, the BatchNorm buffers, logit_scale and the generators are bitwise the saved ones."""
    bs = batches(3)
    a = gps(0, True)
    for b in bs:
        a.step(b)
    torch.cuda.synchronize()
    a.save_state(tmp_path)
    want, want_rng, want_step = graph_buffers(a), rng(), a.global_step
    a.close()
    c = gps(1, True)
    c.step(bs[0])                    # captured on seed-1 weights
    c.load_state(tmp_path)           # in place into the captured step
    assert_same_tensors(graph_buffers(c), want, "graph buffers")
    assert_same_tensors(rng(), want_rng, "generators")
    assert c.global_step == want_step
    # the packed PointNet++ images equal a fresh pack of the loaded weights
    pn = c.module.model.point_encoder.point_feature_extractor
    old = pn._packed
    pn._packed = None
    fresh = pn._pack()
    assert torch.equal(old["sa1"], fresh["sa1"]) and torch.equal(old["sa2"], fresh["sa2"])
    assert all(torch.equal(x, y) for (x, _), (y, _) in zip(old["sa3"], fresh["sa3"]))
    c.close()


def test_eager_round_trip_bitwise(tmp_path):
    bs = batches(3)
    a = gps(0, False)
    for b in bs:
        a.step(b)
    a.save_state(tmp_path)
    want, want_rng = a.state_dict(), rng()
    q = gps(1, False)
    q.load_state(tmp_path)
    got = q.state_dict()
    assert_same_tensors(got["model"], want["model"], "model")
    assert_same_tensors(got["loss"], want["loss"], "loss")
    assert set(got["optimizer"]["state"]) == set(want["optimizer"]["state"])
    for i, s in want["optimizer"]["state"].items():
        assert_same_tensors(got["optimizer"]["state"][i], s, f"optimizer state {i}")
    assert got["scheduler"]["last_epoch"] == want["scheduler"]["last_epoch"] == 3
    assert_same_tensors(rng(), want_rng, "generators")


def test_objcls_graph_round_trip_bitwise(tmp_path):
    bs = obj_batches(3)
    a = objcls(0, True)
    for b in bs:
        a.step(b)
    a.save_state(tmp_path)
    want_model = {k: v.clone() for k, v in a.model.state_dict().items()}
    want_opt = {n: {k: v.clone() for k, v in a.optimizer.state[p].items()} for n, p in a.model.named_parameters()}
    want_rng = rng()
    c = objcls(1, True)
    c.step(bs[0])
    c.load_state(tmp_path)
    assert any("running_mean" in k for k in want_model)
    assert_same_tensors(c.model.state_dict(), want_model, "ObjCls model (running statistics included)")
    for n, p in c.model.named_parameters():
        assert_same_tensors(c.optimizer.state[p], want_opt[n], f"AdamW state of {n}")
    assert_same_tensors(rng(), want_rng, "generators")


def params_of(ps):
    return {n: p.detach().float().clone() for n, p in ps.module.named_parameters() if p.requires_grad}


def close_params(got, want, tol=2e-2):
    """DESIGN.md §2: the wgrad kernels accumulate with atomics, so parameters of two runs agree to the bf16 level only."""
    worst = 0.0
    for n, w in want.items():
        d = (got[n] - w).abs().max().item() / (w.abs().max().item() + 1e-12)
        worst = max(worst, d)
    assert worst < tol, worst
    return worst


@pytest.mark.parametrize("when", ["before_first_step", "after_capture"])
def test_resume_continues(tmp_path, when):
    """3 steps, save, steps 4-6; a fresh step loads the checkpoint and runs steps 4-6 on the same batches.  Step 4's loss
    is bitwise the original's (deterministic forward, restored dropout counter and generators); 5-6 and the parameters
    agree within the gradient-atomics tolerance.  after_capture: the fresh step is captured on other weights first (and,
    since the in-kernel dropout seeds are constants of each capture, both runs are dropout-free) — the next loss must be
    the checkpoint's, which stale packed PointNet++ weights or bf16 shadows would break."""
    nd = when == "after_capture"
    bs = batches(6)
    a = gps(0, True, no_dropout=nd)
    for b in bs[:3]:
        a.step(b)
    a.save_state(tmp_path)
    want = [float(a.step(b)) for b in bs[3:]]
    want_p = params_of(a)
    a.close()
    r = gps(1, True, no_dropout=nd)
    if nd:
        l_own = float(r.step(batches(1, seed=90)[0]))     # capture + one replay on the seed-1 weights
        r.load_state(tmp_path)
    else:
        r.load_state(tmp_path)
    got = [float(r.step(b)) for b in bs[3:]]
    assert got[0] == want[0], (got, want)
    assert np.allclose(got[1:], want[1:], rtol=2e-3), (got, want)
    worst = close_params(params_of(r), want_p)
    print(f"resume {when}: losses {got} vs {want}, worst parameter difference {worst:.2e}")
    if nd:
        assert l_own != got[0]
    r.close()


def test_train_log_continues_from_restored_step(tmp_path):
    from sceneverse_b200 import evaluate
    bs = batches(4)
    a = gps(0, True)
    for b in bs[:3]:
        a.step(b)
    a.save_state(tmp_path)
    a.close()
    r = train.PretrainStep(M.pretrain_config(1, text_features=TF), "cuda", dtype=torch.bfloat16, seed=1, cuda_graph=True,
                           total_steps=50, train_eval=evaluate.PretrainEval(), log_every=4)
    r.load_state(tmp_path)
    r.step(bs[3])
    r.step(bs[0])
    logs = r.logs()
    assert [d["train/step"] for d in logs] == [4, 5]
    assert all(np.isfinite(d["train/total_loss"]) for d in logs)
    r.close()


def test_stage_hand_off(tmp_path):
    """ObjCls -> GPS (vision.args.path) -> ScanRefer / ScanQA (load_pretrain)."""
    o = objcls(0, False)
    for b in obj_batches(2):
        o.step(b)
    o.save_state(tmp_path / "objcls")
    pn_want = {k: v.clone() for k, v in o.model.point_feature_extractor.state_dict().items()}
    cfg = M.pretrain_config(1, text_features=TF)
    cfg["model"]["vision"]["args"]["path"] = str(tmp_path / "objcls")
    g = gps(2, True, cfg=cfg)
    assert_same_tensors(g.module.model.point_encoder.point_feature_extractor.state_dict(), pn_want, "backbone")
    bs = batches(2)
    for b in bs:
        g.step(b)
    g.save_state(tmp_path / "gps")
    shared = {k: v.clone() for k, v in g.module.model.state_dict().items()}
    loss_keys = set(g.module.loss.state_dict())
    g.close()
    assert_same_tensors({k: v for k, v in shared.items() if k.startswith("point_encoder.point_feature_extractor.")},
                        {"point_encoder.point_feature_extractor." + k: v for k, v in pn_want.items()}, "frozen backbone")
    for make, head in ((M.scanrefer_config, "ground_head"), (M.scanqa_config, "qa_head")):
        f = gps(3, True, cfg=make(1, text_features=TF))
        missing, unexpected = f.load_pretrain(tmp_path / "gps")
        assert missing and all(k.startswith(head + ".") for k in missing), missing
        assert set(missing) == {k for k in f.module.model.state_dict() if k.startswith(head + ".")}
        # as in the reference, the pre-training loss module's file (pytorch_model_1.bin) is offered to the model too
        assert set(unexpected) - loss_keys == {k for k in shared if k.startswith("pretrain_head.")}
        mine = f.module.model.state_dict()
        both = [k for k in mine if k in shared]
        assert len(both) == len(mine) - len(missing)
        for k in both:
            assert torch.equal(mine[k].cpu(), shared[k].cpu()), k
        if head == "ground_head":
            assert np.isfinite(float(f.step(bs[0])))
        f.close()
    assert os.path.exists(tmp_path / "gps" / "random_states_0.pkl")
