"""Parity of the native GPS modules with the reference's own modules (goldens: tests/golden/model_gps_stack.npz,
produced by running the UNMODIFIED reference classes on CPU in fp32, oracle/make_golden_model.py).
CPU tests cover the host logic of the attention stack / heads / losses at fp32 (1e-5); the GPU tests run the whole
chain including the native PointNet++ path."""
import json
import os

import numpy as np
import pytest
import torch

from sceneverse_b200 import synthetic, weights
from sceneverse_b200.modules import grounding, heads, losses, registry, vision

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
Z = np.load(os.path.join(GOLDEN, "model_gps_stack.npz"))


def load(m, seed):
    m.load_state_dict(weights.synthetic_state_dict(m, seed=seed))
    return m.eval()


def inputs(device="cpu"):
    d = synthetic.scene_batch(int(Z["data_seed"]), B=2, O=32, P=1024, L=50, Ls=300, min_obj=12)
    t = {k: torch.from_numpy(v).to(device) for k, v in d.items()}
    g = torch.Generator().manual_seed(int(Z["txt_seed"]))
    txt = (torch.randn(2, 50, 768, generator=g) * 0.5).to(device)
    scene_txt = (torch.randn(2, 768, generator=g) * 0.5).to(device)
    return t, txt, scene_txt


def close(got, want, tol, what):
    got = got.detach().float().cpu().numpy()
    scale = np.abs(want[np.isfinite(want)]).max() + 1e-12
    fin = np.isfinite(want)
    assert (np.isfinite(got) == fin).all(), what
    err = np.abs(got[fin] - want[fin]).max() / scale
    assert err < tol, f"{what}: max err / max|ref| = {err:.3e} (tol {tol})"
    return err


@pytest.mark.parametrize("name", ["PointOpenVocabEncoder", "UnifiedSpatialCrossEncoderV2", "UnifiedSpatialCrossEncoderV1",
                                  "EntitySpatialCrossEncoder", "GroundHeadV1", "GroundHead", "PretrainHeadV1",
                                  "OVPretrainHead"])
def test_state_dict_contracts(name):
    want = json.load(open(os.path.join(GOLDEN, "state_dict_shapes.json")))[name]
    tf = weights.synthetic_tensor("text_features", (607, 768))
    kw = {"PointOpenVocabEncoder": dict(freeze=True, text_features=tf),
          "GroundHeadV1": dict(input_size=768, hidden_size=384, sem_cls_size=607)}.get(name, {})
    reg = registry.VISION_REGISTRY if name in registry.VISION_REGISTRY else \
        registry.GROUNDING_REGISTRY if name in registry.GROUNDING_REGISTRY else registry.HEADS_REGISTRY
    m = reg.get(name)(None, **kw)
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == want


def run_stack(device, obj, obj_pre, tol):
    t, txt, scene_txt = inputs(device)
    errs = {}
    with torch.no_grad():
        v2 = load(grounding.UnifiedSpatialCrossEncoderV2(None), 1).to(device)
        t2, o2 = v2(txt, t["txt_masks"], obj, t["obj_locs"], t["obj_masks"])
        errs["v2_txt"] = close(t2, Z["v2_txt"], tol, "V2 txt")
        errs["v2_obj"] = close(o2, Z["v2_obj"], tol, "V2 obj")
        v1 = load(grounding.UnifiedSpatialCrossEncoderV1(None), 2).to(device)
        t1, o1 = v1(txt, t["txt_masks"], obj, t["obj_locs"], t["obj_masks"])
        errs["v1_txt"] = close(t1, Z["v1_txt"], tol, "V1 txt")
        errs["v1_obj"] = close(o1, Z["v1_obj"], tol, "V1 obj")
        en = load(grounding.EntitySpatialCrossEncoder(None), 3).to(device)
        _, oe = en(txt, t["txt_masks"], obj, t["obj_locs"], t["obj_masks"])
        errs["entity"] = close(oe, Z["entity_obj"], tol, "Entity obj")
        gh = load(heads.GroundHeadV1(None, input_size=768, hidden_size=384, sem_cls_size=607), 4).to(device)
        a, b, c, og = gh(t2, o2, obj_pre, t["obj_masks"])
        errs["gh_txt"] = close(a, Z["gh_txt_cls"], tol, "GroundHeadV1 txt_cls")
        close(b[:, :, :64], Z["gh_obj_cls"], tol, "GroundHeadV1 obj_cls")
        close(c[:, :, :64], Z["gh_obj_cls_pre"], tol, "GroundHeadV1 obj_cls_pre")
        errs["og3d"] = close(og, Z["gh_og3d"], tol, "og3d logits")  # north_star: grounding logits within 1e-3
        ph = load(heads.OVPretrainHead(None), 5).to(device)
        lm, ol = ph(t2, o2)
        errs["lm"] = close(lm[:, :, :128], Z["ph_txt_lm_slice"], tol, "LM logits")
        close(lm.sum(-1), Z["ph_txt_lm_rowsum"], tol * 30, "LM logits row sums")
        close(ol[:, :, :64], Z["ph_obj_lm"], tol, "obj LM logits")
        dd = dict(t)
        dd.update(intra_obj_embeds=o2, intra_text_embed=t2[:, 0], inter_obj_embeds=obj, inter_text_embed=txt[:, 0],
                  scene_embed=obj.mean(dim=1), scene_text_embed=scene_txt, og3d_logits=og, txt_lm_cls_logits=lm)
        cfg = {"num_gpu": 1}
        for key, fn in [("loss_within", losses.TextObjWithinBatch(cfg)), ("loss_obj_between", losses.TextObjBetweenBatch(cfg)),
                        ("loss_scene_between", losses.TextSceneBetweenBatch(cfg)), ("loss_og3d", losses.og3d_loss),
                        ("loss_lm", losses.lm_cls_loss)]:
            if isinstance(fn, torch.nn.Module):
                fn = fn.to(device)
            got = float(fn(dd))
            want = float(Z[key])
            assert abs(got - want) <= tol * 10 * max(1.0, abs(want)), (key, got, want)
    return errs


def test_attention_stack_heads_losses_cpu_fp32():
    """Host logic on CPU, fed with the reference's own object embeddings: fp32 tolerance 1e-5 (north_star)."""
    obj = torch.from_numpy(Z["vis_obj"])
    obj_pre = torch.from_numpy(Z["vis_obj_pre"])
    errs = run_stack("cpu", obj, obj_pre, 1e-5)
    print(errs)


def test_calc_pairwise_locs_properties():
    from sceneverse_b200 import ops
    t, _, _ = inputs()
    locs = ops.calc_pairwise_locs(t["obj_locs"][:, :, :3], t["obj_locs"][:, :, 3:])
    assert locs.shape == (2, 32, 32, 5)
    assert torch.allclose(locs[..., 0].amax(dim=(1, 2)), torch.ones(2))          # normalised by the max distance
    assert torch.allclose(locs[..., 1] ** 2 + locs[..., 2] ** 2, torch.ones(2, 32, 32), atol=1e-3)  # sin^2+cos^2 (eps inside sqrt)
    assert torch.allclose(locs[..., 0], locs[..., 0].transpose(1, 2))


@pytest.mark.gpu
def test_full_chain_gpu_generic_fp32():
    """Vision encoder through the reference operator sequence on the native point ops (fp32, TF32 off) + stack: 1e-5 class."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    t, txt, _ = inputs("cuda")
    tf = weights.synthetic_tensor("text_features", (607, 768))
    enc = load(vision.PointOpenVocabEncoder(None, freeze=True, text_features=tf), 0).cuda()
    enc.point_feature_extractor.fused_available = lambda x: False  # force the generic path
    with torch.no_grad():
        obj, obj_pre, sem = enc(t["obj_fts"], t["obj_locs"], t["obj_masks"], t["obj_sem_masks"], t["obj_labels"], 1, 1)
    close(obj_pre, Z["vis_obj_pre"], 2e-5, "PointNet++ embeddings (generic path)")
    close(obj, Z["vis_obj"], 5e-5, "spatial encoder output")
    assert (sem.argmax(-1).cpu().numpy() == Z["vis_sem_cls_argmax"]).mean() > 0.98
    errs = run_stack("cuda", obj, obj_pre, 1e-4)
    print(errs)


@pytest.mark.gpu
def test_full_chain_gpu_fused_bf16():
    """Same chain with the fused wgmma PointNet++ path (bf16 operands): bf16-level tolerance vs the fp32 reference."""
    t, txt, _ = inputs("cuda")
    tf = weights.synthetic_tensor("text_features", (607, 768))
    enc = load(vision.PointOpenVocabEncoder(None, freeze=True, text_features=tf), 0).cuda()
    with torch.no_grad():
        assert enc.point_feature_extractor.fused_available(t["obj_fts"].view(-1, 1024, 6))
        obj, obj_pre, sem = enc(t["obj_fts"], t["obj_locs"], t["obj_masks"], t["obj_sem_masks"], t["obj_labels"], 1, 1)
    e1 = close(obj_pre, Z["vis_obj_pre"], 2e-2, "PointNet++ embeddings (fused bf16)")
    e2 = close(obj, Z["vis_obj"], 2e-2, "spatial encoder output (fused bf16 backbone)")
    print("fused bf16 backbone: obj_pre err", e1, "obj err", e2)
    errs = run_stack("cuda", obj, obj_pre, 2e-2)
    print(errs)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["pretrain", "scanrefer"])
def test_training_step_runs_and_learns(which):
    """BASELINE.json configs[3] / configs[2] at a reduced batch: three optimisation steps on one fixed batch must run
    through every native kernel in the step (sampling, SA-MLP, GEMM chain, attention, CE) and lower the loss."""
    from sceneverse_b200 import model as M, train, _lib
    tf = weights.synthetic_tensor("text_features", (607, 768))
    cfg = M.pretrain_config(1, text_features=tf) if which == "pretrain" else M.scanrefer_config(1, text_features=tf)
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 1
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=3)
    d = synthetic.scene_batch(9, B=4, O=80, P=1024, L=50, Ls=300)
    batch = {k: torch.from_numpy(v).cuda() for k, v in d.items()}
    n0 = _lib.launch_count()
    losses_seen = [float(ps.step(dict(batch))) for _ in range(4)]
    assert all(np.isfinite(losses_seen)), losses_seen
    assert losses_seen[-1] < losses_seen[0], losses_seen
    assert _lib.launch_count() - n0 >= 4 * 10  # native launches per step
    if which == "pretrain":  # the object LM head feeds no loss in all_pretrain.yaml: found once, then frozen
        assert any(n.endswith("pretrain_head.obj_pred_head.transform.dense.weight") for n in ps.unused_parameters)


@pytest.mark.gpu
def test_training_step_cuda_graph_replay():
    """The captured whole-step CUDA graph (forward, losses, backward, clipping, AdamW) trains like the eager step: finite,
    decreasing loss on a fixed batch, new inputs are picked up from the static buffers, the LR schedule advances."""
    from sceneverse_b200 import model as M, train, _lib
    tf = weights.synthetic_tensor("text_features", (607, 768))
    cfg = M.pretrain_config(1, text_features=tf)
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 1
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=3, cuda_graph=True)
    assert ps.graph_mode
    d = synthetic.scene_batch(9, B=4, O=80, P=1024, L=50, Ls=300)
    batch = {k: torch.from_numpy(v).cuda() for k, v in d.items()}
    seen = [float(ps.step(dict(batch))) for _ in range(6)]
    assert all(np.isfinite(seen)), seen
    assert seen[-1] < seen[0], seen
    assert ps.graph is not None and ps.native_launches_per_step >= 40
    lr0 = float(ps.optimizer.param_groups[0]["lr"])
    d2 = synthetic.scene_batch(10, B=4, O=80, P=1024, L=50, Ls=300)
    other = {k: torch.from_numpy(v).cuda() for k, v in d2.items()}
    l_other = float(ps.step(other))
    assert np.isfinite(l_other) and abs(l_other - seen[-1]) > 1e-6       # a different batch went through the graph
    assert float(ps.optimizer.param_groups[0]["lr"]) != lr0 or ps._sched_step > 0
    _lib.gps().sv_dropout_seed_offset(None)                               # do not leak the counter into later tests
    from sceneverse_b200 import ops
    assert len(ops._SHADOW) > 100                                         # bf16 weight shadows were in use
    ops.clear_shadows()


def test_backward_matches_reference_gradients_cpu_fp32():
    """Backward parity with the UNMODIFIED reference (goldens from oracle/make_golden_model.py::golden_gps_backward):
    same synthetic weights and inputs, frozen-backbone features taken from the fixture (the PointNet++ path is CUDA-only
    by design), eval mode, fp32 CPU: every loss term, the gradient norm of all 143 trainable parameters and five gradient
    slices must match — checks the autograd structure of the host logic (detach points, shared weights, masked losses)."""
    G = np.load(os.path.join(GOLDEN, "model_gps_grads.npz"))
    want_norms = json.load(open(os.path.join(GOLDEN, "model_gps_grad_norms.json")))
    d = synthetic.scene_batch(int(G["data_seed"]), B=2, O=16, P=1024, L=50, Ls=300, min_obj=6)
    t = {k: torch.from_numpy(v) for k, v in d.items()}
    g = torch.Generator().manual_seed(int(G["txt_seed"]))
    txt = torch.randn(2, 50, 768, generator=g) * 0.5
    scene_txt = torch.randn(2, 768, generator=g) * 0.5
    tf = weights.synthetic_tensor("text_features", (607, 768))
    mods = {"enc": load(vision.PointOpenVocabEncoder(None, freeze=True, text_features=tf), 0),
            "v2": load(grounding.UnifiedSpatialCrossEncoderV2(None), 1),
            "gh": load(heads.GroundHeadV1(None, input_size=768, hidden_size=384, sem_cls_size=607), 4),
            "ph": load(heads.OVPretrainHead(None), 5),
            "l_within": losses.TextObjWithinBatch({"num_gpu": 1}), "l_obj": losses.TextObjBetweenBatch({"num_gpu": 1}),
            "l_scene": losses.TextSceneBetweenBatch({"num_gpu": 1})}

    class Backbone(torch.nn.Module):          # the frozen PointNet++ output of the reference run
        def forward(self, x):
            return torch.from_numpy(G["pn_out"])
    mods["enc"].point_feature_extractor = Backbone()
    obj, obj_pre, _ = mods["enc"](t["obj_fts"], t["obj_locs"], t["obj_masks"], t["obj_sem_masks"], t["obj_labels"], 1, 1)
    t2, o2 = mods["v2"](txt, t["txt_masks"], obj, t["obj_locs"], t["obj_masks"])
    _, _, _, og = mods["gh"](t2, o2, obj_pre, t["obj_masks"])
    lm, _ = mods["ph"](t2, o2)
    dd = dict(t)
    dd.update(intra_obj_embeds=o2, intra_text_embed=t2[:, 0], inter_obj_embeds=obj, inter_text_embed=txt[:, 0],
              scene_embed=obj.mean(dim=1), scene_text_embed=scene_txt, og3d_logits=og, txt_lm_cls_logits=lm)
    parts = {"lm": losses.lm_cls_loss(dd), "within": mods["l_within"](dd), "obj_between": mods["l_obj"](dd),
             "scene_between": mods["l_scene"](dd), "og3d": losses.og3d_loss(dd)}
    for k, v in parts.items():
        assert abs(float(v) - float(G["loss_" + k])) < 1e-4 * max(1.0, abs(float(G["loss_" + k]))), k
    total = sum(parts.values())
    assert abs(float(total) - float(G["total"])) < 1e-4 * abs(float(G["total"]))
    total.backward()
    got_norms = {}
    for mname, m in mods.items():
        for n, p in m.named_parameters():
            if p.grad is not None:
                got_norms[f"{mname}.{n}"] = float(p.grad.double().norm())
    assert set(got_norms) == set(want_norms), set(got_norms) ^ set(want_norms)
    # gradients that are mathematically zero (key bias under a row-shift-invariant softmax, biases behind masked logits)
    # are fp32 rounding noise of size 1e-8 in both implementations: absolute floor 1e-6
    bad = {k: (got_norms[k], w) for k, w in want_norms.items() if abs(got_norms[k] - w) > 2e-3 * abs(w) + 1e-6}
    assert not bad, bad
    for key in [k for k in G.files if k.startswith("slice:")]:
        mname, n = key[6:].split(".", 1)
        got = dict(mods[mname].named_parameters())[n].grad.reshape(-1)[:96].numpy()
        assert np.abs(got - G[key]).max() <= 1e-4 * (np.abs(G[key]).max() + 1e-8), key



@pytest.mark.gpu
def test_graph_step_matches_eager_step_parameters():
    """One optimisation step through the captured path (flat parameter / gradient / moment buffers, wgrad kernels accumulating
    into the flat gradient, native clip + AdamW) must move every parameter like the eager step (torch autograd accumulation,
    clip_grad_norm_, torch.optim.AdamW) from the same initial state, batch and dropout-free modules."""
    from sceneverse_b200 import model as M, train
    tf = weights.synthetic_tensor("text_features", (607, 768))
    d = synthetic.scene_batch(9, B=4, O=80, P=1024, L=50, Ls=300)
    batch = {k: torch.from_numpy(v).cuda() for k, v in d.items()}

    def make(graph):
        cfg = M.pretrain_config(1, text_features=tf)
        cfg["solver"]["sched"]["args"]["warmup_steps"] = 0      # lr factor 1 from the first step
        ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=3, cuda_graph=graph)
        for m in ps.module.modules():          # no dropout: both paths must be deterministic functions of the batch
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
    # eager reference: one step
    eager.step(dict(batch))
    # graph path: the same single step, run eagerly on the flat state (what the capture records)
    graph.static_batch = {k: v.clone() for k, v in batch.items()}
    from sceneverse_b200 import ops
    graph._make_flat_state()
    graph._raw_step()
    ops.clear_shadows()
    worst = (1.0, None)
    checked = 0
    for (n, pe), (_, pg) in zip(eager.module.named_parameters(), graph.module.named_parameters()):
        if not pe.requires_grad or pe.grad is None:
            continue
        ge = pe.grad.float()
        big = ge.abs() > 0.2 * ge.abs().max()          # coordinates whose gradient is far above the bf16 noise
        if big.sum() == 0 or ge.abs().max() == 0:
            continue
        de, dg = (pe.detach() - p0[n]).float(), (pg.detach() - p0[n]).float()
        # the first AdamW step moves a coordinate by -lr * g / (|g| + eps): same sign and (almost) the same size in both paths
        agree = (torch.sign(de[big]) == torch.sign(dg[big])).float().mean().item()
        ratio = (dg[big].abs().mean() / (de[big].abs().mean() + 1e-20)).item()
        worst = min(worst, (agree, n), key=lambda t: t[0])
        checked += 1
        assert agree > 0.98 and 0.9 < ratio < 1.1, (n, agree, ratio)
    assert checked > 100, checked
    print("GRAPH_VS_EAGER worst sign agreement", worst, "parameters checked", checked)
