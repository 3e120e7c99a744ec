"""Per-scene grounding (model.OpenVocabPerScene, ops.scene_broadcast, evaluate.flatten_per_scene, synthetic.per_scene_batch).

CPU: the model against the unmodified reference OpenVocabPerScene (tests/golden/model_per_scene.npz, oracle/make_golden_per_scene.py)
with the same stub encoders, 2-D batches against OpenVocab, the unsupported combinations, the evaluators' per-scene counts
against the reference's (tests/golden/eval_per_scene.npz), and the checkpoint key sets.
GPU: the U-sum kernel against float64, the bf16 stack against the fixture, the training step (eager, graph, checkpoints) and
the evaluation runner."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_per_scene as G
from sceneverse_b200 import _lib, evaluate, model as M, synthetic, weights
from sceneverse_b200.modules import losses
from sceneverse_b200.modules.registry import LANGUAGE_REGISTRY, VISION_REGISTRY

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TF = weights.synthetic_tensor("text_features", (607, 768))

for _stub in (G.StubLanguageEncoder, G.StubVisionEncoder):
    (LANGUAGE_REGISTRY if "Language" in _stub.__name__ else VISION_REGISTRY).register(_stub)


def stub_cfg(name="OpenVocabPerScene", rows=None, q=G.PER_SCENE_GOLDEN, head_list=("pretrain_head",)):
    """per_scene_pretrain_config with the fixture's stub encoders in place of BERT and the object encoder."""
    cfg = M.per_scene_pretrain_config(1, text_features=TF)
    cfg["model"]["name"] = name
    cfg["model"]["language"] = {"name": "StubLanguageEncoder",
                                "args": {"rows": rows or q["B"] * q["U"], "T": q["T"], "D": q["D"], "seed": q["lang_seed"]}}
    cfg["model"]["vision"] = {"name": "StubVisionEncoder", "args": {"B": q["B"], "O": q["O"], "D": q["D"], "seed": q["obj_seed"]}}
    cfg["model"]["heads"]["head_list"] = list(head_list)
    return cfg


def stub_model(device="cpu", name="OpenVocabPerScene", rows=None):
    q = G.PER_SCENE_GOLDEN
    m = M.build_model(stub_cfg(name, rows))
    m.unified_encoder.load_state_dict(weights.synthetic_state_dict(m.unified_encoder, seed=q["v2_seed"]))
    m.pretrain_head.load_state_dict(weights.synthetic_state_dict(m.pretrain_head, seed=q["head_seed"]))
    return m.to(device).eval()


def run_stack(m, t):
    """Forward of the fixture's batch, its three losses and their backward; (og3d_logits, {loss: value}, {param: grad norm})."""
    ls = {"l_within": losses.TextObjWithinBatch({"num_gpu": 1}), "l_obj": losses.TextObjBetweenBatch({"num_gpu": 1})}
    ls = {k: v.to(t["obj_masks"].device) for k, v in ls.items()}
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=t["obj_masks"].is_cuda):
        dd = m(dict(t))
        parts = {"lm": losses.lm_cls_loss(dd), "within": ls["l_within"](dd), "obj_between": ls["l_obj"](dd)}
        total = sum(parts.values())
    total.backward()
    norms = {n: float(p.grad.double().norm()) for n, p in m.named_parameters() if p.grad is not None}
    norms.update({f"loss.{k}.{n}": float(p.grad.double().norm()) for k, v in ls.items()
                  for n, p in v.named_parameters() if p.grad is not None})
    return dd, parts, total, norms


def fixture_batch(device="cpu"):
    return {k: torch.from_numpy(v).to(device) for k, v in G.per_scene_inputs().items()}


# ---- CPU -----------------------------------------------------------------------------------------------------------------
def test_per_scene_batch_layout():
    B, U, O, T = 3, 5, 12, 20
    d = synthetic.per_scene_batch(7, B=B, U=U, O=O, P=32, T=T, min_obj=4)
    for k in ("txt_ids", "txt_masks", "masked_lm_labels"):
        assert d[k].shape == (B, U, T) and d[k].dtype == np.int64, k
    for k in ("tgt_object_id", "tgt_object_label"):
        assert d[k].shape == (B, U) and d[k].dtype == np.int64, k
    for k in ("is_multiple", "is_hard", "is_view_dependent"):
        assert d[k].shape == (B, U) and d[k].dtype == bool, k
    assert d["obj_fts"].shape == (B, O, 32, 6) and d["obj_masks"].shape == (B, O)
    tgt = d["tgt_object_id"]
    assert np.take_along_axis(d["obj_masks"], tgt, 1).all()                              # a valid object of its scene
    assert (d["tgt_object_label"] == np.take_along_axis(d["obj_labels"], tgt, 1)).all()
    for k in ("tgt_object_id_iou25", "tgt_object_id_iou50"):
        assert d[k].shape == (B, U, O) and np.take_along_axis(d[k], tgt[:, :, None], 2).all()
        assert not (d[k].astype(bool) & ~d["obj_masks"][:, None, :]).any()
    assert (d["tgt_object_id_iou50"] <= d["tgt_object_id_iou25"]).all()
    assert ((d["masked_lm_labels"] != -1).sum(-1) > 0).all()
    s = synthetic.scene_batch(7, B=B, O=O, P=32, L=8, Ls=8, min_obj=4)
    assert all(np.array_equal(d[k], s[k]) for k in ("obj_fts", "obj_locs", "obj_masks", "obj_sem_masks", "obj_labels"))


def test_matches_reference_cpu_fp32():
    """The fixture's forward and backward through the repo's OpenVocabPerScene (fp32 CPU, same stubs, weights and batch):
    og3d_logits and losses within 1e-4, every parameter's gradient norm (the object stub's = the U-sum) within 2e-3 + 1e-6,
    gradient slices within 1e-4 of the slice's largest entry."""
    F = np.load(os.path.join(GOLDEN, "model_per_scene.npz"))
    want_norms = json.load(open(os.path.join(GOLDEN, "model_per_scene_grad_norms.json")))
    m = stub_model()
    dd, parts, total, norms = run_stack(m, fixture_batch())
    og = dd["og3d_logits"].detach().numpy()
    assert og.shape == (2, 4, 16)
    assert np.abs(og - F["og3d_logits"]).max() <= 1e-4 * np.abs(F["og3d_logits"]).max()
    for k, v in parts.items():
        assert abs(float(v.detach()) - float(F["loss_" + k])) <= 1e-4 * abs(float(F["loss_" + k])), k
    assert abs(float(total) - float(F["total"])) <= 1e-4 * abs(float(F["total"]))
    assert set(norms) == set(want_norms), set(norms) ^ set(want_norms)
    assert "point_encoder.feats" in norms and "lang_encoder.feats" in norms
    bad = {k: (norms[k], w) for k, w in want_norms.items() if abs(norms[k] - w) > 2e-3 * abs(w) + 1e-6}
    assert not bad, bad
    params = dict(m.named_parameters())
    for key in [k for k in F.files if k.startswith("slice:")]:
        got = params[key[6:]].grad.reshape(-1)[:96].numpy()
        assert np.abs(got - F[key]).max() <= 1e-4 * np.abs(F[key]).max(), key


def test_two_d_batch_equals_openvocab_without_ground_head():
    """A 2-D batch through OpenVocabPerScene is OpenVocab (no ground head, no scene captions) with the same weights."""
    d = synthetic.scene_batch(12, B=2, O=16, P=16, L=50, Ls=8, min_obj=6)
    t = {k: torch.from_numpy(v) for k, v in d.items()}
    per_scene, plain = stub_model(rows=2), stub_model(name="OpenVocab", rows=2)
    assert type(per_scene) is M.OpenVocabPerScene and type(plain) is M.OpenVocab
    plain.load_state_dict(per_scene.state_dict())
    with torch.no_grad():
        a, b = per_scene(dict(t)), plain(dict(t))
    keys = ("og3d_logits", "txt_lm_cls_logits", "obj_cls_post_logits", "intra_obj_embeds", "intra_text_embed",
            "inter_obj_embeds", "inter_text_embed")
    for k in keys:
        assert torch.equal(a[k], b[k]), k
    assert "scene_embed" not in a and "txt_cls_logits" not in a


@pytest.mark.parametrize("what", ["og3d_loss", "TextSceneBetweenBatch", "answer_loss", "qa_head"])
def test_unsupported_combinations_raise(what):
    cfg = M.per_scene_pretrain_config(1, text_features=TF)
    if what == "qa_head":
        cfg["model"]["heads"] = M.scanqa_config(1)["model"]["heads"]
    else:
        cfg["model"]["loss_list"] = cfg["model"]["loss_list"] + [what]
    with pytest.raises(ValueError, match=what):
        M.build_model(cfg)


def test_unsupported_at_run_time_raise():
    from sceneverse_b200 import train
    with pytest.raises(ValueError, match="per-scene"):
        train.PretrainStep(M.per_scene_pretrain_config(1, text_features=TF), "cpu", train_eval=evaluate.ScanReferEval(device="cpu"))
    with pytest.raises(ValueError, match="per-scene"):
        losses.og3d_loss({"og3d_logits": torch.zeros(2, 3, 4), "tgt_object_id": torch.zeros(2, 3, dtype=torch.int64)})
    with pytest.raises(ValueError, match="per-scene"):
        evaluate.PretrainEval(device="cpu").update({"txt_lm_cls_logits": torch.zeros(6, 5, 7),
                                                    "masked_lm_labels": torch.zeros(2, 3, 5, dtype=torch.int64)})


def test_build_model_and_configs():
    cfg = M.per_scene_pretrain_config(1, text_features=TF)
    c = M.to_cfg(cfg)
    assert c.model.name == "OpenVocabPerScene" and c.data.args.use_scene_cap is False
    assert list(c.model.loss_list) == ["lm_cls_loss", "TextObjWithinBatch", "TextObjBetweenBatch"]
    assert M.to_cfg(M.pretrain_config(1)).model.name == "OpenVocab"
    with pytest.raises(KeyError, match="NoSuchModel"):
        M.build_model(dict(cfg, model=dict(cfg["model"], name="NoSuchModel")))


def test_checkpoint_keys_and_opt_groups_are_shared():
    """OpenVocab and OpenVocabPerScene built from the pre-training configs: identical state-dict keys and shapes and the
    same optimizer groups, so checkpoints and load_pretrain move between them unchanged."""
    torch.manual_seed(0)
    a = M.build_model(M.pretrain_config(1, text_features=TF))
    b = M.build_model(M.per_scene_pretrain_config(1, text_features=TF))
    assert type(a) is M.OpenVocab and type(b) is M.OpenVocabPerScene
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    assert all(sa[k].shape == sb[k].shape for k in sa)
    ga, gb = a.get_opt_params(), b.get_opt_params()
    assert [(len(g["params"]), g["lr"], g["weight_decay"]) for g in ga] == [(len(g["params"]), g["lr"], g["weight_decay"]) for g in gb]
    names_a = {id(p): n for n, p in a.named_parameters()}
    names_b = {id(p): n for n, p in b.named_parameters()}
    assert [[names_a[id(p)] for p in g["params"]] for g in ga] == [[names_b[id(p)] for p in g["params"]] for g in gb]


def test_losses_per_scene_branches_match_flattened_inputs():
    """TextObjWithinBatch / TextObjBetweenBatch on (B*U) rows with (B, O) masks and (B, U) targets equal the 2-D losses
    on the explicitly repeated masks and (B*U, 1) targets."""
    g = torch.Generator().manual_seed(3)
    B, U, O, D = 2, 3, 5, 16
    masks = torch.tensor([[1, 1, 1, 0, 0], [1, 1, 1, 1, 1]], dtype=torch.bool)
    tgt = torch.tensor([[0, 2, 1], [4, 3, 0]])
    d = {"intra_obj_embeds": torch.randn(B * U, O, D, generator=g), "intra_text_embed": torch.randn(B * U, D, generator=g),
         "inter_obj_embeds": torch.randn(B * U, O, D, generator=g), "inter_text_embed": torch.randn(B * U, D, generator=g),
         "obj_masks": masks, "tgt_object_id": tgt}
    flat = dict(d, obj_masks=masks.repeat_interleave(U, 0), tgt_object_id=tgt.reshape(-1, 1))
    w, b = losses.TextObjWithinBatch({"num_gpu": 1}), losses.TextObjBetweenBatch({"num_gpu": 1})
    assert torch.equal(w(d), w(flat)) and torch.equal(b(d), b(flat))


# ---- evaluation ----------------------------------------------------------------------------------------------------------
def eval_meta():
    E = np.load(os.path.join(GOLDEN, "eval_per_scene.npz"))
    return E, json.loads(bytes(E["meta"]).decode())


def eval_batch(E, case, i):
    p = f"{case}:{i}:"
    return {k[len(p):]: torch.from_numpy(E[k]) for k in E.files if k.startswith(p)}


def host_counts(case, d, c):
    """The grounding counters of one flattened per-scene batch, restated with torch on the CPU (tests/test_eval_host.py)."""
    valid = d.get("valid", torch.ones(d["og3d_logits"].shape[0], dtype=torch.bool))
    p = torch.argmax(d["og3d_logits"], -1)
    ok = (p == d["tgt_object_id"][:, 0]) & valid
    c[_lib.EVG_ITEMS] += int(valid.sum())
    c[_lib.EVG_OG_ACC] += int(ok.sum())
    if case == "scanrefer":
        m = d["is_multiple"] & valid
        h25 = d["tgt_object_id_iou25"][torch.arange(len(p)), p].bool() & valid
        h50 = d["tgt_object_id_iou50"][torch.arange(len(p)), p].bool() & valid
        c[_lib.EVG_MULTIPLE] += int(m.sum())
        c[_lib.EVG_IOU25] += int(h25.sum())
        c[_lib.EVG_IOU50] += int(h50.sum())
        c[_lib.EVG_IOU25_MULTIPLE] += int((h25 & m).sum())
        c[_lib.EVG_IOU50_MULTIPLE] += int((h50 & m).sum())
    else:
        c[_lib.EVG_HARD] += int((d["is_hard"] & valid).sum())
        c[_lib.EVG_VIEW_DEP] += int((d["is_view_dependent"] & valid).sum())
        c[_lib.EVG_OG_ACC_HARD] += int((ok & d["is_hard"]).sum())
        c[_lib.EVG_OG_ACC_VIEW_DEP] += int((ok & d["is_view_dependent"]).sum())
    keys = evaluate._obj_logit_keys(d)
    sv = d.get("scene_valid", torch.ones(d["obj_masks"].shape[0], dtype=torch.bool))
    m = d["obj_masks"] & sv[:, None]
    for t, k in enumerate(keys):
        pred = torch.argmax(d[k], 2)
        c[_lib.EVG_OBJ + 2 * t] += int((pred[m] == d["obj_labels"][m]).sum())
        c[_lib.EVG_OBJ + 2 * t + 1] += int(m.sum())
    return keys


@pytest.mark.parametrize("case", ["scanrefer", "referit3d"])
def test_flatten_then_counters_reproduce_reference(case):
    """flatten_per_scene + the counters reproduce the reference evaluators' per-scene batch_metrics(include_count=True) of
    every batch and record() exactly; the B*U-row object logits are skipped, the per-scene ones counted once."""
    E, meta = eval_meta()
    m = meta[case]
    ev = getattr(evaluate, m["evaluator"])(device="cpu")
    total = ev.counters.tolist()
    for i in range(m["batches"]):
        d = eval_batch(E, case, i)
        B, U = d["og3d_logits"].shape[:2]
        flat = evaluate.flatten_per_scene(d)
        assert flat["og3d_logits"].shape == (B * U, d["og3d_logits"].shape[2])
        assert flat["og3d_logits"].data_ptr() == d["og3d_logits"].data_ptr()             # a view
        assert flat["tgt_object_id"].shape == (B * U, 1)
        c = [0.0] * ev.size
        keys = host_counts(case, flat, c)
        assert keys == ["obj_cls_raw_logits"]
        ev._obj_keys = keys
        got = ev.counts_to_metrics(c, include_count=True)
        assert {k: list(v) for k, v in got.items()} == m["batch_metrics"][i], i
        total = [a + b for a, b in zip(total, c)]
    ev.counters = torch.tensor(total, dtype=torch.float64)
    _, rec = ev.record()
    assert set(rec) == set(m["record"])
    for k, v in m["record"].items():
        assert rec[k] == v or abs(rec[k] - v) <= 1e-12 * abs(v), k


def test_flatten_per_scene_valid_and_plain_batches():
    d = {"og3d_logits": torch.zeros(3, 4, 6), "tgt_object_id": torch.zeros(3, 4, dtype=torch.int64),
         "is_hard": torch.zeros(3, 4, dtype=torch.bool), "valid": torch.tensor([True, True, False])}
    f = evaluate.flatten_per_scene(d)
    assert f["valid"].tolist() == [True] * 8 + [False] * 4 and f["scene_valid"] is d["valid"]
    assert f["is_hard"].shape == (12,) and d["og3d_logits"].shape == (3, 4, 6)       # the input dict is not changed
    plain = {"og3d_logits": torch.zeros(3, 6)}
    assert evaluate.flatten_per_scene(plain) == plain


# ---- GPU -----------------------------------------------------------------------------------------------------------------
def usum_case(dtype, B, U, O, D, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(B * U, O, D, generator=g, device="cuda") * torch.exp(torch.randn(B * U, O, D, generator=g, device="cuda")))
    return x.to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("U", [1, 3, 64])
@pytest.mark.parametrize("B,O,D", [(3, 7, 768), (2, 5, 40)])
def test_usum_kernel_vs_float64(dtype, U, B, O, D):
    """The backward of ops.scene_broadcast (sv_colsum_batched) against a float64 sum: |err| <= U 2^-24 sum|g| before the
    output rounding (bf16: plus half an ulp of the result); bitwise equal across two runs.  B*O = 21 / 10 rows, D = 40: not a
    multiple of the 256-column tile."""
    from sceneverse_b200 import ops
    x = torch.zeros(B, O, D, dtype=dtype, device="cuda", requires_grad=True)
    y = ops.scene_broadcast(x, U)
    g = usum_case(dtype, B, U, O, D)
    (dx,) = torch.autograd.grad(y, x, g)
    (dx2,) = torch.autograd.grad(ops.scene_broadcast(x, U), x, g)
    assert dx.dtype == dtype and dx.shape == (B, O, D)
    assert torch.equal(dx, dx2)
    g64 = g.double().view(B, U, O, D)
    want = g64.sum(1)
    bound = U * 2.0 ** -24 * g64.abs().sum(1)
    if dtype == torch.bfloat16:
        bound = bound * (1 + 2.0 ** -8) + 2.0 ** -8 * want.abs()
    err = (dx.double() - want).abs()
    assert (err <= bound).all(), float((err / bound.clamp_min(1e-300)).max())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_scene_broadcast_forward_equals_expand(dtype):
    from sceneverse_b200 import ops
    x = usum_case(dtype, 1, 3, 20, 768).view(3, 20, 768)
    y = ops.scene_broadcast(x, 5)
    assert torch.equal(y, x.unsqueeze(1).expand(3, 5, 20, 768).reshape(15, 20, 768))
    assert torch.equal(ops.scene_broadcast(x.cpu(), 5), y.cpu())


def test_usum_argument_validation():
    lib = _lib.gps()
    fake = 0x1000
    assert lib.sv_colsum_batched(fake, 100, 800, 1, 2, 4, 100, fake, fake, None) == 1        # N % 8
    assert lib.sv_colsum_batched(fake, 96, 804, 1, 2, 4, 96, fake, fake, None) == 1         # batch stride % 8
    assert lib.sv_colsum_batched(None, 96, 0, 1, 0, 4, 96, None, None, None) == 0           # no matrices
    assert lib.sv_colsum_batched_scratch_floats(4, 64, 61440) == 4 * 61440


@pytest.mark.gpu
def test_bf16_stack_matches_reference():
    """The fixture through the native bf16 path (autocast: native V2, LM head and cross-entropy, the U-sum kernel), at the
    bounds of tests/test_zz_reference_gradients_gpu.py."""
    from tests.test_zz_reference_gradients_gpu import FLOOR, LOSS_TOL, NORM_TOL
    F = np.load(os.path.join(GOLDEN, "model_per_scene.npz"))
    want_norms = json.load(open(os.path.join(GOLDEN, "model_per_scene_grad_norms.json")))
    m = stub_model("cuda")
    dd, parts, _, norms = run_stack(m, fixture_batch("cuda"))
    for k, v in parts.items():
        want = float(F["loss_" + k])
        assert abs(float(v.detach()) - want) / max(1.0, abs(want)) < LOSS_TOL, (k, float(v.detach()), want)
    scale = max(want_norms.values())
    bad = {k: (norms.get(k, 0.0), w) for k, w in want_norms.items()
           if abs(norms.get(k, 0.0) - w) > NORM_TOL * abs(w) + FLOOR * scale}
    assert not bad, bad
    og = dd["og3d_logits"].detach().float().cpu().numpy()
    assert np.abs(og - F["og3d_logits"]).max() <= LOSS_TOL * max(1.0, np.abs(F["og3d_logits"]).max())


def _step(graph, seed=3, no_dropout=True):
    from sceneverse_b200 import train
    cfg = M.per_scene_pretrain_config(1, text_features=TF)
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 0
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=seed, cuda_graph=graph, total_steps=50)
    if no_dropout:
        for m in ps.module.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
            if hasattr(m, "dropout") and isinstance(m.dropout, float):
                m.dropout = 0.0
    return ps


def _batch(seed, B=2, U=8, O=24):
    d = synthetic.per_scene_batch(seed, B=B, U=U, O=O, P=1024, T=50, min_obj=6)
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


@pytest.mark.gpu
def test_eager_steps_decrease_loss():
    ps = _step(False)
    assert type(ps.module.model) is M.OpenVocabPerScene
    b = _batch(11)
    got = [float(ps.step(dict(b))) for _ in range(4)]
    assert all(math.isfinite(v) for v in got) and all(y < x for x, y in zip(got, got[1:])), got
    ps.close()


@pytest.mark.gpu
def test_graph_replay_reads_new_batch():
    ps = _step(True)
    a, b = _batch(21), _batch(22)
    float(ps.step(dict(a)))
    ps.module.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        want_b, want_a = float(ps.module(dict(b))[0]), float(ps.module(dict(a))[0])
    ps.module.train()
    n0 = _lib.launch_count()
    lb = float(ps.step(dict(b)))
    assert _lib.launch_count() == n0
    assert abs(lb - want_b) < 0.1 * abs(want_b - want_a) and abs(lb - want_b) < 1e-3 * abs(want_b), (lb, want_b, want_a)
    ps.close()


@pytest.mark.gpu
def test_graph_step_matches_eager_step_parameters():
    from sceneverse_b200 import ops
    b = _batch(9)
    eager, graph = _step(False), _step(True)
    graph.module.load_state_dict(eager.module.state_dict())
    p0 = {n: p.detach().clone() for n, p in eager.module.named_parameters()}
    eager._probe_unused(dict(b))
    graph._probe_unused(dict(b))
    eager.step(dict(b))
    graph.static_batch = {k: v.clone() for k, v in b.items()}
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
    eager.close()
    graph.close()


@pytest.mark.gpu
def test_openvocab_checkpoint_loads_into_per_scene_step(tmp_path):
    """An OpenVocab pre-training checkpoint: every model key loads into the per-scene step through load_pretrain (none
    missing); the only unexpected keys are the pre-training losses' own (their file is offered to the model too)."""
    from sceneverse_b200 import train
    g = train.PretrainStep(M.pretrain_config(1, text_features=TF), "cuda", dtype=torch.bfloat16, seed=0)
    d = synthetic.scene_batch(40, B=2, O=24, P=1024, L=50, Ls=300)
    g.step({k: torch.from_numpy(v).cuda() for k, v in d.items()})
    g.save_state(tmp_path)
    want = {k: v.clone() for k, v in g.module.model.state_dict().items()}
    loss_keys = set(g.module.loss.state_dict())
    g.close()
    ps = _step(True, no_dropout=False)
    missing, unexpected = ps.load_pretrain(tmp_path)
    assert list(missing) == [] and set(unexpected) <= loss_keys, (missing, unexpected)
    got = ps.module.model.state_dict()
    assert set(got) == set(want) and all(torch.equal(got[k], want[k]) for k in want)
    assert math.isfinite(float(ps.step(_batch(41))))
    ps.close()


@pytest.mark.gpu
def test_graph_save_resume_bitwise(tmp_path):
    from tests.test_checkpoint_gpu import assert_same_tensors, graph_buffers, rng
    bs = [_batch(50 + i) for i in range(3)]
    a = _step(True, seed=0, no_dropout=False)
    for b in bs:
        a.step(b)
    torch.cuda.synchronize()
    a.save_state(tmp_path)
    want, want_rng, want_step = graph_buffers(a), rng(), a.global_step
    a.close()
    c = _step(True, seed=1, no_dropout=False)
    c.step(bs[0])
    c.load_state(tmp_path)
    assert_same_tensors(graph_buffers(c), want, "graph buffers")
    assert_same_tensors(rng(), want_rng, "generators")
    assert c.global_step == want_step
    c.close()


def _eval_step(seed=0):
    from sceneverse_b200 import train
    return train.PretrainStep(M.per_scene_pretrain_config(1, text_features=TF), "cuda", dtype=torch.bfloat16, seed=seed)


@pytest.mark.gpu
def test_eval_runner_graph_equals_eager_and_padding_counts_nothing():
    """Per-scene EvalRunner (ScanRefer + ReferIt3D counters): the graph replays equal eager updates of the flattened
    forward; a last batch of 1 scene (padded to 3 by whole scenes) counts only its own U utterances and objects."""
    ps = _eval_step()
    U = 6
    bs = [_batch(60, B=3, U=U), _batch(61, B=3, U=U), _batch(62, B=1, U=U)]
    evs = [evaluate.ScanReferEval(), evaluate.ReferIt3DEval()]
    runner = evaluate.EvalRunner(ps, evs, batch_size=3)
    runner.run(bs)
    got = [ev.counters.cpu().tolist() for ev in evs]
    eager = [evaluate.ScanReferEval(), evaluate.ReferIt3DEval()]
    model = ps.module.model.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for b in bs:
            out = evaluate.flatten_per_scene(model(dict(b)))
            for ev in eager:
                ev.update(out)
    model.train()
    assert got == [ev.counters.cpu().tolist() for ev in eager]
    assert got[0][_lib.EVG_ITEMS] == (3 + 3 + 1) * U
    assert got[0][_lib.EVG_OBJ + 1] == sum(int(b["obj_masks"].sum()) for b in bs)
    runner.run(bs)
    assert [ev.counters.cpu().tolist() for ev in evs] == got
    ps.close()


@pytest.mark.gpu
def test_eval_logits_match_per_utterance_model():
    """Eval mode: the per-scene og3d_logits of B scenes x U utterances against OpenVocab on the same B*U items (each scene's
    objects repeated), same weights, within the bf16 parity bound (GEMM tiling depends on M, so not bitwise)."""
    from sceneverse_b200 import train
    ps = _eval_step()
    cfg = M.pretrain_config(1, text_features=TF)
    cfg["data"]["args"]["use_scene_cap"] = False
    cfg["model"]["loss_list"] = cfg["model"]["vis_loss_list"] = ["lm_cls_loss", "TextObjWithinBatch"]
    plain = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=1)
    plain.module.model.load_state_dict(ps.module.model.state_dict())
    B, U = 2, 8
    b = _batch(70, B=B, U=U)
    flat = {k: v.reshape(B * U, *v.shape[2:]) for k, v in b.items() if k in ("txt_ids", "txt_masks", "masked_lm_labels")}
    for k in ("obj_fts", "obj_locs", "obj_masks", "obj_sem_masks", "obj_labels"):
        flat[k] = b[k].repeat_interleave(U, 0)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        a = ps.module.model.eval()(dict(b))["og3d_logits"].float()
        p = plain.module.model.eval()(dict(flat))["og3d_logits"].float()
    assert a.shape == (B, U, 24)
    err = (a.reshape(B * U, -1) - p).abs().max().item()
    assert err <= 2e-2 * p.abs().max().item(), (err, p.abs().max().item())
    ps.close()
    plain.close()
