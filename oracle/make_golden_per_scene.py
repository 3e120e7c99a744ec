"""ORACLE — TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available (oracle/ref_shims.py):
    python oracle/make_golden_per_scene.py
Per-scene grounding fixtures (tests/golden/model_per_scene.npz, model_per_scene_grad_norms.json, eval_per_scene.npz):

* Model: the UNMODIFIED reference `OpenVocabPerScene.forward` (model/openvocab.py:141-230) on CPU in fp32, eval mode, with the
  reference UnifiedSpatialCrossEncoderV2 and OVPretrainHead (name-keyed synthetic weights, sceneverse_b200/weights.py) and the
  reference lm_cls_loss, TextObjWithinBatch and TextObjBetweenBatch on a synthetic.per_scene_batch (B = 2 scenes, U = 4
  utterances, O = 16 object slots, one scene padded).  BERT and PointNet++ cannot be loaded here, so two stub encoders
  registered in the reference registries stand in for them: seeded learnable tensors of shape (B*U, T, D) for the text and
  (B, O, D) for the objects.  The object stub's gradient is then exactly the sum over each scene's U utterance copies.
  Stored: og3d_logits (B, U, O), every loss term and their total, the gradient norm of every parameter (stubs included) and
  a few gradient slices.
* Evaluation: the UNMODIFIED reference ScanReferEval and ReferIt3DEval `batch_metrics(include_count=True)` of per-scene
  batches (og3d_logits (B, U, O), per-utterance targets and flags, per-scene object logits next to B*U-row ones) and
  `record()` after `update` of all of them.
"""
import importlib
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402
from sceneverse_b200 import synthetic, weights  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
PER_SCENE_GOLDEN = dict(data_seed=4, B=2, U=4, O=16, T=50, D=768, lang_seed=17, obj_seed=18, v2_seed=1, head_seed=5)


def stub_tensor(shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * 0.5


class StubLanguageEncoder(nn.Module):
    """Stands in for BERT: a learnable (rows, T, D) tensor, whatever the token ids."""

    def __init__(self, cfg, rows=8, T=50, D=768, seed=0):
        super().__init__()
        self.feats = nn.Parameter(stub_tensor((rows, T, D), seed))

    def forward(self, txt_ids, txt_masks, **kwargs):
        assert txt_ids.shape == self.feats.shape[:2], (tuple(txt_ids.shape), tuple(self.feats.shape))
        return self.feats


class StubVisionEncoder(nn.Module):
    """Stands in for PointNet++ and the spatial layers: a learnable (B, O, D) tensor as the object features (and as the
    pre-spatial features); no object-class logits."""

    def __init__(self, cfg, B=2, O=16, D=768, seed=0):
        super().__init__()
        self.feats = nn.Parameter(stub_tensor((B, O, D), seed))

    def forward(self, obj_fts, obj_locs, obj_masks, obj_sem_masks, obj_labels, cur_step, total_steps):
        assert obj_masks.shape == self.feats.shape[:2]
        return self.feats, self.feats, None


def per_scene_cfg(q=PER_SCENE_GOLDEN):
    """The model config the fixture's model is built from (attribute access, as the reference reads it)."""
    ns = types.SimpleNamespace
    return ns(
        num_gpu=1, task="Pretrain", solver=ns(lr=5e-4), data=ns(args={}),
        model=ns(name="OpenVocabPerScene", inter="before",
                 language=ns(name="StubLanguageEncoder", args={"rows": q["B"] * q["U"], "T": q["T"], "D": q["D"],
                                                               "seed": q["lang_seed"]}),
                 vision=ns(name="StubVisionEncoder", args={"B": q["B"], "O": q["O"], "D": q["D"], "seed": q["obj_seed"]}),
                 grounding=ns(name="UnifiedSpatialCrossEncoderV2", args={}),
                 heads=ns(head_list=["pretrain_head"], pretrain_head=ns(name="OVPretrainHead", args={}))))


def per_scene_inputs(q=PER_SCENE_GOLDEN):
    d = synthetic.per_scene_batch(q["data_seed"], B=q["B"], U=q["U"], O=q["O"], P=16, T=q["T"], min_obj=6)
    n = d["obj_masks"].sum(1)
    assert (n < q["O"]).sum() == 1, n           # one scene padded, one full
    return d


SLICES = ["point_encoder.feats", "lang_encoder.feats", "unified_encoder.unified_encoder.0.self_attn.in_proj_weight",
          "pretrain_head.lm_pred_head.transform.dense.weight", "pretrain_head.lm_pred_head.decoder.weight"]


def golden_model():
    ref_shims.install()
    from modules.build import GROUNDING_REGISTRY, LANGUAGE_REGISTRY, VISION_REGISTRY  # noqa: F401
    import modules.grounding.unified_encoder  # noqa: F401
    import modules.heads.pretrain_head  # noqa: F401
    LANGUAGE_REGISTRY.register(StubLanguageEncoder)
    VISION_REGISTRY.register(StubVisionEncoder)
    pkg = types.ModuleType("model")                  # skip model/__init__ (objcls and its CLIP / dataset imports)
    pkg.__path__ = [os.path.join(ref_shims.REF_ROOT, "model")]
    sys.modules["model"] = pkg
    OV = importlib.import_module("model.openvocab")
    CL = importlib.import_module("optim.loss.contra_loss")
    LL = importlib.import_module("optim.loss.loss")
    q = PER_SCENE_GOLDEN
    d = per_scene_inputs()
    t = {k: torch.from_numpy(v) for k, v in d.items()}
    cfg = per_scene_cfg()
    with ref_shims.cpu_cuda_identity():
        model = OV.OpenVocabPerScene(cfg)
        model.unified_encoder.load_state_dict(weights.synthetic_state_dict(model.unified_encoder, seed=q["v2_seed"]))
        model.pretrain_head.load_state_dict(weights.synthetic_state_dict(model.pretrain_head, seed=q["head_seed"]))
        model.eval()
        losses = {"l_within": CL.TextObjWithinBatch(cfg), "l_obj": CL.TextObjBetweenBatch(cfg)}
        dd = model(dict(t))
        parts = {"lm": LL.lm_cls_loss(dd), "within": losses["l_within"](dd), "obj_between": losses["l_obj"](dd)}
        total = sum(parts.values())
        total.backward()
    norms = {n: float(p.grad.double().norm()) for n, p in model.named_parameters() if p.grad is not None}
    norms.update({f"loss.{k}.{n}": float(p.grad.double().norm()) for k, m in losses.items()
                  for n, p in m.named_parameters() if p.grad is not None})
    params = dict(model.named_parameters())
    slices = {k: params[k].grad.reshape(-1)[:96].numpy() for k in SLICES}
    np.savez_compressed(os.path.join(OUT, "model_per_scene.npz"), **{k: np.int64(v) for k, v in q.items()},
                        og3d_logits=dd["og3d_logits"].detach().numpy(), total=total.detach().numpy(),
                        **{"loss_" + k: v.detach().numpy() for k, v in parts.items()},
                        **{"slice:" + k: v for k, v in slices.items()})
    json.dump(norms, open(os.path.join(OUT, "model_per_scene_grad_norms.json"), "w"), indent=0, sort_keys=True)
    print("per-scene golden:", {k: float(v) for k, v in parts.items()}, len(norms), "parameter gradients")


# ---- evaluation ----------------------------------------------------------------------------------------------------------
def per_scene_eval_batch(rng, B, U, O=12, C=40, with_iou=True):
    """B scenes x U utterances: og3d_logits (B, U, O) on a coarse grid (ties; padded slots -inf; one all -inf row), per-scene
    object keys and object logits (B, O, C), B*U-row object logits (obj_cls_post_logits, which the evaluators skip)."""
    from oracle.make_golden_eval import _q
    n = rng.integers(3, O + 1, size=B)
    masks = np.arange(O)[None] < n[:, None]
    og = _q(rng, (B, U, O))
    og[~np.broadcast_to(masks[:, None, :], og.shape)] = -np.inf
    og[0, 0, :] = -np.inf
    og[0, 1, :3] = og[0, 1, :3].max()
    d = {"og3d_logits": og, "obj_masks": masks,
         "obj_labels": np.where(masks, rng.integers(0, 8, size=(B, O)), -100).astype(np.int64),
         "tgt_object_id": np.stack([rng.integers(0, k, size=U) for k in n]).astype(np.int64)}
    d["obj_cls_raw_logits"] = _q(rng, (B, O, C), -1, 1)
    d["obj_cls_raw_logits"][:, :, :8] = _q(rng, (B, O, 8), 0, 2)
    d["obj_cls_post_logits"] = _q(rng, (B * U, O, C), -1, 1)
    if with_iou:
        d["tgt_object_id_iou25"] = (rng.random((B, U, O)) < 0.3).astype(np.int64)
        d["tgt_object_id_iou50"] = d["tgt_object_id_iou25"] * (rng.random((B, U, O)) < 0.6)
        d["is_multiple"] = rng.random((B, U)) < 0.5
    else:
        d["is_hard"] = rng.random((B, U)) < 0.4
        d["is_view_dependent"] = rng.random((B, U)) < 0.3
    # the last scene repeats its first utterance, as per_scene_pad fills a scene with too few utterances
    for k in ("og3d_logits", "tgt_object_id", "tgt_object_id_iou25", "tgt_object_id_iou50", "is_multiple", "is_hard",
              "is_view_dependent"):
        if k in d:
            d[k][-1, -1] = d[k][-1, 0]
    return d


EVAL_CASES = {  # name -> (evaluator, with_iou, scenes per batch, utterances per scene)
    "scanrefer": ("ScanReferEval", True, (3, 2), 4),
    "referit3d": ("ReferIt3DEval", False, (2, 3), 5),
}


def golden_eval():
    from oracle import make_golden_eval as E
    mods, _ = E._install()
    out, meta = {}, {}
    with tempfile.TemporaryDirectory() as exp_dir:
        for case, (name, with_iou, sizes, U) in EVAL_CASES.items():
            rng = np.random.default_rng(sum(map(ord, case)) + 1)
            ev = E._evaluator(mods, name, exp_dir)
            per_batch = []
            for i, B in enumerate(sizes):
                d = per_scene_eval_batch(rng, B, U, with_iou=with_iou)
                for k, v in d.items():
                    out[f"{case}:{i}:{k}"] = v
                t = {k: torch.from_numpy(v) for k, v in d.items()}
                bm = ev.batch_metrics(dict(t), include_count=True)
                per_batch.append({k: list(v) for k, v in bm.items()})
                ev.update(dict(t))
            _, rec = ev.record()
            meta[case] = {"evaluator": name, "batches": len(sizes), "batch_metrics": per_batch,
                          "record": {k: float(v) for k, v in rec.items()}}
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), np.uint8)
    np.savez_compressed(os.path.join(OUT, "eval_per_scene.npz"), **out)
    print("eval_per_scene.npz:", {c: m["record"]["target_metric"] for c, m in meta.items()})


if __name__ == "__main__":
    torch.manual_seed(0)
    golden_model()
    golden_eval()
