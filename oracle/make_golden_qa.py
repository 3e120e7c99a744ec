"""ORACLE — TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available (oracle/ref_shims.py):
    python oracle/make_golden_qa.py
Backward parity fixture of the ScanQA fine-tune (tests/golden/model_qa_grads.npz, model_qa_grad_norms.json): the UNMODIFIED
reference UnifiedSpatialCrossEncoderV2 -> QAHeadV1 (8864 answers) -> answer_loss + TextObjWithinBatch with cfg.task =
'ScanQA' (masked BCE over a multi-hot target), eval mode, fp32 CPU, name-keyed synthetic weights
(sceneverse_b200/weights.py).  Same machinery as oracle/make_golden_model.py::golden_gps_backward.
"""
import importlib
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402
from oracle.make_golden_model import OUT, _load  # noqa: E402
from sceneverse_b200 import synthetic  # noqa: E402

QA_GOLDEN = dict(data_seed=41, feat_seed=9, B=2, O=16, L=50, num_answers=8864, v2_seed=1, head_seed=12)


def qa_inputs(q=QA_GOLDEN):
    """The seeded batch (row 0: no answer; row B-1: only the 'no target' placeholder) and encoder input features.  The
    features stand in for the text / object encoders, whose backward golden_gps_backward already pins."""
    d = synthetic.qa_batch(q["data_seed"], "ScanQA", B=q["B"], O=q["O"], L=q["L"], num_answers=q["num_answers"], min_obj=6,
                           edge_rows=True)
    g = torch.Generator().manual_seed(q["feat_seed"])
    txt = torch.randn(q["B"], q["L"], 768, generator=g) * 0.5
    obj = torch.randn(q["B"], q["O"], 768, generator=g) * 0.5
    return d, txt, obj


def golden_qa_backward():
    from modules.build import GROUNDING_REGISTRY
    from modules.heads.qa_head import QAHeadV1
    CL = importlib.import_module("optim.loss.contra_loss")
    LL = importlib.import_module("optim.loss.loss")
    q = QA_GOLDEN
    d, txt, obj = qa_inputs()
    t = {k: torch.from_numpy(v) for k, v in d.items()}
    assert int(t["answer_label"][0].sum()) == 0 and int(t["tgt_object_id"][-1].sum()) == 1
    cfg = types.SimpleNamespace(num_gpu=1, task="ScanQA")
    with ref_shims.cpu_cuda_identity():
        mods = {"v2": _load(GROUNDING_REGISTRY.get("UnifiedSpatialCrossEncoderV2")(None), q["v2_seed"]),
                "qa": _load(QAHeadV1(None, num_answers=q["num_answers"]), q["head_seed"]),
                "l_within": CL.TextObjWithinBatch(cfg)}
        t2, o2 = mods["v2"](txt, t["txt_masks"], obj, t["obj_locs"], t["obj_masks"])
        scores = mods["qa"](o2, t["obj_masks"], t2, t["txt_masks"])
        dd = dict(t)
        dd.update(intra_obj_embeds=o2, intra_text_embed=t2[:, 0], answer_scores=scores)
        parts = {"answer": LL.answer_loss(dd), "within": mods["l_within"](dd)}
        total = sum(parts.values())
        total.backward()
    norms, slices = {}, {}
    for mname, m in mods.items():
        for n, p in m.named_parameters():
            if p.grad is not None:
                norms[f"{mname}.{n}"] = float(p.grad.double().norm())
    for key in ["qa.answer_cls.3.weight", "qa.answer_cls.0.weight", "qa.attflat_visual.mlp.fc.linear.weight",
                "qa.attflat_lang.linear_merge.weight", "v2.unified_encoder.3.self_attn.in_proj_weight"]:
        mname, n = key.split(".", 1)
        slices[key] = dict(mods[mname].named_parameters())[n].grad.reshape(-1)[:96].numpy()
    np.savez_compressed(os.path.join(OUT, "model_qa_grads.npz"), **{k: np.int64(v) for k, v in q.items()},
                        answer_scores=scores.detach().numpy(), total=total.detach().numpy(),
                        **{"loss_" + k: v.detach().numpy() for k, v in parts.items()},
                        **{"slice:" + k: v for k, v in slices.items()})
    json.dump(norms, open(os.path.join(OUT, "model_qa_grad_norms.json"), "w"), indent=0, sort_keys=True)
    print("QA backward golden:", {k: float(v) for k, v in parts.items()}, len(norms), "parameter gradients")


if __name__ == "__main__":
    ref_shims.install()
    torch.manual_seed(0)
    golden_qa_backward()
