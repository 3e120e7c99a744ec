"""ORACLE — TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available (oracle/ref_shims.py):
    python oracle/make_golden_aux_losses.py
Fixture of the reference's object-classification and multi-target grounding losses (tests/golden/aux_losses.npz): the
UNMODIFIED optim/loss/loss.py functions obj_cls_{raw,pre,post}_loss, obj_cls_{pre,post}_loss_{mask,unmask},
og3d_multi_loss and txt_cls_multi_loss in float64 on the CPU, on a seeded synthetic batch, with the gradient of each loss
with respect to the logits it reads.

The batch holds padded object slots (obj_masks False, label -100); -inf og3d logits at the padded objects, as GroundHeadV1
makes them (NaN loss, zero gradient there); object logits stored 608 wide with a zero pad column, as the native linear
writes them (the losses read the first 607 columns); and a second set of semantic masks equal to obj_masks, under which the
`_mask` losses have no member (0 / 0 = NaN).  The inputs are stored in float32, the values the tests feed; the reference
runs on their float64 copies.
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402
from sceneverse_b200 import synthetic  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "aux_losses.npz")
SEEDS = dict(data_seed=17, logit_seed=5, B=3, O=8)
V, W = 607, 608
OBJ_LOSSES = ("obj_cls_raw_loss", "obj_cls_pre_loss", "obj_cls_post_loss", "obj_cls_pre_loss_mask",
              "obj_cls_pre_loss_unmask", "obj_cls_post_loss_mask", "obj_cls_post_loss_unmask")
LOGITS_OF = {"obj_cls_raw_loss": "obj_cls_raw_logits", "og3d_multi_loss": "og3d_logits",
             "txt_cls_multi_loss": "txt_cls_logits"}
for _k in OBJ_LOSSES[1:]:
    LOGITS_OF[_k] = "obj_cls_pre_logits" if "_pre_" in _k else "obj_cls_post_logits"
ALL_LOSSES = OBJ_LOSSES + ("og3d_multi_loss", "txt_cls_multi_loss")


def inputs(s=SEEDS):
    """The batch (numpy): masks, labels, multi-hot targets and every logits tensor in float32."""
    B, O = s["B"], s["O"]
    d = synthetic.scene_batch(s["data_seed"], B=B, O=O, P=16, L=8, Ls=8, min_obj=4, max_obj=O - 2, multi_target=True,
                              multi_label=True)
    g = torch.Generator().manual_seed(s["logit_seed"])
    pre = torch.zeros(B, O, W)
    pre[..., :V] = torch.randn(B, O, V, generator=g) * 3
    post = torch.zeros(B, O, W)
    post[..., :V] = torch.randn(B, O, V, generator=g) * 3
    raw = torch.softmax(torch.randn(B, O, V, generator=g) * 4, dim=2)     # probabilities, as the object encoder gives them
    og3d = (torch.randn(B, O, generator=g) * 2).masked_fill(~torch.from_numpy(d["obj_masks"]), -float("inf"))
    txt = torch.zeros(B, W)
    txt[:, :V] = torch.randn(B, V, generator=g) * 3
    out = {k: d[k] for k in ("obj_masks", "obj_sem_masks", "obj_labels", "tgt_object_id", "tgt_object_label")}
    out.update(obj_sem_masks_none=d["obj_masks"].copy(), obj_cls_raw_logits=raw.numpy(), obj_cls_pre_logits=pre.numpy(),
               obj_cls_post_logits=post.numpy(), og3d_logits=og3d.numpy(), txt_cls_logits=txt.numpy())
    return out


def run(fn, arrays, logits_key, sem_key="obj_sem_masks"):
    """(loss, gradient w.r.t. the stored logits tensor) of one reference loss in float64."""
    leaf = torch.from_numpy(arrays[logits_key]).double().requires_grad_(True)
    dd = {k: torch.from_numpy(arrays[k]) for k in ("obj_masks", "obj_labels", "tgt_object_id", "tgt_object_label")}
    dd["obj_sem_masks"] = torch.from_numpy(arrays[sem_key])
    view = leaf[..., :V] if leaf.shape[-1] == W else leaf
    dd[logits_key] = view
    loss = fn(dd)
    loss.backward()
    return loss.detach().numpy(), leaf.grad.numpy()


def main():
    ref_shims.install()
    LL = importlib.import_module("optim.loss.loss")
    a = inputs()
    m, sem = a["obj_masks"], a["obj_sem_masks"]
    assert (~m).any() and (a["obj_labels"][~m] == -100).all()
    assert (m & ~sem).any() and (m & sem).any() and not (m & ~a["obj_sem_masks_none"]).any()
    assert (a["tgt_object_id"].sum(1) > 1).any()
    res = {k: np.int64(v) for k, v in SEEDS.items()}
    res.update(a)
    for name in ALL_LOSSES:
        loss, grad = run(getattr(LL, name), a, LOGITS_OF[name])
        res["loss:" + name], res["grad:" + name] = loss, grad
    for name in OBJ_LOSSES[3:]:
        loss, grad = run(getattr(LL, name), a, LOGITS_OF[name], sem_key="obj_sem_masks_none")
        res["loss_none:" + name], res["grad_none:" + name] = loss, grad
    assert all(np.isnan(res["loss_none:" + n]) for n in OBJ_LOSSES[3:] if n.endswith("_mask"))
    assert np.isnan(res["loss:og3d_multi_loss"]) and (res["grad:og3d_multi_loss"][~m] == 0).all()
    assert all(np.isfinite(res["loss:" + n]) for n in ALL_LOSSES if n != "og3d_multi_loss")
    np.savez_compressed(OUT, **res)
    print("aux-loss golden:", {n: float(res["loss:" + n]) for n in ALL_LOSSES})


if __name__ == "__main__":
    main()
