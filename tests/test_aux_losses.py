"""The reference's object-classification and multi-target grounding losses (optim/loss/loss.py:12-47, 64-94) without a GPU:
the torch path of every new loss against the reference's own functions in float64 (tests/golden/aux_losses.npz, made by
oracle/make_golden_aux_losses.py), configs naming them, the per-scene checks, argument validation of
sv_masked_cross_entropy_fwd_bwd in a process that sees no CUDA device, and the opt-in multi-hot targets of scene_batch."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from sceneverse_b200 import model as M, ops, synthetic
from sceneverse_b200.modules import losses

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "aux_losses.npz"))
OBJ_LOSSES = ["obj_cls_raw_loss", "obj_cls_pre_loss", "obj_cls_post_loss", "obj_cls_pre_loss_mask", "obj_cls_pre_loss_unmask",
              "obj_cls_post_loss_mask", "obj_cls_post_loss_unmask"]
NEW_LOSSES = OBJ_LOSSES + ["og3d_multi_loss", "txt_cls_multi_loss"]
LOGITS_OF = {"obj_cls_raw_loss": "obj_cls_raw_logits", "og3d_multi_loss": "og3d_logits", "txt_cls_multi_loss": "txt_cls_logits",
             **{k: "obj_cls_pre_logits" if "_pre_" in k else "obj_cls_post_logits" for k in OBJ_LOSSES[1:]}}


def run_fp32(name, sem_key="obj_sem_masks"):
    """(loss, gradient w.r.t. the stored logits) of our loss on float32 copies of the fixture's inputs.  The object logits
    are stored 608 wide: the loss reads the 607-column view, which carries the padded parent as the native linear's does."""
    leaf = torch.from_numpy(G[LOGITS_OF[name]].copy()).requires_grad_(True)
    view = leaf[..., :607] if leaf.shape[-1] == 608 else leaf
    if view is not leaf:
        view._sv_padded = leaf
    dd = {k: torch.from_numpy(G[k].copy()) for k in ("obj_masks", "obj_labels", "tgt_object_id", "tgt_object_label")}
    dd["obj_sem_masks"] = torch.from_numpy(G[sem_key].copy())
    dd[LOGITS_OF[name]] = view
    loss = getattr(losses, name)(dd)
    loss.backward()
    return loss.detach().double().numpy(), leaf.grad.double().numpy()


def assert_matches(got, want, what):
    """fp32 tolerance: the loss within 2e-6 relative; each gradient entry within 1e-5 of the gradient's largest entry.
    NaN exactly where the reference has NaN."""
    (gl, gg), (wl, wg) = got, want
    assert np.isnan(gl) == np.isnan(wl), (what, gl, wl)
    if not np.isnan(wl):
        assert abs(gl - wl) <= 2e-6 * abs(wl), (what, gl, wl)
    assert (np.isnan(gg) == np.isnan(wg)).all(), what
    fin = ~np.isnan(wg)
    if fin.any():
        err = np.abs(gg[fin] - wg[fin]).max()
        assert err <= 1e-5 * np.abs(wg[fin]).max(), (what, err)


@pytest.mark.parametrize("name", NEW_LOSSES)
def test_torch_path_matches_reference_float64(name):
    assert_matches(run_fp32(name), (G["loss:" + name], G["grad:" + name]), name)


@pytest.mark.parametrize("name", [n for n in OBJ_LOSSES if n.endswith(("_mask", "_unmask"))])
def test_mask_split_without_members_is_nan(name):
    """obj_sem_masks == obj_masks: the `_mask` losses have no member (0 / 0 = NaN, gradient NaN), the `_unmask` losses
    are every valid object."""
    got = run_fp32(name, sem_key="obj_sem_masks_none")
    assert_matches(got, (G["loss_none:" + name], G["grad_none:" + name]), name)
    assert np.isnan(got[0]) == name.endswith("_mask")


def test_fixture_edge_cases():
    """What the fixture pins: padded slots with label -100 and zero gradient, -inf og3d logits at the padded objects (NaN
    loss, zero gradient there, finite elsewhere), zero gradient in the pad column of the 608-wide logits."""
    m = G["obj_masks"]
    assert (~m).any() and (G["obj_labels"][~m] == -100).all()
    for name in OBJ_LOSSES:
        g = G["grad:" + name]
        assert (g[~m] == 0).all() and (g[..., 607:] == 0).all(), name       # raw logits are 607 wide: an empty slice
    og = G["grad:og3d_multi_loss"]
    assert np.isnan(G["loss:og3d_multi_loss"]) and np.isinf(G["og3d_logits"][~m]).all()
    assert (og[~m] == 0).all() and np.isfinite(og).all()


def test_og3d_multi_loss_is_finite_without_ground_head():
    """The plain OpenVocab og3d_logits (einsum, no -inf): a finite loss equal to torch's BCE sum / B."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(3, 8, generator=g).requires_grad_(True)
    tgt = torch.from_numpy(G["tgt_object_id"].copy())
    loss = losses.og3d_multi_loss({"og3d_logits": x, "tgt_object_id": tgt})
    want = torch.nn.functional.binary_cross_entropy_with_logits(x.double(), tgt.double(), reduction="sum") / 3
    loss = loss.detach()
    assert torch.isfinite(loss) and abs(float(loss) - float(want)) <= 1e-6 * abs(float(want))


def test_configs_name_the_new_losses():
    from sceneverse_b200.modules.registry import LOSS_REGISTRY  # noqa: F401
    for make, names in ((M.scanrefer_config, ["og3d_loss", "obj_cls_raw_loss", "obj_cls_pre_loss", "obj_cls_post_loss",
                                              "obj_cls_pre_loss_mask", "obj_cls_pre_loss_unmask", "txt_cls_multi_loss"]),
                        (M.pretrain_config, ["lm_cls_loss", "obj_cls_raw_loss", "obj_cls_post_loss", "obj_cls_post_loss_mask",
                                             "obj_cls_post_loss_unmask"]),
                        (M.scanqa_config, ["answer_loss", "og3d_multi_loss"])):
        cfg = M.to_cfg(make(1))
        cfg["model"]["loss_list"] = cfg["model"]["vis_loss_list"] = list(names)
        loss = losses.Loss(cfg.model.loss_list, cfg.model.vis_loss_list, task=cfg.get("task"))
        assert list(loss.loss_fn) == names
        assert all(loss.loss_fn[n] is getattr(losses, n) for n in names if n in NEW_LOSSES)


def test_check_per_scene_for_each_new_loss():
    """The per-scene model (no ground head; obj_cls_post_logits of B*U object rows; (B, U, O) og3d_logits) runs
    obj_cls_raw_loss, whose (B, O, 607) logits match the (B, O) labels, and refuses every other new loss with its reason."""
    for name in NEW_LOSSES:
        cfg = M.per_scene_pretrain_config(1)
        cfg["model"]["loss_list"] = ["lm_cls_loss", name]
        cfg["model"]["vis_loss_list"] = ["lm_cls_loss", name]
        if name == "obj_cls_raw_loss":
            M.check_per_scene(cfg)
            continue
        with pytest.raises(ValueError) as e:
            M.check_per_scene(cfg)
        assert str(e.value) == f"OpenVocabPerScene cannot use '{name}': {M.PER_SCENE_UNSUPPORTED[name]}"


def test_masked_cross_entropy_rejects_bad_arguments():
    x, y, m = torch.zeros(2, 3, 5), torch.zeros(2, 3, dtype=torch.int64), torch.ones(2, 3, dtype=torch.bool)
    with pytest.raises(ValueError, match="mode"):
        ops.masked_cross_entropy(x, y, m, m, mode=3)
    with pytest.raises(ValueError, match="sem_masks"):
        ops.masked_cross_entropy(x, y, m, None, mode=1)
    with pytest.raises(ValueError, match="must be"):
        ops.masked_cross_entropy(x, y[:, :2], m)
    with pytest.raises(ValueError, match="must be"):
        ops.masked_cross_entropy(x.reshape(6, 5), y, m)


_VALIDATION = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from sceneverse_b200 import _lib
lib = _lib.gps()
a = 0x1000      # 16-byte aligned fake address


def ce(x=a, rs=608, bf=1, y=a, om=a, sm=a, mode=1, R=4, V=607, rows=a, sums=a, out=a, cnt=a, g=a, gs=608):
    return lib.sv_masked_cross_entropy_fwd_bwd(x, rs, bf, y, om, sm, mode, R, V, rows, sums, out, cnt, g, gs, None)


out = {"R 0": ce(R=0), "V 0": ce(V=0), "row stride < V": ce(rs=600), "grad stride < V": ce(gs=600),
       "mode -1": ce(mode=-1), "mode 3": ce(mode=3), "mode 1 without sem mask": ce(sm=None),
       "mode 2 without sem mask": ce(mode=2, sm=None), "NULL logits": ce(x=None), "NULL labels": ce(y=None),
       "NULL obj mask": ce(om=None), "NULL rows": ce(rows=None), "NULL sums": ce(sums=None), "NULL out": ce(out=None),
       "NULL counter": ce(cnt=None), "misaligned labels": ce(y=a + 4), "misaligned bf16 logits": ce(x=a + 1),
       "misaligned f32 logits": ce(bf=0, x=a + 2), "misaligned grad": ce(g=a + 1), "misaligned f32 grad": ce(bf=0, g=a + 2),
       "misaligned rows": ce(rows=a + 2), "misaligned sums": ce(sums=a + 1), "misaligned out": ce(out=a + 3),
       "misaligned counter": ce(cnt=a + 2)}
print(json.dumps(out))
"""


def test_masked_ce_entry_point_validates_arguments_without_gpu():
    """sv_masked_cross_entropy_fwd_bwd rejects malformed calls before any launch (1 = SV_ERR_INVALID_ARG).  The calls run in
    a process that sees no CUDA device: a missing check would reach the launch and return 2 instead."""
    res = subprocess.run([sys.executable, "-c", _VALIDATION, ROOT], capture_output=True, text=True, timeout=120,
                         env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    bad = {k: v for k, v in got.items() if v != 1}
    assert len(got) == 24 and not bad, bad


def test_scene_batch_multi_hot_targets_are_opt_in():
    a = synthetic.scene_batch(5, B=6, O=12, P=16, L=10, Ls=10)
    b = synthetic.scene_batch(5, B=6, O=12, P=16, L=10, Ls=10, multi_target=True, multi_label=True)
    c = synthetic.scene_batch(5, B=6, O=12, P=16, L=10, Ls=10, multi_label=True)
    assert "tgt_object_label" not in a and a["tgt_object_id"].shape == (6, 1)
    assert all(np.array_equal(a[k], b[k]) for k in a if k != "tgt_object_id")
    tgt, m, lab = b["tgt_object_id"], b["obj_masks"], b["obj_labels"]
    assert tgt.dtype == np.int64 and tgt.shape == (6, 12) and (tgt[np.arange(6), a["tgt_object_id"][:, 0]] == 1).all()
    assert set(np.unique(tgt.sum(1))) <= {1, 2, 3} and (tgt * ~m).sum() == 0
    assert b["tgt_object_label"].shape == (6, 607) and b["tgt_object_label"].dtype == np.int64
    for i in range(6):
        assert set(np.flatnonzero(b["tgt_object_label"][i])) == set(lab[i][tgt[i] == 1])
        assert list(np.flatnonzero(c["tgt_object_label"][i])) == [lab[i, a["tgt_object_id"][i, 0]]]
    assert np.array_equal(c["tgt_object_id"], a["tgt_object_id"])
