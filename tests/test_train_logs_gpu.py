"""Per-step train logs of train.PretrainStep(train_eval=...): each logged entry against a torch restatement of the
reference evaluator's batch_metrics on what that step computed, the logged losses against that step's loss tensors, no host
synchronisation in graph-mode steps, the ring's overflow, the eager path, and that logging leaves training unchanged."""
import numpy as np
import pytest
import torch

from sceneverse_b200 import evaluate, model as M, ops, synthetic, train, weights
from tests.test_eval_gpu import _train_state

pytestmark = pytest.mark.gpu


def _tf():
    return weights.synthetic_tensor("text_features", (607, 768))


def pretrain_batches(n, B=4):
    return [{k: torch.from_numpy(v).cuda() for k, v in
             synthetic.scene_batch(11 + i, B=B, O=16, P=1024, L=50, Ls=300, min_obj=6).items()} for i in range(n)]


def scanrefer_batches(n, B=4, O=16):
    out = []
    for i in range(n):
        d = synthetic.scene_batch(31 + i, B=B, O=O, P=1024, L=50, min_obj=6)
        rng = np.random.default_rng(i)
        d["tgt_object_id_iou25"] = (rng.random((B, O)) < 0.3).astype(np.int64)
        d["tgt_object_id_iou50"] = d["tgt_object_id_iou25"] * (rng.random((B, O)) < 0.6)
        d["is_multiple"] = rng.random(B) < 0.5
        d["tgt_object_label"] = rng.integers(0, 607, (B, 1))
        out.append({k: torch.from_numpy(np.asarray(v)).cuda() for k, v in d.items()})
    return out


class Stash:
    """Keeps detached views of the data dict and the loss dict of the last forward (views only: holding the autograd graph
    of a warm-up step would break the capture).  In graph mode that is the capture's: its storage stays alive, so every
    replay rewrites it with what that replay computed."""

    def __init__(self, ps):
        fwd = ps.module.loss.forward

        def forward(d):
            total, all_losses = fwd(d)
            self.data = {k: v.detach() for k, v in d.items() if torch.is_tensor(v)}
            self.losses = {k: v.detach() for k, v in all_losses.items()}
            return total, all_losses
        ps.module.loss.forward = forward

    def cpu(self):
        return {k: (v.float().cpu() if v.is_floating_point() else v.cpu()) for k, v in self.data.items() if torch.is_tensor(v)}


def _sum(xs):
    s = 0
    for x in xs:
        s = s + x
    return s


def ref_pretrain_metrics(d):
    """evaluator/pretrain_eval.py:21-67 restated with torch on the CPU (sums left to right, as the reference's Python)."""
    m = {}
    tok = d["masked_lm_labels"] != -1
    if "tgt_object_id" in d:
        m["og_acc"] = (torch.argmax(d["og3d_logits"], -1) == d["tgt_object_id"].squeeze(1)).sum().item() / \
            float(len(d["tgt_object_id"]))
    m["lang_cls_acc_mask"] = torch.sum(torch.argmax(d["txt_lm_cls_logits"], 2)[tok] == d["masked_lm_labels"][tok]).item() / \
        float(tok.sum().item() + 1e-8)
    om, sem = d["obj_masks"], d["obj_sem_masks"]
    for name in ("post", "raw", "pre"):
        k = f"obj_cls_{name}_logits"
        if k not in d:
            continue
        pred = torch.argmax(d[k], 2)
        splits = [("", om)] + ([("_unmask", om * sem), ("_mask", om * sem.logical_not())] if name != "raw" else [])
        for suffix, mm in splits:
            m[f"obj_cls_{name}_acc{suffix}"] = torch.sum(pred[mm] == d["obj_labels"][mm]).item() / float(mm.sum().item() + 1e-8)
    acc = list(m.values())
    m["target_metric"] = float(_sum(acc)) / len(acc)
    m["total_count"] = d["txt_lm_cls_logits"].shape[0]
    return m


def ref_scanrefer_metrics(d):
    """evaluator/scanrefer_eval.py batch_metrics(include_count=False) restated with torch on the CPU."""
    pred = torch.argmax(d["og3d_logits"], -1)
    n = len(pred)
    mult = d["is_multiple"].sum().item()
    i25 = d["tgt_object_id_iou25"][torch.arange(n), pred].bool()
    i50 = d["tgt_object_id_iou50"][torch.arange(n), pred].bool()
    m = {"og_acc_iou25": (i25.sum().item(), n), "og_acc_iou50": (i50.sum().item(), n),
         "og_acc_iou25_unique": ((i25 & ~d["is_multiple"]).sum().item(), n - mult),
         "og_acc_iou50_unique": ((i50 & ~d["is_multiple"]).sum().item(), n - mult),
         "og_acc_iou25_multiple": ((i25 & d["is_multiple"]).sum().item(), mult),
         "og_acc_iou50_multiple": ((i50 & d["is_multiple"]).sum().item(), mult),
         "og_acc": ((pred == d["tgt_object_id"].squeeze(1)).sum().item(), n)}
    if "txt_cls_logits" in d:
        m["txt_acc"] = ((torch.argmax(d["txt_cls_logits"], 1) == d["tgt_object_label"].squeeze(1)).sum().item(), n)
    mask = d["obj_masks"]
    for k, v in d.items():
        if k.endswith("logits") and v.ndim == 3 and v.shape[:2] == d["obj_labels"].shape:
            p = torch.argmax(v, 2)
            m[k.replace("logits", "acc")] = ((p[mask] == d["obj_labels"][mask]).sum().item(), mask.sum().item())
    return {k: v[0] / max(v[1], 1) for k, v in m.items()}


def check_entry(ps, entry, stash, ref, step, loss):
    """entry == the reference trainer's log dict of the step whose outputs `stash` holds."""
    want = {"train/step": step}
    want.update((f"train/{k}", float(v)) for k, v in stash.losses.items())
    want.update((f"train/{k}", v) for k, v in ref(stash.cpu()).items())
    want.update((f"train/lr/group_{i}", lr) for i, lr in enumerate(ps._lrs()))
    assert list(entry) == list(want)
    for k, v in want.items():
        assert entry[k] == v, (k, entry[k], v)
    assert entry["train/total_loss"] == float(loss)


def test_pretrain_graph_logs():
    """Pre-training config, graph mode, PretrainEval: after every replay that step's entry equals the restatement on the
    outputs the replay computed; graph-mode steps do not synchronise the host; a full ring raises instead of dropping."""
    ps = train.PretrainStep(M.pretrain_config(text_features=_tf()), "cuda:0", seed=0, cuda_graph=True,
                            train_eval=evaluate.PretrainEval(), log_every=3)
    try:
        stash = Stash(ps)
        batches = pretrain_batches(3)
        ps.step(batches[0])                          # set-up: probe, eager steps, capture, first replay
        assert len(ps.logs()) == 1
        for i in range(4):
            loss = ps.step(batches[i % 3])
            (entry,) = ps.logs()
            check_entry(ps, entry, stash, ref_pretrain_metrics, i + 2, loss)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for i in range(3):
                ps.step(batches[i])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        with pytest.raises(RuntimeError, match="log_every"):
            ps.step(batches[0])
        logs = ps.logs()
        assert [e["train/step"] for e in logs] == [6, 7, 8]
        loss = ps.step(batches[1])                   # the raise lost nothing and stepped nothing
        (entry,) = ps.logs()
        check_entry(ps, entry, stash, ref_pretrain_metrics, 9, loss)
    finally:
        ps.close()


def test_scanrefer_graph_logs():
    ps = train.PretrainStep(M.scanrefer_config(text_features=_tf()), "cuda:0", seed=0, cuda_graph=True,
                            train_eval=evaluate.ScanReferEval(), log_every=4)
    try:
        stash = Stash(ps)
        batches = scanrefer_batches(2)
        ps.step(batches[0])
        ps.logs()
        for i in range(3):
            loss = ps.step(batches[i % 2])
            (entry,) = ps.logs()
            check_entry(ps, entry, stash, ref_scanrefer_metrics, i + 2, loss)
            assert "train/txt_acc" in entry and "train/obj_cls_post_acc" in entry
    finally:
        ps.close()


def test_missing_batch_key_raises_at_the_first_step():
    ps = train.PretrainStep(M.scanrefer_config(text_features=_tf()), "cuda:0", seed=0, cuda_graph=True,
                            train_eval=evaluate.ScanReferEval())
    try:
        b = scanrefer_batches(1)[0]
        del b["tgt_object_id_iou25"]
        with pytest.raises(KeyError, match="tgt_object_id_iou25"):
            ps.step(b)
    finally:
        ps.close()


def test_eager_logs():
    """Without a graph: the same entries, from the same arithmetic."""
    ps = train.PretrainStep(M.pretrain_config(text_features=_tf()), "cuda:0", seed=0, cuda_graph=False,
                            train_eval=evaluate.PretrainEval(), log_every=2)
    try:
        stash = Stash(ps)
        for i, b in enumerate(pretrain_batches(2)):
            loss = ps.step(b)
            (entry,) = ps.logs()
            check_entry(ps, entry, stash, ref_pretrain_metrics, i + 1, loss)
    finally:
        ps.close()


def test_logging_changes_no_training_state():
    """The same step from the same training state and RNG state, with and without logs: the losses are bitwise equal and
    the generator advances alike.  (The state is copied from the step without logs into the one with them: two separate
    runs differ in the last bits anyway, the weight-gradient reductions use atomics.)"""
    batch = pretrain_batches(1)[0]
    cfg = M.pretrain_config(text_features=_tf())

    calls = ops._dropout_calls[0]

    def two_steps(train_eval):
        ops._dropout_calls[0] = calls        # the in-kernel dropout seeds count calls: both captures draw the same ones
        ps = train.PretrainStep(cfg, "cuda:0", seed=0, cuda_graph=True, train_eval=train_eval, log_every=8)
        for _ in range(2):
            ps.step(dict(batch))
        torch.cuda.synchronize()
        return ps

    plain = two_steps(None)
    state = {k: v.clone() for k, v in _train_state(plain).items()}
    bufs = [b.clone() for b in plain.module.buffers()]
    rng, sched = torch.cuda.get_rng_state(), plain._sched_step
    loss = plain.step(dict(batch)).clone()
    rng_after = torch.cuda.get_rng_state()
    launches = plain.native_launches_per_step
    plain.close()
    del plain
    logged = two_steps(evaluate.PretrainEval())
    try:
        for k, v in _train_state(logged).items():
            v.copy_(state[k])
        for b, s in zip(logged.module.buffers(), bufs):
            b.copy_(s)
        torch.cuda.set_rng_state(rng)
        logged._sched_step = sched
        assert torch.equal(logged.step(dict(batch)), loss)
        assert torch.equal(torch.cuda.get_rng_state(), rng_after)
        assert logged.native_launches_per_step > launches
        assert len(logged.logs()) == 3
    finally:
        logged.close()
