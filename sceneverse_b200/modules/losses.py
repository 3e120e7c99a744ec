"""Losses on the GPS path (reference: optim/loss/loss.py:8-94,111-148; optim/loss/contra_loss.py:11-98;
common/dist_utils.py:131-149)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch import nn

from .. import ops
from .registry import LOSS_REGISTRY


def all_gather(tensors):
    """common/dist_utils.py:131-149: NCCL all-gather of equally shaped tensors, concatenated on dim 0 in rank
    order.  REFERENCE SEMANTICS: the result carries no autograd history (the reference gathers into
    `torch.ones_like` placeholders), so in distributed mode no gradient reaches the embeddings through the gathered
    batch — only `logit_scale` learns from these losses.  Both tensors travel in ONE collective here."""
    world = dist.get_world_size()
    flat = torch.cat([t.detach().reshape(-1) for t in tensors])
    out = torch.empty(world * flat.numel(), dtype=flat.dtype, device=flat.device)
    dist.all_gather_into_tensor(out, flat.contiguous())
    out = out.view(world, -1)
    res, off = [], 0
    for t in tensors:
        n = t.numel()
        res.append(out[:, off:off + n].reshape(world * t.shape[0], *t.shape[1:]))
        off += n
    return res


def og3d_loss(data_dict):
    if data_dict["og3d_logits"].dim() == 3:
        raise ValueError("og3d_loss has no per-scene form: cross-entropy over (B, U, O) logits would treat U as the class axis")
    return ops.cross_entropy(data_dict["og3d_logits"], data_dict["tgt_object_id"].squeeze(1))


def lm_cls_loss(data_dict):
    """loss.py:56-61: cross-entropy over the vocabulary at the masked positions (label -1 = not supervised)."""
    target = data_dict["masked_lm_labels"]
    target = target.view(-1, target.size(-1)) if target.dim() == 3 else target
    return ops.cross_entropy(data_dict["txt_lm_cls_logits"], target, ignore_index=-1)


def answer_loss(data_dict):
    """loss.py:50-53: BCE with logits over the answer vocabulary against the multi-hot `answer_label` (int64, read as
    float), summed and divided by the batch size; all-zero rows (unanswerable questions) still count."""
    return ops.bce_with_logits_sum(data_dict["answer_scores"], data_dict["answer_label"])


def og3d_multi_loss(data_dict):
    """loss.py:12-16: BCE with logits over `og3d_logits` (B, O) against a multi-hot (B, O) `tgt_object_id` read as float,
    summed and divided by B.  GroundHeadV1's og3d_logits are -inf at padded objects (heads.py): torch then gives a NaN loss
    and a zero gradient at those entries, and so does the native kernel; without a ground head the logits are the finite
    einsum of OpenVocab."""
    return ops.bce_with_logits_sum(data_dict["og3d_logits"], data_dict["tgt_object_id"])


def txt_cls_multi_loss(data_dict):
    """loss.py:19-23: BCE with logits over `txt_cls_logits` (B, 607) against a multi-hot (B, 607) `tgt_object_label` read as
    float, summed and divided by B."""
    return ops.bce_with_logits_sum(data_dict["txt_cls_logits"], data_dict["tgt_object_label"])


def obj_cls_raw_loss(data_dict):
    """loss.py:26-31: (CE(obj_cls_raw_logits) * obj_masks).sum() / obj_masks.sum().  The logits are the detached softmax
    probabilities of the object encoder's class head (vision.py), so nothing trains on this loss."""
    return ops.masked_cross_entropy(data_dict["obj_cls_raw_logits"], data_dict["obj_labels"], data_dict["obj_masks"])


def obj_cls_pre_loss(data_dict):
    """loss.py:34-39: (CE(obj_cls_pre_logits) * obj_masks).sum() / obj_masks.sum()."""
    return ops.masked_cross_entropy(data_dict["obj_cls_pre_logits"], data_dict["obj_labels"], data_dict["obj_masks"])


def obj_cls_post_loss(data_dict):
    """loss.py:42-47: (CE(obj_cls_post_logits) * obj_masks).sum() / obj_masks.sum()."""
    return ops.masked_cross_entropy(data_dict["obj_cls_post_logits"], data_dict["obj_labels"], data_dict["obj_masks"])


def obj_cls_pre_loss_mask(data_dict):
    """loss.py:64-70: (CE(obj_cls_pre_logits) * w).sum() / w.sum(), w = obj_masks & ~obj_sem_masks (NaN when no object of
    the batch is semantically masked)."""
    return ops.masked_cross_entropy(data_dict["obj_cls_pre_logits"], data_dict["obj_labels"], data_dict["obj_masks"],
                                    data_dict["obj_sem_masks"], mode=1)


def obj_cls_pre_loss_unmask(data_dict):
    """loss.py:72-78: (CE(obj_cls_pre_logits) * w).sum() / w.sum(), w = obj_masks & obj_sem_masks."""
    return ops.masked_cross_entropy(data_dict["obj_cls_pre_logits"], data_dict["obj_labels"], data_dict["obj_masks"],
                                    data_dict["obj_sem_masks"], mode=2)


def obj_cls_post_loss_mask(data_dict):
    """loss.py:80-86: (CE(obj_cls_post_logits) * w).sum() / w.sum(), w = obj_masks & ~obj_sem_masks (NaN when no object of
    the batch is semantically masked)."""
    return ops.masked_cross_entropy(data_dict["obj_cls_post_logits"], data_dict["obj_labels"], data_dict["obj_masks"],
                                    data_dict["obj_sem_masks"], mode=1)


def obj_cls_post_loss_unmask(data_dict):
    """loss.py:88-94: (CE(obj_cls_post_logits) * w).sum() / w.sum(), w = obj_masks & obj_sem_masks."""
    return ops.masked_cross_entropy(data_dict["obj_cls_post_logits"], data_dict["obj_labels"], data_dict["obj_masks"],
                                    data_dict["obj_sem_masks"], mode=2)


def obj_cls_loss(data_dict, smoothing=0.3):
    """optim/loss/loss.py:96-102 (ObjCls pre-training)."""
    ce = F.cross_entropy(data_dict["obj_logits"].permute(0, 2, 1), data_dict["obj_labels"], reduction='none',
                         label_smoothing=smoothing)
    return (ce * data_dict["obj_masks"]).sum() / data_dict["obj_masks"].sum()


def _num_gpu(cfg):
    return cfg["num_gpu"] if isinstance(cfg, dict) else cfg.num_gpu


def _task(cfg):
    return cfg.get("task") if isinstance(cfg, dict) else getattr(cfg, "task", None)


@LOSS_REGISTRY.register()
class TextObjWithinBatch(nn.Module):
    """contra_loss.py:11-38.  Default: cross-entropy over the valid objects against one target id (B, 1).  task 'ScanQA':
    masked BCE with logits over all object slots against a multi-hot (B, O) target (several objects, or the masked
    'no target' placeholder slot), weight = obj_masks, summed and divided by B.  Per scene (B*U object rows, (B, O) masks,
    (B, U) targets): each scene's mask repeated for its U utterances, cross-entropy over the B*U rows."""

    def __init__(self, cfg):
        super().__init__()
        self.distributed = _num_gpu(cfg) > 1
        self.bce = _task(cfg) in ["ScanQA"]

    def forward(self, data_dict):
        obj_feats = ops.l2_normalize(data_dict["intra_obj_embeds"])
        text_feats = ops.l2_normalize(data_dict["intra_text_embed"])
        logits = torch.einsum("bod,bd->bo", obj_feats, text_feats)
        masks = data_dict["obj_masks"]
        if obj_feats.shape[0] != masks.shape[0]:
            # per scene (contra_loss.py:24-27): B*U rows against (B, O) masks and (B, U) targets
            if self.bce:
                raise ValueError("TextObjWithinBatch(task='ScanQA') has no per-scene form")
            U = obj_feats.shape[0] // masks.shape[0]
            masks = masks.unsqueeze(1).expand(masks.shape[0], U, masks.shape[1]).reshape(-1, masks.shape[1])
            logits = logits.masked_fill(masks.logical_not(), -float('inf'))
            return F.cross_entropy(logits, data_dict["tgt_object_id"].reshape(-1))
        if self.bce:
            labels = data_dict["tgt_object_id"]
            if labels.dim() != 2 or labels.shape != logits.shape:
                raise ValueError(f"TextObjWithinBatch(task='ScanQA') needs a multi-hot tgt_object_id of shape (B, O) = "
                                 f"{tuple(logits.shape)}, got {tuple(labels.shape)} (a (B, 1) target id is the "
                                 "cross-entropy form of the other tasks)")
            return ops.bce_with_logits_sum(logits, labels, weight=data_dict["obj_masks"])
        logits = logits.masked_fill(data_dict["obj_masks"].logical_not(), -float('inf'))
        return F.cross_entropy(logits, data_dict["tgt_object_id"].squeeze(-1))


class _SymmetricInfoNCE(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.distributed = _num_gpu(cfg) > 1
        # single-process run with the DISTRIBUTED autograd semantics (the gathered negatives of common/dist_utils.py:131-149
        # carry no gradient): what one rank of a data-parallel job computes, minus the exchange — the equal-work baseline
        # of the scaling curve (bench.py)
        self.emulate_dist = bool(cfg.get("emulate_dist", False)) if isinstance(cfg, dict) else bool(getattr(cfg, "emulate_dist", False))
        self.logit_scale = nn.Parameter((torch.ones([]) * np.log(1 / 0.07)).exp())

    def info_nce(self, a_feats, text_feats):
        logit_scale = torch.clamp(self.logit_scale, max=100)
        fused = None
        if self.distributed and a_feats.is_cuda and dist.is_initialized() and dist.get_backend() == "nccl":
            from .. import fused_gather
            fused = fused_gather.get(a_feats.shape[0], a_feats.shape[1], a_feats.device)
        if fused is not None:
            # one kernel: normalise both sets and store them into every rank's buffer over NVLink (detached, like the
            # reference's gather)
            a_feats, text_feats = fused(a_feats, text_feats)
        else:
            a_feats = ops.l2_normalize(a_feats)
            text_feats = ops.l2_normalize(text_feats)
            if self.distributed:
                a_feats, text_feats = all_gather([a_feats, text_feats])
            elif self.emulate_dist:
                a_feats, text_feats = a_feats.detach(), text_feats.detach()
        labels = torch.arange(text_feats.shape[0], device=text_feats.device)
        t2a = logit_scale * text_feats @ a_feats.t()
        a2t = logit_scale * a_feats @ text_feats.t()
        return (F.cross_entropy(t2a, labels) + F.cross_entropy(a2t, labels)) / 2


@LOSS_REGISTRY.register()
class TextObjBetweenBatch(_SymmetricInfoNCE):
    def forward(self, data_dict):
        labels = data_dict["tgt_object_id"]
        obj_feats = data_dict["inter_obj_embeds"]
        if obj_feats.shape[0] != labels.shape[0]:
            labels = labels.reshape(-1, 1)          # per scene (contra_loss.py:55-56): (B, U) -> (B*U, 1)
        tgt = obj_feats[torch.arange(labels.size(0), device=labels.device), labels[:, 0], :]
        return self.info_nce(tgt, data_dict["inter_text_embed"])


@LOSS_REGISTRY.register()
class TextSceneBetweenBatch(_SymmetricInfoNCE):
    def forward(self, data_dict):
        return self.info_nce(data_dict["scene_embed"], data_dict["scene_text_embed"])


class Loss(nn.Module):
    """optim/loss/loss.py:111-148 list-loss container (cfg.model.loss_list / vis_loss_list); `task` (cfg.task) reaches the
    registry losses' cfg (TextObjWithinBatch switches to its BCE form for 'ScanQA')."""

    def __init__(self, loss_list, vis_loss_list=None, num_gpu=1, emulate_dist=False, task=None):
        super().__init__()
        self.selected_keys = list(loss_list)
        self.all_keys = list(dict.fromkeys(list(vis_loss_list or []) + self.selected_keys))
        self.loss_fn = {}
        for k in self.all_keys:
            if k in globals() and callable(globals()[k]) and not isinstance(globals()[k], type):
                self.loss_fn[k] = globals()[k]
            else:
                self.loss_fn[k] = LOSS_REGISTRY.get(k)({"num_gpu": num_gpu, "emulate_dist": emulate_dist, "task": task})
                setattr(self, k, self.loss_fn[k])

    def forward(self, data_dict):
        all_losses = {k: fn(data_dict) for k, fn in self.loss_fn.items()}
        total = sum(all_losses[k] for k in self.selected_keys)
        all_losses["total_loss"] = total
        return total, all_losses
