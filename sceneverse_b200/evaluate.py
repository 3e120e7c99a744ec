"""Evaluation (reference: evaluator/build.py:10-53 `BaseEvaluator`, scanrefer_eval.py, referit3d_eval.py, scanqa_eval.py,
sqa3d_eval.py, objcls_eval.py, pretrain_eval.py; trainer/openvocab_trainer.py:48-62 `eval_step`).

Each evaluator keeps its metrics as one float64 counter vector on the device (layouts: include/svgps.h SV_EV*).  `update`
launches the metric kernels of csrc/eval_metrics.cu, which add one batch into it: no host synchronisation, so the updates of
an epoch can be replayed from a CUDA graph (`EvalRunner`).  `record` reads the vector once (after one all_reduce(SUM) when
several ranks evaluate) and builds the reference's dictionary: integer totals divided by counts, or, for SQA3DEval, its
batch-size-weighted average of per-batch ratios, accumulated on the device in the reference's float64 order.
`counts_to_metrics` turns one batch's counter values into `batch_metrics`; train.PretrainStep's per-step logs use it too.

Not supported (NotImplementedError): `cfg.eval.save` (results.json).  Per-scene batches (model.OpenVocabPerScene: B scenes x U
utterances, og3d_logits (B, U, O)) are counted by the grounding evaluators after `flatten_per_scene`, which EvalRunner applies;
PretrainEval has no per-scene form.
An item whose `valid` entry is False (the padding of a last partial batch) counts nothing."""
import math

import torch
import torch.distributed as dist

from . import _lib

__all__ = ["ScanReferEval", "ReferIt3DEval", "ScanQAEval", "SQA3DEval", "PretrainObjEval", "PretrainEval", "EvalRunner",
           "flatten_per_scene"]


def _is_bf16(t):
    if t.dtype not in (torch.bfloat16, torch.float32):
        raise TypeError(f"logits must be bf16 or f32, got {t.dtype}")
    return 1 if t.dtype == torch.bfloat16 else 0


def _rows(t, what):
    """A (B, C) tensor read in place: unit stride along the row, any row stride (padded vocabularies)."""
    if t.dim() != 2 or t.stride(1) != 1:
        raise ValueError(f"{what} must be 2-D with unit stride along its rows, got shape {tuple(t.shape)} strides {t.stride()}")
    return t


def _i64(t, what):
    if t.dtype != torch.int64:
        raise TypeError(f"{what} must be int64, got {t.dtype}")
    return t.contiguous()


def _bytes(t):
    if t is None:
        return None
    return (t if t.dtype in (torch.bool, torch.uint8) else t.bool()).contiguous()


def _save_flag(cfg):
    ev = getattr(cfg, "eval", None) if not isinstance(cfg, dict) else cfg.get("eval")
    if ev is None:
        return False
    return bool(ev.get("save", False) if isinstance(ev, dict) else getattr(ev, "save", False))


def _obj_logit_keys(data_dict):
    """The keys every reference evaluator turns into `*_acc`: 3-D `*logits` whose first two dims match obj_labels."""
    shape = data_dict["obj_labels"].shape
    return [k for k, v in data_dict.items() if k.endswith("logits") and torch.is_tensor(v) and v.ndim == 3
            and v.shape[:2] == shape]


_PER_SCENE_ITEM_KEYS = ("og3d_logits", "tgt_object_id_iou25", "tgt_object_id_iou50", "is_multiple", "is_hard",
                        "is_view_dependent")


def flatten_per_scene(data_dict):
    """A per-scene data dict (og3d_logits (B, U, O)) as B*U grounding items, as evaluator/scanrefer_eval.py:15-21 and
    referit3d_eval.py:15-20 flatten it before counting: og3d_logits, tgt_object_id_iou25 / 50 (B*U, O); is_multiple, is_hard,
    is_view_dependent (B*U); tgt_object_id, tgt_object_label (B*U, 1).  These are views (safe inside a CUDA graph).  A
    per-scene `valid` (B) is repeated over U and kept as `scene_valid` for the per-scene object keys (obj_labels, obj_masks
    and the (B, O, C) object logits), which stay as they are; object logits of B*U rows are not counted.  Duplicate
    utterances (per_scene_pad fills every scene to U) count like any other.  Returns a new dict; a 2-D batch is returned
    as a copy."""
    d = dict(data_dict)
    og = d["og3d_logits"]
    if og.dim() != 3:
        return d
    B, U = og.shape[:2]
    for k in _PER_SCENE_ITEM_KEYS:
        if k in d:
            d[k] = d[k].flatten(0, 1)
    for k in ("tgt_object_id", "tgt_object_label"):
        if k in d:
            d[k] = d[k].reshape(B * U, 1)
    if d.get("valid") is not None:
        d["scene_valid"] = d["valid"]
        d["valid"] = d["valid"].unsqueeze(1).expand(B, U).reshape(B * U)
    return d


def _launch_obj_cls(tensors, data_dict, valid, counters, split=None):
    """Masked-argmax hits of up to three (B, O, C) logits tensors; pairs (hits, count) from counters[0], or with a (B, O)
    split mask three pairs per tensor (all masked objects, those in the split, those outside it)."""
    labels = _i64(data_dict["obj_labels"], "obj_labels")
    masks = _bytes(data_dict["obj_masks"])
    B, O, C = tensors[0].shape
    n = len(tensors)
    for t in tensors:
        if t.shape != (B, O, C) or t.stride(2) != 1:
            raise ValueError(f"object logits must share one (B, O, C) shape with unit stride along C, got {tuple(t.shape)}")
    arr = lambda ct, vals: (ct * n)(*vals)  # noqa: E731
    import ctypes
    ptrs = arr(ctypes.c_void_p, [t.data_ptr() for t in tensors])
    bf = arr(ctypes.c_int, [_is_bf16(t) for t in tensors])
    rs = arr(ctypes.c_longlong, [t.stride(1) for t in tensors])
    its = arr(ctypes.c_longlong, [t.stride(0) for t in tensors])
    if split is not None and tuple(split.shape) != (B, O):
        raise ValueError(f"the split mask must be {(B, O)}, got {tuple(split.shape)}")
    _lib.call(_lib.gps(), "sv_eval_obj_cls", labels.device, n, ptrs, bf, rs, its, B, O, C, labels.data_ptr(), masks.data_ptr(),
              _lib.ptr(split), _lib.ptr(valid), counters.data_ptr())


class _CounterEvaluator:
    """BaseEvaluator with the metrics as device counters.  Subclasses define `kind`, `target_metric`, `_launch(data_dict,
    valid, counters)` and `_metrics(c)` -> {key: (value, count)} from a list of counter values."""
    kind = None
    target_metric = None

    def __init__(self, cfg=None, accelerator=None, device=None, **kwargs):
        if _save_flag(cfg):
            raise NotImplementedError(f"{type(self).__name__}: cfg.eval.save (writing results.json) is not supported")
        self.accelerator = accelerator
        self.save = False
        self.best_result = -math.inf
        self.device = torch.device(device if device is not None else "cuda")
        self.size = _lib.gps().sv_eval_counters_size(self.kind)
        self.counters = torch.zeros(self.size, dtype=torch.float64, device=self.device)
        self.eval_dict = {}
        self.reset()

    def _initial(self):
        return torch.zeros(self.size, dtype=torch.float64)

    def reset(self):
        """Zero the counters in place (a captured graph keeps adding into the same buffer)."""
        self.counters.copy_(self._initial())
        self.eval_dict = {}

    def update(self, data_dict):
        self._launch(data_dict, _bytes(data_dict.get("valid")), self.counters)

    def _batch_counts(self, data_dict):
        c = self._initial().to(self.device)
        self._launch(data_dict, _bytes(data_dict.get("valid")), c)
        return c.tolist()

    def batch_metrics(self, data_dict, include_count=False):
        return self.counts_to_metrics(self._batch_counts(data_dict), include_count)

    def counts_to_metrics(self, c, include_count=False):
        """`batch_metrics` of one batch from its counter values `c` (a list of floats): the one host arithmetic shared by the
        eager `batch_metrics` and the per-step train logs (train.PretrainStep.logs)."""
        metrics = self._metrics(c)
        if not include_count:
            return {k: v[0] / max(v[1], 1) for k, v in metrics.items()}
        return metrics

    def _reduced(self):
        c = self.counters
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            c = c.clone()
            dist.all_reduce(c, op=dist.ReduceOp.SUM)
        return c.tolist()

    def record(self):
        self.eval_dict = {k: v[0] / max(v[1], 1) for k, v in self._metrics(self._reduced()).items()}
        self.eval_dict["target_metric"] = self.eval_dict[self.target_metric]
        is_best = self.eval_dict["target_metric"] > self.best_result
        if is_best:
            self.best_result = self.eval_dict["target_metric"]
        self.eval_dict["best_result"] = self.best_result
        return is_best, self.eval_dict


class _GroundingEval(_CounterEvaluator):
    kind = _lib.EVAL_GROUNDING
    uses_iou = False

    def __init__(self, *a, **k):
        self._txt = False
        self._obj_keys = []
        super().__init__(*a, **k)

    def _launch(self, data_dict, valid, counters):
        og = data_dict["og3d_logits"]
        if og.ndim == 3:
            raise NotImplementedError(f"{type(self).__name__}: per-scene (3-D) og3d_logits are counted after "
                                      "evaluate.flatten_per_scene(data_dict)")
        if og.dim() != 2:
            raise ValueError(f"og3d_logits must be (B, O), got {tuple(og.shape)}")
        B, O = og.shape
        tgt = _i64(data_dict["tgt_object_id"], "tgt_object_id").reshape(-1)
        iou25 = iou50 = None
        if self.uses_iou:
            iou25 = _rows(_i64(data_dict["tgt_object_id_iou25"], "tgt_object_id_iou25"), "tgt_object_id_iou25")
            iou50 = _rows(_i64(data_dict["tgt_object_id_iou50"], "tgt_object_id_iou50"), "tgt_object_id_iou50")
            if iou25.shape != iou50.shape:
                raise ValueError("tgt_object_id_iou25 and tgt_object_id_iou50 must have one shape")
        txt = data_dict.get("txt_cls_logits")
        label = None
        if txt is not None:
            txt = _rows(txt, "txt_cls_logits")
            label = _i64(data_dict["tgt_object_label"], "tgt_object_label").reshape(-1)
            self._txt = True
        # ScanRefer splits by is_multiple, ReferIt3D by is_hard and is_view_dependent
        split_keys = ("is_multiple",) if self.uses_iou else ("is_hard", "is_view_dependent")
        flags = [_bytes(data_dict.get(k)) if k in split_keys else None for k in ("is_multiple", "is_hard", "is_view_dependent")]
        _lib.call(_lib.gps(), "sv_eval_grounding", og.device, og.data_ptr(), _is_bf16(og), og.stride(0), og.stride(1), B, O,
                  tgt.data_ptr(), _lib.ptr(iou25), _lib.ptr(iou50), iou25.stride(0) if iou25 is not None else 0, _lib.ptr(txt),
                  _is_bf16(txt) if txt is not None else 0, txt.stride(0) if txt is not None else 0,
                  txt.shape[1] if txt is not None else 0, _lib.ptr(label), *[_lib.ptr(f) for f in flags], _lib.ptr(valid),
                  counters.data_ptr())
        keys = _obj_logit_keys(data_dict)
        if len(keys) > 3:
            raise NotImplementedError(f"at most three object logits tensors, got {keys}")
        if keys:
            if self._obj_keys and keys != self._obj_keys:
                raise ValueError(f"object logits changed between batches: {self._obj_keys} -> {keys}")
            self._obj_keys = keys
            if "scene_valid" in data_dict:        # flatten_per_scene: the object keys are per scene
                valid = _bytes(data_dict["scene_valid"])
            _launch_obj_cls([data_dict[k] for k in keys], data_dict, valid, counters[_lib.EVG_OBJ:])

    def _obj_metrics(self, c, m):
        for i, k in enumerate(self._obj_keys):
            m[k.replace("logits", "acc")] = (int(c[_lib.EVG_OBJ + 2 * i]), int(c[_lib.EVG_OBJ + 2 * i + 1]))
        return m


class ScanReferEval(_GroundingEval):
    """evaluator/scanrefer_eval.py: og_acc_iou25 / 50 (all, unique, multiple), og_acc, txt_acc, obj_cls_*_acc."""
    target_metric = "og_acc_iou25"
    uses_iou = True

    def _metrics(self, c):
        n, mult = int(c[_lib.EVG_ITEMS]), int(c[_lib.EVG_MULTIPLE])
        i25, i50 = int(c[_lib.EVG_IOU25]), int(c[_lib.EVG_IOU50])
        i25m, i50m = int(c[_lib.EVG_IOU25_MULTIPLE]), int(c[_lib.EVG_IOU50_MULTIPLE])
        m = {"og_acc_iou25": (i25, n), "og_acc_iou50": (i50, n),
             "og_acc_iou25_unique": (i25 - i25m, n - mult), "og_acc_iou50_unique": (i50 - i50m, n - mult),
             "og_acc_iou25_multiple": (i25m, mult), "og_acc_iou50_multiple": (i50m, mult),
             "og_acc": (int(c[_lib.EVG_OG_ACC]), n)}
        if self._txt:
            m["txt_acc"] = (int(c[_lib.EVG_TXT_ACC]), n)
        return self._obj_metrics(c, m)


class ReferIt3DEval(_GroundingEval):
    """evaluator/referit3d_eval.py (Nr3D, Sr3D, MultiScan): og_acc and its easy / hard, view-dependent / -independent splits."""
    target_metric = "og_acc"

    def _metrics(self, c):
        n, hard, vd = int(c[_lib.EVG_ITEMS]), int(c[_lib.EVG_HARD]), int(c[_lib.EVG_VIEW_DEP])
        ok, ok_h, ok_v = int(c[_lib.EVG_OG_ACC]), int(c[_lib.EVG_OG_ACC_HARD]), int(c[_lib.EVG_OG_ACC_VIEW_DEP])
        m = {"og_acc_easy": (ok - ok_h, n - hard), "og_acc_hard": (ok_h, hard),
             "og_acc_view_dep": (ok_v, vd), "og_acc_view_indep": (ok - ok_v, n - vd), "og_acc": (ok, n)}
        if self._txt:
            m["txt_acc"] = (int(c[_lib.EVG_TXT_ACC]), n)
        return self._obj_metrics(c, m)


class PretrainObjEval(_CounterEvaluator):
    """evaluator/objcls_eval.py: masked top-1 accuracy of obj_logits."""
    kind = _lib.EVAL_OBJ_CLS
    target_metric = "accuracy"

    def _launch(self, data_dict, valid, counters):
        _launch_obj_cls([data_dict["obj_logits"]], data_dict, valid, counters)

    def _metrics(self, c):
        return {"accuracy": (int(c[_lib.EVO_HIT]), int(c[_lib.EVO_COUNT]))}


def _launch_answers(data_dict, valid, counters, with_type):
    s = _rows(data_dict["answer_scores"], "answer_scores")
    B, A = s.shape
    label = _i64(data_dict["answer_label"], "answer_label")
    if tuple(label.shape) != (B, A):
        raise ValueError(f"answer_label must be {(B, A)}, got {tuple(label.shape)}")
    qtype = _i64(data_dict["sqa_type"], "sqa_type").reshape(-1) if with_type else None
    _lib.call(_lib.gps(), "sv_eval_answers", s.device, s.data_ptr(), _is_bf16(s), s.stride(0), B, A, label.data_ptr(),
              _lib.ptr(qtype), _lib.ptr(valid), counters.data_ptr())


class ScanQAEval(_CounterEvaluator):
    """evaluator/scanqa_eval.py: ans1_acc (EM@1), ans10_acc (EM@10), obj_cls_*_acc."""
    kind = _lib.EVAL_ANSWERS
    target_metric = "ans1_acc"

    def __init__(self, *a, **k):
        self._obj_key = None
        super().__init__(*a, **k)

    def _launch(self, data_dict, valid, counters):
        _launch_answers(data_dict, valid, counters, with_type=False)
        keys = _obj_logit_keys(data_dict)
        if len(keys) > 1:
            raise NotImplementedError(f"{type(self).__name__}: one object logits tensor is supported, got {keys}")
        if keys:
            self._obj_key = keys[0]
            _launch_obj_cls([data_dict[keys[0]]], data_dict, valid, counters[_lib.EVA_OBJ_HIT:])

    def _metrics(self, c):
        n = int(c[_lib.EVA_ITEMS])
        m = {"ans1_acc": (int(c[_lib.EVA_ANS1]), n), "ans10_acc": (int(c[_lib.EVA_ANS10]), n)}
        if self._obj_key is not None:
            m[self._obj_key.replace("logits", "acc")] = (int(c[_lib.EVA_OBJ_HIT]), int(c[_lib.EVA_OBJ_COUNT]))
        return m


def _type_count(n):
    """count_type of sqa3d_eval.py:87-89: 1e-10, then + 1 per item, each addition rounded."""
    x = 1e-10
    for _ in range(int(n)):
        x += 1
    return x


class SQA3DEval(_CounterEvaluator):
    """evaluator/sqa3d_eval.py.  Its `update` stores each batch's ratios times the batch size (the type accuracies times the
    type counts, which start at 1e-10) and `record` divides their sums by the totals: obj_cls_raw_acc is therefore a
    batch-size-weighted mean of per-batch ratios, not hits over masked objects.  The device keeps exactly those float64 sums
    (sv_eval_sqa3d_batch after every batch), so `record` returns the reference's values."""
    kind = _lib.EVAL_ANSWERS
    target_metric = "ans1_acc"
    KEYS = ["target_metric", "obj_cls_raw_acc", "ans1_acc", "ans10_acc"] + [f"type{k}_acc" for k in range(6)]

    def __init__(self, cfg=None, task_name=None, device=None, **kwargs):
        self.task_name = task_name
        super().__init__(cfg, None, device=device)

    def _initial(self):
        c = torch.zeros(self.size, dtype=torch.float64)
        c[_lib.EVA_Q_TYPE_COUNT:_lib.EVA_Q_TYPE_COUNT + _lib.EVA_NTYPES] = 1e-10   # self.type_count's start
        return c

    def reset(self):
        super().reset()
        self.eval_dict = {k: [] for k in self.KEYS}

    def _launch(self, data_dict, valid, counters):
        _launch_answers(data_dict, valid, counters, with_type=True)
        _launch_obj_cls([data_dict["obj_cls_raw_logits"]], data_dict, valid, counters[_lib.EVA_OBJ_HIT:])
        _lib.call(_lib.gps(), "sv_eval_sqa3d_batch", counters.device, counters.data_ptr())

    def batch_metrics(self, data_dict):
        return self.counts_to_metrics(self._batch_counts(data_dict))

    def counts_to_metrics(self, c, include_count=False):
        n = int(c[_lib.EVA_ITEMS])
        m = {"ans1_acc": c[_lib.EVA_ANS1] / float(n), "ans10_acc": c[_lib.EVA_ANS10] / float(n),
             "obj_cls_raw_acc": c[_lib.EVA_OBJ_HIT] / float(c[_lib.EVA_OBJ_COUNT])}
        for k in range(_lib.EVA_NTYPES):
            cnt = _type_count(c[_lib.EVA_TYPE_ITEMS + k])
            m[f"type{k}_acc"] = int(c[_lib.EVA_TYPE_ANS1 + k]) / cnt
            m[f"type{k}_count"] = cnt
        m["target_metric"] = m["ans1_acc"]
        m["total_count"] = n
        return m

    def record(self, split="val"):
        c = self._reduced()
        total = int(c[_lib.EVA_ITEMS])
        sums = {"target_metric": c[_lib.EVA_Q_ANS1], "ans1_acc": c[_lib.EVA_Q_ANS1], "ans10_acc": c[_lib.EVA_Q_ANS10],
                "obj_cls_raw_acc": c[_lib.EVA_Q_OBJ]}
        self.eval_dict = {}
        for k in self.KEYS:
            if "type" in k:
                self.eval_dict[k] = c[_lib.EVA_Q_TYPE + int(k[4])] / c[_lib.EVA_Q_TYPE_COUNT + int(k[4])]
            else:
                self.eval_dict[k] = sums[k] / total
        is_best = self.eval_dict["target_metric"] > self.best_result
        if is_best:
            self.best_result = self.eval_dict["target_metric"]
        return is_best, self.eval_dict


def _sum_left_to_right(xs):
    """The builtin sum of the reference's Python 3.9: one rounded addition per item, in order (from Python 3.12 on, sum()
    compensates the rounding)."""
    total = 0
    for x in xs:
        total = total + x
    return total


class PretrainEval(_CounterEvaluator):
    """evaluator/pretrain_eval.py: og_acc, lang_cls_acc_mask (masked-LM accuracy over the tokens whose masked_lm_labels is not
    -1) and obj_cls_{post,raw,pre}_acc, the post / pre ones also over obj_masks & obj_sem_masks (`_unmask`) and
    obj_masks & ~obj_sem_masks (`_mask`); each key only if its input is in the batch.  Its arithmetic is kept as it is:
    og_acc = hits / B with no mask (the plain einsum's padded slots can win), every other accuracy hits / (count + 1e-8)
    (0.0 for a batch with no labelled token), target_metric = the mean of the batch's accuracies.  `update` stores metric x
    total_count per batch and `record` divides the sums by the total count (a key never seen records 0.0); the device keeps
    exactly those float64 sums (sv_eval_pretrain_batch after every batch), so `record` returns the reference's values.  Sums
    are left to right, as the builtin sum of the reference's pinned Python 3.9 adds them."""
    kind = _lib.EVAL_PRETRAIN
    target_metric = "target_metric"
    KEYS = ["target_metric", "og_acc", "lang_cls_acc_mask", "obj_cls_post_acc", "obj_cls_pre_acc", "obj_cls_raw_acc",
            "obj_cls_pre_acc_unmask", "obj_cls_pre_acc_mask", "obj_cls_post_acc_unmask", "obj_cls_post_acc_mask"]
    OBJ = (("obj_cls_post_logits", _lib.EVP_HAS_POST), ("obj_cls_raw_logits", _lib.EVP_HAS_RAW),
           ("obj_cls_pre_logits", _lib.EVP_HAS_PRE))

    def __init__(self, *a, **k):
        self.present = 0           # SV_EVP_HAS_* bits of the last batch: which keys batch_metrics reports
        super().__init__(*a, **k)

    def _launch(self, data_dict, valid, counters):
        if data_dict["masked_lm_labels"].dim() == 3 or ("og3d_logits" in data_dict and data_dict["og3d_logits"].dim() == 3):
            raise ValueError("PretrainEval has no per-scene form: the per-scene model's B*U logits rows do not match its "
                             "(B, O) object masks and (B, U) targets")
        lm = data_dict["txt_lm_cls_logits"]
        labels = _i64(data_dict["masked_lm_labels"], "masked_lm_labels")
        if lm.dim() != 3 or lm.stride(2) != 1 or lm.stride(0) != lm.shape[1] * lm.stride(1):
            raise ValueError("txt_lm_cls_logits must be (B, L, V) with unit stride along V and rows of one pitch, got shape "
                             f"{tuple(lm.shape)} strides {lm.stride()}")
        B, L, V = lm.shape
        if tuple(labels.shape) != (B, L):
            raise ValueError(f"masked_lm_labels must be {(B, L)}, got {tuple(labels.shape)}")
        present = 0
        if "tgt_object_id" in data_dict:
            og = data_dict["og3d_logits"]
            if og.dim() != 2 or og.shape[0] != B:
                raise ValueError(f"og3d_logits must be ({B}, O), got {tuple(og.shape)}")
            tgt = _i64(data_dict["tgt_object_id"], "tgt_object_id").reshape(-1)
            _lib.call(_lib.gps(), "sv_eval_grounding", og.device, og.data_ptr(), _is_bf16(og), og.stride(0), og.stride(1), B,
                      og.shape[1], tgt.data_ptr(), None, None, 0, None, 0, 0, 0, None, None, None, None, _lib.ptr(valid),
                      counters[_lib.EVP_OG:].data_ptr())
            present |= _lib.EVP_HAS_OG
        obj = [(k, bit) for k, bit in self.OBJ if k in data_dict]
        if obj:
            present |= sum(bit for _, bit in obj)
            # the split is only reported for post / pre; raw alone needs no obj_sem_masks
            sem = data_dict["obj_sem_masks"] if present & (_lib.EVP_HAS_POST | _lib.EVP_HAS_PRE) else \
                data_dict.get("obj_sem_masks", data_dict["obj_masks"])
            _launch_obj_cls([data_dict[k] for k, _ in obj], data_dict, valid, counters[_lib.EVP_OBJ:], split=_bytes(sem))
        _lib.call(_lib.gps(), "sv_eval_lm_acc", lm.device, lm.data_ptr(), _is_bf16(lm), lm.stride(1), B * L, V, L,
                  labels.data_ptr(), _lib.ptr(valid), counters.data_ptr())
        _lib.call(_lib.gps(), "sv_eval_pretrain_batch", counters.device, counters.data_ptr(), present)
        self.present = present

    def counts_to_metrics(self, c, include_count=False):
        n = int(c[_lib.EVP_ITEMS])
        acc = lambda k: int(c[k]) / float(int(c[k + 1]) + 1e-8)  # noqa: E731
        m = {}
        if self.present & _lib.EVP_HAS_OG:
            m["og_acc"] = int(c[_lib.EVP_OG + _lib.EVG_OG_ACC]) / float(n)
        m["lang_cls_acc_mask"] = acc(_lib.EVP_LM_HIT)
        t = _lib.EVP_OBJ
        for name, bit in ((k[:-len("logits")], b) for k, b in self.OBJ):
            if self.present & bit:
                m[name + "acc"] = acc(t)
                if bit != _lib.EVP_HAS_RAW:
                    m[name + "acc_unmask"] = acc(t + 2)
                    m[name + "acc_mask"] = acc(t + 4)
                t += 6
        all_acc = list(m.values())
        m["target_metric"] = float(_sum_left_to_right(all_acc)) / len(all_acc)
        m["total_count"] = n
        return m

    def record(self):
        c = self._reduced()
        total = int(c[_lib.EVP_ITEMS])
        self.eval_dict = {k: c[_lib.EVP_Q + i] / total for i, k in enumerate(self.KEYS)}
        is_best = self.eval_dict["target_metric"] > self.best_result
        if is_best:
            self.best_result = self.eval_dict["target_metric"]
        return is_best, self.eval_dict


class EvalRunner:
    """Inference of one batch shape for evaluation: `forward` (model in eval mode, no_grad, bf16 autocast) and the metric
    kernels of `evaluators` captured into ONE CUDA graph from static input buffers, replayed once per batch.

    forward: a callable data_dict -> data_dict (the model), or a train.PretrainStep / train.ObjClsStep, whose model is used as
    it is: the bf16 weight shadows that training keeps current are what the native linears read, so no weight is copied.
    `run(batches)` evaluates an iterable of batches (dicts of device tensors, at most `batch_size` items each; a smaller last
    batch is padded by repeating its first item, with `valid` False for the padding) and returns `record()` of every
    evaluator.  With a per-scene model (txt_ids (B, U, T)) an item is a scene: a partial batch is padded by whole scenes and
    the output goes through `flatten_per_scene` before the evaluators.  The model's train / eval mode is restored afterwards; the run writes no parameter and no optimizer state."""

    def __init__(self, forward, evaluators, batch_size, dtype=torch.bfloat16):
        if isinstance(getattr(forward, "module", None), torch.nn.Module) and hasattr(forward.module, "model"):
            model = forward.module.model                     # train.PretrainStep: StepModule(model, loss)
        elif not isinstance(forward, torch.nn.Module) and isinstance(getattr(forward, "model", None), torch.nn.Module):
            model = forward.model                            # train.ObjClsStep
        else:
            model = forward if isinstance(forward, torch.nn.Module) else None
        self.model = model
        self.forward = model if model is not None else forward
        self.evaluators = list(evaluators)
        self.B = int(batch_size)
        self.dtype = dtype
        self.graph = self.static = self.valid = None

    def _run_eager(self, batch):
        with torch.autocast("cuda", dtype=self.dtype, enabled=self.dtype != torch.float32):
            out = self.forward(dict(batch))
        out["valid"] = batch["valid"]
        og = out.get("og3d_logits")
        if og is not None and og.dim() == 3:
            out = flatten_per_scene(out)          # per-scene model: B scenes x U utterances
        for ev in self.evaluators:
            ev.update(out)

    def _capture(self, batch):
        dev = next(v for v in batch.values() if torch.is_tensor(v)).device
        self.static = {k: torch.zeros((self.B,) + tuple(v.shape[1:]), dtype=v.dtype, device=dev)
                       for k, v in batch.items() if torch.is_tensor(v)}
        self.static["valid"] = torch.zeros(self.B, dtype=torch.bool, device=dev)
        self._fill(batch)
        saved = [ev.counters.clone() for ev in self.evaluators]
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):           # warm-up: lazy allocations and tensor maps outside the graph pool
            for _ in range(2):
                self._run_eager(self.static)
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        for ev, s in zip(self.evaluators, saved):
            ev.counters.copy_(s)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._run_eager(self.static)

    def _fill(self, batch):
        n = None
        for k, dst in self.static.items():
            if k == "valid":
                continue
            src = batch[k]
            n = src.shape[0]
            if n > self.B or n < 1 or tuple(src.shape[1:]) != tuple(dst.shape[1:]):
                raise ValueError(f"batch key {k!r}: shape {tuple(src.shape)} does not fit the runner's {tuple(dst.shape)}")
            dst[:n].copy_(src, non_blocking=True)
            if n < self.B:
                dst[n:].copy_(src[:1].expand((self.B - n,) + tuple(src.shape[1:])), non_blocking=True)
        self.static["valid"][:n].fill_(True)
        self.static["valid"][n:].fill_(False)

    def step(self, batch):
        """Add one batch to the evaluators' counters (no host synchronisation)."""
        if self.graph is None:
            self._capture(batch)
        else:
            self._fill(batch)
        self.graph.replay()

    def run(self, batches, reset=True):
        was = self.model.training if self.model is not None else None
        if self.model is not None:
            self.model.eval()
        try:
            if reset:
                for ev in self.evaluators:
                    ev.reset()
            with torch.no_grad():
                for batch in batches:
                    self.step(batch)
            return [ev.record() for ev in self.evaluators]
        finally:
            if self.model is not None and was:
                self.model.train()
