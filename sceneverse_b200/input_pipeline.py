"""Device-side input pipeline (SURVEY.md §8 f2): the `data_dict` of one training step built ON THE GPU from ragged raw scene
data, replacing the dataloader-worker loops of data/datasets/base.py:697-741 (`_obj_processing_post`),
data/datasets/dataset_wrapper.py:38-111 (padding, masks) and data/data_utils.py:76-121 (`random_word`, `random_point_cloud`).

Input (what a scan loader hands over after reading the files): every object's raw points concatenated (total, 6) [xyz rgb],
a CSR offset per object SLOT (B * max_obj_len + 1; padded slots are empty ranges), the tokenised captions.  Output: the keys
`OpenVocab.forward` consumes, same dtypes and padding conventions as the reference (padded objects = all-ones points, zero
locs, label -100, mask False).  Randomness is a counter hash of (seed, index): reproducible and order independent.

The training split of a config is augmented as the reference's dataset does it (`AugSpec`, `prepare_objects_aug`): with a
`data_aug` block, data/datasets/data_augmentor.py + base.py:742-776 `_obj_processing_aug`; without one, `_obj_processing_post`
with its `rot_aug` quarter turn (data/data_utils.py:163-178)."""
import math
from collections.abc import Mapping
from dataclasses import dataclass
from typing import Optional, Tuple

import torch

from . import _lib


def prepare_objects(raw_points, slot_offsets, B, O, P=1024, seed=0, return_indices=False):
    """raw_points (total,6) f32 cuda, slot_offsets (B*O+1) int64 cuda -> obj_fts (B,O,P,6) f32, obj_locs (B,O,6) f32,
    obj_masks (B,O) bool [, sample indices (B,O,P) i32]."""
    assert raw_points.is_cuda and raw_points.dtype == torch.float32 and raw_points.dim() == 2 and raw_points.shape[1] == 6
    assert slot_offsets.dtype == torch.int64 and slot_offsets.numel() == B * O + 1
    raw_points, slot_offsets = raw_points.contiguous(), slot_offsets.contiguous()
    dev = raw_points.device
    fts = torch.empty((B, O, P, 6), dtype=torch.float32, device=dev)
    locs = torch.empty((B, O, 6), dtype=torch.float32, device=dev)
    masks = torch.empty((B, O), dtype=torch.uint8, device=dev)
    idx = torch.empty((B, O, P), dtype=torch.int32, device=dev) if return_indices else None
    # the post path without quarter turns; slots_per_item >= 1 keeps a batch without object slots (O = 0) valid
    _lib.call(_lib.pointops(), "sv_scene_prep_rot_f32", dev, raw_points.data_ptr(), slot_offsets.data_ptr(), B * O, max(O, 1),
              P, int(seed) & 0x7FFFFFFFFFFFFFFF, None, None, fts.data_ptr(), locs.data_ptr(), None, masks.data_ptr(),
              _lib.ptr(idx))
    out = (fts, locs, masks.bool())
    return out + (idx,) if return_indices else out


@dataclass(frozen=True)
class RotationSpec:
    """One `rotation` block of data_augmentor.py: angle i is value[i] times a quarter turn (axis_align) or U[-pi, pi)."""
    value: Tuple[float, float, float]
    axis_align: bool
    shuffle: bool


@dataclass(frozen=True)
class AugSpec:
    """Which object-processing path runs and which augmentations it applies.

    path "aug": the config has a `data_aug` block (base.py:247-253, 964-972), every field below may be set.
    path "post": no `data_aug`; only `rot_aug` (a quarter turn per item, train split) applies."""
    path: str = "post"
    rot_aug: bool = False
    flip: bool = False
    scaling: Optional[Tuple[float, float]] = None
    scene_translation: Optional[Tuple[float, float, float]] = None
    scene_rotation: Optional[RotationSpec] = None
    color_jitter: bool = False
    obj_translation: Optional[Tuple[float, float, float]] = None
    obj_rotation: Optional[RotationSpec] = None
    jitter: Optional[float] = None
    pts_shuffle: bool = False

    @classmethod
    def from_config(cls, data_aug, rot_aug=False, split="train"):
        """Restates how the reference picks the path and builds `DataAugmentor`'s queue.  `data_aug` may be a plain mapping or
        an attribute-style config (hydra's DictConfig).  An augmentation runs only on the train split, when it is named in
        `aug_list` and present in the block, and when `check_key` enables it (None / bool / `enabled`; a missing entry counts
        as absent).  `p` is not consulted: the reference's blocks are DictConfigs, not dicts, so its `check_p` is always true.
        `order_shuffle` (a permutation nothing reads) and `accord_to_size` (never read) are accepted and ignored."""
        if not data_aug:
            return cls(path="post", rot_aug=bool(rot_aug) and split == "train")
        if split != "train":
            return cls(path="aug")
        aug_list = _cfg_get(data_aug, "aug_list")
        if aug_list is None or isinstance(aug_list, (str, bytes)):
            raise ValueError(f"data_aug.aug_list must be a list of augmentation names, got {aug_list!r}")
        kw = {}
        for aug in aug_list:
            if not _cfg_has(data_aug, aug):
                continue
            block = _cfg_get(data_aug, aug)
            if aug == "scene_aug":
                if _check_key(_cfg_get(block, "translation")):
                    kw["scene_translation"] = _vec3(_cfg_get(_cfg_get(block, "translation"), "value"), "scene_aug.translation.value")
                if _check_key(_cfg_get(block, "scaling")):
                    kw["scaling"] = _pair(_cfg_get(_cfg_get(block, "scaling"), "value"), "scene_aug.scaling.value")
                kw["flip"] = bool(_check_key(_cfg_get(block, "flip")))
                if _check_key(_cfg_get(block, "rotation")):
                    kw["scene_rotation"] = _rotation(_cfg_get(block, "rotation"), "scene_aug.rotation")
                kw["color_jitter"] = bool(_check_key(_cfg_get(block, "color_jitter")))
            elif aug == "obj_aug":
                if _check_key(_cfg_get(block, "translation")):
                    kw["obj_translation"] = _vec3(_cfg_get(_cfg_get(block, "translation"), "value"), "obj_aug.translation.value")
                if _check_key(_cfg_get(block, "rotation")):
                    kw["obj_rotation"] = _rotation(_cfg_get(block, "rotation"), "obj_aug.rotation")
                if _check_key(_cfg_get(block, "random_jitter")):
                    v = _number(_cfg_get(_cfg_get(block, "random_jitter"), "value"), "obj_aug.random_jitter.value")
                    if v < 0:
                        raise ValueError(f"obj_aug.random_jitter.value must be >= 0, got {v}")
                    kw["jitter"] = v
                kw["pts_shuffle"] = bool(_check_key(_cfg_get(block, "pts_shuffle")))
            else:
                raise ValueError(f"unknown augmentation {aug!r} in data_aug.aug_list (known: scene_aug, obj_aug)")
        return cls(path="aug", **kw)

    def params(self):
        """The C-side `sv_aug_params` of the aug path."""
        p = _lib.AugParams()
        f = 0
        if self.flip:
            f |= _lib.AUG_FLIP
        if self.scaling is not None:
            f |= _lib.AUG_SCALE
            p.scale_lo, p.scale_hi = self.scaling
        if self.scene_translation is not None:
            f |= _lib.AUG_SCENE_TRANS
            p.scene_trans[:] = self.scene_translation
        if self.scene_rotation is not None:
            f |= _lib.AUG_SCENE_ROT
            p.scene_rot[:] = self.scene_rotation.value
            p.scene_rot_axis_align, p.scene_rot_shuffle = int(self.scene_rotation.axis_align), int(self.scene_rotation.shuffle)
        if self.color_jitter:
            f |= _lib.AUG_COLOR
        if self.obj_translation is not None:
            f |= _lib.AUG_OBJ_TRANS
            p.obj_trans[:] = self.obj_translation
        if self.obj_rotation is not None:
            f |= _lib.AUG_OBJ_ROT
            p.obj_rot[:] = self.obj_rotation.value
            p.obj_rot_axis_align, p.obj_rot_shuffle = int(self.obj_rotation.axis_align), int(self.obj_rotation.shuffle)
        if self.jitter is not None:
            f |= _lib.AUG_JITTER
            p.jitter = self.jitter
        if self.pts_shuffle:
            f |= _lib.AUG_PTS_SHUFFLE
        p.flags = f
        return p


def _cfg_has(cfg, key):
    if cfg is None or isinstance(cfg, (bool, int, float, str)):
        return False
    if isinstance(cfg, Mapping) or hasattr(cfg, "keys"):
        return key in cfg
    return hasattr(cfg, key)


def _cfg_get(cfg, key, default=None):
    if not _cfg_has(cfg, key):
        return default
    if isinstance(cfg, Mapping) or hasattr(cfg, "keys"):
        return cfg[key]
    return getattr(cfg, key)


def _check_key(key):
    """data_augmentor.py DataAugmentor.check_key."""
    if key is None:
        return False
    if isinstance(key, bool):
        return key
    if isinstance(key, dict):
        return key.get("enabled", True)
    if _cfg_has(key, "enabled"):
        return _cfg_get(key, "enabled")
    return True


def _number(v, what):
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
        raise ValueError(f"{what} must be a finite number, got {v!r}")
    return float(v)


def _seq(v, n, what):
    if v is None or isinstance(v, (str, bytes, Mapping)) or not hasattr(v, "__len__") or len(v) != n:
        raise ValueError(f"{what} must be a list of {n} numbers, got {v!r}")
    return tuple(_number(x, what) for x in v)


def _vec3(v, what):
    return _seq(v, 3, what)


def _pair(v, what):
    return _seq(v, 2, what)


def _rotation(block, what):
    return RotationSpec(_vec3(_cfg_get(block, "value"), what + ".value"), bool(_cfg_get(block, "axis_align", False)),
                        bool(_cfg_get(block, "shuffle", False)))


def prepare_objects_aug(raw_points, slot_offsets, B, O, P, spec, seed, want_boxes=False, draws=None, return_draws=False):
    """The object tensors of one batch with the augmentation `spec` (AugSpec) of a training split.

    raw_points (total,6) f32 cuda, slot_offsets (B*O+1) int64 cuda (O slots per item, empty range = padded slot) ->
    obj_fts (B,O,P,6) f32, obj_locs (B,O,6) f32, obj_masks (B,O) bool [, obj_boxes (B,O,6) f32 if want_boxes]
    [, draws if return_draws].

    The random values come from `seed`, or from `draws` (replay):
      aug path:  {"item": (B,25) f64, "obj": (B,O,12) f64, "index": (B,O,P) i32, "noise": (B,O,P,3) f32 (with jitter)}
                 (table layouts in include/svpointops.h; index = the raw index of each output point, subsample and shuffle
                 composed; noise = the standard normals of its jitter);
      post path: {"quarter_turns": (B,) i32 in 0..3, "index": (B,O,P) i32}.
    `return_draws` returns the dict that was used; passing it back as `draws` reproduces the output bit for bit."""
    assert raw_points.is_cuda and raw_points.dtype == torch.float32 and raw_points.dim() == 2 and raw_points.shape[1] == 6
    assert slot_offsets.dtype == torch.int64 and slot_offsets.numel() == B * O + 1
    if spec.path not in ("aug", "post"):
        raise ValueError(f"unknown object-processing path {spec.path!r}")
    raw_points, slot_offsets = raw_points.contiguous(), slot_offsets.contiguous()
    dev = raw_points.device
    fts = torch.empty((B, O, P, 6), dtype=torch.float32, device=dev)
    locs = torch.empty((B, O, 6), dtype=torch.float32, device=dev)
    masks = torch.empty((B, O), dtype=torch.uint8, device=dev)
    boxes = torch.empty((B, O, 6), dtype=torch.float32, device=dev) if want_boxes else None
    seed = int(seed) & 0x7FFFFFFFFFFFFFFF
    lib = _lib.pointops()

    def given(key, shape, dtype):
        t = draws.get(key)
        if t is None or tuple(t.shape) != shape or t.dtype != dtype or t.device != dev:
            raise ValueError(f"draws[{key!r}] must be a {dtype} tensor of shape {shape} on {dev}")
        return t.contiguous()

    if spec.path == "post":
        if draws is not None:
            qt, idx_in = given("quarter_turns", (B,), torch.int32), given("index", (B, O, P), torch.int32)
        else:
            qt, idx_in = None, None
            if spec.rot_aug:
                qt = torch.empty(B, dtype=torch.int32, device=dev)
                _lib.call(lib, "sv_quarter_turn_draw", dev, B, seed, qt.data_ptr())
        idx_out = torch.empty((B, O, P), dtype=torch.int32, device=dev) if return_draws else None
        _lib.call(lib, "sv_scene_prep_rot_f32", dev, raw_points.data_ptr(), slot_offsets.data_ptr(), B * O, O, P, seed,
                  _lib.ptr(qt), _lib.ptr(idx_in), fts.data_ptr(), locs.data_ptr(), _lib.ptr(boxes), masks.data_ptr(),
                  _lib.ptr(idx_out))
        used = {"quarter_turns": qt if qt is not None else torch.zeros(B, dtype=torch.int32, device=dev),
                "index": idx_out}
    else:
        params = spec.params()
        jitter = spec.jitter is not None
        if draws is not None:
            item, obj = given("item", (B, _lib.AUG_ITEM_STRIDE), torch.float64), given("obj", (B, O, _lib.AUG_OBJ_STRIDE), torch.float64)
            idx_in = given("index", (B, O, P), torch.int32)
            noise_in = given("noise", (B, O, P, 3), torch.float32) if jitter else None
        else:
            item = torch.empty((B, _lib.AUG_ITEM_STRIDE), dtype=torch.float64, device=dev)
            obj = torch.empty((B, O, _lib.AUG_OBJ_STRIDE), dtype=torch.float64, device=dev)
            idx_in = noise_in = None
            _lib.call(lib, "sv_aug_draw", dev, params, B, O, seed, item.data_ptr(), obj.data_ptr())
        idx_out = torch.empty((B, O, P), dtype=torch.int32, device=dev) if return_draws else None
        noise_out = torch.empty((B, O, P, 3), dtype=torch.float32, device=dev) if return_draws and jitter else None
        _lib.call(lib, "sv_scene_prep_aug_f32", dev, raw_points.data_ptr(), slot_offsets.data_ptr(), B, O, P, params,
                  item.data_ptr(), obj.data_ptr(), _lib.ptr(idx_in), _lib.ptr(noise_in), seed, fts.data_ptr(), locs.data_ptr(),
                  _lib.ptr(boxes), masks.data_ptr(), _lib.ptr(idx_out), _lib.ptr(noise_out))
        used = {"item": item, "obj": obj, "index": idx_out}
        if jitter:
            used["noise"] = noise_out
    out = (fts, locs, masks.bool())
    if want_boxes:
        out += (boxes,)
    return out + (used,) if return_draws else out


def mask_tokens(txt_ids, txt_masks, mask_ratio=0.15, mask_token_id=103, vocab_size=30522, seed=0):
    """BERT masked-LM corruption: (B,L) int64 ids / masks -> (masked ids, labels with -1 = not supervised)."""
    assert txt_ids.is_cuda and txt_ids.dtype == torch.int64 and txt_masks.dtype == torch.int64 and txt_ids.shape == txt_masks.shape
    ids, am = txt_ids.contiguous(), txt_masks.contiguous()
    out, lab = torch.empty_like(ids), torch.empty_like(ids)
    _lib.call(_lib.pointops(), "sv_token_mask", ids.device, ids.data_ptr(), am.data_ptr(), ids.numel(), float(mask_ratio),
              int(mask_token_id), int(vocab_size), int(seed) & 0x7FFFFFFFFFFFFFFF, out.data_ptr(), lab.data_ptr())
    return out, lab


def mask_objects(obj_masks, drop_ratio=0.1, seed=0):
    """random_point_cloud: (B,O) bool -> (B,O) bool, True = keep the object's semantic features."""
    v = obj_masks.to(torch.uint8).contiguous()
    out = torch.empty_like(v)
    _lib.call(_lib.pointops(), "sv_coin_mask", v.device, v.data_ptr(), v.numel(), float(drop_ratio),
              int(seed) & 0x7FFFFFFFFFFFFFFF, out.data_ptr())
    return out.bool()


def build_data_dict(raw_points, slot_offsets, obj_labels, txt_ids, txt_masks, tgt_object_id, B, O, P=1024, seed=0,
                    txt_mask_ratio=0.15, pc_mask_ratio=0.1, scene_txt_ids=None, scene_txt_masks=None, augment=None,
                    want_boxes=False):
    """Everything `OpenVocab.forward` + the losses read, in three launches.  obj_labels: (B,O) int64 with -100 on padded slots
    (dataset_wrapper.py:70-71); tgt_object_id (B,1) int64.  augment: an AugSpec (`AugSpec.from_config(cfg.data_aug,
    cfg.data.args.rot_aug, split)`) processes the objects as that config's split does; None keeps the plain post path of
    `prepare_objects`.  want_boxes adds "obj_boxes" (B,O,6) = [box centre, size]."""
    if augment is None and not want_boxes:
        fts, locs, masks = prepare_objects(raw_points, slot_offsets, B, O, P, seed)
    else:
        objs = prepare_objects_aug(raw_points, slot_offsets, B, O, P, augment if augment is not None else AugSpec(), seed,
                                   want_boxes=want_boxes)
        fts, locs, masks = objs[:3]
    ids, labels = mask_tokens(txt_ids, txt_masks, txt_mask_ratio, seed=seed + 1)
    d = {"obj_fts": fts, "obj_locs": locs, "obj_masks": masks, "obj_sem_masks": mask_objects(masks, pc_mask_ratio, seed + 2),
         "obj_labels": obj_labels, "txt_ids": ids, "txt_masks": txt_masks, "masked_lm_labels": labels, "tgt_object_id": tgt_object_id}
    if want_boxes:
        d["obj_boxes"] = objs[3]
    if scene_txt_ids is not None:
        d["scene_txt_ids"], d["scene_txt_masks"] = scene_txt_ids, scene_txt_masks
    return d


def grounding_targets(points, cand_offsets, item_offsets, cand_labels, tgt_label, O, seed=0, gt_points=None, gt_offsets=None,
                      gt_index=None, return_iou=False):
    """Evaluation targets of a grounding batch (base.py:387-454), csrc/eval_targets.cu.

    points (total, 6) f32 cuda: every candidate object's raw points; cand_offsets (n_cand + 1) int64 cuda: one CSR range per
    candidate (>= 1 point each); item_offsets (B + 1) int64 on the HOST: the candidates of each item; cand_labels (n_cand)
    int64 cuda; tgt_label (B,) int64 cuda.  pred mode: gt_points / gt_offsets (B + 1, cuda) hold each item's ground-truth
    object.  gt mode: gt_index (B,) int64 cuda = the target candidate of each item (after the caller's wall / floor /
    ceiling filter).  Returns slot_map (B, O) int32 (-1 = empty slot), tgt_object_id (B, 1), tgt_object_id_iou25 and
    tgt_object_id_iou50 (B, O) int64 [, per-candidate IoU (n_cand,) f32]."""
    item_offsets = torch.as_tensor(item_offsets, dtype=torch.int64).cpu()
    B = item_offsets.numel() - 1
    counts = item_offsets[1:] - item_offsets[:-1]
    if B < 1 or int(item_offsets[0]) != 0 or bool((counts < 0).any()):
        raise ValueError("item_offsets must start at 0 and be non-decreasing")
    n_cand = int(item_offsets[-1])
    assert points.is_cuda and points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 6
    assert cand_offsets.dtype == torch.int64 and cand_offsets.numel() == n_cand + 1
    assert cand_labels.dtype == torch.int64 and cand_labels.numel() == n_cand and tgt_label.numel() == B
    if (gt_index is None) == (gt_points is None):
        raise ValueError("pass gt_points / gt_offsets (pred mode) or gt_index (gt mode)")
    dev = points.device
    slot_map = torch.empty((B, O), dtype=torch.int32, device=dev)
    tgt = torch.empty((B, 1), dtype=torch.int64, device=dev)
    iou25 = torch.empty((B, O), dtype=torch.int64, device=dev)
    iou50 = torch.empty((B, O), dtype=torch.int64, device=dev)
    iou = torch.empty(max(n_cand, 1), dtype=torch.float32, device=dev) if return_iou else None
    cand_offsets, cand_labels, tgt_label = cand_offsets.contiguous(), cand_labels.contiguous(), tgt_label.contiguous()
    if gt_points is not None:
        gt_points, gt_offsets = gt_points.contiguous(), gt_offsets.contiguous()
        assert gt_offsets.dtype == torch.int64 and gt_offsets.numel() == B + 1
    else:
        gt_index = gt_index.contiguous()
        assert gt_index.dtype == torch.int64 and gt_index.numel() == B
    item_dev = item_offsets.to(dev)
    _lib.call(_lib.pointops(), "sv_grounding_targets_f32", dev, points.data_ptr(), cand_offsets.data_ptr(), item_dev.data_ptr(),
              _lib.ptr(gt_points), _lib.ptr(gt_offsets), _lib.ptr(gt_index), cand_labels.data_ptr(), tgt_label.data_ptr(), B, O,
              int(counts.max()), int(seed) & 0x7FFFFFFFFFFFFFFF, slot_map.data_ptr(), tgt.data_ptr(), iou25.data_ptr(),
              iou50.data_ptr(), _lib.ptr(iou))
    out = (slot_map, tgt, iou25, iou50)
    return out + (iou[:n_cand],) if return_iou else out


def kept_objects(points, cand_offsets, item_offsets, slot_map):
    """The points of the candidates `slot_map` keeps, slot by slot, and the (B*O + 1) slot_offsets over them that
    prepare_objects / prepare_objects_aug consume (empty range = padded slot)."""
    B, O = slot_map.shape
    dev = points.device
    base = torch.as_tensor(item_offsets, dtype=torch.int64)[:-1].to(dev)
    sm = slot_map.long()
    cand = (base[:, None] + sm.clamp(min=0)).reshape(-1)
    starts = cand_offsets[cand]
    lens = (cand_offsets[cand + 1] - starts) * (sm.reshape(-1) >= 0)
    slot_offsets = torch.zeros(B * O + 1, dtype=torch.int64, device=dev)
    slot_offsets[1:] = lens.cumsum(0)
    total = int(slot_offsets[-1])
    src = torch.repeat_interleave(starts - slot_offsets[:-1], lens, output_size=total) + torch.arange(total, device=dev)
    return points[src], slot_offsets


def build_eval_dict(points, cand_offsets, item_offsets, cand_labels, tgt_label, txt_ids, txt_masks, O, P=1024, seed=0,
                    augment=None, gt_points=None, gt_offsets=None, gt_index=None):
    """The evaluation batch of ScanFamilyDatasetWrapperOld (dataset_wrapper.py:147-195) on the device: the targets and crop of
    `grounding_targets`, the kept objects processed as `augment` says (`AugSpec.from_config(cfg.data_aug, rot_aug,
    split="val")`; None = the plain post path), boxes, no masked-LM corruption and obj_sem_masks = obj_masks."""
    slot_map, tgt, iou25, iou50 = grounding_targets(points, cand_offsets, item_offsets, cand_labels, tgt_label, O, seed,
                                                    gt_points, gt_offsets, gt_index)
    kept, slot_offsets = kept_objects(points, cand_offsets, item_offsets, slot_map)
    B = slot_map.shape[0]
    fts, locs, masks, boxes = prepare_objects_aug(kept, slot_offsets, B, O, P, augment if augment is not None else AugSpec(),
                                                  seed, want_boxes=True)
    base = torch.as_tensor(item_offsets, dtype=torch.int64)[:-1].to(points.device)
    sm = slot_map.long()
    labels = torch.where(sm >= 0, cand_labels[(base[:, None] + sm.clamp(min=0))], torch.full_like(sm, -100))
    return {"obj_fts": fts, "obj_locs": locs, "obj_boxes": boxes, "obj_masks": masks, "obj_sem_masks": masks.clone(),
            "obj_labels": labels, "txt_ids": txt_ids, "txt_masks": txt_masks, "tgt_object_id": tgt,
            "tgt_object_label": tgt_label.reshape(B, 1), "tgt_object_id_iou25": iou25, "tgt_object_id_iou50": iou50}
