"""ORACLE — TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available (oracle/ref_shims.py):
    python oracle/make_golden_aug.py
Fixtures of the augmented object processing (tests/golden/input_aug_*.npz, described in tests/golden/INPUT_AUG.md): the
UNMODIFIED reference data/datasets/data_augmentor.py `DataAugmentor` and base.py `ScanBase._obj_processing_aug` / `_obj_processing_post` (called
unbound on a stub `self`), seeded with np.random.  What the run draws is recorded without editing the reference: the augmentor
instance's `update_data_dict` (the aug_dict), `subsample_fn` (np.random.choice), `jitter_fn` (np.random.randn) and
`pts_shuffle_fn` (np.random.permutation) are wrapped, and for the post path np.random.randint / choice.  The draws are stored in
the table layout of include/svpointops.h so that `prepare_objects_aug(..., draws=...)` replays them.

The config block is passed as an attribute-style mapping that is not a dict, as hydra passes a DictConfig.  Each item is one
reference call on its real objects; padded slots are filled as dataset_wrapper.py pads (points 1.0, locs / boxes 0).
"""
import contextlib
import copy
import importlib.util
import json
import os
import sys
import types
from collections.abc import Mapping

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden")

SHIPPED = {   # configs/final/all_pretrain.yaml data_aug (the block of every shipped pre-train / grounding config)
    "aug_list": ["scene_aug"],
    "scene_aug": {
        "translation": {"enabled": False, "value": [1.0, 1.0, 1.0], "p": 1.0},
        "scaling": {"enabled": False, "p": 1.0, "value": [0.9, 1.1]},
        "flip": {"enabled": False, "p": 0.5},
        "rotation": {"enabled": True, "p": 1.0, "axis_align": True, "value": [0.0, 0.0, 1.0], "shuffle": True},
        "color_jitter": False,
        "order_shuffle": False},
    "obj_aug": {
        "translation": {"enabled": False, "value": [0.1, 0.1, 0.1], "p": 1.0},
        "rotation": {"enabled": False, "p": 1.0, "axis_align": False, "value": [0.0, 0.0, 0.1], "shuffle": True},
        "random_jitter": {"enabled": False, "value": 0.01, "accord_to_size": False, "p": 1.0},
        "pts_shuffle": True}}


def all_on(obj_axis_align):
    """Every option of both blocks enabled (p < 1 on some: the reference never consults it)."""
    return {
        "aug_list": ["scene_aug", "obj_aug"],
        "scene_aug": {
            "translation": {"enabled": True, "value": [0.5, 0.5, 0.2], "p": 1.0},
            "scaling": {"enabled": True, "p": 0.5, "value": [0.9, 1.1]},
            "flip": {"enabled": True, "p": 0.5},
            "rotation": {"enabled": True, "p": 1.0, "axis_align": obj_axis_align, "value": [0.1, 0.2, 1.0], "shuffle": True},
            "color_jitter": True,
            "order_shuffle": True},
        "obj_aug": {
            "translation": {"enabled": True, "value": [0.1, 0.1, 0.1], "p": 1.0},
            "rotation": {"enabled": True, "p": 1.0, "axis_align": obj_axis_align,
                         "value": [0.3, 0.2, 1.0] if obj_axis_align else [0.1, 0.1, 0.1], "shuffle": True},
            "random_jitter": {"enabled": True, "value": 0.01, "accord_to_size": False, "p": 1.0},
            "pts_shuffle": True}}


class AttrCfg(Mapping):
    """Attribute-style, non-dict mapping (what DictConfig looks like to data_augmentor.py)."""

    def __init__(self, d):
        object.__setattr__(self, "_d", {k: AttrCfg(v) if isinstance(v, dict) else v for k, v in d.items()})

    def __getitem__(self, k):
        return self._d[k]

    def __iter__(self):
        return iter(self._d)

    def __len__(self):
        return len(self._d)

    def __getattr__(self, k):
        if k.startswith("_"):
            raise AttributeError(k)
        try:
            return self._d[k]
        except KeyError:
            raise AttributeError(k) from None


def load_reference():
    """data/datasets/base.py and data_augmentor.py without running the packages' __init__ (which imports every dataset)."""
    if REF not in sys.path:
        sys.path.insert(0, REF)
    for name in ("jsonlines",):
        sys.modules.setdefault(name, types.ModuleType(name))
    for pkg, path in (("data", os.path.join(REF, "data")), ("data.datasets", os.path.join(REF, "data", "datasets"))):
        if pkg not in sys.modules:
            m = types.ModuleType(pkg)
            m.__path__ = [path]
            sys.modules[pkg] = m

    def load(name, path):
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod

    aug = load("data.datasets.data_augmentor", os.path.join(REF, "data", "datasets", "data_augmentor.py"))
    base = load("data.datasets.base", os.path.join(REF, "data", "datasets", "base.py"))
    return aug.DataAugmentor, base.ScanBase


@contextlib.contextmanager
def recording(name, sink):
    real = getattr(np.random, name)

    def rec(*a, **k):
        r = real(*a, **k)
        sink.append(np.array(r))
        return r
    setattr(np.random, name, rec)
    try:
        yield
    finally:
        setattr(np.random, name, real)


def wrap(fn, name, sink):
    def wrapped(*a, **k):
        with recording(name, sink):
            return fn(*a, **k)
    return wrapped


def scene(rng, B, O, P, n_pad_last):
    """Per item O slots: n > P, n = P, n = 1, n < P, n > P, then padding (more of it in the last item)."""
    counts = np.zeros((B, O), np.int64)
    for b in range(B):
        c = [rng.integers(P + 1, 4 * P), P, 1, rng.integers(2, P), rng.integers(P + 1, 3 * P)][:O]
        n_real = O - (n_pad_last if b == B - 1 else 1)
        counts[b, :n_real] = c[:n_real]
    off = np.concatenate([[0], np.cumsum(counts.reshape(-1))]).astype(np.int64)
    raw = np.empty((off[-1], 6), np.float32)
    for s in range(B * O):
        n = off[s + 1] - off[s]
        if n:
            ctr = rng.uniform(-4, 4, 3)
            ext = rng.uniform(0.1, 2.0, 3)
            raw[off[s]:off[s + 1], :3] = (ctr + rng.uniform(-0.5, 0.5, (n, 3)) * ext).astype(np.float32)
            raw[off[s]:off[s + 1], 3:] = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    return raw, off, counts


def run_aug(DataAugmentor, ScanBase, cfg, split, raw, off, counts, P, seed):
    B, O = counts.shape
    np.random.seed(seed)
    item = np.zeros((B, 25))
    obj = np.zeros((B, O, 12))
    index = np.full((B, O, P), -1, np.int32)
    noise = np.zeros((B, O, P, 3), np.float32)
    fts = np.ones((B, O, P, 6), np.float32)
    locs, boxes = np.zeros((B, O, 6), np.float32), np.zeros((B, O, 6), np.float32)
    eye = np.eye(3).reshape(-1)
    for b in range(B):
        aug = DataAugmentor(AttrCfg(cfg), split)
        dicts, subs, jits, perms = [], [], [], []
        orig_update = aug.update_data_dict
        aug.update_data_dict = lambda dd, ad: (dicts.append(copy.deepcopy(ad)), orig_update(dd, ad))[1]
        aug.subsample_fn = wrap(DataAugmentor.subsample_fn, "choice", subs)
        aug.jitter_fn = wrap(DataAugmentor.jitter_fn, "randn", jits)
        aug.pts_shuffle_fn = wrap(DataAugmentor.pts_shuffle_fn, "permutation", perms)
        stub = types.SimpleNamespace(augmentor=aug, num_points=P)
        n_obj = int((counts[b] > 0).sum())
        objs = [raw[off[b * O + i]:off[b * O + i + 1]].copy() for i in range(n_obj)]
        f, l, bx, _ = ScanBase._obj_processing_aug(stub, objs, list(range(n_obj)), is_need_bbox=True)
        ad = dicts[0]
        item[b, 0:9] = ad["scene_flip"].reshape(-1) if ad["scene_flip"] is not None else eye
        item[b, 9] = ad["scene_scale"] if ad["scene_scale"] is not None else 1.0
        item[b, 10:13] = ad["scene_trans"] if ad["scene_trans"] is not None else 0.0
        item[b, 13:22] = ad["scene_rot"].reshape(-1) if ad["scene_rot"] is not None else eye
        item[b, 22:25] = ad["rgb_delta"] if ad["rgb_delta"] is not None else 0.0
        for i in range(O):
            obj[b, i, 3:12] = eye
        for i in range(n_obj):
            if ad["obj_trans"] and ad["obj_trans"][i] is not None:
                obj[b, i, 0:3] = ad["obj_trans"][i]
            if ad["obj_rot"] and ad["obj_rot"][i] is not None:
                obj[b, i, 3:12] = ad["obj_rot"][i].reshape(-1)
            perm = perms[i] if perms else np.arange(P)
            index[b, i] = subs[i][perm]
            if jits:
                noise[b, i] = jits[i][perm].astype(np.float32)
        fts[b, :n_obj] = f.numpy()
        locs[b, :n_obj] = l.numpy()
        boxes[b, :n_obj] = bx.numpy()
    flip_types = [{(-1, 1): 0, (1, -1): 1, (-1, -1): 2, (1, 1): 3}[(int(item[b, 0]), int(item[b, 4]))] for b in range(B)]
    angles = np.round(np.arctan2(item[:, 14], item[:, 13]) / (np.pi / 2)).astype(int) % 4
    return dict(item=item, obj=obj, index=index, noise=noise, obj_fts=fts, obj_locs=locs, obj_boxes=boxes), flip_types, angles


def run_post(ScanBase, raw, off, counts, P, seed):
    B, O = counts.shape
    np.random.seed(seed)
    qt = np.zeros(B, np.int32)
    index = np.full((B, O, P), -1, np.int32)
    fts = np.ones((B, O, P, 6), np.float32)
    locs, boxes = np.zeros((B, O, 6), np.float32), np.zeros((B, O, 6), np.float32)
    for b in range(B):
        ints, choices = [], []
        n_obj = int((counts[b] > 0).sum())
        objs = [raw[off[b * O + i]:off[b * O + i + 1]].copy() for i in range(n_obj)]
        stub = types.SimpleNamespace(split="train", num_points=P)
        with recording("randint", ints), recording("choice", choices):
            f, l, bx, _ = ScanBase._obj_processing_post(stub, objs, list(range(n_obj)), is_need_bbox=True, rot_aug=True)
        qt[b] = int(ints[0])
        for i in range(n_obj):
            index[b, i] = choices[i]
        fts[b, :n_obj] = f.numpy()
        locs[b, :n_obj] = l.numpy()
        boxes[b, :n_obj] = bx.numpy()
    return dict(quarter_turns=qt, index=index, obj_fts=fts, obj_locs=locs, obj_boxes=boxes)


def _jitter_on(cfg):
    return "obj_aug" in cfg["aug_list"] and cfg["obj_aug"]["random_jitter"]["enabled"]


def save(name, raw, off, counts, P, cfg, split, rot_aug, path, res):
    B, O = counts.shape
    if not (cfg and _jitter_on(cfg)):
        res.pop("noise", None)
    np.savez_compressed(os.path.join(OUT, name), raw=raw, offsets=off, B=B, O=O, P=P, config=json.dumps(cfg), split=split,
             rot_aug=rot_aug, path=path, obj_masks=(counts > 0), **res)
    print(name, {k: v.shape for k, v in res.items()})


def main():
    torch.set_num_threads(1)
    DataAugmentor, ScanBase = load_reference()
    B, O, P = 8, 6, 128
    # shipped block, train: all four scene angles among the items
    for seed in range(100):
        raw, off, counts = scene(np.random.default_rng(100 + seed), B, O, P, 3)
        res, _, angles = run_aug(DataAugmentor, ScanBase, SHIPPED, "train", raw, off, counts, P, seed)
        if len(set(angles.tolist())) == 4:
            break
    print("shipped angles (quarter turns)", angles.tolist())
    save("input_aug_shipped_train.npz", raw, off, counts, P, SHIPPED, "train", False, "aug", res)
    # shipped block, val: the augmentor queue is empty
    raw, off, counts = scene(np.random.default_rng(7), 4, O, P, 2)
    res, _, _ = run_aug(DataAugmentor, ScanBase, SHIPPED, "val", raw, off, counts, P, 3)
    save("input_aug_shipped_val.npz", raw, off, counts, P, SHIPPED, "val", False, "aug", res)
    # every option on, object / scene rotation axis-aligned and free: every flip type among the items
    for tag, align in (("align", True), ("free", False)):
        cfg = all_on(align)
        for seed in range(100):
            raw, off, counts = scene(np.random.default_rng(200 + seed), B, O, P, 2)
            res, flips, _ = run_aug(DataAugmentor, ScanBase, cfg, "train", raw, off, counts, P, seed)
            if len(set(flips)) == 4:
                break
        print(tag, "flip types", flips)
        save(f"input_aug_all_{tag}.npz", raw, off, counts, P, cfg, "train", False, "aug", res)
    # post path with rot_aug (ScanQA / SQA3D): every quarter turn among the items
    for seed in range(100):
        raw, off, counts = scene(np.random.default_rng(300 + seed), B, O, P, 2)
        res = run_post(ScanBase, raw, off, counts, P, seed)
        if len(set(res["quarter_turns"].tolist())) == 4:
            break
    print("post quarter turns", res["quarter_turns"].tolist())
    save("input_aug_post_rot.npz", raw, off, counts, P, None, "train", True, "post", res)


if __name__ == "__main__":
    main()
