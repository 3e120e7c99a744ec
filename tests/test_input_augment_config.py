"""`AugSpec.from_config` on the config blocks stored with the augmentation fixtures (tests/golden/input_aug_*.npz): which path
the reference's dataset takes and which augmentations its `DataAugmentor` queues (data/datasets/base.py:247-253,
data/datasets/data_augmentor.py)."""
import copy
import json
import os
from collections.abc import Mapping

import numpy as np
import pytest

from sceneverse_b200 import _lib
from sceneverse_b200.input_pipeline import AugSpec, RotationSpec

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def block(name):
    return json.loads(str(np.load(os.path.join(GOLDEN, f"input_aug_{name}.npz"))["config"]))


class AttrCfg(Mapping):
    """Attribute-style mapping that is not a dict, like hydra's DictConfig."""

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


@pytest.mark.parametrize("wrap", [dict, AttrCfg])
def test_shipped_block_is_one_scene_quarter_turn(wrap):
    spec = AugSpec.from_config(wrap(block("shipped_train")), rot_aug=False, split="train")
    assert spec == AugSpec(path="aug", scene_rotation=RotationSpec((0.0, 0.0, 1.0), True, True))
    assert spec.params().flags == _lib.AUG_SCENE_ROT
    # obj_aug is in the block but not in aug_list: pts_shuffle: True does not run
    assert not spec.pts_shuffle


@pytest.mark.parametrize("wrap", [dict, AttrCfg])
def test_every_option_block(wrap):
    for name, align in (("all_align", True), ("all_free", False)):
        cfg = block(name)
        spec = AugSpec.from_config(wrap(cfg), split="train")
        assert spec.path == "aug" and spec.flip and spec.color_jitter and spec.pts_shuffle
        assert spec.scaling == (0.9, 1.1) and spec.scene_translation == (0.5, 0.5, 0.2) and spec.obj_translation == (0.1, 0.1, 0.1)
        assert spec.jitter == 0.01
        assert spec.scene_rotation.axis_align == align and spec.obj_rotation.axis_align == align and spec.obj_rotation.shuffle
        assert spec.params().flags == 511


def test_post_path_and_rot_aug():
    assert AugSpec.from_config(None, rot_aug=True, split="train") == AugSpec(path="post", rot_aug=True)
    assert AugSpec.from_config({}, rot_aug=True, split="train") == AugSpec(path="post", rot_aug=True)
    assert AugSpec.from_config(None, rot_aug=False, split="train") == AugSpec(path="post")
    for split in ("val", "test"):
        assert AugSpec.from_config(None, rot_aug=True, split=split) == AugSpec(path="post")


def test_p_is_not_consulted():
    cfg = block("all_align")
    zero = copy.deepcopy(cfg)
    for b in ("scene_aug", "obj_aug"):
        for v in zero[b].values():
            if isinstance(v, dict):
                v["p"] = 0.0
    assert AugSpec.from_config(AttrCfg(zero)) == AugSpec.from_config(AttrCfg(cfg))
    assert AugSpec.from_config(zero) == AugSpec.from_config(cfg)


def test_non_train_splits_turn_everything_off():
    for name in ("shipped_train", "all_align"):
        for split in ("val", "test"):
            assert AugSpec.from_config(AttrCfg(block(name)), split=split) == AugSpec(path="aug")
    assert AugSpec.from_config(AttrCfg(block("shipped_val")), split="val") == AugSpec(path="aug")


def test_check_key_semantics():
    cfg = block("all_align")
    cfg["obj_aug"]["pts_shuffle"] = None                     # None: off
    cfg["scene_aug"]["flip"] = {"p": 1.0}                    # a block without `enabled`: on
    cfg["scene_aug"]["color_jitter"] = {"enabled": False}
    del cfg["obj_aug"]["translation"]                        # absent: off
    spec = AugSpec.from_config(AttrCfg(cfg))
    assert not spec.pts_shuffle and spec.flip and not spec.color_jitter and spec.obj_translation is None
    only_obj = block("all_align")
    del only_obj["scene_aug"]                                # listed but not in the block: skipped
    spec = AugSpec.from_config(AttrCfg(only_obj))
    assert spec.scene_rotation is None and not spec.flip and spec.obj_rotation is not None


@pytest.mark.parametrize("path,value", [
    (("scene_aug", "scaling", "value"), [0.9]),
    (("scene_aug", "scaling", "value"), [0.9, 1.0, 1.1]),
    (("scene_aug", "scaling", "value"), "0.9,1.1"),
    (("scene_aug", "scaling", "value"), [0.9, float("nan")]),
    (("obj_aug", "random_jitter", "value"), -0.01),
    (("obj_aug", "random_jitter", "value"), "0.01"),
    (("scene_aug", "translation", "value"), [1.0, 1.0]),
    (("obj_aug", "rotation", "value"), [0.1, None, 0.1]),
    (("aug_list",), ["scene_aug", "mystery_aug"]),
    (("aug_list",), "scene_aug"),
])
def test_malformed_blocks_raise(path, value):
    cfg = block("all_align")
    d = cfg
    for k in path[:-1]:
        d = d[k]
    d[path[-1]] = value
    if path == ("aug_list",):
        cfg["mystery_aug"] = {}
    with pytest.raises(ValueError):
        AugSpec.from_config(AttrCfg(cfg))
