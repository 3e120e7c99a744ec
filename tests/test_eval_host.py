"""Evaluation on the host (no GPU): the numpy-1.26 IoU restatement against the unmodified reference helpers, and the
counter -> metric-dictionary code of sceneverse_b200.evaluate against every golden `record()` of the unmodified evaluators
(tests/golden/eval_*.npz, oracle/make_golden_eval.py)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_eval as G
from sceneverse_b200 import _lib, evaluate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def boxes():
    Z = np.load(os.path.join(GOLDEN, "eval_boxes.npz"))
    ci = np.concatenate([[0], np.cumsum(Z["cand_len"])])
    gi = np.concatenate([[0], np.cumsum(Z["gt_len"])])
    return Z, [(Z["cand"][ci[i]:ci[i + 1]], Z["gt"][gi[i]:gi[i + 1]]) for i in range(len(Z["names"]))]


def test_iou_restatements_match_the_reference_helpers():
    """numpy-2 restatement == the unmodified helpers run under numpy 2 (bitwise); the numpy-1.26 restatement gives the same
    flags on every case off the thresholds, and the cases where the two flows disagree are all within a few ulps of one."""
    Z, cases = boxes()
    for i, (c, g) in enumerate(cases):
        assert np.float32(G.iou_np2(c, g)) == np.float32(Z["iou_reference_np2"][i]), Z["names"][i]
        assert G.iou_np126(c, g) == Z["iou_np126"][i], Z["names"][i]
    ref, r126 = Z["iou_reference_np2"], Z["iou_np126"]
    differ = set(Z["differ"].tolist())
    for i, name in enumerate(Z["names"]):
        same = (ref[i] >= 0.25) == (r126[i] >= 0.25) and (ref[i] >= 0.5) == (r126[i] >= 0.5)
        assert same == (i not in differ), name
        if not name.startswith(("x0.", "shift0.")):
            assert same, name
    assert differ, "the fixture should hold a case where the two flows give different flags"


def test_crop_priority():
    hit = [0, 1, 0, 0, 1, 0, 0, 0]
    lab = [3, 3, 5, 3, 9, 5, 3, 3]
    assert G.crop_priority(hit, lab, 3, 4) == ([0, 1, 3, 4], 0)
    assert G.crop_priority(hit, lab, 7, 4) == ([1, 4], 2)
    assert G.crop_priority(hit, lab, 3, 8) == (list(range(8)), 0)
    assert G.crop_priority([1] * 8, lab, 3, 3) == ([5, 6, 7], 0)     # more hits than slots: the last O (target = last)


# ---- counters restated on the host from the fixture batches ---------------------------------------------------------------
def meta():
    M = np.load(os.path.join(GOLDEN, "eval_metrics.npz"))
    return M, json.loads(bytes(M["meta"]).decode())


def batch(M, case, i):
    p = f"{case}:{i}:"
    return {k[len(p):]: torch.from_numpy(M[k]) for k in M.files if k.startswith(p)}


def rank_hit(s, lab, k):
    """a labelled answer among the first k (scores descending, NaN first, ties: lower index first)"""
    key = np.where(np.isnan(s), np.inf, s)
    order = sorted(range(len(s)), key=lambda j: (-key[j], j))
    return any(lab[j] == 1 for j in order[:k])


def topk_hit(s, lab, k):
    """the reference: torch.topk (CPU), whose choice among tied scores at the boundary is its own"""
    return any(lab[j] == 1 for j in torch.topk(torch.from_numpy(s), k)[1].tolist())


def host_counters(case, d, c, hit10=rank_hit):
    """What the metric kernels add for one batch, restated with torch on the CPU; hit10=topk_hit counts the top-10 hits as
    the reference does."""
    valid = torch.ones(len(next(iter(d.values()))), dtype=torch.bool)
    if case in ("scanrefer", "referit3d"):
        p = torch.argmax(d["og3d_logits"], -1)
        ok = p == d["tgt_object_id"][:, 0]
        c[_lib.EVG_ITEMS] += len(p)
        c[_lib.EVG_OG_ACC] += int(ok.sum())
        c[_lib.EVG_TXT_ACC] += int((torch.argmax(d["txt_cls_logits"], 1) == d["tgt_object_label"][:, 0]).sum())
        if case == "scanrefer":
            m = d["is_multiple"]
            h25 = d["tgt_object_id_iou25"][torch.arange(len(p)), p].bool()
            h50 = d["tgt_object_id_iou50"][torch.arange(len(p)), p].bool()
            c[_lib.EVG_MULTIPLE] += int(m.sum())
            c[_lib.EVG_IOU25] += int(h25.sum())
            c[_lib.EVG_IOU50] += int(h50.sum())
            c[_lib.EVG_IOU25_MULTIPLE] += int((h25 & m).sum())
            c[_lib.EVG_IOU50_MULTIPLE] += int((h50 & m).sum())
        else:
            c[_lib.EVG_HARD] += int(d["is_hard"].sum())
            c[_lib.EVG_VIEW_DEP] += int(d["is_view_dependent"].sum())
            c[_lib.EVG_OG_ACC_HARD] += int((ok & d["is_hard"]).sum())
            c[_lib.EVG_OG_ACC_VIEW_DEP] += int((ok & d["is_view_dependent"]).sum())
        keys = evaluate._obj_logit_keys(d)
        base = _lib.EVG_OBJ
    elif case == "objcls":
        keys, base = ["obj_logits"], 0
    else:
        s, lab = d["answer_scores"].numpy(), d["answer_label"].numpy()
        for b in range(len(s)):
            h1, h10 = rank_hit(s[b], lab[b], 1), hit10(s[b], lab[b], 10)
            c[_lib.EVA_ITEMS] += 1
            c[_lib.EVA_ANS1] += h1
            c[_lib.EVA_ANS10] += h10
            if case == "sqa3d":
                t = int(d["sqa_type"][b])
                c[_lib.EVA_TYPE_ITEMS + t] += 1
                c[_lib.EVA_TYPE_ANS1 + t] += h1
        keys, base = ["obj_cls_raw_logits"], _lib.EVA_OBJ_HIT
    m = d["obj_masks"] & valid[:, None]
    for t, k in enumerate(keys):
        pred = torch.argmax(d[k], 2)
        c[base + 2 * t] += int((pred[m] == d["obj_labels"][m]).sum())
        c[base + 2 * t + 1] += int(m.sum())
    if case == "sqa3d":
        sqa3d_batch(c)
    return keys


def sqa3d_batch(c):
    """Host restatement of sqa3d_batch_kernel (csrc/eval_metrics.cu)."""
    snap = c[_lib.EVA_SNAPSHOT:_lib.EVA_SNAPSHOT + _lib.EVA_SNAPSHOT]
    n = c[_lib.EVA_ITEMS] - snap[_lib.EVA_ITEMS]
    if n > 0:
        d = lambda k: c[k] - snap[k]  # noqa: E731
        c[_lib.EVA_Q_ANS1] += d(_lib.EVA_ANS1) / n * n
        c[_lib.EVA_Q_ANS10] += d(_lib.EVA_ANS10) / n * n
        if d(_lib.EVA_OBJ_COUNT) > 0:
            c[_lib.EVA_Q_OBJ] += d(_lib.EVA_OBJ_HIT) / d(_lib.EVA_OBJ_COUNT) * n
        for t in range(6):
            cnt = evaluate._type_count(d(_lib.EVA_TYPE_ITEMS + t))
            c[_lib.EVA_Q_TYPE + t] += d(_lib.EVA_TYPE_ANS1 + t) / cnt * cnt
            c[_lib.EVA_Q_TYPE_COUNT + t] += cnt
    c[_lib.EVA_SNAPSHOT:_lib.EVA_SNAPSHOT * 2] = c[:_lib.EVA_SNAPSHOT]


def close(a, b):
    return a == b or abs(a - b) <= 1e-12 * max(abs(a), abs(b))


@pytest.mark.parametrize("case", list(G.CASES))
def test_record_from_counters_matches_golden(case):
    M, meta_ = meta()
    m = meta_[case]
    ev = getattr(evaluate, m["evaluator"])(device="cpu")
    c = ev.counters.tolist()
    for i in range(m["batches"]):
        d = batch(M, case, i)
        keys = host_counters(case, d, c, hit10=topk_hit)
        if case in ("scanrefer", "referit3d"):
            ev._txt, ev._obj_keys = True, keys
        elif case == "scanqa":
            ev._obj_key = keys[0]
    ev.counters = torch.tensor(c, dtype=torch.float64)
    _, rec = ev.record()
    want = m["record"]
    assert set(rec) == set(want)
    for k in want:
        assert close(float(rec[k]), want[k]), (k, rec[k], want[k])


def test_save_and_per_scene_logits_raise():
    with pytest.raises(NotImplementedError):
        evaluate.ScanReferEval({"eval": {"save": True}}, None, device="cpu")
    ev = evaluate.ScanReferEval(device="cpu")
    with pytest.raises(NotImplementedError):
        ev.update({"og3d_logits": torch.zeros(2, 3, 4), "tgt_object_id": torch.zeros(2, 3, dtype=torch.int64)})
