"""ORACLE — TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available (oracle/ref_shims.py):
    python oracle/make_golden_eval.py
Writes tests/golden/eval_metrics.npz and tests/golden/eval_boxes.npz (described in tests/golden/EVAL.md).

* Metrics: the UNMODIFIED reference evaluators (evaluator/scanrefer_eval.py, referit3d_eval.py, scanqa_eval.py,
  sqa3d_eval.py, objcls_eval.py) on CPU over seeded batches with logits ties, padded -inf slots, a NaN row, top-10 ties away
  from and at the boundary and a partial last batch: every batch's `batch_metrics(include_count=True)` and the `record()`
  dictionary after `update` of all batches.  Stand-ins: `omegaconf.open_dict`, `common.misc.gather_dict` (one process: the
  identity), empty `data` / `evaluator` packages so that only the modules named here are imported, and SQA3DEval's
  `__init__` without its answer-vocabulary file.
* Boxes: `convert_pc_to_box` -> `construct_bbox_corners` -> `eval_ref_one_sample` (data/data_utils.py) on boxes a few ulps
  either side of IoU 0.25 and 0.5, one-point, disjoint and nested boxes, next to the restatements below of the numpy-1.26
  flow (the reference's pinned numpy) and of the numpy-2 flow (what runs here).
"""
import importlib
import importlib.util
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


# ---- restatements (no reference code) -----------------------------------------------------------------------------------
def box_np126(pts):
    """(lo, hi) of the corner box, dtypes of numpy 1.26 scalar arithmetic (value-independent promotion of all-scalar ops):
    xmin..zmax              np.float32   (np.min / np.max of the f32 points)
    xmin + xmax             np.float32   (both f32)
    (xmin + xmax) / 2       float64      (f32 with a Python int promotes; halving is exact)
    xmax - xmin             np.float32
    sx / 2, -sx / 2         float64      (exact)
    corners = vstack(...)   float64 array; corners[k] + center[k]: float64, rounded once
    min / max over corners  float64"""
    mn, mx = pts[:, :3].min(0).astype(np.float32), pts[:, :3].max(0).astype(np.float32)
    c = (mn + mx).astype(np.float32).astype(np.float64) / 2
    h = (mx - mn).astype(np.float32).astype(np.float64) / 2
    a, b = h + c, (-h) + c
    return np.minimum(a, b), np.maximum(a, b)


def box_np2(pts):
    """The same under numpy 2 (NEP 50): every step stays float32."""
    mn, mx = pts[:, :3].min(0).astype(np.float32), pts[:, :3].max(0).astype(np.float32)
    c = ((mn + mx) / np.float32(2)).astype(np.float32)
    h = ((mx - mn) / np.float32(2)).astype(np.float32)
    a, b = (h + c).astype(np.float32), ((-h) + c).astype(np.float32)
    return np.minimum(a, b), np.maximum(a, b)


def iou_of(b1, b2, dt):
    """box3d_iou: xA = max(mins), xB = min(maxs), inter = prod(max(xB - xA, 0)) left to right, volumes left to right,
    inter / (v1 + v2 - inter + 1e-8), all in dtype dt (float64 under numpy 1.26, float32 under numpy 2)."""
    (lo1, hi1), (lo2, hi2) = b1, b2
    d = np.maximum(np.minimum(hi1, hi2) - np.maximum(lo1, lo2), dt(0)).astype(dt)
    inter = dt(dt(d[0] * d[1]) * d[2])
    e1, e2 = (hi1 - lo1).astype(dt), (hi2 - lo2).astype(dt)
    v1, v2 = dt(dt(e1[0] * e1[1]) * e1[2]), dt(dt(e2[0] * e2[1]) * e2[2])
    return dt(inter / dt(dt(dt(v1 + v2) - inter) + dt(1e-8)))


def iou_np126(cand, gt):
    return iou_of(box_np126(cand), box_np126(gt), np.float64)


def iou_np2(cand, gt):
    return iou_of(box_np2(cand), box_np2(gt), np.float32)


def crop_priority(hit25, labels, tgt_label, O):
    """base.py:420-437 with the documented cap: the candidates chosen before the random draw, and how many the draw adds.
    (1) the IoU-25 hits (the target is the last of them; the last O if there are more), (2) candidates with the target label
    in index order until O are kept.  n <= O keeps everything."""
    n = len(labels)
    if n <= O:
        return list(range(n)), 0
    hits = [i for i in range(n) if hit25[i]][-O:]
    chosen = set(hits)
    for k in range(n):
        if len(chosen) >= O:
            break
        if k not in chosen and labels[k] == tgt_label:
            chosen.add(k)
    return sorted(chosen), O - len(chosen)


# ---- the unmodified reference ----------------------------------------------------------------------------------------------
def _install():
    ref_shims.install()
    om = sys.modules["omegaconf"]
    if not hasattr(om, "open_dict"):
        import contextlib
        om.open_dict = contextlib.nullcontext
    misc = types.ModuleType("common.misc")
    misc.gather_dict = lambda accelerator, d: d          # one process
    import common  # noqa: F401  (the reference's package; misc itself needs `accelerate`)
    sys.modules["common.misc"] = misc
    for pkg in ("data", "data.datasets", "evaluator"):     # skip the package __init__s (datasets, every evaluator)
        m = types.ModuleType(pkg)
        m.__path__ = [os.path.join(ref_shims.REF_ROOT, *pkg.split("."))]
        sys.modules[pkg] = m
    return {n: importlib.import_module("evaluator." + n) for n in
            ("build", "scanrefer_eval", "referit3d_eval", "scanqa_eval", "sqa3d_eval", "objcls_eval")}, \
        importlib.import_module("data.data_utils")


def _q(rng, shape, lo=-4, hi=4):
    """Scores on a coarse grid (multiples of 1/4, exact in bf16): plenty of ties."""
    return (rng.integers(lo * 4, hi * 4 + 1, size=shape) / 4.0).astype(np.float32)


def grounding_batch(rng, B, O=12, C=607, nan_row=None, with_iou=True):
    n = rng.integers(3, O + 1, size=B)
    masks = np.arange(O)[None] < n[:, None]
    d = {"og3d_logits": _q(rng, (B, O)), "obj_masks": masks,
         "obj_labels": np.where(masks, rng.integers(0, 8, size=(B, O)), -100).astype(np.int64),
         "tgt_object_id": np.array([[rng.integers(0, k + 1)] for k in n], np.int64),
         "txt_cls_logits": _q(rng, (B, C), -1, 1), "tgt_object_label": rng.integers(0, 4, size=(B, 1)).astype(np.int64)}
    d["og3d_logits"][~masks] = -np.inf                       # padded slots, as the grounding head masks them
    d["og3d_logits"][0, :] = -np.inf                         # an all -inf row: argmax 0
    d["og3d_logits"][1, :3] = d["og3d_logits"][1, :3].max()  # a tie for the maximum
    if nan_row is not None:
        d["og3d_logits"][nan_row, 2] = np.nan
    for k in ("obj_cls_post_logits", "obj_cls_pre_logits", "obj_cls_raw_logits"):
        d[k] = _q(rng, (B, O, C), -1, 1)
        d[k][:, :, :8] = _q(rng, (B, O, 8), 0, 2)             # ties among the first classes, the labels' range
    if nan_row is not None:
        d["obj_cls_raw_logits"][nan_row, 0, 5] = np.nan
    if with_iou:
        d["tgt_object_id_iou25"] = (rng.random((B, O)) < 0.3).astype(np.int64)
        d["tgt_object_id_iou50"] = d["tgt_object_id_iou25"] * (rng.random((B, O)) < 0.6)
        d["is_multiple"] = rng.random(B) < 0.5
    else:
        d["is_hard"] = rng.random(B) < 0.4
        d["is_view_dependent"] = rng.random(B) < 0.3
    return d


def answers_batch(rng, B, A, O=12, types=False, nan_row=None):
    s = _q(rng, (B, A))
    lab = np.zeros((B, A), np.int64)
    for b in range(B):
        if b % 5 != 4:                                       # some questions have no answer
            lab[b, rng.choice(A, size=int(rng.integers(1, 4)), replace=False)] = 1
    # row 0: the only correct answer ties with three others straddling rank 10 (lower index first: rank 9)
    # row 1: the same tie with the correct answer at the highest index (rank 12: a miss by the rule)
    # row 2: tie for the top score, correct answer at the lower index
    for b, pos in ((0, 0), (1, 3)):
        top = np.arange(9) + 10
        s[b] = -5.0
        s[b, top] = 10.0 + np.arange(9)
        tie = np.array([20, 21, 22, 23])
        s[b, tie] = 5.0
        lab[b] = 0
        lab[b, tie[pos]] = 1
    s[2, [30, 31]] = 9.5
    lab[2] = 0
    lab[2, 30] = 1
    if nan_row is not None:
        s[nan_row, 7] = np.nan
    n = rng.integers(3, O + 1, size=B)
    masks = np.arange(O)[None] < n[:, None]
    d = {"answer_scores": s, "answer_label": lab, "obj_masks": masks,
         "obj_labels": np.where(masks, rng.integers(0, 8, size=(B, O)), -100).astype(np.int64)}
    d["obj_cls_raw_logits"] = _q(rng, (B, O, 607), -1, 1)
    d["obj_cls_raw_logits"][:, :, :8] = _q(rng, (B, O, 8), 0, 2)
    if types:
        d["sqa_type"] = rng.integers(0, 6, size=B).astype(np.int64)
        d["sqa_type"][0] = 5
    return d


def objcls_batch(rng, B, O=12):
    n = rng.integers(3, O + 1, size=B)
    masks = np.arange(O)[None] < n[:, None]
    lg = _q(rng, (B, O, 607), -1, 1)
    lg[:, :, :8] = _q(rng, (B, O, 8), 0, 2)
    return {"obj_logits": lg, "obj_masks": masks,
            "obj_labels": np.where(masks, rng.integers(0, 8, size=(B, O)), -100).astype(np.int64)}


CASES = {  # name -> (evaluator, batch maker, batch sizes: the last one partial)
    "scanrefer": ("ScanReferEval", lambda r, B, i: grounding_batch(r, B, nan_row=3 if i == 1 else None), (8, 8, 5)),
    "referit3d": ("ReferIt3DEval", lambda r, B, i: grounding_batch(r, B, nan_row=3 if i == 0 else None, with_iou=False),
                  (8, 8, 3)),
    "scanqa": ("ScanQAEval", lambda r, B, i: answers_batch(r, B, 300, nan_row=4 if i == 1 else None), (8, 8, 6)),
    "sqa3d": ("SQA3DEval", lambda r, B, i: answers_batch(r, B, 706, types=True), (8, 8, 5)),
    "objcls": ("PretrainObjEval", lambda r, B, i: objcls_batch(r, B), (8, 8, 3)),
}


def _evaluator(mods, name, exp_dir):
    cfg = types.SimpleNamespace(eval=types.SimpleNamespace(save=False), exp_dir=exp_dir)
    if name == "SQA3DEval":
        cls = mods["sqa3d_eval"].SQA3DEval
        ev = cls.__new__(cls)                     # __init__ without the answer-vocabulary file: the same state
        ev.eval_dict = {k: [] for k in ['target_metric', 'obj_cls_raw_acc', 'ans1_acc', 'ans10_acc'] +
                        [f"type{i}_acc" for i in range(6)]}
        ev.total_count = 0
        ev.type_count = {f"type{i}_count": 1e-10 for i in range(6)}
        ev.best_result = -np.inf
        ev.save = False
        return ev
    mod = {"ScanReferEval": "scanrefer_eval", "ReferIt3DEval": "referit3d_eval", "ScanQAEval": "scanqa_eval",
           "PretrainObjEval": "objcls_eval"}[name]
    return getattr(mods[mod], name)(cfg, None)


def golden_metrics(mods):
    out, meta = {}, {}
    with tempfile.TemporaryDirectory() as exp_dir:
        for case, (name, make, sizes) in CASES.items():
            rng = np.random.default_rng(sum(map(ord, case)))
            ev = _evaluator(mods, name, exp_dir)
            per_batch = []
            for i, B in enumerate(sizes):
                d = make(rng, B, i)
                for k, v in d.items():
                    out[f"{case}:{i}:{k}"] = v
                t = {k: torch.from_numpy(v) for k, v in d.items()}
                if name == "SQA3DEval":
                    bm = ev.batch_metrics(dict(t))
                else:
                    bm = ev.batch_metrics(dict(t), include_count=True)
                per_batch.append({k: (list(v) if isinstance(v, tuple) else v) for k, v in bm.items()})
                ev.update(dict(t))
            _, rec = ev.record()
            meta[case] = {"evaluator": name, "batches": len(sizes), "batch_metrics": per_batch,
                          "record": {k: float(v) for k, v in rec.items()}}
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), np.uint8)
    np.savez_compressed(os.path.join(OUT, "eval_metrics.npz"), **out)
    print("eval_metrics.npz:", {c: m["record"].get("target_metric") for c, m in meta.items()})


def box_cases():
    """(name, candidate points, gt points): boxes at IoU 0.25 / 0.5 +- a few ulps, degenerate and disjoint boxes."""
    cases = []
    gt = np.array([[3.7, -1.3, 0.2, 0, 0, 0], [4.7, -0.3, 1.2, 0, 0, 0]], np.float32)     # an offset unit cube
    for target in (0.25, 0.5):
        s0 = np.float32(target)
        for k in range(-4, 5):
            s = s0
            for _ in range(abs(k)):
                s = np.nextafter(s, np.float32(np.inf if k > 0 else -np.inf))
            # nested box: x extent s of the unit cube's, same y and z
            x1 = np.float32(gt[0, 0] + s)
            cand = np.array([[gt[0, 0], gt[0, 1], gt[0, 2], 0, 0, 0], [x1, gt[1, 1], gt[1, 2], 0, 0, 0]], np.float32)
            cases.append((f"x{target}_{k:+d}", cand, gt))
            # shifted box: overlap fraction near the threshold along x
            sh = np.float32(gt[0, 0] + (1 - s))
            cand2 = cand.copy()
            cand2[:, 0] = [sh, sh + np.float32(1)]
            cases.append((f"shift{target}_{k:+d}", cand2, gt))
    rng = np.random.default_rng(5)
    cases.append(("one_point", gt[:1].copy(), gt))
    cases.append(("one_point_both", gt[:1].copy(), gt[:1].copy()))
    cases.append(("disjoint", gt + np.array([5, 0, 0, 0, 0, 0], np.float32), gt))
    inner = np.array([[3.9, -1.1, 0.4, 0, 0, 0], [4.5, -0.5, 1.0, 0, 0, 0]], np.float32)
    cases.append(("nested_inner", inner, gt))
    cases.append(("nested_outer", gt, inner))
    cases.append(("identical", gt.copy(), gt))
    for i in range(24):                                  # random clouds, off the thresholds
        c = rng.uniform(-3, 3, size=3)
        e = rng.uniform(0.2, 2, size=3)
        a = np.concatenate([c + rng.uniform(-0.5, 0.5, size=(50, 3)) * e, rng.uniform(-1, 1, (50, 3))], 1)
        b = np.concatenate([c + rng.uniform(-0.5, 0.5, size=(60, 3)) * e * rng.uniform(0.7, 1.3, 3) + rng.normal(0, 0.2, 3),
                            rng.uniform(-1, 1, (60, 3))], 1)
        cases.append((f"random{i}", a.astype(np.float32), b.astype(np.float32)))
    return cases


def golden_boxes(du):
    names, pts, gts, ref, r126, r2 = [], [], [], [], [], []
    for name, cand, gt in box_cases():
        c1, s1 = du.convert_pc_to_box(cand)
        c2, s2 = du.convert_pc_to_box(gt)
        iou = du.eval_ref_one_sample(du.construct_bbox_corners(c1, s1), du.construct_bbox_corners(c2, s2))
        names.append(name)
        pts.append(cand)
        gts.append(gt)
        ref.append(float(iou))
        r126.append(float(iou_np126(cand, gt)))
        r2.append(float(iou_np2(cand, gt)))
    ref, r126, r2 = np.array(ref), np.array(r126), np.array(r2)
    assert np.array_equal(ref.astype(np.float32), r2.astype(np.float32)), "the numpy-2 restatement is not the reference here"
    flags = lambda v: np.stack([v >= 0.25, v >= 0.5], 1)  # noqa: E731
    differ = np.nonzero((flags(r126) != flags(ref)).any(1))[0]
    print("boxes:", len(names), "cases; numpy-1.26 and numpy-2 flags differ on", [names[i] for i in differ])
    np.savez_compressed(os.path.join(OUT, "eval_boxes.npz"), names=np.array(names), cand=np.concatenate(pts),
                        gt=np.concatenate(gts), cand_len=np.array([len(p) for p in pts]),
                        gt_len=np.array([len(g) for g in gts]),
                        iou_reference_np2=ref, iou_np126=r126, iou_np2=r2, differ=differ.astype(np.int64))


if __name__ == "__main__":
    mods, du = _install()
    torch.manual_seed(0)
    golden_metrics(mods)
    golden_boxes(du)
