"""ORACLE — TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available (oracle/ref_shims.py):
    python oracle/make_golden_pretrain_eval.py
Writes tests/golden/eval_pretrain.npz (described in tests/golden/EVAL_PRETRAIN.md).

The UNMODIFIED reference `PretrainEval` (evaluator/pretrain_eval.py) on CPU over seeded batches on the coarse score grid of
make_golden_eval (plenty of ties): every batch's `batch_metrics` and the `record()` dictionary after `update` of all batches.
The masked-LM vocabulary is 1,000 wide (the full 30,522 is checked on the GPU against torch.argmax).  Logits are stored as
float16, which holds every value of the grid exactly (and NaN); the tests widen them to float32, as the reference saw them.

The evaluator sums Python floats with the builtin `sum` (target_metric, record).  The reference pins Python 3.9, whose `sum`
adds left to right; from Python 3.12 on `sum` compensates the rounding (Neumaier), which can change the last bit.  The
fixture records both: `batch_metrics` / `record` with the module's `sum` bound to the left-to-right sum of the pinned
interpreter (the one stand-in), and `record_compensated` from the same evaluator as this interpreter runs it.
"""
import importlib
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_eval as G  # noqa: E402

V, L, O, C = 1000, 6, 10, 48


def pretrain_batch(rng, B, shape, no_label=False, no_sem=None, specials=False):
    """shape 'pretrain': og3d, LM, post and raw object logits (OVPretrainHead); 'finetune': also pre.  no_sem: 'all' (no
    sem-masked object in the batch) or 'item' (item 0 has none).  specials: tie rows, NaN rows and an all-negative row."""
    lm = G._q(rng, (B, L, V))
    lab = np.where(rng.random((B, L)) < 0.25, rng.integers(0, V, (B, L)), -1).astype(np.int64)
    if no_label:
        lab[:] = -1
    elif (lab == -1).all():
        lab[0, 0] = 3
    for b, t in zip(*np.nonzero(lab != -1)):
        u = rng.random()
        if u < 0.35:
            lm[b, t, lab[b, t]] = lm[b, t].max()          # a tie for the maximum: a hit only if no lower index ties
        elif u < 0.6:
            lm[b, t, lab[b, t]] = 4.25                    # the unique maximum
    if specials:
        lm[0, 0], lab[0, 0] = -4.0, 17                    # every column ties: index 0 wins, a miss
        lm[0, 1, :] = -4.0
        lm[0, 1, [5, 9]], lab[0, 1] = 2.0, 9               # two tied maxima, the label at the higher index: a miss
        lm[0, 2, :] = -4.0
        lm[0, 2, [5, 9]], lab[0, 2] = 2.0, 5               # ... at the lower index: a hit
        lm[1, 0, [40, 700]], lab[1, 0] = np.nan, 40        # first NaN wins: a hit
        lm[1, 1, [40, 700]], lab[1, 1] = np.nan, 700       # second NaN: a miss
        lm[1, 1, 3] = 4.25
        lm[1, 2] = G._q(rng, (V,), -4, -1)                 # every logit negative
        lab[1, 2] = int(np.argmax(lm[1, 2]))
    n = rng.integers(3, O + 1, size=B)
    masks = np.arange(O)[None] < n[:, None]
    sem = masks & (rng.random((B, O)) > 0.25)
    if no_sem == "all":
        sem[:] = False
    elif no_sem == "item":
        sem[0] = False
    d = {"txt_lm_cls_logits": lm, "masked_lm_labels": lab, "og3d_logits": G._q(rng, (B, O)),
         "tgt_object_id": np.array([[rng.integers(0, k)] for k in n], np.int64), "obj_masks": masks, "obj_sem_masks": sem,
         "obj_labels": np.where(masks, rng.integers(0, 8, size=(B, O)), -100).astype(np.int64)}
    d["og3d_logits"][1, :4] = d["og3d_logits"][1].max()   # a tie for the maximum (padded slots take part: no mask)
    for k in ("obj_cls_post_logits", "obj_cls_raw_logits") + (("obj_cls_pre_logits",) if shape == "finetune" else ()):
        d[k] = G._q(rng, (B, O, C), -1, 1)
        d[k][:, :, :8] = G._q(rng, (B, O, 8), 0, 2)        # ties among the first classes, the labels' range
    if specials:
        d["obj_cls_post_logits"][2, 0, 6] = np.nan
    return d


CASES = {  # name -> (batch maker, batch sizes); the pretrain case ends in a partial batch
    "pretrain": (lambda r, B, i: pretrain_batch(r, B, "pretrain", specials=i == 0), (8, 8, 5)),
    "finetune": (lambda r, B, i: pretrain_batch(r, B, "finetune", specials=i == 1), (8, 6)),
    "no_label": (lambda r, B, i: pretrain_batch(r, B, "pretrain", no_label=i == 0), (6, 6)),
    "no_sem": (lambda r, B, i: pretrain_batch(r, B, "finetune", no_sem="all" if i == 0 else "item"), (6, 6)),
}


def stored(k, v):
    return v.astype(np.float16) if k.endswith("logits") else v


def loaded(v):
    return v.astype(np.float32) if v.dtype == np.float16 else v


def sum_left_to_right(xs, start=0):
    """Python 3.9's builtin sum over floats: one rounded addition per item, in order."""
    for x in xs:
        start = start + x
    return start


def run(mod, batches):
    ev = mod.PretrainEval(types.SimpleNamespace(), types.SimpleNamespace(device="cpu"))
    per_batch = []
    for d in batches:
        t = {k: torch.from_numpy(loaded(v)) for k, v in d.items()}
        per_batch.append(ev.batch_metrics(dict(t)))
        ev.update(dict(t))
    _, rec = ev.record()
    return per_batch, {k: float(v) for k, v in rec.items()}


def main():
    G._install()
    mod = importlib.import_module("evaluator.pretrain_eval")
    out, meta = {}, {}
    for case, (make, sizes) in CASES.items():
        rng = np.random.default_rng(sum(map(ord, case)) + 7)
        batches = [{k: stored(k, v) for k, v in make(rng, B, i).items()} for i, B in enumerate(sizes)]
        for i, d in enumerate(batches):
            for k, v in d.items():
                out[f"{case}:{i}:{k}"] = v
        mod.sum = sum_left_to_right
        per_batch, rec = run(mod, batches)
        del mod.sum
        _, rec_compensated = run(mod, batches)
        meta[case] = {"batches": len(sizes), "batch_metrics": per_batch, "record": rec,
                      "record_compensated": rec_compensated}
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), np.uint8)
    path = os.path.join(G.OUT, "eval_pretrain.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes:", {c: m["record"]["target_metric"] for c, m in meta.items()})


if __name__ == "__main__":
    main()
