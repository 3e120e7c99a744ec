"""PretrainEval on the host (no GPU): its count -> metric arithmetic (`counts_to_metrics`, `record`) and the per-step train-log
dictionary, from counters restated with torch on the CPU, against every golden `batch_metrics` and `record()` of the
unmodified reference evaluator (tests/golden/eval_pretrain.npz, oracle/make_golden_pretrain_eval.py)."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_pretrain_eval as GP
from sceneverse_b200 import _lib, evaluate, train

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def meta():
    M = np.load(os.path.join(GOLDEN, "eval_pretrain.npz"))
    return M, json.loads(bytes(M["meta"]).decode())


def batch(M, case, i):
    p = f"{case}:{i}:"
    return {k[len(p):]: torch.from_numpy(GP.loaded(M[k])) for k in M.files if k.startswith(p)}


def host_counters(d, c, valid=None):
    """What PretrainEval's kernels add for one batch (the integer words, then the float64 bookkeeping), restated with torch
    on the CPU.  Returns the SV_EVP_HAS_* bits of the batch."""
    B = d["masked_lm_labels"].shape[0]
    valid = torch.ones(B, dtype=torch.bool) if valid is None else valid
    c[_lib.EVP_ITEMS] += int(valid.sum())
    lab = d["masked_lm_labels"]
    m = (lab != -1) & valid[:, None]
    pred = torch.argmax(d["txt_lm_cls_logits"].float(), 2)
    c[_lib.EVP_LM_HIT] += int((pred[m] == lab[m]).sum())
    c[_lib.EVP_LM_COUNT] += int(m.sum())
    present = 0
    if "tgt_object_id" in d:
        ok = (torch.argmax(d["og3d_logits"].float(), -1) == d["tgt_object_id"][:, 0]) & valid
        c[_lib.EVP_OG + _lib.EVG_ITEMS] += int(valid.sum())
        c[_lib.EVP_OG + _lib.EVG_OG_ACC] += int(ok.sum())
        present |= _lib.EVP_HAS_OG
    om = d["obj_masks"] & valid[:, None]
    sem = d.get("obj_sem_masks", d["obj_masks"])
    t = _lib.EVP_OBJ
    for k, bit in evaluate.PretrainEval.OBJ:
        if k in d:
            present |= bit
            hit = torch.argmax(d[k].float(), 2) == d["obj_labels"]
            for s, mm in enumerate((om, om & sem, om & ~sem)):
                c[t + 2 * s] += int((hit & mm).sum())
                c[t + 2 * s + 1] += int(mm.sum())
            t += 6
    pretrain_batch(c, present)
    return present


def pretrain_batch(c, present):
    """Host restatement of pretrain_batch_kernel (csrc/eval_metrics.cu)."""
    S, Q = _lib.EVP_SNAPSHOT, _lib.EVP_Q
    d = lambda k: c[k] - c[S + k]  # noqa: E731
    n = d(_lib.EVP_ITEMS)
    if n > 0:
        acc = lambda k: d(k) / (d(k + 1) + 1e-8)  # noqa: E731
        vals = []
        if present & _lib.EVP_HAS_OG:
            vals.append((_lib.EVP_Q_OG, d(_lib.EVP_OG + _lib.EVG_OG_ACC) / n))
        vals.append((_lib.EVP_Q_LM, acc(_lib.EVP_LM_HIT)))
        t = _lib.EVP_OBJ
        for bit, q in ((_lib.EVP_HAS_POST, (_lib.EVP_Q_POST, _lib.EVP_Q_POST_UNMASK, _lib.EVP_Q_POST_MASK)),
                       (_lib.EVP_HAS_RAW, (_lib.EVP_Q_RAW,)),
                       (_lib.EVP_HAS_PRE, (_lib.EVP_Q_PRE, _lib.EVP_Q_PRE_UNMASK, _lib.EVP_Q_PRE_MASK))):
            if present & bit:
                vals += [(qk, acc(t + 2 * s)) for s, qk in enumerate(q)]
                t += 6
        s = 0.0
        for qk, v in vals:
            c[Q + qk] += v * n
            s += v
        c[Q + _lib.EVP_Q_TARGET] += s / len(vals) * n
    c[S:2 * S] = c[:S]


def test_layout_mirrors_the_library():
    assert _lib.gps().sv_eval_counters_size(_lib.EVAL_PRETRAIN) == _lib.EVP_SIZE
    assert _lib.EVP_Q == 2 * _lib.EVP_SNAPSHOT and _lib.EVP_SNAPSHOT == _lib.EVP_OBJ + 18


@pytest.mark.parametrize("case", list(GP.CASES))
def test_batch_metrics_from_counts_match_golden(case):
    """Every batch: the counts restated on the CPU, through PretrainEval.counts_to_metrics, give the reference's
    batch_metrics exactly, keys in its order."""
    M, m = meta()
    ev = evaluate.PretrainEval(device="cpu")
    for i, want in enumerate(m[case]["batch_metrics"]):
        c = [0.0] * _lib.EVP_SIZE
        ev.present = host_counters(batch(M, case, i), c)
        got = ev.counts_to_metrics(c)
        assert list(got) == list(want), (case, i)
        assert got == want, (case, i)


@pytest.mark.parametrize("case", list(GP.CASES))
def test_record_from_counters_matches_golden(case):
    """The float64 sums kept as sv_eval_pretrain_batch keeps them give the reference's record() bitwise."""
    M, m = meta()
    ev = evaluate.PretrainEval(device="cpu")
    c = [0.0] * _lib.EVP_SIZE
    for i in range(m[case]["batches"]):
        ev.present = host_counters(batch(M, case, i), c)
    ev.counters = torch.tensor(c, dtype=torch.float64)
    is_best, rec = ev.record()
    assert is_best and list(rec) == list(m[case]["record"])
    assert rec == m[case]["record"]
    # Python 3.12's compensated sum() (the fixture's second run) differs from the reference's pinned 3.9 in the last bits only
    for k, v in m[case]["record_compensated"].items():
        assert math.isclose(rec[k], v, rel_tol=1e-15, abs_tol=0.0), (k, rec[k], v)


@pytest.mark.parametrize("case", list(GP.CASES))
def test_step_log_entry_matches_reference_batch_metrics(case):
    """A train-log ring row holding a batch's counts reads back as the reference trainer's log dictionary: train/step, the
    losses, train/<key> of the reference's batch_metrics (same keys, same values) and train/lr/group_i."""
    M, m = meta()
    ev = evaluate.PretrainEval(device="cpu")
    log = train.TrainLog(ev, ["lm_cls_loss", "total_loss"], 4, "cpu")
    rows = []
    for i, want in enumerate(m[case]["batch_metrics"]):
        c = [0.0] * _lib.EVP_SIZE
        ev.present = host_counters(batch(M, case, i), c)
        rows.append([float(i + 1), 0.5 + i, 1.25 + i] + c)
        log.end_step(i + 1, [1e-5 * (i + 1), 2e-4])
    log.ring[:len(rows)] = torch.tensor(rows, dtype=torch.float64)
    out = log.read()
    assert len(out) == len(rows) and log.read() == []
    for i, (entry, want) in enumerate(zip(out, m[case]["batch_metrics"])):
        expect = {"train/step": i + 1, "train/lm_cls_loss": 0.5 + i, "train/total_loss": 1.25 + i}
        expect.update((f"train/{k}", v) for k, v in want.items())
        expect.update({"train/lr/group_0": 1e-5 * (i + 1), "train/lr/group_1": 2e-4})
        assert list(entry) == list(expect) and entry == expect, (case, i)


def test_log_ring_overflow_raises():
    log = train.TrainLog(evaluate.PretrainEval(device="cpu"), ["total_loss"], 2, "cpu")
    for s in (1, 2):
        log.begin_step()
        log.end_step(s, [])
    with pytest.raises(RuntimeError, match="log_every"):
        log.begin_step()
