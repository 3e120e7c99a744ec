"""Evaluation throughput on one GPU: items/s of `evaluate.EvalRunner` (eval-mode forward + metric kernels replayed from one
CUDA graph) against an eager no_grad forward followed by a restatement of the reference's `batch_metrics`, with its host
synchronisations (evaluator/scanrefer_eval.py, scanqa_eval.py), on the same model and batch; and the metric kernels alone.

    python scripts/time_eval.py [--steps K] [--warmup W] [--out FILE]

Workloads: ScanRefer eval at 64 and 256 items per step (the yaml's per-GPU batch size), ScanQA at 32; 80 object slots x 1024
points, 50 text tokens, inputs resident on the device, synthetic weights.  Prints one JSON line per measurement with the
card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def scanrefer_batch(B):
    """64 synthetic scenes, tiled up to B items, with the ScanRefer eval keys."""
    from sceneverse_b200 import synthetic
    d = synthetic.scene_batch(42, B=64, O=80, P=1024, L=50, Ls=8)
    rng = np.random.default_rng(7)
    d["tgt_object_id_iou25"] = (rng.random((64, 80)) < 0.05).astype(np.int64)
    d["tgt_object_id_iou50"] = d["tgt_object_id_iou25"] * (rng.random((64, 80)) < 0.5)
    d["is_multiple"] = rng.random(64) < 0.5
    d["tgt_object_label"] = rng.integers(0, 607, (64, 1))
    reps = (B + 63) // 64
    return {k: torch.from_numpy(np.concatenate([np.asarray(v)] * reps)[:B]).cuda() for k, v in d.items()
            if k not in ("scene_txt_ids", "scene_txt_masks", "masked_lm_labels")}


def scanqa_batch(B):
    from sceneverse_b200 import synthetic
    d = synthetic.qa_batch(42, "ScanQA", B=B, O=80, P=1024, L=50, Ls=8, num_answers=8864)
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()
            if k not in ("scene_txt_ids", "scene_txt_masks", "masked_lm_labels")}


def scanrefer_metrics_with_syncs(d):
    """evaluator/scanrefer_eval.py batch_metrics: the same tensor operations and `.item()` reads."""
    m = {}
    og_pred = torch.argmax(d["og3d_logits"], dim=-1)
    total = len(og_pred)
    mult = d["is_multiple"].sum().item()
    i25 = d["tgt_object_id_iou25"][torch.arange(total, device=og_pred.device), og_pred].to(bool)
    i50 = d["tgt_object_id_iou50"][torch.arange(total, device=og_pred.device), og_pred].to(bool)
    m["og_acc_iou25"], m["og_acc_iou50"] = i25.sum().item(), i50.sum().item()
    m["og_acc_iou25_multiple"] = (i25 & d["is_multiple"]).sum().item()
    m["og_acc_iou50_multiple"] = (i50 & d["is_multiple"]).sum().item()
    m["og_acc"] = (og_pred == d["tgt_object_id"].squeeze(1)).sum().item()
    m["txt_acc"] = (torch.argmax(d["txt_cls_logits"], dim=1) == d["tgt_object_label"].squeeze(1)).sum().item()
    gt, mask = d["obj_labels"], d["obj_masks"]
    for k in list(d.keys()):
        if k.endswith("logits") and d[k].ndim == 3 and d[k].shape[:2] == gt.shape:
            pred = torch.argmax(d[k], dim=2)
            m[k.replace("logits", "acc")] = ((pred[mask] == gt[mask]).sum().item(), mask.sum().item())
    return m, mult


def scanqa_metrics_with_syncs(d):
    """evaluator/scanqa_eval.py batch_metrics: argmax, topk and the Python loop over every item and its top 10."""
    c1 = c10 = 0
    choice_1 = d["answer_scores"].argmax(dim=-1)
    choice_10 = torch.topk(d["answer_scores"].detach(), 10, -1)[1]
    for i in range(d["answer_label"].shape[0]):
        if d["answer_label"][i, choice_1[i]] == 1:
            c1 += 1
        for j in range(10):
            if d["answer_label"][i, choice_10[i, j]] == 1:
                c10 += 1
                break
    gt, mask = d["obj_labels"], d["obj_masks"]
    pred = torch.argmax(d["obj_cls_raw_logits"], dim=2)
    return c1, c10, (pred[mask] == gt[mask]).sum().item()


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def time_workload(name, B, args):
    from sceneverse_b200 import evaluate, model as M, ops, train, weights
    tf = weights.synthetic_tensor("text_features", (607, 768))
    cfg = M.scanrefer_config(text_features=tf) if name == "scanrefer" else M.scanqa_config(text_features=tf)
    ps = train.PretrainStep(cfg, "cuda", seed=1)
    ops.register_shadows(ps.module)          # the bf16 weight copies a training run keeps current
    data = scanrefer_batch(B) if name == "scanrefer" else scanqa_batch(B)
    ev = evaluate.ScanReferEval() if name == "scanrefer" else evaluate.ScanQAEval()
    runner = evaluate.EvalRunner(ps, [ev], batch_size=B)
    model = ps.module.model
    model.eval()
    with torch.no_grad():
        ms_graph = timed(lambda: runner.step(data), args.steps, args.warmup)

        def eager():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = model(dict(data))
            (scanrefer_metrics_with_syncs if name == "scanrefer" else scanqa_metrics_with_syncs)(out)
        ms_eager = timed(eager, args.steps, args.warmup)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(dict(data))
        out["valid"] = torch.ones(B, dtype=torch.bool, device="cuda")
        ms_kernels = timed(lambda: ev.update(out), 10 * args.steps, args.warmup)
    model.train()
    ops.clear_shadows()
    return {"workload": name, "items_per_step": B, "graph_ms": round(ms_graph, 3),
            "graph_items_per_s": round(B * 1e3 / ms_graph, 1), "eager_with_syncs_ms": round(ms_eager, 3),
            "eager_items_per_s": round(B * 1e3 / ms_eager, 1), "metric_kernels_ms": round(ms_kernels, 4),
            "steps": args.steps, "card": card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_eval.py measures on a GPU; none is visible")
    rows = []
    for name, B in (("scanrefer", 64), ("scanrefer", 256), ("scanqa", 32)):
        rows.append(time_workload(name, B, args))
        print(json.dumps(rows[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
