"""Cost of the per-step train logs (`train.PretrainStep(train_eval=...)`) on one GPU, in one process.

    python scripts/time_train_logs.py [--steps K] [--pairs N] [--read-every R] [--out FILE]

* GPS pre-training step at the bench shape (64 scenes x 80 objects x 1024 points, bf16, one CUDA graph) without logs and
  with PretrainEval logs read by `logs()` every R steps; ScanRefer fine-tune step (same shape) without and with
  ScanReferEval logs.  The two steps of a workload are built side by side and timed alternately, N windows of K steps each
  (CUDA events around the window; the `logs()` reads, which synchronise the host, are inside it).  One resident batch.
* The metric kernels alone (CUDA events over 200 launches): the masked-LM argmax over a (3200, 30528) bf16 LM-head buffer
  with V = 30522 and about 15 % labelled rows, the object splits over (64, 80, 607) post and raw logits, and all of
  PretrainEval's kernels of one step.
* The reference's pattern: an eager step followed by pretrain_eval.py's batch_metrics with its `.item()` reads.
Prints one JSON line per measurement with the card's name and power limit."""
import argparse
import gc
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


def gps_batch():
    import bench
    d = bench.make_scene_batches(1, bench.SCENES, 0)[0]
    return {k: torch.from_numpy(np.asarray(v)).cuda() for k, v in d.items()}


def scanrefer_batch():
    d = {k: v for k, v in gps_batch().items() if k not in ("scene_txt_ids", "scene_txt_masks")}
    B, O = d["obj_masks"].shape
    g = torch.Generator(device="cuda").manual_seed(7)
    d["tgt_object_id_iou25"] = (torch.rand((B, O), device="cuda", generator=g) < 0.05).long()
    d["tgt_object_id_iou50"] = d["tgt_object_id_iou25"] * (torch.rand((B, O), device="cuda", generator=g) < 0.5)
    d["is_multiple"] = torch.rand(B, device="cuda", generator=g) < 0.5
    d["tgt_object_label"] = torch.randint(0, 607, (B, 1), device="cuda", generator=g)
    return d


def events_ms(fn, n):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0.record()
    for i in range(n):
        fn(i)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / n


def time_steps(name, cfg, batch, make_eval, args):
    from sceneverse_b200 import train
    steps = {"no_logs": train.PretrainStep(cfg, "cuda", seed=0, cuda_graph=True),
             "logs": train.PretrainStep(cfg, "cuda", seed=0, cuda_graph=True, train_eval=make_eval(),
                                        log_every=args.read_every)}
    for st in steps.values():
        for _ in range(3):          # set-up and warm-up replays
            st.step(batch)
    steps["logs"].logs()
    res = {k: [] for k in steps}
    for _ in range(args.pairs):
        for k, st in steps.items():
            def one(i, st=st, k=k):
                st.step(batch)
                if k == "logs" and (i + 1) % args.read_every == 0:
                    st.logs()
            res[k].append(round(events_ms(one, args.steps), 3))
    row = {"workload": name, "ms_per_step": res, "read_every": args.read_every, "steps_per_window": args.steps,
           "native_launches_per_step": {k: int(st.native_launches_per_step) for k, st in steps.items()},
           "card": card()}
    steps["logs"].step(batch)
    row["last_log"] = {k: v for k, v in steps["logs"].logs()[-1].items() if "/lr/" not in k}
    for st in steps.values():
        st.close()
    return row


def time_kernels(args):
    from sceneverse_b200 import _lib, evaluate
    V, B, L, O, C = 30522, 64, 50, 80, 607
    g = torch.Generator(device="cuda").manual_seed(0)
    lm = torch.zeros((B * L, 30528), dtype=torch.bfloat16, device="cuda")
    lm[:, :V] = torch.randn((B * L, V), device="cuda", generator=g).to(torch.bfloat16)
    labels = torch.where(torch.rand(B * L, device="cuda", generator=g) < 0.15,
                         torch.randint(0, V, (B * L,), device="cuda", generator=g), -1).view(B, L)
    masks = torch.rand((B, O), device="cuda", generator=g) < 0.6
    d = {"txt_lm_cls_logits": lm.view(B, L, -1)[..., :V], "masked_lm_labels": labels,
         "og3d_logits": torch.randn((B, O), device="cuda", generator=g).to(torch.bfloat16),
         "tgt_object_id": torch.randint(0, O, (B, 1), device="cuda", generator=g), "obj_masks": masks,
         "obj_sem_masks": masks & (torch.rand((B, O), device="cuda", generator=g) < 0.75),
         "obj_labels": torch.randint(0, C, (B, O), device="cuda", generator=g),
         "obj_cls_post_logits": torch.randn((B, O, C), device="cuda", generator=g).to(torch.bfloat16),
         "obj_cls_raw_logits": torch.randn((B, O, C), device="cuda", generator=g).to(torch.bfloat16)}
    ev = evaluate.PretrainEval()
    c = ev.counters
    n = args.kernel_launches
    labelled = int((labels != -1).sum())

    def lm_only(i):
        _lib.call(_lib.gps(), "sv_eval_lm_acc", lm.device, lm.data_ptr(), 1, lm.stride(0), B * L, V, L, labels.data_ptr(),
                  None, c.data_ptr())
    ms_lm = events_ms(lm_only, n)
    ms_obj = events_ms(lambda i: evaluate._launch_obj_cls([d["obj_cls_post_logits"], d["obj_cls_raw_logits"]], d, None,
                                                          c[_lib.EVP_OBJ:], split=d["obj_sem_masks"]), n)
    ms_all = events_ms(lambda i: ev._launch(d, None, c), n)
    lm_bytes = labelled * V * 2 + B * L * 8
    return {"workload": "metric_kernels", "launches": n, "lm_rows": B * L, "lm_labelled_rows": labelled,
            "lm_argmax_ms": round(ms_lm, 4), "lm_argmax_GBps": round(lm_bytes / ms_lm / 1e6, 1),
            "obj_splits_ms": round(ms_obj, 4), "pretrain_eval_step_kernels_ms": round(ms_all, 4), "card": card()}


def ref_metrics_with_syncs(d):
    """evaluator/pretrain_eval.py:21-67: the same tensor operations and `.item()` reads (post and raw logits)."""
    m = {}
    tok = d["masked_lm_labels"] != -1
    m["og_acc"] = (torch.argmax(d["og3d_logits"], -1) == d["tgt_object_id"].squeeze(1)).sum().item() / \
        float(len(d["tgt_object_id"]))
    m["lang_cls_acc_mask"] = torch.sum(torch.argmax(d["txt_lm_cls_logits"], 2)[tok] == d["masked_lm_labels"][tok]).item() / \
        float(tok.sum().item() + 1e-8)
    om, sem = d["obj_masks"], d["obj_sem_masks"]
    for k, splits in (("obj_cls_post_logits", (om, om * sem, om * sem.logical_not())), ("obj_cls_raw_logits", (om,))):
        for mm in splits:
            m[k + str(len(m))] = torch.sum(torch.argmax(d[k], 2)[mm] == d["obj_labels"][mm]).item() / \
                float(mm.sum().item() + 1e-8)
    return m


def time_reference_pattern(cfg, batch, args):
    from sceneverse_b200 import train
    st = train.PretrainStep(cfg, "cuda", seed=0)
    for _ in range(3):
        st.step(dict(batch))
    steps = max(args.steps // 2, 5)
    ms_eager = events_ms(lambda i: st.step(dict(batch)), steps)

    def with_metrics(i):
        d = dict(batch)
        st.step(d)                   # the eager step fills d with the model's outputs
        ref_metrics_with_syncs(d)
    ms_ref = events_ms(with_metrics, steps)
    return {"workload": "gps_pretrain_eager_reference_metrics", "eager_step_ms": round(ms_eager, 3),
            "eager_step_plus_reference_batch_metrics_ms": round(ms_ref, 3), "steps": steps, "card": card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--read-every", type=int, default=50)
    ap.add_argument("--kernel-launches", type=int, default=200)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_train_logs.py measures on a GPU; none is visible")
    from sceneverse_b200 import evaluate, model as M, weights
    tf = weights.synthetic_tensor("text_features", (607, 768))
    rows = [time_kernels(args)]
    print(json.dumps(rows[-1]), flush=True)
    gps = gps_batch()
    rows.append(time_steps("gps_pretrain", M.pretrain_config(text_features=tf), gps, evaluate.PretrainEval, args))
    print(json.dumps(rows[-1]), flush=True)
    gc.collect()
    torch.cuda.empty_cache()
    rows.append(time_steps("scanrefer", M.scanrefer_config(text_features=tf), scanrefer_batch(), evaluate.ScanReferEval, args))
    print(json.dumps(rows[-1]), flush=True)
    gc.collect()
    torch.cuda.empty_cache()
    rows.append(time_reference_pattern(M.pretrain_config(text_features=tf), gps, args))
    print(json.dumps(rows[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
