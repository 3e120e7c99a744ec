"""Per-scene grounding against per-utterance grounding on one GPU, alternated in one process:

* training: the per-scene pre-training step (OpenVocabPerScene, B = 4 scenes x U = 64 utterances, one CUDA graph) against the
  OpenVocab step on the same 256 utterances as 256 one-utterance scenes (each scene's objects repeated, same losses, no scene
  captions): ms per step, utterances/s, native launches per step;
* evaluation: the per-scene EvalRunner (16 scenes x 64 utterances, ScanReferEval) against the per-utterance runner on the same
  1,024 items (16 batches of 64);
* the U-sum kernel alone (the backward of ops.scene_broadcast at B = 4, U = 64, O = 80, D = 768, bf16): CUDA events, GB/s
  against the 3.35 TB/s of the H100 SXM data sheet.

    python scripts/time_per_scene.py [--steps K] [--rounds R] [--out FILE]

80 object slots x 1024 points, 50 text tokens, synthetic weights and inputs resident on the device.  Prints one JSON line per
measurement with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def per_scene_batch(seed, B, U):
    from sceneverse_b200 import synthetic
    d = synthetic.per_scene_batch(seed, B=B, U=U, O=80, P=1024, T=50)
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def as_utterances(b):
    """The same utterances as one-utterance scenes: every per-utterance key flattened, each scene's objects repeated."""
    B, U = b["txt_ids"].shape[:2]
    out = {}
    for k, v in b.items():
        if k.startswith("obj_"):
            out[k] = v.repeat_interleave(U, 0)
        elif k in ("tgt_object_id", "tgt_object_label"):
            out[k] = v.reshape(B * U, 1)
        else:
            out[k] = v.reshape(B * U, *v.shape[2:])
    return out


def time_steps(step, batch, k):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(k):
        step(batch)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_per_scene.py measures on the GPU"
    from sceneverse_b200 import evaluate, model as M, native, train, weights
    gpu = card()
    lines = []

    def emit(d):
        d["card"] = gpu
        print(json.dumps(d), flush=True)
        lines.append(d)
        if a.out:
            with open(a.out, "w") as f:
                json.dump(lines, f, indent=1)

    tf = weights.synthetic_tensor("text_features", (607, 768))
    B, U = 4, 64
    ps_cfg = M.per_scene_pretrain_config(1, text_features=tf)
    pu_cfg = M.pretrain_config(1, text_features=tf)
    pu_cfg["data"]["args"]["use_scene_cap"] = False
    pu_cfg["model"]["loss_list"] = pu_cfg["model"]["vis_loss_list"] = list(ps_cfg["model"]["loss_list"])
    # ---- the U-sum kernel ----------------------------------------------------------------------------------------------
    O, D = 80, 768
    g = torch.randn(B, U, O * D, device="cuda").to(torch.bfloat16)
    for _ in range(10):
        native.colsum_batched(g)
    n = 200
    for r in range(a.rounds):
        us = time_steps(lambda x: native.colsum_batched(x), g, n) * 1e3
        nbytes = (B * U * O * D + B * O * D) * 2
        emit({"what": "usum_kernel", "round": r, "B": B, "U": U, "O": O, "D": D, "dtype": "bf16", "us": round(us, 2),
              "GB_per_s": round(nbytes / us * 1e-3, 1), "share_of_3.35TB_per_s": round(nbytes / us * 1e6 / HBM_BYTES_PER_S, 3)})
    # ---- evaluation ----------------------------------------------------------------------------------------------------
    S, n_items = 16, 16 * 64
    scene = per_scene_batch(2, S, U)
    utter = as_utterances(scene)
    ps = train.PretrainStep(ps_cfg, "cuda", seed=0)
    pu = train.PretrainStep(pu_cfg, "cuda", seed=0)
    pu.module.model.load_state_dict(ps.module.model.state_dict())
    runners = {"per_scene": (evaluate.EvalRunner(ps, [evaluate.ScanReferEval()], batch_size=S), [scene]),
               "per_utterance": (evaluate.EvalRunner(pu, [evaluate.ScanReferEval()], batch_size=64),
                                 [{k: v[i:i + 64] for k, v in utter.items()} for i in range(0, n_items, 64)])}
    for runner, bs in runners.values():
        runner.run(bs)                          # capture
    for r in range(a.rounds):
        for name, (runner, bs) in runners.items():
            ms = time_steps(lambda _: runner.run(bs), None, a.steps)
            emit({"what": "eval", "path": name, "round": r, "ms_per_1024_utterances": round(ms, 3),
                  "utterances_per_s": round(n_items / ms * 1e3, 1),
                  "og_acc_iou25": runner.evaluators[0].eval_dict.get("og_acc_iou25")})
    ps.close()
    pu.close()
    del runners, scene, utter
    torch.cuda.empty_cache()
    # ---- training ------------------------------------------------------------------------------------------------------
    scene = per_scene_batch(1, B, U)
    batches = {"per_scene": scene, "per_utterance": as_utterances(scene)}
    cfgs = {"per_scene": ps_cfg, "per_utterance": pu_cfg}
    # one captured step alive at a time: a capture re-registers the process-wide bf16 weight shadows, so a second captured
    # step would free memory the first one's graph still reads; each round builds, captures, times and closes each path
    for r in range(a.rounds):
        for name in ("per_scene", "per_utterance"):
            st = train.PretrainStep(cfgs[name], "cuda", seed=0, cuda_graph=True)
            st.step(batches[name])              # probe, set-up steps, capture, first replay
            st.step(batches[name])
            ms = time_steps(st.step, batches[name], a.steps)
            emit({"what": "train_step", "path": name, "round": r, "ms": round(ms, 3), "utterances": B * U,
                  "utterances_per_s": round(B * U / ms * 1e3, 1), "native_launches_per_step": st.native_launches_per_step,
                  "loss": float(st.static_loss)})
            st.close()
            del st
            torch.cuda.empty_cache()
    del batches


if __name__ == "__main__":
    main()
