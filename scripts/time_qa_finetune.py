"""ms/step and scenes/s of the ScanQA and SQA3D fine-tune steps (model.scanqa_config / sqa3d_config) on one GPU, CUDA-graph
mode, B scenes of O object slots x 1024 points and L text tokens per step, inputs resident on the device:

    python scripts/time_qa_finetune.py [--steps K] [--warmup W] [--batch 32] [--profile] [--out FILE]

Prints one JSON line per config with the native kernel launches replayed per step, the card's name and its power limit.
--profile instead runs the QA head and its losses alone (forward + backward, bf16 autocast, training mode) under
torch.profiler and lists every CUDA kernel by name and by whether it comes from the project's libraries."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def batch(config, B, O, L, seed):
    from sceneverse_b200 import synthetic
    task, A = ("ScanQA", 8864) if config == "scanqa" else ("SQA3D", 706)
    d = synthetic.qa_batch(seed, task, B=B, O=O, P=1024, L=L, Ls=8, num_answers=A)
    d.pop("scene_txt_ids"), d.pop("scene_txt_masks")       # no scene captions in the QA configs
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def time_config(config, args):
    from sceneverse_b200 import model as M, train, weights
    tf = weights.synthetic_tensor("text_features", (607, 768))
    cfg = (M.scanqa_config if config == "scanqa" else M.sqa3d_config)(1, text_features=tf)
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=1, cuda_graph=True)
    data = batch(config, args.batch, args.objects, args.tokens, 42)
    for _ in range(args.warmup):
        ps.step(data)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.steps):
        loss = ps.step(data)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.steps
    res = {"config": config, "ms_per_step": round(ms, 3), "scenes_per_s": round(args.batch * 1e3 / ms, 1),
           "batch": args.batch, "objects": args.objects, "tokens": args.tokens, "steps": args.steps,
           "native_launches_per_step": int(ps.native_launches_per_step), "loss": float(loss), "card": card()}
    ps.close()
    return res


def profile(args):
    """Kernels of the QA head + answer_loss + ScanQA TextObjWithinBatch alone, forward and backward."""
    from torch.profiler import ProfilerActivity, profile as prof
    from sceneverse_b200 import ops, weights
    from sceneverse_b200.modules import heads, losses
    out = {}
    for config in ("scanqa", "sqa3d"):
        A = 8864 if config == "scanqa" else 706
        head = heads.QAHeadV1(None, num_answers=A)
        head.load_state_dict(weights.synthetic_state_dict(head, seed=11))
        head = head.cuda().train()
        loss = losses.Loss(["answer_loss"] + (["TextObjWithinBatch"] if config == "scanqa" else []),
                           task="ScanQA" if config == "scanqa" else "SQA3D")
        d = batch(config, args.batch, args.objects, args.tokens, 7)
        g = torch.Generator(device="cuda").manual_seed(0)
        obj = torch.randn(args.batch, args.objects, 768, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
        txt = torch.randn(args.batch, args.tokens, 768, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)

        def run():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                dd = dict(d, answer_scores=head(obj, d["obj_masks"], txt, d["txt_masks"]), intra_obj_embeds=obj,
                          intra_text_embed=txt[:, 0])
                total, _ = loss(dd)
            total.backward()
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            run()
            torch.cuda.synchronize()
        names = {}
        for e in p.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and e.name and not e.name.startswith(("Memcpy", "Memset")):
                names[e.name] = names.get(e.name, 0) + 1
        vendor = ("at::", "cutlass", "cublas", "xmma", "nvjet", "gemv", "splitK", "cudnn")     # ATen / cuBLAS kernel names
        aten = {k: v for k, v in names.items() if any(s in k for s in vendor)}
        native = {k: v for k, v in names.items() if k not in aten}
        out[config] = {"native_kernels": native, "aten_kernels": aten, "n_native": sum(native.values()),
                       "n_aten": sum(aten.values())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--objects", type=int, default=80)
    ap.add_argument("--tokens", type=int, default=50)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_qa_finetune.py needs a CUDA device")
    torch.cuda.set_device(0)
    results = [profile(args)] if args.profile else [time_config(c, args) for c in ("scanqa", "sqa3d")]
    for r in results:
        print(json.dumps(r))
    if args.out:
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
