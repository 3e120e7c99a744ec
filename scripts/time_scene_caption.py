"""Scene-caption encoder of the GPS pre-training step, full last layer against the CLS-only last layer, in one process.

The step reads only row 0 of each caption's last hidden state (`scene_text_embed`).  This times BERT-4L in training mode
(dropout on, bf16 autocast, eager) on 64 synthetic captions of 300 tokens (lengths 8..300, synthetic.scene_batch) through
`BERTLanguageEncoder(ids, masks)[:, 0]` and `BERTLanguageEncoder(ids, masks, cls_only=True)`: forward and backward
separately, CUDA events over many calls, the two arms alternated.  The calls are eager, so the event times include the
host's launch overhead, which at this size hides the difference.  Then one torch.profiler pass per arm sums device time
per kernel name (`kernel_ms_total`, `kernel_ms_removed`): that is the work the CLS-only layer removed, launch by launch.

    python scripts/time_scene_caption.py [--iters 30] [--rounds 3] [--out DIR]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from sceneverse_b200 import model as M, synthetic  # noqa: E402
from sceneverse_b200.modules.layers import route_linears  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to DIR/time_scene_caption.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_scene_caption.py needs a CUDA device")
    torch.manual_seed(0)
    enc = route_linears(M.BERTLanguageEncoder(None)).cuda().train()
    d = synthetic.scene_batch(0, B=64, O=8, P=16, L=8, Ls=300)
    ids, masks = (torch.from_numpy(d[k]).cuda() for k in ("scene_txt_ids", "scene_txt_masks"))
    proj = torch.randn(64, 768, device="cuda")
    arms = {"full": lambda: enc(ids, masks)[:, 0], "cls_only": lambda: enc(ids, masks, cls_only=True)}

    def fwd(arm):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return arms[arm]()

    def bwd(emb):
        (emb.float() * proj).sum().backward()

    def timed(arm):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3 * args.iters)]
        f = b = 0.0
        for i in range(args.iters):
            e0, e1, e2 = ev[3 * i:3 * i + 3]
            e0.record()
            emb = fwd(arm)
            e1.record()
            bwd(emb)
            e2.record()
            enc.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        for i in range(args.iters):
            e0, e1, e2 = ev[3 * i:3 * i + 3]
            f += e0.elapsed_time(e1)
            b += e1.elapsed_time(e2)
        return f / args.iters, b / args.iters

    for arm in arms:          # warm-up: modules, GEMM configurations, allocator
        for _ in range(3):
            bwd(fwd(arm))
            enc.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    res = {"gpu": torch.cuda.get_device_name(), "captions": 64, "tokens": 300,
           "lengths": [int(masks.sum(1).min()), int(masks.sum(1).max())], "iters": args.iters}
    for r in range(args.rounds):
        for arm in arms:
            f, b = timed(arm)
            res.setdefault(f"{arm}_fwd_ms", []).append(round(f, 4))
            res.setdefault(f"{arm}_bwd_ms", []).append(round(b, 4))

    # device time per kernel name, one profiled forward + backward per arm (a separate pass: tracing slows the host)
    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    for arm in arms:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                bwd(fwd(arm))
                enc.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
        kernels[arm] = {e.key: [e.count, e.device_time_total / 5e3]      # ms per forward + backward
                        for e in prof.key_averages() if e.device_time_total > 0}
    names = set(kernels["full"]) | set(kernels["cls_only"])
    rows = sorted(((kernels["full"].get(n, [0, 0.0])[1] - kernels["cls_only"].get(n, [0, 0.0])[1], n) for n in names),
                  reverse=True)
    res["kernel_ms_removed"] = [
        {"kernel": n[:90], "full_ms": round(kernels["full"].get(n, [0, 0.0])[1], 4),
         "cls_only_ms": round(kernels["cls_only"].get(n, [0, 0.0])[1], 4),
         "launches_full": kernels["full"].get(n, [0])[0] // 5, "launches_cls_only": kernels["cls_only"].get(n, [0])[0] // 5}
        for delta, n in rows if abs(delta) >= 0.005]
    res["kernel_ms_total"] = {arm: round(sum(v[1] for v in kernels[arm].values()), 4) for arm in arms}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_scene_caption.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
