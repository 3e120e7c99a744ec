"""Cost of a checkpoint of the GPS pre-training step on one GPU, in one process.

    python scripts/time_checkpoint.py [--steps K] [--windows N] [--out FILE]

GPS step at the bench shape (64 scenes x 80 objects x 1024 points, bf16, one CUDA graph), one resident batch:
* the step time before the save: N windows of K replays (CUDA events around each window);
* `save_state` and `load_state` wall time (host clock, the device synchronised before and after) and the size of each
  file written; the directory is a temporary one;
* the step time of the replays right after the load into the same, already captured step (in place), N windows of K.
Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def windows(ps, batch, steps, n):
    out = []
    for _ in range(n):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        for _ in range(steps):
            ps.step(batch)
        t1.record()
        torch.cuda.synchronize()
        out.append(round(t0.elapsed_time(t1) / steps, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_checkpoint.py needs a CUDA device")
    import bench
    from sceneverse_b200 import model as M, train, weights
    d = bench.make_scene_batches(1, bench.SCENES, 0)[0]
    batch = {k: torch.from_numpy(np.asarray(v)).cuda() for k, v in d.items()}
    cfg = M.pretrain_config(1, text_features=weights.synthetic_tensor("text_features", (607, 768)))
    ps = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=0, cuda_graph=True)
    for _ in range(3):                      # set-up, capture and warm-up replays
        ps.step(batch)
    before = windows(ps, batch, args.steps, args.windows)
    with tempfile.TemporaryDirectory() as tmp:
        torch.cuda.synchronize()
        t = time.perf_counter()
        ps.save_state(tmp)
        torch.cuda.synchronize()
        save_s = time.perf_counter() - t
        sizes = {f: os.path.getsize(os.path.join(tmp, f)) for f in sorted(os.listdir(tmp))}
        t = time.perf_counter()
        ps.load_state(tmp)
        torch.cuda.synchronize()
        load_s = time.perf_counter() - t
    after = windows(ps, batch, args.steps, args.windows)
    row = {"workload": "gps_pretrain_checkpoint", "shape": f"{bench.SCENES}x{bench.OBJS}x{bench.PTS} bf16 graph",
           "card": card(), "save_state_s": round(save_s, 3), "load_state_s": round(load_s, 3),
           "bytes": sizes, "total_mb": round(sum(sizes.values()) / 2 ** 20, 1),
           "ms_per_step_before_save": before, "ms_per_step_after_load": after,
           "median_before": float(np.median(before)), "median_after": float(np.median(after)),
           "native_launches_per_step": int(ps.native_launches_per_step)}
    line = json.dumps(row)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    ps.close()


if __name__ == "__main__":
    main()
