"""ms/step and objects/s of train.ObjClsStep (config C2) at 64 objects x 1024 points per GPU, one process per GPU:

    python -m torch.distributed.run --nproc-per-node N scripts/time_objcls_dp.py [--generic] [--steps K] [--warmup W]

N = 1: plain BatchNorm2d on the native path (what bench.py --workload objcls runs).  N > 1: SyncBatchNorm; by default the
native statistics exchange with graph A | NCCL all-reduce | graph B, with --generic the torch SyncBatchNorm operator sequence
(fp32 cuDNN convolutions) under eager DDP, i.e. the path the model took before the native exchange existed.  Rank 0 prints one
JSON line with the nvidia-smi clock sample of the timed region, the card's name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--generic", action="store_true", help="N > 1: torch SyncBatchNorm on the generic path under DDP")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from bench import ClockSampler
    from sceneverse_b200 import pn_train, synthetic, train, weights
    if args.generic:
        pn_train.exchange_for = lambda net, device: False if any(
            isinstance(m, torch.nn.SyncBatchNorm) for m in net.modules()) else None
    tf = weights.synthetic_tensor("text_features", (607, 768))
    OBJ = 64
    batches = []
    for i in range(3):
        d = synthetic.scene_batch(42 + rank + 1000 * i, B=1, O=OBJ, P=1024, all_valid=True)
        batches.append({k: torch.from_numpy(d[k]).to(dev) for k in ("obj_fts", "obj_labels", "obj_masks")})
    step = train.ObjClsStep(dev, tf.to(dev), dtype=torch.bfloat16, seed=1234, cuda_graph=True, num_gpu=world)
    for i in range(args.warmup):
        step.step(dict(batches[i % 3]))
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(local) as cs:
        t0.record()
        for i in range(args.steps):
            loss = step.step(dict(batches[i % 3]))
        t1.record()
        torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.steps
    ms_t = torch.tensor([ms], device=dev)
    if world > 1:
        dist.all_reduce(ms_t, op=dist.ReduceOp.MAX)          # the step of the slowest rank
    if rank == 0:
        gpu = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        path = "plain BatchNorm2d, native" if world == 1 else ("torch SyncBatchNorm, generic, DDP" if args.generic else
                                                              "native SyncBatchNorm exchange, graph | all-reduce | graph")
        print(json.dumps({"metric": "ObjCls pre-train objects/sec (64 objects x 1024 points per GPU)", "world": world,
                          "path": path, "cuda_graph": bool(step.graph_mode), "ms_per_step": round(float(ms_t), 3),
                          "objects_per_s": round(OBJ * world * 1000.0 / float(ms_t), 1), "steps": args.steps,
                          "warmup": args.warmup, "loss": float(loss), "gpu": gpu, "clocks": cs.summary()}))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
