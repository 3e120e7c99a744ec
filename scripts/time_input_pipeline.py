"""Times the device-side object processing of one GPS batch: 64 scenes x 80 object slots x 1024 points, seeded raw counts
of 500-6000 points per object.

    python scripts/time_input_pipeline.py [--iters 100] [--warmup 10]

Paths: `prepare_objects` (the plain post path), the aug path with the shipped `data_aug` block (scene z quarter turn), the aug
path with every option on, and the post path with the `rot_aug` quarter turn.  Each is timed with CUDA events over --iters
launches after --warmup, draw kernel included.  The bandwidth figure is a byte model against the 3.35 TB/s HBM3 data-sheet peak
of the H100 SXM: every raw row a path reads whole (24 B) + the P gathered rows + the P written rows of every slot."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

PEAK_BW = 3.35e12
SHIPPED = {"aug_list": ["scene_aug"],
           "scene_aug": {"translation": {"enabled": False, "value": [1.0, 1.0, 1.0], "p": 1.0},
                         "scaling": {"enabled": False, "p": 1.0, "value": [0.9, 1.1]}, "flip": {"enabled": False, "p": 0.5},
                         "rotation": {"enabled": True, "p": 1.0, "axis_align": True, "value": [0.0, 0.0, 1.0], "shuffle": True},
                         "color_jitter": False, "order_shuffle": False},
           "obj_aug": {"translation": {"enabled": False, "value": [0.1, 0.1, 0.1], "p": 1.0},
                       "rotation": {"enabled": False, "p": 1.0, "axis_align": False, "value": [0.0, 0.0, 0.1], "shuffle": True},
                       "random_jitter": {"enabled": False, "value": 0.01, "accord_to_size": False, "p": 1.0},
                       "pts_shuffle": True}}
ALL_ON = {"aug_list": ["scene_aug", "obj_aug"],
          "scene_aug": {"translation": {"enabled": True, "value": [0.5, 0.5, 0.2]}, "scaling": {"enabled": True, "value": [0.9, 1.1]},
                        "flip": {"enabled": True}, "rotation": {"enabled": True, "axis_align": True, "value": [0.0, 0.0, 1.0],
                                                                 "shuffle": True},
                        "color_jitter": True, "order_shuffle": True},
          "obj_aug": {"translation": {"enabled": True, "value": [0.1, 0.1, 0.1]},
                      "rotation": {"enabled": True, "axis_align": False, "value": [0.0, 0.0, 0.1], "shuffle": True},
                      "random_jitter": {"enabled": True, "value": 0.01}, "pts_shuffle": True}}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - informational only
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert args.iters >= 50
    from sceneverse_b200 import input_pipeline as ip
    B, O, P = 64, 80, 1024
    counts = np.random.default_rng(0).integers(500, 6001, size=B * O)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    raw = torch.randn(int(off[-1]), 6, generator=torch.Generator().manual_seed(0)).cuda()
    offc = torch.from_numpy(off).cuda()
    S, rows = B * O, int(off[-1])
    per_slot = S * P * 24 * 2   # gathered rows + written rows
    shipped, all_on, post_rot = ip.AugSpec.from_config(SHIPPED), ip.AugSpec.from_config(ALL_ON), ip.AugSpec.from_config(None, True)
    paths = [
        ("prepare_objects", lambda i: ip.prepare_objects(raw, offc, B, O, P, seed=i), rows * 24 + per_slot),
        ("aug shipped block", lambda i: ip.prepare_objects_aug(raw, offc, B, O, P, shipped, seed=i,
                                                               want_boxes=True), per_slot),
        ("aug every option", lambda i: ip.prepare_objects_aug(raw, offc, B, O, P, all_on, seed=i,
                                                              want_boxes=True), rows * 24 + per_slot),
        ("post rot_aug", lambda i: ip.prepare_objects_aug(raw, offc, B, O, P, post_rot, seed=i,
                                                          want_boxes=True), rows * 24 + per_slot),
    ]
    print(f"card: {card()}")
    print(f"batch: {B} scenes x {O} slots x {P} points, {rows} raw points ({rows * 24 / 1e6:.1f} MB)")
    for name, fn, nbytes in paths:
        for i in range(args.warmup):
            fn(i)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for i in range(args.iters):
            fn(i)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / args.iters
        print(f"{name:20s} {ms * 1e3:8.1f} us   {nbytes / 1e6:7.1f} MB modelled   {nbytes / (ms * 1e-3) / 1e12:5.2f} TB/s "
              f"({100 * nbytes / (ms * 1e-3) / PEAK_BW:4.1f} % of 3.35 TB/s)")


if __name__ == "__main__":
    main()
