"""GPS pre-training with the object encoder unfrozen (model.pretrain_unfreeze_config, all_pretrain_unfreeze.yaml) against the
frozen step of bench.py (model.pretrain_config), alternated in one process on one GPU:

* each round builds, captures, times and closes the frozen step, then the unfrozen one (one captured step alive at a time:
  a capture re-registers the process-wide bf16 weight shadows);
* per arm: ms per step (CUDA events over --steps replays, 3 input batches rotated as in bench.py), scenes/s, native launches
  per replay, peak device memory of the arm, the final loss;
* --profile DIR: afterwards, one eager unfrozen step under torch.profiler (CUDA activities), and the device time of every
  kernel summed by name into DIR/pretrain_unfreeze_kernels.json (the top 40 are printed).

    python scripts/time_pretrain_unfreeze.py [--steps K] [--rounds R] [--out FILE] [--profile DIR]

64 scenes x 80 object slots x 1024 points, 50 + 300 text tokens, bf16, synthetic weights and inputs resident on the device.
Prints one JSON line per measurement with the card's name and power limit."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default=None, metavar="DIR")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_pretrain_unfreeze.py measures on the GPU"
    import bench
    from sceneverse_b200 import model as M, train, weights
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
    batches = [{k: torch.from_numpy(v).cuda() for k, v in b.items()}
               for b in bench.make_scene_batches(3, bench.SCENES, 42)]
    cfgs = {"frozen": M.pretrain_config(1, text_features=tf), "unfrozen": M.pretrain_unfreeze_config(1, text_features=tf)}
    for r in range(a.rounds):
        for name, cfg in cfgs.items():
            torch.cuda.reset_peak_memory_stats()
            st = train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=1234, cuda_graph=True)
            for i in range(3):                  # probe, set-up steps, capture, first replays
                st.step(dict(batches[i % 3]))
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            for i in range(a.steps):
                loss = st.step(dict(batches[i % 3]))
            e.record()
            torch.cuda.synchronize()
            ms = s.elapsed_time(e) / a.steps
            emit({"what": "gps_pretrain_step", "arm": name, "round": r, "ms": round(ms, 3),
                  "scenes_per_s": round(bench.SCENES / ms * 1e3, 1), "native_launches_per_step": st.native_launches_per_step,
                  "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2), "loss": float(loss),
                  "scenes": bench.SCENES, "objects": bench.OBJS, "points": bench.PTS})
            st.close()
            del st, loss
            torch.cuda.empty_cache()
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        st = train.PretrainStep(cfgs["unfrozen"], "cuda", dtype=torch.bfloat16, seed=1234)
        for i in range(2):
            st.step(dict(batches[i]))
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            st.step(dict(batches[2]))
            torch.cuda.synchronize()
        per = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                n, t = per.get(ev.name, (0, 0.0))
                per[ev.name] = (n + 1, t + ev.device_time_total / 1e3)
        rows = sorted(({"kernel": k, "calls": n, "ms": round(t, 4)} for k, (n, t) in per.items()), key=lambda d: -d["ms"])
        os.makedirs(a.profile, exist_ok=True)
        with open(os.path.join(a.profile, "pretrain_unfreeze_kernels.json"), "w") as f:
            json.dump({"card": gpu, "step": "unfrozen, eager", "total_ms": round(sum(d["ms"] for d in rows), 3),
                       "kernels": rows}, f, indent=1)
        emit({"what": "profile_unfrozen_eager_step", "device_ms_total": round(sum(d["ms"] for d in rows), 3),
              "top": rows[:40]})
        st.close()


if __name__ == "__main__":
    main()
