"""Cost of the reference's auxiliary object-classification losses (optim/loss/loss.py:26-47, 64-94) on one GPU:

    python scripts/time_aux_losses.py [--steps K] [--rounds N] [--warmup W] [--batch 64] [--out FILE]

* ScanRefer step (model.scanrefer_config, B scenes x 80 objects x 1024 points, bf16, one CUDA graph), `og3d_loss` alone
  against `og3d_loss + obj_cls_raw_loss + obj_cls_pre_loss + obj_cls_post_loss`;
* GPS pre-training step (model.pretrain_config) with and without `obj_cls_post_loss{,_mask,_unmask}`;
  the two variants of each step are built in one process and timed in alternating rounds (median reported), with their
  native launches per step and the peak device memory each added;
* the masked cross-entropy alone over a (5120, 608) bf16 tensor (607 classes in padded rows), CUDA events: the native kernel,
  the native op forward + backward (kernel + in-place scale), and the reference's torch expression (permute, cross-entropy
  with reduction='none', mask, sum, divide, backward), with the kernel's achieved bytes/s against the H100 SXM data-sheet
  3.35 TB/s.
Prints one JSON line per measurement with the card's name and power limit."""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
AUX_REFER = ["og3d_loss", "obj_cls_raw_loss", "obj_cls_pre_loss", "obj_cls_post_loss"]
AUX_PRETRAIN = ["obj_cls_post_loss", "obj_cls_post_loss_mask", "obj_cls_post_loss_unmask"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def batch(B, seed):
    from sceneverse_b200 import synthetic
    d = synthetic.scene_batch(seed, B=B, O=80, P=1024, L=50, Ls=300)
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def make_step(config, losses):
    from sceneverse_b200 import model as M, train, weights
    tf = weights.synthetic_tensor("text_features", (607, 768))
    cfg = getattr(M, config)(1, text_features=tf)
    cfg["model"]["loss_list"] = cfg["model"]["vis_loss_list"] = list(losses)
    return train.PretrainStep(cfg, "cuda", dtype=torch.bfloat16, seed=1, cuda_graph=True)


def time_steps(ps, data, steps):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        ps.step(data)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def compare_steps(name, config, variants, args):
    """Both variants of one step, built one after the other in this process, timed in alternating rounds."""
    data = batch(args.batch, 42)
    if config == "scanrefer_config":
        data = {k: v for k, v in data.items() if not k.startswith("scene_txt")}
    built, peak = {}, {}
    for label, losses in variants.items():
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        ps = make_step(config, losses)
        for _ in range(args.warmup):
            ps.step(data)
        torch.cuda.synchronize()
        built[label] = ps
        peak[label] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    times = {label: [] for label in variants}
    for _ in range(args.rounds):
        for label, ps in built.items():
            times[label].append(time_steps(ps, data, args.steps))
    out = []
    for label, ps in built.items():
        ms = statistics.median(times[label])
        out.append({"measure": name, "variant": label, "losses": variants[label], "ms_per_step": round(ms, 3),
                    "ms_rounds": [round(t, 3) for t in times[label]], "scenes_per_s": round(args.batch * 1e3 / ms, 1),
                    "batch": args.batch, "native_launches_per_step": int(ps.native_launches_per_step),
                    "peak_mem_gib_added": round(peak[label], 2), "card": card()})
        ps.close()
    built.clear()
    gc.collect()
    torch.cuda.empty_cache()
    return out


def time_kernel(args):
    from sceneverse_b200 import _lib, ops
    dev = torch.device("cuda", 0)
    R, V, W = 5120, 607, 608
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.zeros(R, W, device=dev)
    x[:, :V] = torch.randn(R, V, device=dev, generator=g) * 3
    x = x.to(torch.bfloat16).view(64, 80, W)
    obj = torch.rand(64, 80, device=dev, generator=g) < 0.7
    sem = obj & (torch.rand(64, 80, device=dev, generator=g) > 0.25)
    y = torch.randint(0, V, (64, 80), device=dev, generator=g).masked_fill(~obj, -100)
    rows, sums, out = torch.empty(R, device=dev), torch.empty(2, device=dev), torch.empty((), device=dev)
    grad = torch.empty(R, W, dtype=torch.bfloat16, device=dev)
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    lib = _lib.gps()
    stream = torch.cuda.current_stream().cuda_stream
    obj_u8, sem_u8 = obj.view(torch.uint8), sem.view(torch.uint8)

    def kernel():
        st = lib.sv_masked_cross_entropy_fwd_bwd(x.data_ptr(), W, 1, y.data_ptr(), obj_u8.data_ptr(), sem_u8.data_ptr(), 0, R,
                                                 V, rows.data_ptr(), sums.data_ptr(), out.data_ptr(), counter.data_ptr(),
                                                 grad.data_ptr(), W, stream)
        _lib.check(lib, st, "sv_masked_cross_entropy_fwd_bwd")

    leaf = x.clone().requires_grad_(True)

    def native_op():
        view = leaf[..., :V]
        view._sv_padded = leaf
        leaf.grad = None
        ops.masked_cross_entropy(view, y, obj).backward()

    xt = x[..., :V].clone().requires_grad_(True)

    def reference():
        xt.grad = None
        loss = (F.cross_entropy(xt.permute(0, 2, 1), y, reduction='none') * obj).sum() / obj.sum()
        loss.backward()

    def timed(fn, n):
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(n):
            fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / n * 1e3          # microseconds

    n = args.kernel_iters
    res = {"measure": "masked_ce_kernel", "rows": R, "classes": V, "row_width": W, "dtype": "bf16",
           "live_rows": int(obj.sum())}
    res["us_kernel"] = round(timed(kernel, n), 2)
    res["us_native_fwd_bwd"] = round(timed(native_op, n), 2)
    res["us_torch_reference_fwd_bwd"] = round(timed(reference, n), 2)
    # logits read and gradient written in full (rows of weight 0 are not read, so this is an upper bound on what is read),
    # labels, the two mask bytes, and the per-row losses written and read back by the last CTA
    nbytes = R * W * 2 * 2 + R * 8 + R * 2 + R * 4 * 2
    res["bytes"] = nbytes
    res["kernel_tb_per_s"] = round(nbytes / (res["us_kernel"] * 1e-6) / 1e12, 3)
    res["kernel_fraction_of_3_35_tb_s"] = round(nbytes / (res["us_kernel"] * 1e-6) / HBM_BYTES_PER_S, 3)
    res["card"] = card()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--kernel-iters", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_aux_losses.py needs a CUDA device")
    torch.cuda.set_device(0)
    from sceneverse_b200 import model as M
    results = [time_kernel(args)]
    print(json.dumps(results[-1]), flush=True)
    for r in compare_steps("scanrefer_step", "scanrefer_config", {"og3d_loss": ["og3d_loss"], "og3d+aux": AUX_REFER}, args):
        results.append(r)
        print(json.dumps(r), flush=True)
    base = M.pretrain_config(1)["model"]["loss_list"]
    for r in compare_steps("pretrain_step", "pretrain_config", {"shipped": base, "shipped+obj_cls_post": base + AUX_PRETRAIN},
                           args):
        results.append(r)
        print(json.dumps(r), flush=True)
    if args.out:
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
