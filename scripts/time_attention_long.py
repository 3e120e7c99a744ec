"""Timing of the long attention entries (sv_attention_fwd_long_bf16 / sv_attention_bwd_long_bf16) above 384 tokens.

For plain, gated (one gate per head) and dropout attention at L = Lq = Lk in {385, 512, 1024, 2048}, head dim 64, 12
heads, and B scenes chosen so that every launch has at least 4096 CTAs (about 10 waves of 3 CTAs on 132 SMs): CUDA-event
time of 100 launches after 10 warm-up launches, forward and backward separately, and the rate from the FLOP model below
against the H100 SXM data-sheet peak of 989 dense BF16 TFLOP/s.  Then L = 384 on the resident forward entry against the
long one, alternated in the same process.  The card's name, power limit and maximum SM clock are read in the same run.

FLOP model (tensor-core work the algorithm needs; the kernels' recomputation is not counted):
  forward  4 B H Lq Lk 64   (S = Q K^T and O = P V: 2 Lq Lk 64 each)
  backward 10 B H Lq Lk 64  (S recomputed, dP = dO V^T, dV = P^T dO, dQ = dS K, dK = dS^T Q: 2 Lq Lk 64 each)

Needs a CUDA device: without one it exits with an error, it never times anything else.
    python scripts/time_attention_long.py [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

PEAK_TFLOPS = 989.0     # H100 SXM, dense BF16, data sheet (700 W card)
H, E = 12, 768
LENGTHS = (385, 512, 1024, 2048)
WARMUP, ITERS = 10, 100


def fwd_flops(B, L):
    return 4 * B * H * L * L * 64


def bwd_flops(B, L):
    return 10 * B * H * L * L * 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def time_ms(fn):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(ITERS):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / ITERS


def case(variant, L, g):
    from sceneverse_b200 import native
    B = max(1, -(-4096 // (H * ((L + 63) // 64))))
    q, k, v, go = (torch.randn(B, L, E, device="cuda", generator=g).bfloat16() for _ in range(4))
    mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    mask[1::2, (3 * L) // 4:] = True            # every other scene pads its last quarter
    kw = dict(key_padding_mask=mask, long=True)
    if variant == "gated":
        # uniform pairwise geometry in [-1, 1): sv_pairwise_locs_f32 stops at 1024 objects, the kernels do not
        kw.update(spatial_w=torch.randn(B, L, H * 6, device="cuda", generator=g), spatial_heads=H,
                  pairwise_locs=torch.rand(B, L, L, 5, device="cuda", generator=g) * 2 - 1)
    p = 0.1 if variant == "dropout" else 0.0
    out, lse = native.attention(q, k, v, H, return_lse=True, dropout_p=p, seed=7, **kw)
    bkw = {n: kw[n] for n in ("key_padding_mask", "long")}
    if variant == "gated":
        bkw.update(spatial_w=kw["spatial_w"], pairwise_locs=kw["pairwise_locs"])
    f = time_ms(lambda: native.attention(q, k, v, H, return_lse=True, dropout_p=p, seed=7, **kw))
    bw = time_ms(lambda: native.attention_backward(q, k, v, out, go, lse, H, dropout_p=p, seed=7, **bkw))
    ff, bf = fwd_flops(B, L) / f / 1e9, bwd_flops(B, L) / bw / 1e9
    return {"variant": variant, "L": L, "B": B, "H": H, "ctas": B * H * ((L + 63) // 64),
            "fwd_ms": round(f, 4), "fwd_tflops": round(ff, 1), "fwd_peak_share": round(ff / PEAK_TFLOPS, 3),
            "bwd_ms": round(bw, 4), "bwd_tflops": round(bf, 1), "bwd_peak_share": round(bf / PEAK_TFLOPS, 3)}


def resident_vs_long(g, rounds=5):
    """L = 384 plain forward, resident entry against long entry, alternated; per-round times and medians."""
    from sceneverse_b200 import native
    L = 384
    B = -(-4096 // (H * 6))
    q, k, v = (torch.randn(B, L, E, device="cuda", generator=g).bfloat16() for _ in range(3))
    res = {"resident_ms": [], "long_ms": []}
    for _ in range(rounds):
        res["resident_ms"].append(round(time_ms(lambda: native.attention(q, k, v, H, long=False)), 4))
        res["long_ms"].append(round(time_ms(lambda: native.attention(q, k, v, H, long=True)), 4))
    med = {n: sorted(t)[len(t) // 2] for n, t in res.items()}
    return {"L": L, "B": B, "H": H, **res, "resident_median_ms": med["resident_ms"], "long_median_ms": med["long_ms"],
            "fwd_tflops_resident": round(fwd_flops(B, L) / med["resident_ms"] / 1e9, 1),
            "fwd_tflops_long": round(fwd_flops(B, L) / med["long_ms"] / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_attention_long.py needs a CUDA device; nothing was measured")
    torch.cuda.set_device(0)
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card(), "flop_model": {"forward": "4 B H Lq Lk 64", "backward": "10 B H Lq Lk 64"},
           "peak_tflops": PEAK_TFLOPS, "cases": []}
    for variant in ("plain", "gated", "dropout"):
        for L in LENGTHS:
            r = case(variant, L, g)
            print(json.dumps(r), flush=True)
            res["cases"].append(r)
    res["resident_vs_long_384"] = resident_vs_long(g)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
