"""Times every GEMM shape of the GPS pre-training step (64 scenes: BERT at 300 and 50 tokens, the joint / spatial layers, the
LM head) in all three directions on the native kernel family, with the epilogues the step uses, and prints TFLOP/s against
the dense bf16 data-sheet peak (989 TFLOP/s, H100 SXM at 700 W).

    python scripts/time_gemm_shapes.py [--iters 20] [--force 0|1|2|4] [--out FILE]

Per shape and direction: the time with the epilogue (CUDA events over --iters launches after warm-up), the time with the
epilogue body switched off (sv_gemm_force_ctas bit 8: the difference is the part of the epilogue the MMAs do not hide)."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

PEAK = 989e12
# (name, M tokens, N out, K in, activation of this layer, activation whose derivative the dgrad epilogue applies)
SHAPES = [
    ("bert300.qkv", 19200, 2304, 768, None, None), ("bert300.out", 19200, 768, 768, None, None),
    ("bert300.ffn1", 19200, 3072, 768, "gelu", None), ("bert300.ffn2", 19200, 768, 3072, None, "gelu"),
    ("joint130.qkv", 8320, 2304, 768, None, None), ("joint130.ffn1", 8320, 2048, 768, "relu", None),
    ("joint130.ffn2", 8320, 768, 2048, None, "relu"),
    ("spatial80.qkv", 5120, 2304, 768, None, None), ("spatial80.ffn1", 5120, 2048, 768, "relu", None),
    ("spatial80.ffn2", 5120, 768, 2048, None, "relu"),
    ("bert50.qkv", 3200, 2304, 768, None, None), ("bert50.ffn1", 3200, 3072, 768, "gelu", None),
    ("bert50.ffn2", 3200, 768, 3072, None, "gelu"), ("lm_head", 3200, 30528, 768, None, None),
]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - informational only
        q = f"nvidia-smi unavailable ({e})"
    return q


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--force", type=int, default=0, help="tile width: 0 heuristic, 1 / 2 / 4 = 64 / 128 / 192 columns")
    ap.add_argument("--out", default=None, help="also write the table as JSON")
    args = ap.parse_args()
    from sceneverse_b200 import native
    assert torch.cuda.is_available(), "time_gemm_shapes.py measures on the GPU; there is no CPU path"
    dev = torch.device("cuda", 0)
    print("card:", card(), flush=True)
    rows = []
    g = torch.Generator(device=dev).manual_seed(1234)

    def rnd(*s, scale=0.5):
        return (torch.randn(*s, device=dev, generator=g) * scale).bfloat16()

    for name, M, N, K, act, dact in SHAPES:
        x, w, b = rnd(M, K), rnd(N, K, scale=K ** -0.5), torch.randn(N, device=dev, generator=g)
        gy, aux = rnd(M, N), rnd(M, K, scale=1.5)
        dw, db = torch.zeros(N, K, device=dev), torch.zeros(N, device=dev)
        flop = 2.0 * M * N * K
        fns = {
            "fwd": lambda: native.linear_fwd(x, w, b, act, want_pre=act == "gelu"),
            "dgrad": lambda: native.linear_dgrad(gy, w, act=dact, aux=aux if dact else None),
            "wgrad": lambda: native.linear_wgrad(gy, x, dw=dw, db=db, accumulate=True),
        }
        for d, fn in fns.items():
            native.gemm_force_ctas(args.force)
            ms = timed(fn, args.iters)
            native.gemm_force_ctas(args.force | (1 << 8))
            ms_noepi = timed(fn, args.iters)
            native.gemm_force_ctas(args.force)
            r = {"shape": name, "dir": d, "M": M, "N": N, "K": K, "ms": round(ms, 4), "tflops": round(flop / ms / 1e9, 1),
                 "pct_peak": round(100 * flop / ms / 1e9 / (PEAK / 1e12), 1), "ms_no_epilogue": round(ms_noepi, 4),
                 "exposed_epilogue_pct": round(100 * (ms - ms_noepi) / ms, 1)}
            rows.append(r)
            print(f"{name:15s} {d:5s} {M:6d} x {N:5d} x {K:5d}  {ms:8.4f} ms  {r['tflops']:6.1f} TFLOP/s ({r['pct_peak']:5.1f} %)"
                  f"  no-epilogue {ms_noepi:8.4f} ms (exposed {r['exposed_epilogue_pct']:5.1f} %)", flush=True)
    native.gemm_force_ctas(0)
    tot = sum(r["ms"] for r in rows)
    print(f"sum over shapes (one launch each): {tot:.3f} ms")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card(), "force": args.force, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
