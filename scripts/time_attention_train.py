"""Forward+backward timing of the native attention kernels at the GPS training shapes (B = 64 scenes): the four attention
configurations of the pre-training step (each runs in four layers), then plain shapes against SDPA."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from sceneverse_b200 import native, ops
B, H, E = 64, 12, 768
quick = len(sys.argv) > 1 and sys.argv[1] == "quick"
def t(fn, n=20):
    if quick:
        fn(); torch.cuda.synchronize(); return 0.0
    for _ in range(3): fn()
    torch.cuda.synchronize(); a=torch.cuda.Event(True); c=torch.cuda.Event(True); a.record()
    for _ in range(n): fn()
    c.record(); torch.cuda.synchronize(); return a.elapsed_time(c)/n
g = torch.Generator(device="cuda").manual_seed(0)
def rnd(*s): return torch.randn(*s, device="cuda", generator=g)
res = {}
# (name, L, key-padding mask, spatial gate, dropout): BERT over scene captions and over utterances, the joint
# object-language self-attention, the gated spatial self-attention of the object encoder
STEP = [("bert300", 300, True, False, 0.1), ("bert50", 50, True, False, 0.1), ("joint130", 130, False, False, 0.1),
        ("spatial80", 80, True, True, 0.0)]
for name, L, masked, gated, p in STEP:
    q, k, v, go = (rnd(B, L, E).bfloat16() for _ in range(4))
    kw = {}
    if masked:
        lens = torch.randint(1, L + 1, (B,), device="cuda", generator=g)
        kw["key_padding_mask"] = torch.arange(L, device="cuda")[None] >= lens[:, None]
    bkw = dict(kw, dropout_p=p, seed=5)
    if gated:
        bkw.update(spatial_w=rnd(B, L, H * 6), pairwise_locs=ops.calc_pairwise_locs(rnd(B, L, 3), None))
    fkw = dict(bkw, spatial_heads=H) if gated else bkw
    res[f"{name}_fwd"] = t(lambda: native.attention(q, k, v, H, return_lse=True, **fkw), n=100)
    out, lse = native.attention(q, k, v, H, return_lse=True, **fkw)
    res[f"{name}_bwd"] = t(lambda: native.attention_backward(q, k, v, out, go, lse, H, **bkw), n=100)
# block skipping (csrc/attn_common.cuh) at the scene-caption shape: captions of 8..300 tokens, the length distribution of
# synthetic.scene_batch, with every fully masked key block skipped (default) against every block visited; alternated
q, k, v, go = (rnd(B, 300, E).bfloat16() for _ in range(4))
lens = torch.randint(8, 301, (B,), device="cuda", generator=g)
cap = dict(key_padding_mask=torch.arange(300, device="cuda")[None] >= lens[:, None], dropout_p=0.1, seed=5)
for rep in range(1 if quick else 3):
    for tag, visit_all in (("skip", 0), ("all", 1)):
        native.attention_visit_all_blocks(visit_all)
        f = t(lambda: native.attention(q, k, v, H, return_lse=True, **cap), n=100)
        out, lse = native.attention(q, k, v, H, return_lse=True, **cap)
        bw = t(lambda: native.attention_backward(q, k, v, out, go, lse, H, **cap), n=100)
        for key, val in ((f"bert300_len8to300_{tag}_fwd", f), (f"bert300_len8to300_{tag}_bwd", bw)):
            res[key] = min(res.get(key, val), val)
native.attention_visit_all_blocks(0)
for name, Lq, Lk in [("joint130", 130, 130), ("self80", 80, 80), ("cross80x50", 80, 50)]:
    q = rnd(B, Lq, E).bfloat16(); k = rnd(B, Lk, E).bfloat16(); v = rnd(B, Lk, E).bfloat16(); go = rnd(B, Lq, E).bfloat16()
    for p in (0.0, 0.1):
        res[f"{name}_fwd_p{p}"] = t(lambda: native.attention(q, k, v, H, return_lse=True, dropout_p=p, seed=5))
        out, lse = native.attention(q, k, v, H, return_lse=True, dropout_p=p, seed=5)
        res[f"{name}_bwd_p{p}"] = t(lambda: native.attention_backward(q, k, v, out, go, lse, H, dropout_p=p, seed=5))
        if quick: continue
        qh, kh, vh = (x.view(B, -1, H, 64).transpose(1, 2).detach().requires_grad_(True) for x in (q, k, v))
        goh = go.view(B, Lq, H, 64).transpose(1, 2)
        res[f"{name}_sdpa_fwd_p{p}"] = t(lambda: F.scaled_dot_product_attention(qh, kh, vh, dropout_p=p))
        def fb():
            o = F.scaled_dot_product_attention(qh, kh, vh, dropout_p=p)
            o.backward(goh)
        res[f"{name}_sdpa_fwdbwd_p{p}"] = t(fb)
print(json.dumps({k: round(v, 4) for k, v in res.items()}))
