"""Attention forward / backward at the tail shapes of the 64-row work units and the 16-column last key / query block:
row counts around multiples of 64, key counts around multiples of 16 and 64, the gated backward away from L = 80, scene x
head counts that do not divide the SM count, and run-to-run determinism of the backward."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g) * scale


def _reference(q, k, v, go, H, mask):
    B, Lq, E = q.shape
    Lk = k.shape[1]
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    qh = qf.view(B, Lq, H, 64).transpose(1, 2)
    kh = kf.view(B, Lk, H, 64).transpose(1, 2)
    vh = vf.view(B, Lk, H, 64).transpose(1, 2)
    att = ((qh @ kh.transpose(-1, -2)) * 0.125).masked_fill(mask[:, None, None, :], float("-inf")).softmax(-1)
    out = (att @ vh).transpose(1, 2).reshape(B, Lq, E)
    out.backward(go.float())
    return out.detach(), qf.grad, kf.grad, vf.grad


def _rel(a, b):
    # the floor keeps gradients that are exactly zero in the reference (one key: softmax = 1, dq = 0) from failing on noise
    return (a.float() - b).abs().max().item() / (b.abs().max().item() + 1e-3)


@pytest.mark.parametrize("Lq", [64, 65, 127, 128, 129, 192, 193, 320, 384])
@pytest.mark.parametrize("Lk", [1, 15, 16, 17, 63, 65, 79, 81, 144, 145, 304, 384])
def test_attention_tail_shapes(Lq, Lk):
    from sceneverse_b200 import native
    B, H = 2, 5                                      # 10 (scene, head) pairs: no divisor of the SM count
    q, k, v, go = (rand(B, L, H * 64, seed=s).bfloat16() for s, L in ((1, Lq), (2, Lk), (3, Lk), (4, Lq)))
    mask = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    mask[1, (Lk + 1) // 2:] = True
    out, lse = native.attention(q, k, v, H, key_padding_mask=mask, return_lse=True)
    dq, dk, dv, _ = native.attention_backward(q, k, v, out, go, lse, H, key_padding_mask=mask)
    want = _reference(q, k, v, go, H, mask)
    for got, w, name in zip((out, dq, dk, dv), want, ("out", "dq", "dk", "dv")):
        assert _rel(got, w) < 3e-2, (name, _rel(got, w))


@pytest.mark.parametrize("L", [17, 50, 130])
def test_spatial_attention_backward_tail_shapes_with_mask(L):
    from sceneverse_b200 import ops
    B, H, E = 3, 12, 768
    q, k, v = (rand(B, L, E, seed=s).bfloat16().requires_grad_(True) for s in (1, 2, 3))
    sw = rand(B, L, H * 6, seed=4).requires_grad_(True)
    locs = ops.calc_pairwise_locs(rand(B, L, 3, seed=6, scale=2.0), None)
    mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    mask[1, L // 2:] = True
    out, _ = ops.spatial_attention(q, k, v, sw, locs, H, H, key_padding_mask=mask)
    assert isinstance(out.grad_fn, ops._AttentionFn._backward_cls)
    out.float().square().sum().backward()
    g_native = [t.grad.clone() for t in (q, k, v, sw)]
    for t in (q, k, v, sw):
        t.grad = None
    out2, _ = ops._spatial_attention_torch(q.float(), k.float(), v.float(), sw, locs, H, H, key_padding_mask=mask)
    out2.float().square().sum().backward()
    for a, b in zip(g_native, (q.grad, k.grad, v.grad, sw.grad)):
        assert (a.float() - b.float()).abs().max().item() <= 5e-2 * b.float().abs().max().item() + 1e-6


def test_attention_backward_is_deterministic():
    from sceneverse_b200 import native, ops
    B, H, L = 7, 12, 130
    q, k, v, go = (rand(B, L, H * 64, seed=s).bfloat16() for s in (1, 2, 3, 4))
    mask = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    mask[2, 77:] = True
    sw = rand(B, L, H * 6, seed=5)
    locs = ops.calc_pairwise_locs(rand(B, L, 3, seed=6, scale=2.0), None)
    for gate, p in ((False, 0.1), (True, 0.0)):
        kw = dict(key_padding_mask=mask, dropout_p=p, seed=99)
        if gate:
            kw.update(spatial_w=sw, pairwise_locs=locs)
        out, lse = native.attention(q, k, v, H, return_lse=True, spatial_heads=H if gate else 0, **kw)
        first = native.attention_backward(q, k, v, out, go, lse, H, **kw)
        for _ in range(3):
            again = native.attention_backward(q, k, v, out, go, lse, H, **kw)
            for x, y in zip(first, again):
                assert (x is None and y is None) or torch.equal(x, y)
