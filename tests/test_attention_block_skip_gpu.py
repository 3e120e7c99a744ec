"""Block skipping in the attention kernels (csrc/attn_common.cuh): a 64-key block whose keys are all masked is never
visited, and a backward key-row unit whose 64 keys are all masked writes zero dK / dV rows without loading anything.
Skipping on (default) against skipping off (sv_attention_visit_all_blocks(1)) must give the same out, lse and
dq | dk | dv bit for bit (torch.equal: a zero may change sign), for prefix masks, masks with a dead interior block,
fully masked scenes, dropout on and off, and the spatial gate.  Every gradient buffer starts as NaN, so a row a skipped
unit fails to write shows."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

B, H = 6, 3
E = H * 64


def rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g) * scale


@pytest.fixture
def visit_all():
    from sceneverse_b200 import native
    yield native.attention_visit_all_blocks
    native.attention_visit_all_blocks(0)


def _mask(kind, L):
    """(B, L) bool, True = masked.  Scene 0 is fully masked in every kind."""
    m = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    m[0] = True
    if kind == "prefix":          # caption-style lengths 1, 2, 17, L // 2 + 3, L
        for b, n in zip(range(1, B), (1, 2, min(17, L), L // 2 + 3, L)):
            m[b, n:] = True
    elif kind == "interior":      # live keys only in the first and the last key block (and one scene all live)
        m[1:B - 1] = True
        m[1:B - 1, :5] = False
        m[1:B - 1, L - 3:] = False
        if L > 70:
            m[2, 64:70] = False
    return m


def _backward(q, k, v, out, go, lse, mask, p, gate, packed):
    """sv_attention_bwd_strided_bf16 called directly with NaN-filled outputs (dq | dk | dv as slices of one packed
    gradient when `packed`)."""
    from sceneverse_b200 import _lib, native
    Lq, Lk = q.shape[1], k.shape[1]
    nan = dict(dtype=torch.bfloat16, device="cuda")
    if packed:
        pg = torch.full((B, Lq, 3 * E), math.nan, **nan)
        dq, dk, dv, d_rs = pg[..., :E], pg[..., E:2 * E], pg[..., 2 * E:], 3 * E
    else:
        dq, dk, dv, d_rs = torch.full((B, Lq, E), math.nan, **nan), torch.full((B, Lk, E), math.nan, **nan), \
            torch.full((B, Lk, E), math.nan, **nan), E
    sw, locs = gate if gate is not None else (None, None)
    dsw = torch.full_like(sw, math.nan) if sw is not None else None
    dvec = torch.full((B, H, Lq), math.nan, device="cuda")
    lib = _lib.gps()
    st = lib.sv_attention_bwd_strided_bf16(
        q.data_ptr(), q.stride(0), q.stride(1), k.data_ptr(), k.stride(0), k.stride(1), v.data_ptr(), v.stride(0),
        v.stride(1), out.data_ptr(), go.data_ptr(), _lib.ptr(native._mask_bytes(mask)), _lib.ptr(sw), _lib.ptr(locs),
        lse.data_ptr(), B, H, Lq, Lk, 0.125, dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), d_rs, _lib.ptr(dsw),
        dvec.data_ptr(), p, 11, torch.cuda.current_stream().cuda_stream)
    _lib.check(lib, st, "sv_attention_bwd_strided_bf16")
    return [dq, dk, dv, dvec] + ([dsw] if dsw is not None else [])


def _run(q, k, v, go, mask, p, gate, packed):
    from sceneverse_b200 import native
    kw = dict(key_padding_mask=mask, dropout_p=p, seed=11)
    if gate is not None:
        kw.update(spatial_w=gate[0], pairwise_locs=gate[1])
    out, lse = native.attention(q, k, v, H, return_lse=True, spatial_heads=H if gate is not None else 0, **kw)
    return [out, lse] + _backward(q, k, v, out, go, lse, mask, p, gate, packed)


def _inputs(Lq, Lk, packed):
    if packed:   # self-attention on a packed projection, gradients into one packed buffer (the BERT / joint layers)
        qkv = rand(B, Lq, 3 * E, seed=1).bfloat16()
        q, k, v = qkv[..., :E], qkv[..., E:2 * E], qkv[..., 2 * E:]
    else:
        q, k, v = (rand(B, L, E, seed=s).bfloat16() for s, L in ((1, Lq), (2, Lk), (3, Lk)))
    return q, k, v, rand(B, Lq, E, seed=4).bfloat16()


def _compare(visit_all, Lq, Lk, kind, p, gated, packed):
    from sceneverse_b200 import ops
    q, k, v, go = _inputs(Lq, Lk, packed)
    mask = _mask(kind, Lk)
    gate = None
    if gated:
        gate = (rand(B, Lq, H * 6, seed=5, scale=2.0), ops.calc_pairwise_locs(rand(B, Lk, 3, seed=6, scale=2.0), None))
    visit_all(1)
    want = _run(q, k, v, go, mask, p, gate, packed)
    visit_all(0)
    got = _run(q, k, v, go, mask, p, gate, packed)
    names = ["out", "lse", "dq", "dk", "dv", "dvec", "dsw"]
    for n, a, b in zip(names, got, want):
        assert not a.isnan().any(), n
        assert torch.equal(a, b), (n, (a.float() - b.float()).abs().max().item())
    # the fully masked scene: zero output and gradients, lse = +inf
    assert (got[0][0] == 0).all() and torch.isinf(got[1][0]).all()
    for g in got[2:5]:
        assert (g[0] == 0).all()
    # masked keys get zero dk / dv rows
    assert (got[3][mask] == 0).all() and (got[4][mask] == 0).all()


@pytest.mark.parametrize("L", [50, 80, 130, 300])
@pytest.mark.parametrize("kind", ["prefix", "interior"])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_skip_matches_full_sweep_self_attention(visit_all, L, kind, p):
    _compare(visit_all, L, L, kind, p, gated=False, packed=True)


@pytest.mark.parametrize("L", [50, 80, 130, 300])
@pytest.mark.parametrize("kind", ["prefix", "interior"])
def test_skip_matches_full_sweep_gated(visit_all, L, kind):
    _compare(visit_all, L, L, kind, 0.0, gated=True, packed=False)


@pytest.mark.parametrize("Lq,Lk", [(1, 300), (50, 300), (300, 80), (129, 130)])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_skip_matches_full_sweep_cross_attention(visit_all, Lq, Lk, p):
    _compare(visit_all, Lq, Lk, "prefix", p, gated=False, packed=False)


def test_skipped_blocks_are_not_read(visit_all):
    """The switch changes what the kernels read: NaN planted in the keys of the fully masked blocks of one scene reaches
    its output and dQ only when every block is visited; with skipping they are never read, and the results are those of
    the same inputs without the NaN."""
    from sceneverse_b200 import native
    L = 300
    q, k, v, go = _inputs(L, L, False)
    mask = _mask("prefix", L)                    # scene 3: 17 live keys, key blocks 1..4 fully masked
    poisoned = k.clone()
    poisoned[3, 64:] = math.nan
    mask_kw = dict(key_padding_mask=mask)

    def run(kk):
        out, lse = native.attention(q, kk, v, H, return_lse=True, **mask_kw)
        return out, _backward(q, kk, v, out, go, lse, mask, 0.0, None, False)[0]

    visit_all(0)
    clean, poison = run(k), run(poisoned)
    for a, b in zip(poison, clean):
        assert torch.equal(a, b)
    visit_all(1)
    out, dq = run(poisoned)
    assert out[3].isnan().any() and dq[3].isnan().any()
    others = [b for b in range(B) if b != 3]
    assert torch.equal(out[others], clean[0][others])


def test_skip_matches_full_sweep_caption_lengths(visit_all):
    """The scene-caption shape of the pre-training step: 64 captions of 8..300 tokens, 12 heads, dropout 0.1."""
    from sceneverse_b200 import native
    Bc, Hc, L = 64, 12, 300
    Ec = Hc * 64
    qkv = rand(Bc, L, 3 * Ec, seed=7).bfloat16()
    q, k, v = qkv[..., :Ec], qkv[..., Ec:2 * Ec], qkv[..., 2 * Ec:]
    go = rand(Bc, L, Ec, seed=8).bfloat16()
    g = torch.Generator(device="cuda").manual_seed(9)
    lens = torch.randint(8, L + 1, (Bc,), device="cuda", generator=g)
    mask = torch.arange(L, device="cuda")[None] >= lens[:, None]
    res = []
    for on in (1, 0):
        visit_all(on)
        out, lse = native.attention(q, k, v, Hc, key_padding_mask=mask, return_lse=True, dropout_p=0.1, seed=3)
        pg = torch.full((Bc, L, 3 * Ec), float("nan"), dtype=torch.bfloat16, device="cuda")
        native.attention_backward(q, k, v, out, go, lse, Hc, key_padding_mask=mask, dropout_p=0.1, seed=3, packed_grad=pg)
        res.append((out, lse, pg))
    for a, b in zip(*res):
        assert not a.isnan().any()
        assert torch.equal(a, b)
