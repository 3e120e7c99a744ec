"""Kernels launched over a prefix of a sequence's rows (sv_attention_fwd_rows_bf16 / sv_attention_bwd_rows_bf16,
sv_layer_norm_fwd_rows / sv_layer_norm_bwd_rows): the CLS-only last BERT layer of the scene captions.

* Attention with one query, the first row of each scene of a packed (B, 300, 3E) projection (a strided view), against all
  300 keys with a padding mask, dropout off and on: within the float64 bound of tests/test_attention_fp64_gpu.py; out,
  lse and dq row 0 equal to row 0 of the 300-query launch; dk | dv equal to that launch's when only row 0 of dO is
  non-zero; dq rows 1.. written as zeros; skipping fully masked key blocks on against off.
* The dropout masks of the new key arguments are rows of the full launch's masks: attention weights (through the
  float64 check with row 0 of the full mask) and LayerNorm outputs.
"""
import math
import types

import pytest
import torch

from tests import test_attention_fp64_gpu as fp64

pytestmark = pytest.mark.gpu

L, H = 300, 12
E = H * 64


def _packed(dropout, lengths=None):
    """float64-test inputs at Lq = Lk = 300 (scene 1 masks its second half of keys), their q | k | v packed into one
    (B, L, 3E) projection, and the 1-query view of them: q = qkv[:, :1, :E], dO = row 0 of dO, keep = row 0 of the mask."""
    x = fp64.inputs(L, L, H, dropout=dropout, B=2 if lengths is None else len(lengths))
    if lengths is not None:
        x.mask = torch.arange(L, device="cuda")[None, :] >= torch.tensor(lengths, device="cuda")[:, None]
    qkv = torch.cat([x.q, x.k, x.v], -1)
    x1 = types.SimpleNamespace(**vars(x))
    x1.q, x1.k, x1.v = qkv[:, :1, :E], qkv[..., E:2 * E], qkv[..., 2 * E:]
    x1.go = x.go[:, :1].contiguous()
    x1.keep = None if x.keep is None else x.keep[:, :, :1].contiguous()
    return x, x1, qkv


def _run_rows(x1):
    from sceneverse_b200 import native
    p = fp64.P_DROP if x1.keep is not None else 0.0
    out, lse = native.attention(x1.q, x1.k, x1.v, H, key_padding_mask=x1.mask, return_lse=True, dropout_p=p, seed=fp64.SEED,
                                seq_rows=L)
    B = x1.q.shape[0]
    pg = torch.full((B, L, 3 * E), math.nan, dtype=torch.bfloat16, device="cuda")
    dq, dk, dv, _ = native.attention_backward(x1.q, x1.k, x1.v, out, x1.go, lse, H, key_padding_mask=x1.mask, dropout_p=p,
                                              seed=fp64.SEED, packed_grad=pg, seq_rows=L)
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv)


@pytest.mark.parametrize("dropout", [False, True])
def test_one_query_of_packed_projection_within_fp64_bound(dropout):
    from sceneverse_b200 import native
    x, x1, qkv = _packed(dropout)
    got = _run_rows(x1)
    assert not any(t.isnan().any() for t in got.values())
    assert not got["dq"][:, 1:].any(), "dq rows past the query must be zero"
    fp64.check(x1, dict(got, dq=got["dq"][:, :1]), f"1-query packed L={L} dropout={dropout}")
    # the same bits as row 0 of the 300-query launch (same masks), and, when only row 0 of dO is non-zero, its dk | dv
    go0 = torch.zeros_like(x.go)
    go0[:, :1] = x.go[:, :1]
    p = fp64.P_DROP if dropout else 0.0
    qv = qkv[..., :E]
    out, lse = native.attention(qv, x1.k, x1.v, H, key_padding_mask=x.mask, return_lse=True, dropout_p=p, seed=fp64.SEED)
    assert torch.equal(out[:, :1], got["out"]) and torch.equal(lse[:, :, :1], got["lse"])
    full = torch.full(qkv.shape, math.nan, dtype=torch.bfloat16, device="cuda")
    dq, dk, dv, _ = native.attention_backward(qv, x1.k, x1.v, out, go0, lse, H, key_padding_mask=x.mask, dropout_p=p,
                                              seed=fp64.SEED, packed_grad=full)
    assert torch.equal(dq, got["dq"]), "dq differs from the 300-query launch"
    assert torch.equal(dk, got["dk"]) and torch.equal(dv, got["dv"]), "dk / dv differ from the 300-query launch"


@pytest.mark.parametrize("dropout", [False, True])
def test_one_query_block_skip_matches_full_sweep(dropout):
    """Caption-style lengths (one scene fully masked, others from 1 key to all 300): skipping the fully masked key blocks
    gives the bits of the full sweep."""
    from sceneverse_b200 import native
    _, x1, _ = _packed(dropout, lengths=[0, 1, 8, 64, 65, 130, 299, 300])
    try:
        native.attention_visit_all_blocks(1)
        want = _run_rows(x1)
    finally:
        native.attention_visit_all_blocks(0)
    got = _run_rows(x1)
    for name in want:
        assert not got[name].isnan().any(), name
        assert torch.equal(got[name], want[name]), name
    assert (got["out"][0] == 0).all() and torch.isinf(got["lse"][0]).all()
    assert (got["dk"][x1.mask] == 0).all() and (got["dv"][x1.mask] == 0).all()


def test_layer_norm_row_key_stride_draws_rows_of_full_launch():
    """LayerNorm over rows 0, L, 2L, ... with row_key_stride = L: outputs and all gradients equal those rows of the launch
    over every row (same dropout masks, same per-row arithmetic)."""
    from sceneverse_b200 import ops
    B, D, p = 64, 768, 0.1
    g = torch.Generator(device="cuda").manual_seed(3)
    x, r, go = (torch.randn(B, L, D, device="cuda", generator=g).bfloat16() for _ in range(3))
    w, b = 1.0 + 0.1 * torch.randn(D, device="cuda", generator=g), 0.1 * torch.randn(D, device="cuda", generator=g)

    def run(xx, rr, gg, stride):
        xx, rr = xx.clone().requires_grad_(True), rr.clone().requires_grad_(True)
        ww, bb = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
        y = ops._LayerNormFn.apply(xx, rr, ww, bb, 1e-12, p, 12345, stride)
        y.backward(gg)
        return y, xx.grad, rr.grad

    go_row0 = torch.zeros_like(go)
    go_row0[:, 0] = go[:, 0]
    full = run(x, r, go_row0, 1)
    rows = run(x[:, :1].contiguous(), r[:, :1].contiguous(), go[:, :1].contiguous(), L)
    for name, a, c in zip(("y", "dx", "dresidual"), full, rows):
        assert torch.equal(a[:, :1], c), name
    dropped = (rows[0] != run(x[:, :1].contiguous(), r[:, :1].contiguous(), go[:, :1].contiguous(), 1)[0]).any()
    assert dropped, "row_key_stride must change the mask of rows past the first"
