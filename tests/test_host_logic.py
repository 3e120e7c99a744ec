"""CPU checks of the host-side logic added around the native kernels (no GPU, no native library calls):
dispatch fallbacks of ops.py, the flat-gradient helpers of train.py, the dropout-mask restatement used by the GPU tests."""
import numpy as np
import torch
import torch.nn.functional as F

from sceneverse_b200 import ops, train


def test_layer_norm_cpu_formulation_matches_reference_block_tail():
    """transformers.py:145-154: tgt = norm(tgt + dropout(tgt2)); with p = 0 the fused op must equal the plain formula."""
    g = torch.Generator().manual_seed(0)
    x, r = torch.randn(4, 7, 48, generator=g), torch.randn(4, 7, 48, generator=g)
    w, b = torch.randn(48, generator=g), torch.randn(48, generator=g)
    got = ops.layer_norm(x, w, b, 1e-5, residual=r)
    assert torch.allclose(got, F.layer_norm(r + x, (48,), w, b, 1e-5), atol=1e-6)
    assert torch.allclose(ops.layer_norm(x, w, b, 1e-12), F.layer_norm(x, (48,), w, b, 1e-12), atol=1e-6)


def test_padded_vocab_linear_cpu_is_plain_linear():
    g = torch.Generator().manual_seed(1)
    h, W, b = torch.randn(5, 16, generator=g), torch.randn(37, 16, generator=g), torch.randn(37, generator=g)
    out = ops.padded_vocab_linear(h, W, b)
    assert out.shape == (5, 37) and not hasattr(out, "_sv_padded")
    assert torch.allclose(out, F.linear(h, W, b), atol=1e-6)
    labels = torch.tensor([0, 36, -1, 5, -1])
    assert torch.allclose(ops.cross_entropy(out, labels, ignore_index=-1), F.cross_entropy(out, labels, ignore_index=-1))


def test_linear_on_cpu_stays_on_the_torch_path():
    x = torch.randn(3, 16, requires_grad=True)
    lin = torch.nn.Linear(16, 8)
    y = ops.linear(x, lin.weight, lin.bias, activation="relu")
    assert torch.allclose(y, F.relu(lin(x)))
    assert "LinearFn" not in type(y.grad_fn.next_functions[0][0]).__name__


def test_flat_grads_views_and_clipping_match_clip_grad_norm():
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 3))
    ref = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 3))
    ref.load_state_dict(net.state_dict())
    fg = train.FlatGrads(list(net.parameters()))
    x = torch.randn(9, 6)
    for _ in range(2):
        fg.zero()
        ref.zero_grad()
        (net(x) ** 2).sum().backward()
        (ref(x) ** 2).sum().backward()
        assert all(p.grad.data_ptr() >= fg.flat.data_ptr() for p in net.parameters())     # still views of the flat buffer
        for p, q in zip(net.parameters(), ref.parameters()):
            assert torch.allclose(p.grad, q.grad, rtol=1e-5, atol=1e-7)
    fg.all_reduce_mean()      # no process group: must be a no-op


def test_weight_shadow_registry_ignores_foreign_and_cpu_parameters():
    lin = torch.nn.Linear(8, 8)
    ops.clear_shadows()
    ops.register_shadows(lin)                      # CPU parameters are not shadowed
    assert len(ops._SHADOW) == 0
    assert ops._bf16_of(lin.weight).dtype == torch.bfloat16
    ops.refresh_shadows()                          # empty registry: no-op


def test_dropout_mask_restatement_statistics():
    """The numpy restatement of the in-kernel counter hash (used by the GPU tests to feed torch the same mask) keeps
    1 - p of the weights, differs between rows and between seeds, and is reproducible."""
    from tests.test_attention_gpu import _dropout_keep
    a = _dropout_keep(123, 1, 2, 64, 128, 0.25)
    b = _dropout_keep(123, 1, 2, 64, 128, 0.25)
    c = _dropout_keep(124, 1, 2, 64, 128, 0.25)
    assert a.shape == (1, 2, 64, 128) and np.array_equal(a, b) and not np.array_equal(a, c)
    assert abs(a.mean() - 0.75) < 0.02
    assert not np.array_equal(a[0, 0, 0], a[0, 0, 1])


def test_attention_mask_bytes_is_a_view_for_bool_masks():
    """native._mask_bytes: bool key-padding masks reach the kernels as their own bytes (no cast kernel); other dtypes keep
    the 'non-zero = ignore' meaning."""
    import torch
    from sceneverse_b200 import native
    m = torch.tensor([[True, False, True], [False, False, True]])
    b = native._mask_bytes(m)
    assert b.dtype == torch.uint8 and b.data_ptr() == m.data_ptr() and b.tolist() == [[1, 0, 1], [0, 0, 1]]
    assert native._mask_bytes(None) is None
    f = torch.tensor([[2.0, 0.0, -1.0]])
    assert native._mask_bytes(f).tolist() == [[1, 0, 1]]
    t = m.t()                                     # non-contiguous: made contiguous, values kept
    assert native._mask_bytes(t).tolist() == [[1, 0], [0, 0], [1, 1]]
