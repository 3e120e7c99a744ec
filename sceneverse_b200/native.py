"""Thin torch-tensor front-ends of the libsvgps kernels (allocation, stream, status checks)."""
import torch

from . import _lib

_ACT = {None: 0, "none": 0, "relu": 1, "gelu": 2}


def gemm(a, w, bias=None, act=None, residual=None, out_dtype=torch.bfloat16, rowmax=0):
    """epilogue(a @ w.T): a (M,K) bf16, w (N,K) bf16 (nn.Linear layout), bias (N) f32 -> (M,N) (or (M/16,N) with rowmax=16).
    Rows may be strided (last dim contiguous, stride % 8 == 0)."""
    assert a.is_cuda and a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and a.dim() == 2 and w.dim() == 2
    assert a.stride(1) == 1 and w.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    out = torch.empty((M // rowmax if rowmax else M, N), dtype=out_dtype, device=a.device)
    if bias is not None:
        bias = bias.float().contiguous()
    if residual is not None:
        residual = residual.to(out_dtype).contiguous()
    _lib.call(_lib.gps(), "sv_gemm_bf16", a.device, a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), M, N, K,
              _lib.ptr(bias), _ACT[act], _lib.ptr(residual), out.data_ptr(), N, 1 if out_dtype == torch.float32 else 0, rowmax)
    return out


def _mask_bytes(mask):
    """(B, L) key-padding mask as the uint8 bytes the kernels read: a bool tensor already IS one byte of 0 / 1 per element,
    so it is re-viewed, not copied (32 cast kernels per training step otherwise)."""
    if mask is None:
        return None
    if mask.dtype == torch.bool:
        return mask.contiguous().view(torch.uint8)
    return (mask != 0).contiguous().view(torch.uint8)


RESIDENT_MAX = 384    # Lq and Lk of sv_attention_{fwd,bwd}_rows_bf16 (include/svgps.h)
LONG_MAX = 2048       # Lq and Lk of sv_attention_{fwd,bwd}_long_bf16


def _long_entry(long, Lq, Lk):
    """None: the long entry exactly when a length exceeds the resident entries' RESIDENT_MAX."""
    return (Lq > RESIDENT_MAX or Lk > RESIDENT_MAX) if long is None else bool(long)


def attention(q, k, v, num_heads, key_padding_mask=None, spatial_w=None, spatial_heads=0, pairwise_locs=None,
              return_lse=False, dropout_p=0.0, seed=0, seq_rows=None, long=None):
    """Fused attention forward: q (B,Lq,E), k/v (B,Lk,E) bf16 (views with a contiguous last dim are fine), head dim 64.
    key_padding_mask (B,Lk) bool, True = ignore.  spatial_w (B,Lq,spatial_heads*6) + pairwise_locs (B,Lq,Lk,5) switch on the
    MultiHeadAttentionSpatial 'cond' gate.  seq_rows (default Lq): the queries are the first Lq rows of a sequence of
    seq_rows rows and draw that sequence's dropout masks.  long: True = sv_attention_fwd_long_bf16 (K / V streamed, Lq, Lk
    <= 2048), False = sv_attention_fwd_rows_bf16 (K / V resident, Lk <= 384), None = the long entry only when Lq or Lk
    exceeds 384.  Returns (B,Lq,E) bf16."""
    B, Lq, E = q.shape
    Lk = k.shape[1]
    entry = "sv_attention_fwd_long_bf16" if _long_entry(long, Lq, Lk) else "sv_attention_fwd_rows_bf16"
    assert E == num_heads * 64 and q.dtype == k.dtype == v.dtype == torch.bfloat16
    assert q.stride(2) == 1 and k.stride(2) == 1 and v.stride(2) == 1
    out = torch.empty((B, Lq, E), dtype=torch.bfloat16, device=q.device)
    kpm = _mask_bytes(key_padding_mask)
    sw = locs = None
    if spatial_w is not None:
        sw = spatial_w.float().contiguous()
        locs = pairwise_locs.float().contiguous()
    lse = torch.empty((B, num_heads, Lq), dtype=torch.float32, device=q.device) if return_lse else None
    _lib.call(_lib.gps(), entry, q.device,
              q.data_ptr(), q.stride(0), q.stride(1), k.data_ptr(), k.stride(0), k.stride(1), v.data_ptr(), v.stride(0),
              v.stride(1), out.data_ptr(), out.stride(0), out.stride(1), _lib.ptr(kpm), _lib.ptr(sw), int(spatial_heads),
              _lib.ptr(locs), B, num_heads, Lq, Lk, 0.125, _lib.ptr(lse), float(dropout_p), int(seed),
              Lq if seq_rows is None else int(seq_rows))
    return (out, lse) if return_lse else out


def attention_backward(q, k, v, out, grad_out, lse, num_heads, key_padding_mask=None, spatial_w=None, pairwise_locs=None,
                       dropout_p=0.0, seed=0, packed_grad=None, seq_rows=None, long=None):
    """Gradients of `attention` (gate requires one weight set per head).  Returns (dq, dk, dv, d_spatial_w or None).
    seq_rows as in `attention`: dq is then (B, seq_rows, E), its rows past Lq zero.  long as in `attention`:
    sv_attention_bwd_long_bf16 (Lq, Lk <= 2048) or sv_attention_bwd_rows_bf16 (<= 384).
    packed_grad: a (B, L, 3E) bf16 buffer (self-attention on a packed QKV projection, L = Lk = seq_rows): dq / dk / dv are
    written straight into its three column slices and returned as views."""
    B, Lq, E = q.shape
    Lk = k.shape[1]
    seq_rows = Lq if seq_rows is None else int(seq_rows)
    dev = q.device
    grad_out = grad_out.to(torch.bfloat16).contiguous()
    out = out.contiguous()
    if packed_grad is not None:
        assert seq_rows == Lk and packed_grad.shape == (B, Lk, 3 * E) and packed_grad.is_contiguous() and \
            packed_grad.dtype == torch.bfloat16
        dq, dk, dv = packed_grad[..., :E], packed_grad[..., E:2 * E], packed_grad[..., 2 * E:]
        d_rs = 3 * E
    else:
        dq = torch.empty((B, seq_rows, E), dtype=torch.bfloat16, device=dev)
        dk = torch.empty((B, Lk, E), dtype=torch.bfloat16, device=dev)
        dv = torch.empty((B, Lk, E), dtype=torch.bfloat16, device=dev)
        d_rs = E
    dvec = torch.empty((B, num_heads, Lq), dtype=torch.float32, device=dev)
    kpm = _mask_bytes(key_padding_mask)
    sw = locs = dsw = None
    if spatial_w is not None:
        sw, locs = spatial_w.float().contiguous(), pairwise_locs.float().contiguous()
        dsw = torch.empty_like(sw)
    entry = "sv_attention_bwd_long_bf16" if _long_entry(long, Lq, Lk) else "sv_attention_bwd_rows_bf16"
    _lib.call(_lib.gps(), entry, dev,
              q.data_ptr(), q.stride(0), q.stride(1), k.data_ptr(), k.stride(0), k.stride(1), v.data_ptr(), v.stride(0),
              v.stride(1), out.data_ptr(), grad_out.data_ptr(), _lib.ptr(kpm), _lib.ptr(sw), _lib.ptr(locs), lse.data_ptr(),
              B, num_heads, Lq, Lk, 0.125, dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), d_rs, _lib.ptr(dsw), dvec.data_ptr(),
              float(dropout_p), int(seed), seq_rows)
    return dq, dk, dv, dsw


def colsum(x):
    """Column sums of a (R, N) bf16 / f32 matrix (rows may be strided) -> (N,) f32; deterministic native kernel."""
    assert x.is_cuda and x.dim() == 2 and x.stride(1) == 1 and x.dtype in (torch.bfloat16, torch.float32)
    R, N = x.shape
    lib = _lib.gps()
    out = torch.empty(N, dtype=torch.float32, device=x.device)
    scratch = torch.empty(lib.sv_colsum_scratch_floats(N), dtype=torch.float32, device=x.device)
    _lib.call(lib, "sv_colsum", x.device, x.data_ptr(), x.stride(0), 1 if x.dtype == torch.bfloat16 else 0, R, N, out.data_ptr(),
              scratch.data_ptr())
    return out


def colsum_batched(x):
    """Column sums of each (R, N) matrix of a (B, R, N) bf16 / f32 tensor (rows and matrices may be strided) -> (B, N) in x's
    dtype, fp32 accumulation in a fixed order; deterministic native kernel."""
    assert x.is_cuda and x.dim() == 3 and x.stride(2) == 1 and x.dtype in (torch.bfloat16, torch.float32)
    B, R, N = x.shape
    lib = _lib.gps()
    out = torch.empty((B, N), dtype=x.dtype, device=x.device)
    scratch = torch.empty(lib.sv_colsum_batched_scratch_floats(B, R, N), dtype=torch.float32, device=x.device)
    _lib.call(lib, "sv_colsum_batched", x.device, x.data_ptr(), x.stride(1), x.stride(0), 1 if x.dtype == torch.bfloat16 else 0,
              B, R, N, out.data_ptr(), scratch.data_ptr())
    return out


def gemm_ex(a, b, a_transposed=False, b_transposed=False, bias=None, act=None, out_dtype=torch.bfloat16):
    """epilogue(A . B^T) with operands optionally given transposed in memory (no copies):
    a: (M,K), or (K,M) when a_transposed;  b: (N,K), or (K,N) when b_transposed.  bf16 in, bf16 / f32 out (M,N)."""
    assert a.is_cuda and a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.dim() == 2 and b.dim() == 2
    assert a.stride(1) == 1 and b.stride(1) == 1
    M, K = (a.shape[1], a.shape[0]) if a_transposed else a.shape
    N, Kb = (b.shape[1], b.shape[0]) if b_transposed else b.shape
    assert K == Kb, (a.shape, b.shape)
    out = torch.empty((M, N), dtype=out_dtype, device=a.device)
    if bias is not None:
        bias = bias.float().contiguous()
    _lib.call(_lib.gps(), "sv_gemm_bf16_ex", a.device, a.data_ptr(), a.stride(0), 1 if a_transposed else 0, b.data_ptr(),
              b.stride(0), 1 if b_transposed else 0, M, N, K, _lib.ptr(bias), _ACT[act], None, out.data_ptr(), N,
              1 if out_dtype == torch.float32 else 0, 0)
    return out


def _rows_ok(t):
    return t.dim() == 2 and t.stride(1) == 1 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0


def linear_fwd(x, w, bias=None, act=None, dropout_p=0.0, seed=0, out_dtype=torch.bfloat16, want_pre=False, n_out=None,
               out=None):
    """out = dropout(act(x @ w[:n].T + bias)): x (M,K) bf16, w (N,K) bf16, bias (N) f32.  `out` may be a wider buffer
    (M, Np >= N): only the first N columns are written.  want_pre: also return the pre-activation (bf16, same layout)."""
    assert x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and _rows_ok(x) and _rows_ok(w), (x.shape, x.stride(), w.shape)
    M, K = x.shape
    N = w.shape[0] if n_out is None else n_out
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=x.device)
    pre = torch.empty_like(out) if want_pre else None
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
    _lib.call(_lib.gps(), "sv_linear_fwd_bf16", x.device, x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), M, N, K,
              _lib.ptr(bias), _ACT[act], float(dropout_p), int(seed), out.data_ptr(), out.stride(0),
              1 if out.dtype == torch.float32 else 0, _lib.ptr(pre))
    return (out, pre) if want_pre else out


def linear_dgrad(g, w, act=None, aux=None, dropout_p=0.0, seed=0, n_red=None, out_dtype=torch.bfloat16):
    """dx (M,Kin) = (g (M,N) @ w (N,Kin)) * act'(aux) [* dropout mask]; n_red > w.shape[0]: g carries zero pad columns."""
    assert g.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and _rows_ok(g) and _rows_ok(w)
    M = g.shape[0]
    N = g.shape[1] if n_red is None else n_red
    Kin = w.shape[1]
    dx = torch.empty((M, Kin), dtype=out_dtype, device=g.device)
    if aux is not None:
        assert aux.dtype == torch.bfloat16 and aux.shape == (M, Kin) and aux.stride(1) == 1
    _lib.call(_lib.gps(), "sv_linear_dgrad_bf16", g.device, g.data_ptr(), g.stride(0), w.data_ptr(), w.stride(0), M, N, Kin,
              _ACT[act], _lib.ptr(aux), aux.stride(0) if aux is not None else 0, float(dropout_p), int(seed), dx.data_ptr(),
              dx.stride(0), 1 if out_dtype == torch.float32 else 0)
    return dx


def linear_wgrad(g, x, n_out=None, dw=None, db=None, want_db=False, accumulate=False):
    """dw (N,Kin) f32 (+)= g[:, :N].T @ x, db (N) f32 (+)= g[:, :N].sum(0).  accumulate=True adds into the given dw / db (the
    flat gradient buffer), otherwise they are (allocated and) overwritten."""
    assert g.dtype == torch.bfloat16 and x.dtype == torch.bfloat16 and _rows_ok(g) and _rows_ok(x) and g.shape[0] == x.shape[0]
    M, Kin = x.shape
    N = g.shape[1] if n_out is None else n_out
    if dw is None:
        assert not accumulate
        dw = torch.empty((N, Kin), dtype=torch.float32, device=g.device)
    if db is None and want_db:
        assert not accumulate
        db = torch.empty(N, dtype=torch.float32, device=g.device)
    assert dw.dtype == torch.float32 and dw.stride(1) == 1 and dw.shape == (N, Kin)
    _lib.call(_lib.gps(), "sv_linear_wgrad_bf16", g.device, g.data_ptr(), g.stride(0), x.data_ptr(), x.stride(0), M, N, Kin,
              dw.data_ptr(), dw.stride(0), _lib.ptr(db), 1 if accumulate else 0)
    return dw, db


def act_bwd(g, aux, act):
    """g * act'(aux): (M,N) bf16; relu: aux = forward output, gelu: aux = pre-activation."""
    assert g.dtype == torch.bfloat16 and aux.dtype == torch.bfloat16 and g.shape == aux.shape and _rows_ok(g) and _rows_ok(aux)
    out = torch.empty((g.shape[0], g.shape[1]), dtype=torch.bfloat16, device=g.device)
    _lib.call(_lib.gps(), "sv_act_bwd_bf16", g.device, g.data_ptr(), g.stride(0), aux.data_ptr(), aux.stride(0), _ACT[act],
              g.shape[0], g.shape[1], out.data_ptr(), out.stride(0))
    return out


def embedding_bwd(grad_out, ids, dw, padding_idx=-1):
    """dw[ids] += grad_out: grad_out (..., D) bf16 | f32, ids (...) int64, dw (V, D) f32 contiguous (accumulated into)."""
    D = grad_out.shape[-1]
    g2 = grad_out.reshape(-1, D)
    if g2.stride(1) != 1:
        g2 = g2.contiguous()
    ids = ids.reshape(-1).contiguous()
    assert ids.dtype == torch.int64 and dw.dtype == torch.float32 and dw.is_contiguous() and dw.shape[1] == D
    assert g2.dtype in (torch.bfloat16, torch.float32) and g2.shape[0] == ids.numel()
    _lib.call(_lib.gps(), "sv_embedding_bwd", g2.device, g2.data_ptr(), g2.stride(0), 1 if g2.dtype == torch.bfloat16 else 0,
              ids.data_ptr(), ids.numel(), D, dw.shape[0], int(padding_idx if padding_idx is not None else -1), dw.data_ptr())
    return dw


def attention_visit_all_blocks(on):
    """1 = the attention kernels sweep every key block, 0 (default) = skip the fully masked ones (svgps.h)."""
    _lib.check(_lib.gps(), _lib.gps().sv_attention_visit_all_blocks(int(on)), "sv_attention_visit_all_blocks")


def gemm_force_ctas(n):
    """0 = heuristic, 1 / 2 / 4 = tiles of 64 / 128 / 192 output columns; bits 8.. are timing-only profiling switches
    (svgps.h)."""
    _lib.check(_lib.gps(), _lib.gps().sv_gemm_force_ctas(int(n)), "sv_gemm_force_ctas")
