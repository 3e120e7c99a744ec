"""Operator dispatch of the attention stack.  Each op has ONE implementation per device class:
CUDA tensors go to the native library where a kernel exists (no silent fallback: if the library is
missing the call raises) and to cuBLAS/ATen for the rest; CPU tensors are only accepted for
shape/contract tests of the host logic.  `NATIVE` lists which ops are hand-written kernels.
"""
import math

import torch
import torch.nn.functional as F

NATIVE = {"linear": True,               # every nn.Linear: native wgmma GEMM forward / dgrad / wgrad with fused epilogues
          "attention": True,            # nn.MultiheadAttention core incl. attention dropout: native wgmma forward + backward
          "spatial_attention": True,    # MultiHeadAttentionSpatial core: native wgmma forward and backward
          "calc_pairwise_locs": True,
          "cross_entropy": True,        # masked-LM / grounding CE: fused native forward+gradient
          "layer_norm": True,           # dropout + residual add + LayerNorm: one native pass per direction
          "l2_normalize": True,         # F.normalize of the contrastive heads: one native kernel per direction
          "bce_with_logits": True,      # QA answer loss / ScanQA within-batch loss: fused native forward+gradient
          "attention_pool": True,       # AttFlat pooling of the QA head (one glimpse): one native kernel per direction
          "scene_broadcast": True}      # per-scene object features over U utterances: native U-sum backward


_dropout_calls = [0]


def _next_dropout_seed():
    """Deterministic per-call seed of the in-kernel attention dropout: torch's global seed + a call counter (no host
    sync, CUDA-graph safe); each call then hashes (seed, b, h, i, j)."""
    _dropout_calls[0] += 1
    return (torch.initial_seed() * 0x9E3779B1 + _dropout_calls[0] * 0x85EBCA6B) & 0x7FFFFFFFFFFFFFFF


ATTENTION_MAX_LEN = 2048   # queries and keys of the native attention (native.LONG_MAX: the long entries above 384)


def _native_ok(*tensors):
    return all(t.is_cuda and t.dtype == torch.bfloat16 for t in tensors)


class _AttentionFn(torch.autograd.Function):
    """Fused wgmma attention: native forward (keeps the per-query log-sum-exp) and native backward (two kernels that
    recompute P).  spatial_n_head must equal n_head when a gate is given (one weight set per head)."""

    @staticmethod
    def forward(ctx, q, k, v, sw, locs, kpm, n_head, spatial_n_head, dropout_p=0.0, seed=0):
        from . import native
        out, lse = native.attention(q, k, v, n_head, key_padding_mask=kpm, spatial_w=sw, spatial_heads=spatial_n_head,
                                    pairwise_locs=locs, return_lse=True, dropout_p=dropout_p, seed=seed)
        ctx.save_for_backward(q, k, v, out, lse, sw, locs, kpm)
        ctx.n_head, ctx.drop = n_head, (dropout_p, seed)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        from . import native
        q, k, v, out, lse, sw, locs, kpm = ctx.saved_tensors
        dq, dk, dv, dsw = native.attention_backward(q, k, v, out, grad_out, lse, ctx.n_head, key_padding_mask=kpm,
                                                    spatial_w=sw, pairwise_locs=locs, dropout_p=ctx.drop[0], seed=ctx.drop[1])
        return dq, dk, dv, dsw, None, None, None, None, None, None


class _AttentionPackedFn(torch.autograd.Function):
    """Self-attention on a PACKED projection qkv (B,L,3E) = [q | k | v]: the kernels read the three column slices through
    strided TMA maps and the backward writes dq | dk | dv into ONE packed gradient, so the projection's backward is a
    single dgrad + a single wgrad GEMM (no split / cat / add kernels in between).  The queries are the first `query_rows`
    rows (all L for plain self-attention); the dropout masks are those of the same rows of the L-query call, and the packed
    gradient's dq rows past them are zero."""

    @staticmethod
    def forward(ctx, qkv, sw, locs, kpm, n_head, spatial_n_head, dropout_p, seed, query_rows):
        from . import native
        E = qkv.shape[-1] // 3
        q, k, v = qkv[:, :query_rows, :E], qkv[..., E:2 * E], qkv[..., 2 * E:]
        out, lse = native.attention(q, k, v, n_head, key_padding_mask=kpm, spatial_w=sw, spatial_heads=spatial_n_head,
                                    pairwise_locs=locs, return_lse=True, dropout_p=dropout_p, seed=seed,
                                    seq_rows=qkv.shape[1])
        ctx.save_for_backward(qkv, out, lse, sw, locs, kpm)
        ctx.n_head, ctx.drop, ctx.query_rows = n_head, (dropout_p, seed), query_rows
        return out

    @staticmethod
    def backward(ctx, grad_out):
        from . import native
        qkv, out, lse, sw, locs, kpm = ctx.saved_tensors
        E = qkv.shape[-1] // 3
        q, k, v = qkv[:, :ctx.query_rows, :E], qkv[..., E:2 * E], qkv[..., 2 * E:]
        dqkv = torch.empty(qkv.shape, dtype=torch.bfloat16, device=qkv.device)
        _, _, _, dsw = native.attention_backward(q, k, v, out, grad_out, lse, ctx.n_head, key_padding_mask=kpm, spatial_w=sw,
                                                 pairwise_locs=locs, dropout_p=ctx.drop[0], seed=ctx.drop[1], packed_grad=dqkv,
                                                 seq_rows=qkv.shape[1])
        return dqkv, dsw, None, None, None, None, None, None, None


def _packed_ok(qkv, num_heads):
    E = qkv.shape[-1] // 3
    return qkv.is_cuda and qkv.dtype == torch.bfloat16 and qkv.dim() == 3 and qkv.shape[-1] == 3 * E and E == num_heads * 64 \
        and qkv.is_contiguous() and qkv.shape[1] <= ATTENTION_MAX_LEN


def attention_packed(qkv, num_heads, key_padding_mask=None, dropout_p=0.0, query_rows=None):
    """Self-attention on qkv (B,L,3E) = [q | k | v] -> (B,L,E).  query_rows = n < L: only the first n rows attend (to all
    L keys) -> (B,n,E), with the dropout masks those rows have in the full call (native path)."""
    L = qkv.shape[1]
    n = L if query_rows is None else int(query_rows)
    if _packed_ok(qkv, num_heads):
        return _AttentionPackedFn.apply(qkv, None, None, key_padding_mask, num_heads, 0, float(dropout_p),
                                        _next_dropout_seed() if dropout_p > 0.0 else 0, n)
    q, k, v = qkv.chunk(3, dim=-1)
    return attention(q[:, :n], k, v, num_heads, key_padding_mask=key_padding_mask, dropout_p=dropout_p)


def spatial_attention_packed(qkv, spatial_weights, pairwise_locs, n_head, spatial_n_head, key_padding_mask=None):
    """MultiHeadAttentionSpatial core on a packed projection; returns (out, None)."""
    if _packed_ok(qkv, n_head) and spatial_n_head == n_head:
        return _AttentionPackedFn.apply(qkv, spatial_weights.float(), pairwise_locs.float(), key_padding_mask, n_head,
                                        spatial_n_head, 0.0, 0, qkv.shape[1]), None
    q, k, v = qkv.chunk(3, dim=-1)
    return spatial_attention(q, k, v, spatial_weights, pairwise_locs, n_head, spatial_n_head, key_padding_mask=key_padding_mask)


class _SpatialAttentionRecomputeFn(torch.autograd.Function):
    """Native forward, torch-recompute backward: only for a gate shared across heads (spatial_multihead=False)."""

    @staticmethod
    def forward(ctx, q, k, v, sw, locs, kpm, n_head, spatial_n_head):
        from . import native
        ctx.save_for_backward(q, k, v, sw, locs, kpm)
        ctx.heads = (n_head, spatial_n_head)
        return native.attention(q, k, v, n_head, key_padding_mask=kpm, spatial_w=sw, spatial_heads=spatial_n_head,
                                pairwise_locs=locs)

    @staticmethod
    def backward(ctx, grad_out):
        q, k, v, sw, locs, kpm = ctx.saved_tensors
        n_head, spatial_n_head = ctx.heads
        with torch.enable_grad():
            qq, kk, vv, ss = (t.detach().float().requires_grad_(True) for t in (q, k, v, sw))
            out, _ = _spatial_attention_torch(qq, kk, vv, ss, locs, n_head, spatial_n_head, kpm)
            gq, gk, gv, gs = torch.autograd.grad(out, (qq, kk, vv, ss), grad_out.float())
        return gq.to(q.dtype), gk.to(k.dtype), gv.to(v.dtype), gs.to(sw.dtype), None, None, None, None


DIRECT_GRAD = [False]   # set by train.PretrainStep: parameter gradients live in one flat fp32 buffer that the wgrad
                        # kernels may accumulate into directly (red.global.add) instead of returning a tensor that
                        # autograd's AccumulateGrad adds with one more elementwise launch per parameter

# bf16 shadows of fp32 parameters, refreshed once per step with ONE multi-tensor copy (train.PretrainStep) instead of one
# cast kernel per weight and per bias inside every linear (autocast's behaviour: ~200 tiny launches per step)
_SHADOW = {}
_SHADOW_LISTS = [[], []]   # (bf16 destinations, fp32 sources)


def register_shadows(module):
    """Create a bf16 shadow for every floating-point parameter of `module` that the bf16 linears read."""
    for p in module.parameters():
        if p.is_cuda and p.dtype == torch.float32 and p.dim() >= 1 and id(p) not in _SHADOW:
            s = torch.empty_like(p, dtype=torch.bfloat16)
            _SHADOW[id(p)] = (s, p)        # the strong reference to p keeps its id from being reused
            _SHADOW_LISTS[0].append(s)
            _SHADOW_LISTS[1].append(p.detach())
    refresh_shadows()


def register_shadow_views(pairs):
    """pairs of (parameter, bf16 view): the shadows are slices of one flat bf16 buffer that the fused optimizer kernel
    rewrites together with the parameters (train.FlatState) — nothing to refresh."""
    for p, s in pairs:
        _SHADOW[id(p)] = (s, p)


def refresh_shadows():
    """Must run after every parameter update and before the next forward that should use the shadows."""
    if _SHADOW_LISTS[0]:
        torch._foreach_copy_(_SHADOW_LISTS[0], _SHADOW_LISTS[1])


def clear_shadows():
    _SHADOW.clear()
    _SHADOW_LISTS[0].clear()
    _SHADOW_LISTS[1].clear()
    _PACKS.clear()


# sibling projections (q | k | v) whose weights / biases are adjacent in the flat buffers of train.FlatState:
# ids of the weights -> ([3E,K] bf16 shadow view, [3E,K] gradient view, [3E] fp32 bias view, [3E] bias-gradient view)
_PACKS = {}


def register_pack(weights, biases, wviews, bviews):
    _PACKS[tuple(id(w) for w in weights)] = (wviews[0], wviews[1], bviews[2], bviews[1], list(weights) + list(biases))


def _bf16_of(p):
    e = _SHADOW.get(id(p))
    return e[0] if e is not None and e[1] is p else p.detach().to(torch.bfloat16)


def _round8(n):
    return (n + 7) // 8 * 8


def _rows_bf16(t, K):
    """(..., K) -> (M, K) bf16 with a contiguous last dim, 16-byte aligned rows (what a TMA tensor map needs)."""
    t2 = t.reshape(-1, K)
    if t2.dtype != torch.bfloat16:
        t2 = t2.to(torch.bfloat16)
    if t2.stride(1) != 1 or t2.stride(0) % 8 or t2.data_ptr() % 16:
        t2 = t2.contiguous()
    return t2


def _direct(p):
    """May the wgrad kernel accumulate straight into p.grad?"""
    return DIRECT_GRAD[0] and p is not None and p.is_leaf and p.grad is not None and p.grad.dtype == torch.float32 and \
        p.grad.is_contiguous()


def _f32(b):
    return None if b is None else b.detach().float().contiguous()


def _wgrad(g2, x2, weight, bias, n_out, k_in):
    """Weight / bias gradient of one linear: accumulated in place into the flat gradient buffer when allowed (returns
    (None, None)), else returned as fresh fp32 tensors."""
    from . import native
    if _direct(weight) and (bias is None or _direct(bias)) and x2.shape[1] == k_in:
        native.linear_wgrad(g2, x2, n_out=n_out, dw=weight.grad, db=bias.grad if bias is not None else None, accumulate=True)
        return None, None
    dw, db = native.linear_wgrad(g2, x2, n_out=n_out, want_db=bias is not None)
    return (dw if x2.shape[1] == k_in else dw[:, :k_in].contiguous()), db


class _LinearFn(torch.autograd.Function):
    """y = act(x W^T + b) on the native wgmma GEMM in all three directions (csrc/gemm.cu): forward with the bias /
    activation epilogue, dgrad with the weight read as a transposed operand, wgrad split over the tokens with the bias
    gradient riding in the same main loop.  The returned tensor is (..., round8(N)) wide (pad columns zero) so that its
    gradient arrives with 16-byte rows; `linear` slices it.  An input width that is not a multiple of 8 (the 6-d box
    embedding, transformers.py loc_layers) is zero-padded on the fly."""

    @staticmethod
    def forward(ctx, x, weight, bias, act):
        from . import native
        N, K = weight.shape
        wb = _bf16_of(weight)
        x2 = _rows_bf16(x, K)
        Kp = _round8(K)
        if Kp != K:
            x2 = F.pad(x2, (0, Kp - K))
            wb = F.pad(wb, (0, Kp - K))
        Np = _round8(N)
        assert act is None or Np == N
        M = x2.shape[0]
        y = torch.empty((*x.shape[:-1], Np), dtype=torch.bfloat16, device=x.device)   # returned as is: not a view
        out = y.view(M, Np)
        if Np != N:
            out[:, N:].zero_()
        need_grad = any(ctx.needs_input_grad[:3])
        pre = None
        if act == "gelu" and need_grad:
            _, pre = native.linear_fwd(x2, wb, _f32(bias), act, out=out, n_out=N, want_pre=True)
        else:
            native.linear_fwd(x2, wb, _f32(bias), act, out=out, n_out=N)
        ctx.save_for_backward(x2, wb, out.detach() if act == "relu" else pre)
        ctx.params = (weight, bias)
        ctx.meta = (x.shape, x.dtype, act, N, K)
        return y

    @staticmethod
    def backward(ctx, g):
        from . import native
        x2, wb, aux = ctx.saved_tensors
        weight, bias = ctx.params
        in_shape, in_dtype, act, N, K = ctx.meta
        Np = _round8(N)
        g2 = _rows_bf16(g, Np)
        if act is not None:
            g2 = native.act_bwd(g2, aux, act)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = native.linear_dgrad(g2, wb, n_red=N)      # the true class count: the weight has no pad rows to read
            if dx.shape[1] != K:
                dx = dx[:, :K]
            dx = dx.reshape(in_shape).to(in_dtype)
        if ctx.needs_input_grad[1] or (bias is not None and ctx.needs_input_grad[2]):
            dw, db = _wgrad(g2, x2, weight, bias, N, K)
        return dx, dw, db, None


class _FFNFn(torch.autograd.Function):
    """y = dropout_p(act(x W1^T + b1)) W2^T + b2 — the feed-forward block of every transformer layer of the stack
    (transformers.py:135-154,300-316; BertIntermediate + BertOutput.dense) as 2 + 4 native GEMMs: activation and dropout
    live in the first GEMM's epilogue (the mask is a counter hash, nothing is stored), their derivative in the epilogue of
    the second layer's dgrad."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, act, p, seed):
        from . import native
        H, K = w1.shape
        N = w2.shape[0]
        wb1, wb2 = _bf16_of(w1), _bf16_of(w2)
        x2 = _rows_bf16(x, K)
        need_grad = any(ctx.needs_input_grad[:5])
        pre = None
        if act == "gelu" and need_grad:
            h, pre = native.linear_fwd(x2, wb1, _f32(b1), act, dropout_p=p, seed=seed, want_pre=True)
        else:
            h = native.linear_fwd(x2, wb1, _f32(b1), act, dropout_p=p, seed=seed)
        y = torch.empty((*x.shape[:-1], N), dtype=torch.bfloat16, device=x.device)
        native.linear_fwd(h, wb2, _f32(b2), out=y.view(-1, N))
        ctx.save_for_backward(x2, wb1, wb2, h, pre)
        ctx.params = (w1, b1, w2, b2)
        ctx.meta = (x.shape, x.dtype, act, p, seed)
        return y

    @staticmethod
    def backward(ctx, g):
        from . import native
        x2, wb1, wb2, h, pre = ctx.saved_tensors
        w1, b1, w2, b2 = ctx.params
        in_shape, in_dtype, act, p, seed = ctx.meta
        H, K = w1.shape
        N = w2.shape[0]
        g2 = _rows_bf16(g, N)
        # dL/d(pre-activation of layer 1): dgrad of layer 2 with the activation / dropout derivative in the epilogue
        dpre = native.linear_dgrad(g2, wb2, act=act, aux=h if act == "relu" else pre, dropout_p=p, seed=seed)
        dw2, db2 = _wgrad(g2, h, w2, b2, N, H)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = native.linear_dgrad(dpre, wb1).reshape(in_shape).to(in_dtype)
        dw1, db1 = _wgrad(dpre, x2, w1, b1, H, K)
        return dx, dw1, db1, dw2, db2, None, None, None


class _PackedLinearFn(torch.autograd.Function):
    """[y1 | y2 | ...] = x [W1; W2; ...]^T + [b1 | b2 | ...]: sibling projections of one input (w_qs / w_ks / w_vs of
    MultiHeadAttentionSpatial, transformers.py:190-192; query / key / value of BertSelfAttention) as ONE GEMM per direction.
    With train.FlatState the stacked weight, bias and their gradients are views of the flat buffers (no copies, the wgrad
    accumulates in place); otherwise the stack is concatenated per call."""

    @staticmethod
    def forward(ctx, x, *params):
        from . import native
        n = len(params) // 2
        ws, bs = params[:n], params[n:]
        pack = _PACKS.get(tuple(id(w) for w in ws))
        if pack is not None:
            wb, bias = pack[0], pack[2]
        else:
            wb = torch.cat([_bf16_of(w) for w in ws], 0)
            bias = torch.cat([b.detach().float() for b in bs], 0)
        K = wb.shape[1]
        x2 = _rows_bf16(x, K)
        y = torch.empty((*x.shape[:-1], wb.shape[0]), dtype=torch.bfloat16, device=x.device)
        native.linear_fwd(x2, wb, bias, out=y.view(-1, wb.shape[0]))
        ctx.save_for_backward(x2, wb)
        ctx.params, ctx.pack, ctx.meta = params, pack, (x.shape, x.dtype)
        return y

    @staticmethod
    def backward(ctx, g):
        from . import native
        x2, wb = ctx.saved_tensors
        params, pack = ctx.params, ctx.pack
        n = len(params) // 2
        in_shape, in_dtype = ctx.meta
        g2 = _rows_bf16(g, wb.shape[0])
        dx = native.linear_dgrad(g2, wb).reshape(in_shape).to(in_dtype) if ctx.needs_input_grad[0] else None
        if pack is not None and all(_direct(p) for p in params):
            native.linear_wgrad(g2, x2, dw=pack[1], db=pack[3], accumulate=True)
            return (dx,) + (None,) * len(params)
        dw, db = native.linear_wgrad(g2, x2, want_db=True)
        rows = [w.shape[0] for w in params[:n]]
        return (dx,) + tuple(dw.split(rows, 0)) + tuple(db.split(rows, 0))


def linear_packed(x, linears):
    """cat([lin(x) for lin in linears], -1) for nn.Linear modules with bias that share the input width."""
    ws = [l.weight for l in linears]
    if _native_linear_ok(x, ws[0]) and all(l.bias is not None and l.weight.shape[0] % 8 == 0 for l in linears) and \
            ws[0].shape[1] % 8 == 0:
        return _PackedLinearFn.apply(x, *ws, *[l.bias for l in linears])
    return torch.cat([linear(x, l.weight, l.bias) for l in linears], dim=-1)


class _EmbeddingFn(torch.autograd.Function):
    """nn.Embedding lookup whose backward is ONE native scatter-add (csrc/train_ops.cu embedding_bwd_kernel, fp32 red.add)
    instead of ATen's sort + segmented reduction (8 kernels); tiny tables (token types) use masked column sums, where every
    row would hit the same few addresses."""

    @staticmethod
    def forward(ctx, ids, weight, padding_idx):
        ctx.save_for_backward(ids)
        ctx.weight, ctx.padding_idx = weight, padding_idx
        return F.embedding(ids, weight, padding_idx)

    @staticmethod
    def backward(ctx, g):
        from . import native
        (ids,) = ctx.saved_tensors
        weight, pad = ctx.weight, ctx.padding_idx
        direct = _direct(weight)
        dw = weight.grad if direct else torch.zeros_like(weight, dtype=torch.float32)
        g2 = g.reshape(-1, g.shape[-1])
        if weight.shape[0] <= 4:
            flat = ids.reshape(-1)
            total = native.colsum(g2 if g2.dtype in (torch.bfloat16, torch.float32) else g2.float())
            rest = torch.zeros_like(total)
            for v in range(1, weight.shape[0]):
                part = native.colsum((g2 * (flat == v).unsqueeze(1).to(g2.dtype)).contiguous())
                rest += part            # the padding row's tokens too: row 0 gets total - rest
                if pad is None or v != pad:
                    dw[v] += part
            if pad is None or pad != 0:
                dw[0] += total - rest
        else:
            native.embedding_bwd(g2, ids, dw, padding_idx=-1 if pad is None else pad)
        return None, (None if direct else dw), None


def embedding(ids, weight, padding_idx=None):
    if weight.is_cuda and weight.dtype == torch.float32 and torch.is_grad_enabled() and weight.requires_grad and ids.dtype == torch.int64:
        return _EmbeddingFn.apply(ids, weight, padding_idx)
    return F.embedding(ids, weight, padding_idx)


def _native_linear_ok(x, weight):
    return x.is_cuda and weight.is_cuda and weight.dim() == 2 and x.numel() > 0 and weight.dtype in (torch.float32, torch.bfloat16) \
        and (x.dtype == torch.bfloat16 or _autocast_on())


def linear(x, weight, bias=None, activation=None):
    """y = act(x W^T + b).  CUDA under bf16 (tensor dtype or autocast): the native GEMM family, training and inference;
    anything else (CPU host-logic tests, the fp32 parity path): the torch formulation."""
    if activation not in (None, "relu", "gelu"):
        raise ValueError(activation)
    if _native_linear_ok(x, weight):
        N = weight.shape[0]
        fuse = activation if N % 8 == 0 else None
        y = _LinearFn.apply(x, weight, bias, fuse)
        if y.shape[-1] != N:
            y = y[..., :N]
        if fuse is None and activation is not None:
            y = F.relu(y) if activation == "relu" else F.gelu(y)
        return y
    y = F.linear(x, weight, bias)
    if activation == "relu":
        y = F.relu(y)
    elif activation == "gelu":
        y = F.gelu(y)
    return y


def ffn(x, w1, b1, w2, b2, activation="relu", dropout_p=0.0):
    """linear2(dropout(act(linear1(x)))); dropout_p = 0 outside training (the caller decides)."""
    if _native_linear_ok(x, w1) and w1.shape[0] % 8 == 0 and w1.shape[1] % 8 == 0 and w2.shape[0] % 8 == 0 and \
            b1 is not None and b2 is not None and activation in ("relu", "gelu"):
        return _FFNFn.apply(x, w1, b1, w2, b2, activation, float(dropout_p), _next_dropout_seed() if dropout_p > 0.0 else 0)
    h = linear(x, w1, b1, activation=activation)
    if dropout_p > 0.0:
        h = F.dropout(h, dropout_p, True)
    return linear(h, w2, b2)


def calc_pairwise_locs(obj_centers, obj_whls, eps=1e-10, pairwise_rel_type='center', spatial_dist_norm=True,
                       spatial_dim=5):
    """modules/utils.py:38-87, 'center' relation (the one GPS uses): (B,O,3) -> (B,O,O,5)
    [dist/max_dist, dz/dist, dist2d/dist, dy/dist2d, dx/dist2d]; the max-distance normaliser includes padded objects."""
    if pairwise_rel_type != 'center':
        raise NotImplementedError(pairwise_rel_type)
    if obj_centers.is_cuda and obj_centers.dtype == torch.float32 and spatial_dim == 5 and not obj_centers.requires_grad \
            and obj_centers.stride(2) == 1 and obj_centers.stride(0) == obj_centers.size(1) * obj_centers.stride(1):
        from . import _lib
        B, O, _ = obj_centers.shape
        out = torch.empty((B, O, O, 5), dtype=torch.float32, device=obj_centers.device)
        _lib.call(_lib.gps(), "sv_pairwise_locs_f32", obj_centers.device, obj_centers.data_ptr(), obj_centers.stride(1), B, O,
                  float(eps), 1 if spatial_dist_norm else 0, out.data_ptr())
        return out
    d = obj_centers[:, :, None, :] - obj_centers[:, None, :, :]
    dist = torch.sqrt((d ** 2).sum(3) + eps)
    if spatial_dist_norm:
        max_d = dist.reshape(dist.size(0), -1).max(dim=1)[0]
        norm = dist / max_d[:, None, None]
    else:
        norm = dist
    if spatial_dim == 1:
        return norm.unsqueeze(3)
    dist2d = torch.sqrt((d[..., :2] ** 2).sum(3) + eps)
    locs = torch.stack([norm, d[..., 2] / dist, dist2d / dist, d[..., 1] / dist2d, d[..., 0] / dist2d], dim=3)
    return locs[..., 1:] if spatial_dim == 4 else locs


def attention(q, k, v, num_heads, key_padding_mask=None, dropout_p=0.0):
    """Scaled-dot-product attention on packed heads: q (B,Lq,E), k/v (B,Lk,E) -> (B,Lq,E).
    key_padding_mask (B,Lk) bool, True = ignore (nn.MultiheadAttention convention).
    bf16 CUDA tensors run on the native wgmma kernels (head dim 64, <= 2048 queries and keys: K / V resident up to 384,
    streamed above) and an unsupported bf16 shape RAISES: there is no silent library fallback on the product path.  fp32
    tensors (CPU host-logic tests, the fp32 parity path on the GPU) use the torch formulation."""
    B, Lq, E = q.shape
    Lk, hd = k.shape[1], E // num_heads
    if _native_ok(q, k, v):
        if hd != 64 or Lk > ATTENTION_MAX_LEN or Lq > ATTENTION_MAX_LEN:
            raise NotImplementedError(f"native attention supports head dim 64 and at most {ATTENTION_MAX_LEN} queries and "
                                      f"keys (got head dim {hd}, Lq {Lq}, Lk {Lk})")
        needs_grad = torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad)
        if not needs_grad and dropout_p == 0.0:
            from . import native
            return native.attention(q, k, v, num_heads, key_padding_mask=key_padding_mask)
        return _AttentionFn.apply(q, k, v, None, None, key_padding_mask, num_heads, 0, float(dropout_p),
                                  _next_dropout_seed() if dropout_p > 0.0 else 0)
    qh = q.view(B, Lq, num_heads, hd).transpose(1, 2)
    kh = k.view(B, Lk, num_heads, hd).transpose(1, 2)
    vh = v.view(B, Lk, num_heads, hd).transpose(1, 2)
    mask = None
    if key_padding_mask is not None:
        mask = key_padding_mask.logical_not()[:, None, None, :]
    out = F.scaled_dot_product_attention(qh, kh, vh, attn_mask=mask, dropout_p=dropout_p)
    return out.transpose(1, 2).reshape(B, Lq, E)


def spatial_attention(q, k, v, spatial_weights, pairwise_locs, n_head, spatial_n_head, key_padding_mask=None):
    """bf16 CUDA tensors -> fused wgmma kernels, forward and backward (attention map not returned: every reference caller
    discards it); the GPS configurations use one gate per head (spatial_multihead=True), a gate shared across heads keeps the
    native forward with a recomputed backward.  An unsupported bf16 shape raises.  fp32 tensors -> the torch formulation
    below (CPU host-logic tests, fp32 parity path)."""
    if _native_ok(q, k, v):
        if q.shape[-1] // n_head != 64 or k.shape[1] > ATTENTION_MAX_LEN or q.shape[1] > ATTENTION_MAX_LEN:
            raise NotImplementedError(f"native spatial attention supports head dim 64 and at most {ATTENTION_MAX_LEN} "
                                      f"objects (got head dim {q.shape[-1] // n_head}, Lq {q.shape[1]}, Lk {k.shape[1]})")
        fn = _AttentionFn if spatial_n_head == n_head else _SpatialAttentionRecomputeFn
        out = fn.apply(q, k, v, spatial_weights.float(), pairwise_locs.float(), key_padding_mask, n_head, spatial_n_head)
        return out, None
    return _spatial_attention_torch(q, k, v, spatial_weights, pairwise_locs, n_head, spatial_n_head, key_padding_mask)


def _spatial_attention_torch(q, k, v, spatial_weights, pairwise_locs, n_head, spatial_n_head, key_padding_mask=None):
    """Core of MultiHeadAttentionSpatial 'cond' (transformers.py:188-237):
    softmax(log(clamp(sigmoid(w . loc + b), 1e-6)) + q k^T / sqrt(dh)) v, masked keys excluded.
    q,k,v (B,L,E) already projected; spatial_weights (B,L,spatial_n_head*(d+1)), per head [bias, w_1..w_d];
    pairwise_locs (B,L,T,d).  Returns (out (B,L,E), attn (H,B,L,T))."""
    B, L, E = q.shape
    T, hd = k.shape[1], E // n_head
    d = pairwise_locs.shape[-1]
    qh = q.view(B, L, n_head, hd).permute(2, 0, 1, 3)
    kh = k.view(B, T, n_head, hd).permute(2, 0, 1, 3)
    vh = v.view(B, T, n_head, hd).permute(2, 0, 1, 3)
    attn = torch.einsum('hblk,hbtk->hblt', qh, kh) / math.sqrt(hd)
    sw = spatial_weights.view(B, L, spatial_n_head, d + 1).permute(2, 0, 1, 3)
    if spatial_n_head == 1:
        sw = sw.expand(n_head, -1, -1, -1)
    loc = torch.sigmoid(torch.einsum('hbld,bltd->hblt', sw[..., 1:], pairwise_locs) + sw[..., :1])
    if key_padding_mask is not None:
        m = key_padding_mask[None, :, None, :]
        attn = attn.masked_fill(m, float('-inf'))
        loc = loc.masked_fill(m, 0)
    fused = torch.softmax(torch.log(torch.clamp(loc, min=1e-6)) + attn, 3)
    out = torch.einsum('hblt,hbtv->hblv', fused, vh).permute(1, 2, 0, 3).reshape(B, L, E)
    return out, fused


class _CrossEntropyFn(torch.autograd.Function):
    """mean cross-entropy over the rows whose label != ignore_index; forward and gradient come from ONE native launch.
    n_classes < logits.shape[1]: the trailing columns are padding (padded-vocabulary logits): ignored by the loss, zero in
    the gradient, which keeps the padded row stride so the backward GEMMs stay 16-byte aligned."""

    @staticmethod
    def forward(ctx, logits2d, labels, ignore_index, n_classes):
        from . import _lib
        R, W = logits2d.shape
        V = n_classes if n_classes else W
        if labels.dtype != torch.int64:
            raise RuntimeError(f"cross_entropy: expected int64 labels, got {labels.dtype}")
        loss_rows = torch.empty(R, dtype=torch.float32, device=logits2d.device)
        need_grad = logits2d.requires_grad
        grad = torch.empty((R, W), dtype=logits2d.dtype, device=logits2d.device) if need_grad else None
        _lib.call(_lib.gps(), "sv_cross_entropy_fwd_bwd_strided", logits2d.device, logits2d.data_ptr(), logits2d.stride(0),
                  1 if logits2d.dtype == torch.bfloat16 else 0, labels.data_ptr(), R, V, int(ignore_index), loss_rows.data_ptr(),
                  _lib.ptr(grad), W)
        # same validity predicate as the kernel: a label outside [0, V) that is not ignore_index contributes nothing
        count = ((labels != ignore_index) & (labels >= 0) & (labels < V)).sum().float()
        ctx.save_for_backward(grad, count)
        ctx.scaled = False
        return loss_rows.sum() / count        # every row ignored: 0 / 0 = nan, like torch

    @staticmethod
    def backward(ctx, gout):
        grad, count = ctx.saved_tensors
        return _scale_saved_grad(ctx, "cross_entropy", grad, gout, count), None, None, None


def _scale_saved_grad(ctx, what, grad, gout, divisor):
    """grad *= gout / divisor for the gradient a fused loss forward saved.  The (R, V) gradient (195 MB for the LM head) is
    scaled IN PLACE: one pass instead of a second tensor of that size; a second backward through the same node
    (retain_graph) would scale it twice, so it is refused."""
    if ctx.scaled:
        raise RuntimeError(f"ops.{what}: backward through the same graph twice is not supported (the saved "
                           "gradient buffer is consumed in place)")
    ctx.scaled = True
    scale = (gout.float() / divisor).reshape(1).contiguous()
    if grad.is_contiguous() and grad.numel() % 8 == 0 and grad.data_ptr() % 16 == 0:
        from . import _lib
        _lib.call(_lib.gps(), "sv_scale_inplace", grad.device, grad.data_ptr(), grad.numel(),
                  1 if grad.dtype == torch.bfloat16 else 0, scale.data_ptr())
        return grad
    return grad.mul_(scale.to(grad.dtype))


_BCE_COUNTERS = {}


def _bce_counter(device):
    """The zero-initialised completion counter of sv_bce_logits_fwd_bwd on `device` (the kernel leaves it at zero)."""
    c = _BCE_COUNTERS.get(device)
    if c is None:
        c = _BCE_COUNTERS[device] = torch.zeros(1, dtype=torch.int32, device=device)
    return c


class _BCEWithLogitsFn(torch.autograd.Function):
    """sum of binary cross-entropy with logits over (R, C) divided by R; loss and gradient from ONE native launch.  n_classes <
    logits.shape[1]: the trailing columns are padding (padded-vocabulary rows), ignored by the loss and zero in the gradient.
    The backward scales the saved gradient in place, as _CrossEntropyFn does."""

    @staticmethod
    def forward(ctx, logits2d, labels2d, weight_u8, n_classes):
        from . import _lib
        R, W = logits2d.shape
        dev = logits2d.device
        loss_rows = torch.empty(R, dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        grad = torch.empty((R, W), dtype=logits2d.dtype, device=dev) if logits2d.requires_grad else None
        _lib.call(_lib.gps(), "sv_bce_logits_fwd_bwd", dev, logits2d.data_ptr(), logits2d.stride(0),
                  1 if logits2d.dtype == torch.bfloat16 else 0, labels2d.data_ptr(), _lib.ptr(weight_u8), R, n_classes,
                  loss_rows.data_ptr(), loss.data_ptr(), _bce_counter(dev).data_ptr(), _lib.ptr(grad), W)
        ctx.save_for_backward(grad)
        ctx.rows, ctx.scaled = R, False
        return loss

    @staticmethod
    def backward(ctx, gout):
        (grad,) = ctx.saved_tensors
        return _scale_saved_grad(ctx, "bce_with_logits_sum", grad, gout, ctx.rows), None, None, None


def bce_with_logits_sum(logits, labels, weight=None):
    """F.binary_cross_entropy_with_logits(logits, labels.float(), weight=weight, reduction='sum') / logits.shape[0] for
    (R, C) logits and labels (optim/loss/loss.py:50-53 `answer_loss`; the ScanQA form of TextObjWithinBatch,
    contra_loss.py:33-34).  CUDA bf16 / f32 logits with int64 labels and a bool / uint8 weight: the fused native kernel,
    reading a padded-vocabulary row (ops.padded_vocab_linear) in place and returning the gradient in that padded layout;
    anything else: the torch formulation."""
    if logits.dim() != 2 or labels.shape != logits.shape or (weight is not None and weight.shape != logits.shape):
        raise ValueError(f"bce_with_logits_sum: logits {tuple(logits.shape)}, labels {tuple(labels.shape)} and weight "
                         f"{None if weight is None else tuple(weight.shape)} must be the same (R, C)")
    R, C = logits.shape
    src = logits
    padded = getattr(logits, "_sv_padded", None)
    if padded is not None and padded.is_cuda and padded.dim() == 2 and padded.shape[0] == R and padded.is_contiguous():
        src = padded
    native = src.is_cuda and src.dtype in (torch.bfloat16, torch.float32) and src.stride(1) == 1 and R > 0 and C > 0 and \
        labels.is_cuda and labels.dtype == torch.int64 and \
        (weight is None or (weight.is_cuda and weight.dtype in (torch.bool, torch.uint8)))
    if native:
        w = None if weight is None else weight.contiguous().view(torch.uint8)
        return _BCEWithLogitsFn.apply(src, labels.contiguous(), w, C)
    return F.binary_cross_entropy_with_logits(logits, labels.float(), weight=weight, reduction='sum') / logits.shape[0]


_MASKED_CE_COUNTERS = {}


class _MaskedCrossEntropyFn(torch.autograd.Function):
    """sum_r w_r CE_r / sum_r w_r over (R, W) logits; loss, weight sum and unscaled gradient from ONE native launch
    (sv_masked_cross_entropy_fwd_bwd).  n_classes < W: the trailing columns are padding, ignored by the loss and zero in the
    gradient.  The backward divides the saved gradient in place by the device weight sum, as _CrossEntropyFn does."""

    @staticmethod
    def forward(ctx, logits2d, labels, obj_u8, sem_u8, mode, n_classes):
        from . import _lib
        R, W = logits2d.shape
        dev = logits2d.device
        counter = _MASKED_CE_COUNTERS.get(dev)
        if counter is None:       # zero-initialised; the kernel leaves it at zero
            counter = _MASKED_CE_COUNTERS[dev] = torch.zeros(1, dtype=torch.int32, device=dev)
        loss_rows = torch.empty(R, dtype=torch.float32, device=dev)
        sums = torch.empty(2, dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        grad = torch.empty((R, W), dtype=logits2d.dtype, device=dev) if logits2d.requires_grad else None
        _lib.call(_lib.gps(), "sv_masked_cross_entropy_fwd_bwd", dev, logits2d.data_ptr(), logits2d.stride(0),
                  1 if logits2d.dtype == torch.bfloat16 else 0, labels.data_ptr(), obj_u8.data_ptr(), _lib.ptr(sem_u8),
                  int(mode), R, n_classes, loss_rows.data_ptr(), sums.data_ptr(), loss.data_ptr(), counter.data_ptr(),
                  _lib.ptr(grad), W)
        ctx.save_for_backward(grad, sums[1])
        ctx.scaled = False
        return loss

    @staticmethod
    def backward(ctx, gout):
        grad, wsum = ctx.saved_tensors
        return _scale_saved_grad(ctx, "masked_cross_entropy", grad, gout, wsum), None, None, None, None, None


def _masked_cross_entropy_torch(logits, labels, obj_masks, sem_masks, mode):
    """The reference's expression (optim/loss/loss.py:26-47, 64-94), unchanged."""
    ce = F.cross_entropy(logits.permute(0, 2, 1), labels, reduction='none')
    if mode == 0:
        return (ce * obj_masks).sum() / obj_masks.sum()
    sem = sem_masks.logical_not() if mode == 1 else sem_masks
    return (ce * obj_masks * sem).sum() / (obj_masks * sem).sum()


def masked_cross_entropy(logits, labels, obj_masks, sem_masks=None, mode=0):
    """The object-classification losses of optim/loss/loss.py: (F.cross_entropy(logits.permute(0, 2, 1), labels,
    reduction='none') * w).sum() / w.sum() for (B, O, V) logits, (B, O) int64 labels (-100 = padded slot) and (B, O) bool
    masks, with w = obj_masks (mode 0), obj_masks & ~sem_masks (mode 1, the `_mask` losses) or obj_masks & sem_masks (mode 2,
    the `_unmask` losses).  w.sum() = 0 gives NaN, as in the reference.  CUDA bf16 / f32 logits: one native launch
    (sv_masked_cross_entropy_fwd_bwd), reading a padded-vocabulary row (`_sv_padded`) in place and returning the gradient in
    that layout, no gradient buffer when the logits need none; anything else: the reference's torch expression."""
    if mode not in (0, 1, 2):
        raise ValueError(f"masked_cross_entropy: mode must be 0, 1 or 2, got {mode!r}")
    if mode != 0 and sem_masks is None:
        raise ValueError("masked_cross_entropy: modes 1 and 2 need sem_masks")
    if logits.dim() != 3 or labels.shape != logits.shape[:2] or obj_masks.shape != labels.shape or \
            (sem_masks is not None and sem_masks.shape != labels.shape):
        raise ValueError(f"masked_cross_entropy: logits {tuple(logits.shape)} must be (B, O, V) with labels "
                         f"{tuple(labels.shape)}, obj_masks {tuple(obj_masks.shape)} and sem_masks "
                         f"{None if sem_masks is None else tuple(sem_masks.shape)} all (B, O)")
    B, O, V = logits.shape
    src = logits
    padded = getattr(logits, "_sv_padded", None)
    if padded is not None and padded.dim() == 3 and padded.shape[:2] == (B, O) and padded.is_contiguous():
        src = padded
    src2d = src.reshape(B * O, src.shape[-1]) if src.stride(-1) == 1 else None
    native = src2d is not None and src2d.is_cuda and src2d.dtype in (torch.bfloat16, torch.float32) and \
        src2d.stride(1) == 1 and B * O > 0 and labels.is_cuda and labels.dtype == torch.int64 and \
        obj_masks.is_cuda and obj_masks.dtype in (torch.bool, torch.uint8) and \
        (mode == 0 or (sem_masks.is_cuda and sem_masks.dtype in (torch.bool, torch.uint8)))
    if not native:
        return _masked_cross_entropy_torch(logits, labels, obj_masks, sem_masks, mode)
    obj_u8 = obj_masks.contiguous().view(torch.uint8).reshape(-1)
    sem_u8 = None if mode == 0 else sem_masks.contiguous().view(torch.uint8).reshape(-1)
    return _MaskedCrossEntropyFn.apply(src2d, labels.reshape(-1).contiguous(), obj_u8, sem_u8, mode, V)


class _AttentionPoolFn(torch.autograd.Function):
    """pooled = sum_l softmax_l(masked score) x_l for one glimpse (modules/heads/qa_head.py:57-69), one native launch per
    direction.  `scores` is the PADDED (B, L, 8) output of the N = 1 score linear; its gradient is returned in that layout."""

    @staticmethod
    def forward(ctx, scores, x, pad_mask_u8):
        from . import _lib
        B, L, D = x.shape
        p = torch.empty((B, L), dtype=torch.float32, device=x.device)
        pooled = torch.empty((B, D), dtype=torch.bfloat16, device=x.device)
        _lib.call(_lib.gps(), "sv_attn_pool_fwd", x.device, scores.data_ptr(), scores.shape[-1], x.data_ptr(), x.stride(0),
                  x.stride(1), _lib.ptr(pad_mask_u8), B, L, D, p.data_ptr(), pooled.data_ptr())
        ctx.save_for_backward(x, p, pad_mask_u8)
        ctx.score_w = scores.shape[-1]
        return pooled

    @staticmethod
    def backward(ctx, g):
        from . import _lib
        x, p, mask = ctx.saved_tensors
        B, L, D = x.shape
        g = g.to(torch.bfloat16)
        if g.stride(1) != 1 or g.stride(0) % 8 or g.data_ptr() % 16:
            g = g.contiguous()
        dx = torch.empty((B, L, D), dtype=torch.bfloat16, device=x.device)
        dscore = torch.empty((B, L, ctx.score_w), dtype=torch.bfloat16, device=x.device)
        _lib.call(_lib.gps(), "sv_attn_pool_bwd", x.device, g.data_ptr(), g.stride(0), p.data_ptr(), x.data_ptr(), x.stride(0),
                  x.stride(1), _lib.ptr(mask), B, L, D, dx.data_ptr(), dscore.data_ptr(), ctx.score_w)
        return dscore, dx, None


def _attention_pool_torch(att, x, pad_mask):
    if pad_mask is not None:
        att = att.masked_fill(pad_mask.unsqueeze(2), -1e9)
    att = torch.softmax(att.float(), dim=1).to(x.dtype)
    return torch.einsum("blg,bld->bgd", att, x).flatten(1)                      # glimpse-major, like the reference's cat


def attention_pool(scores, x, pad_mask=None):
    """AttFlat's pooling (modules/heads/qa_head.py:57-69): scores (B, L, G) of the score MLP, x (B, L, D) tokens, pad_mask
    (B, L) bool, True = padding -> (B, G*D), the softmax over L in fp32 with masked scores set to -1e9.  CUDA under bf16 with
    G = 1 and scores from ops.padded_vocab_linear (the padded parent is read in place): one native kernel per direction;
    otherwise (CPU, the fp32 parity path, G > 1, shapes the kernels reject) the torch formulation."""
    padded = getattr(scores, "_sv_padded", None)
    B, L, D = x.shape
    if padded is not None and scores.shape[-1] == 1 and padded.dim() == 3 and padded.shape[:2] == (B, L) and \
            padded.is_contiguous() and padded.dtype == torch.bfloat16 and x.is_cuda and D % 8 == 0 and 1 <= L <= 8192 and \
            B > 0 and (x.dtype == torch.bfloat16 or (_autocast_on() and x.dtype == torch.float32)) and \
            (pad_mask is None or (pad_mask.is_cuda and pad_mask.dtype == torch.bool and pad_mask.shape == (B, L))):
        xb = x if x.dtype == torch.bfloat16 else x.to(torch.bfloat16)
        if xb.stride(2) != 1 or xb.stride(1) % 8 or xb.stride(0) % 8 or xb.data_ptr() % 16:
            xb = xb.contiguous()
        m = None if pad_mask is None else pad_mask.contiguous().view(torch.uint8)
        return _AttentionPoolFn.apply(padded, xb, m)
    return _attention_pool_torch(scores, x, pad_mask)


def padded_vocab_linear(h, weight, bias):
    """(..., K) -> (..., V) logits of a wide classifier (BERT LM head, modules/heads/pretrain_head.py:22-32: decoder + bias).
    On the native path the GEMM writes rows padded to a multiple of 8 classes (16-byte rows, pad columns zero); the returned
    tensor is the (..., :V) view and carries the padded parent as `_sv_padded`, which ops.cross_entropy uses to produce the
    gradient directly in the padded layout the backward GEMMs read."""
    V = weight.shape[0]
    if _native_linear_ok(h, weight):
        lp = _LinearFn.apply(h, weight, bias, None)
        if lp.shape[-1] == V:
            # no pad columns: nothing to carry (and `lp._sv_padded = lp` would be a reference cycle that keeps the whole
            # autograd graph alive until the next garbage collection — fatal for a CUDA-graph capture that follows)
            return lp
        out = lp[..., :V]
        out._sv_padded = lp
        return out
    return linear(h, weight, bias)


class _LayerNormFn(torch.autograd.Function):
    """y = LayerNorm(residual + dropout(x)) in one native pass; the backward regenerates the dropout mask and produces
    d(x), d(residual), d(gamma), d(beta) (gamma / beta partial sums reduced in a fixed order).  Row r draws the dropout
    mask of row r * key_stride."""

    @staticmethod
    def forward(ctx, x, residual, gamma, beta, eps, p, seed, key_stride=1):
        from . import _lib
        D = x.shape[-1]
        x2 = x.reshape(-1, D)
        R = x2.shape[0]
        r2 = residual.reshape(-1, D) if residual is not None else None
        need_s = r2 is not None or p > 0.0
        y = torch.empty_like(x2)
        s = torch.empty_like(x2) if need_s else None
        stats = torch.empty((2, R), dtype=torch.float32, device=x.device)
        _lib.call(_lib.gps(), "sv_layer_norm_fwd_rows", x.device, x2.data_ptr(), _lib.ptr(r2),
                  1 if x.dtype == torch.bfloat16 else 0, R, D, gamma.data_ptr(), beta.data_ptr(), float(eps), float(p), int(seed),
                  y.data_ptr(), _lib.ptr(s), stats[0].data_ptr(), stats[1].data_ptr(), int(key_stride))
        ctx.save_for_backward(s if need_s else x2, gamma, stats)
        ctx.meta = (float(p), int(seed), residual is not None, x.shape, int(key_stride))
        ctx.params = (gamma, beta)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, g):
        from . import _lib
        s, gamma, stats = ctx.saved_tensors
        p, seed, has_res, shape, key_stride = ctx.meta
        R, D = s.shape
        g2 = g.reshape(R, D).to(s.dtype).contiguous()
        ds = torch.empty_like(s)
        dx = torch.empty_like(s) if p > 0.0 else None
        pg, pb = ctx.params
        direct = _direct(pg) and _direct(pb)        # gamma / beta gradients accumulate straight into the flat buffer
        dgb = None if direct else torch.empty((2, D), dtype=torch.float32, device=s.device)
        dg_t, db_t = (pg.grad, pb.grad) if direct else (dgb[0], dgb[1])
        lib = _lib.gps()
        scratch = torch.empty(lib.sv_layer_norm_scratch_floats(D), dtype=torch.float32, device=s.device)
        _lib.call(lib, "sv_layer_norm_bwd_rows", s.device, g2.data_ptr(), s.data_ptr(), 1 if s.dtype == torch.bfloat16 else 0,
                  R, D, gamma.data_ptr(), stats[0].data_ptr(), stats[1].data_ptr(), p, seed, ds.data_ptr(), _lib.ptr(dx),
                  dg_t.data_ptr(), db_t.data_ptr(), 1 if direct else 0, scratch.data_ptr(), key_stride)
        d_x = (dx if dx is not None else ds).view(shape)
        return d_x, (ds.view(shape) if has_res else None), (None if direct else dgb[0]), (None if direct else dgb[1]), None, \
            None, None, None


def _autocast_on():
    try:
        return torch.is_autocast_enabled("cuda")
    except TypeError:
        return torch.is_autocast_enabled()


def layer_norm(x, weight, bias, eps=1e-5, residual=None, dropout_p=0.0, row_key_stride=1):
    """LayerNorm(residual + dropout(x)) * weight + bias over the last dimension (post-norm block tail of
    transformers.py:145-154,311-315; plain LayerNorm with residual=None, dropout_p=0).  The caller passes dropout_p = 0
    outside training.  CUDA: one native kernel, I/O in bf16 under autocast / for bf16 inputs (statistics in fp32), else
    fp32; row r of the flattened input draws the dropout mask of row r * row_key_stride (the first token of each sequence
    of a (B, L, D) tensor: x of shape (B, 1, D), row_key_stride = L).  CPU: the torch formulation."""
    D = x.shape[-1]
    if x.is_cuda and D % 8 == 0 and 8 <= D <= 1024 and weight is not None and bias is not None and x.numel() > 0 and \
            x.dtype in (torch.bfloat16, torch.float32, torch.float16):
        low = x.dtype != torch.float32 or (residual is not None and residual.dtype != torch.float32) or _autocast_on()
        dt = torch.bfloat16 if low else torch.float32
        x_ = x.to(dt).contiguous()
        r_ = None
        if residual is not None:
            r_ = residual.to(dt).expand_as(x_).contiguous()
        return _LayerNormFn.apply(x_, r_, weight.float().contiguous(), bias.float().contiguous(), eps, float(dropout_p),
                                  _next_dropout_seed() if dropout_p > 0.0 else 0, row_key_stride)
    s = x if dropout_p == 0.0 else F.dropout(x, dropout_p, True)
    if residual is not None:
        s = residual + s
    return F.layer_norm(s, (D,), weight, bias, eps)


class _L2NormalizeFn(torch.autograd.Function):
    """y = x / max(||x||_2, eps) over the last dimension (csrc/layer_norm.cu l2norm_fwd / l2norm_bwd)."""

    @staticmethod
    def forward(ctx, x, eps):
        from . import _lib
        D = x.shape[-1]
        x2 = x.reshape(-1, D).contiguous()
        R = x2.shape[0]
        y = torch.empty_like(x2)
        norm = torch.empty(R, dtype=torch.float32, device=x.device)
        _lib.call(_lib.gps(), "sv_l2norm_fwd", x.device, x2.data_ptr(), int(x2.dtype == torch.bfloat16), R, D, float(eps),
                  y.data_ptr(), norm.data_ptr())
        ctx.save_for_backward(y, norm)
        ctx.eps, ctx.shape = float(eps), x.shape
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, grad):
        from . import _lib
        y, norm = ctx.saved_tensors
        R, D = y.shape
        g2 = grad.reshape(R, D).to(y.dtype).contiguous()
        dx = torch.empty_like(y)
        _lib.call(_lib.gps(), "sv_l2norm_bwd", y.device, g2.data_ptr(), y.data_ptr(), norm.data_ptr(),
                  int(y.dtype == torch.bfloat16), R, D, ctx.eps, dx.data_ptr())
        return dx.view(ctx.shape), None


def l2_normalize(x, eps=1e-12):
    """F.normalize(x, dim=-1, p=2, eps=eps) (the contrastive heads of optim/loss/contra_loss.py:29-30,59-60,86-87).  CUDA, bf16 / fp32,
    last dimension a multiple of 8 up to 1024: one native kernel per direction; otherwise torch."""
    D = x.shape[-1]
    if x.is_cuda and x.dtype in (torch.bfloat16, torch.float32) and D % 8 == 0 and 8 <= D <= 1024 and x.numel() > 0:
        return _L2NormalizeFn.apply(x, eps)
    return F.normalize(x, dim=-1, p=2, eps=eps)


def cross_entropy(logits, labels, ignore_index=-100):
    """F.cross_entropy(logits.permute(0, 2, 1) / logits, labels, ignore_index=...) with the class dimension LAST in
    `logits` ((..., V) with (...) matching labels).  CUDA bf16/f32 -> fused native kernel; otherwise torch."""
    V = logits.shape[-1]
    padded = getattr(logits, "_sv_padded", None)
    if padded is not None and padded.is_cuda and padded.shape[:-1] == logits.shape[:-1] and padded.is_contiguous():
        return _CrossEntropyFn.apply(padded.view(-1, padded.shape[-1]), labels.reshape(-1).contiguous(), ignore_index, V)
    if logits.is_cuda and logits.dtype in (torch.bfloat16, torch.float32) and logits.stride(-1) == 1:
        l2 = logits.reshape(-1, V)
        if l2.stride(1) == 1:
            return _CrossEntropyFn.apply(l2, labels.reshape(-1).contiguous(), ignore_index, 0)
    return F.cross_entropy(logits.reshape(-1, V).float(), labels.reshape(-1), ignore_index=ignore_index)


class _SceneBroadcastFn(torch.autograd.Function):
    """(B, O, D) -> (B*U, O, D): forward one expand copy, backward the sum over the U copies of each scene
    (csrc/colsum.cu sv_colsum_batched: fp32 accumulation in a fixed order, written in the gradient's dtype)."""

    @staticmethod
    def forward(ctx, x, U):
        B = x.shape[0]
        ctx.shape = (B, int(U)) + tuple(x.shape[1:])
        return x.unsqueeze(1).expand(ctx.shape).reshape((B * U,) + tuple(x.shape[1:]))

    @staticmethod
    def backward(ctx, g):
        from . import native
        B, U = ctx.shape[:2]
        rest = ctx.shape[2:]
        g3 = g.reshape(B, U, -1).contiguous()
        if g3.dtype not in (torch.bfloat16, torch.float32):
            g3 = g3.float()
        elif g3.data_ptr() % 16:
            g3 = g3.clone()
        return native.colsum_batched(g3).view((B,) + rest).to(g.dtype), None


def scene_broadcast(x, U):
    """The per-scene repeat of model/openvocab.py:170-173 (reference): (B, O, D) object features -> (B*U, O, D), every scene's
    rows repeated for its U utterances (row b*U + u = x[b]).  CUDA: the gradient is summed over U by one native reduction;
    otherwise torch.  A tensor that needs no gradient can be expanded as a view instead."""
    if x.is_cuda:
        return _SceneBroadcastFn.apply(x, int(U))
    B = x.shape[0]
    return x.unsqueeze(1).expand((B, int(U)) + tuple(x.shape[1:])).reshape((B * int(U),) + tuple(x.shape[1:]))
