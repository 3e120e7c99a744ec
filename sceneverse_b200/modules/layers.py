"""Attention / transformer layers of the GPS stack (reference: modules/layers/transformers.py,
modules/utils.py).  Same constructor arguments, forward contracts and parameter names
(SURVEY.md §8b: `self_attn.{w_qs,w_ks,w_vs,fc,lang_cond_fc}`, `self_attn.{in_proj_weight,in_proj_bias,
out_proj.*}`, `linear1/2`, `norm1/2/3`), so reference checkpoints load unchanged.

The arithmetic is routed through `sceneverse_b200.ops` (fused CUDA where a native kernel exists);
everything here is host-side composition.
"""
import copy
import math

import torch
import torch.nn.functional as F
from torch import nn

from .. import ops


def get_activation_fn(activation_type):
    if activation_type not in ["relu", "gelu", "glu"]:
        raise RuntimeError(f"activation function currently support relu/gelu, not {activation_type}")
    return getattr(F, activation_type)


class Linear(nn.Linear):
    """nn.Linear (same parameters / state_dict) routed through ops.linear (native bias gradient, fp32 weight gradient)."""

    def forward(self, x):
        return ops.linear(x, self.weight, self.bias)


class Embedding(nn.Embedding):
    """nn.Embedding (same parameters / state_dict) whose backward is the native scatter-add (ops.embedding)."""

    def forward(self, ids):
        if self.max_norm is not None or self.sparse or self.scale_grad_by_freq:
            return super().forward(ids)
        return ops.embedding(ids, self.weight, self.padding_idx)


def route_linears(module):
    """Re-class every plain nn.Linear / nn.Embedding below `module` (incl. third-party sub-modules such as the HF BERT
    blocks) so that their arithmetic goes through sceneverse_b200.ops."""
    for m in module.modules():
        if type(m) is nn.Linear:
            m.__class__ = Linear
        elif type(m) is nn.Embedding:
            m.__class__ = Embedding
    return module


class LayerNorm(nn.LayerNorm):
    """nn.LayerNorm (same parameters / state_dict) whose forward is the fused native dropout + residual + LayerNorm:
    norm(x, residual=r, dropout_p=p) == LayerNorm(r + dropout(x)); row_key_stride as in ops.layer_norm."""

    def forward(self, x, residual=None, dropout_p=0.0, row_key_stride=1):
        return ops.layer_norm(x, self.weight, self.bias, self.eps, residual=residual, dropout_p=dropout_p,
                              row_key_stride=row_key_stride)


def get_mlp_head(input_size, hidden_size, output_size, dropout=0):
    """modules/utils.py:18-25 (note LayerNorm eps=1e-12)."""
    return nn.Sequential(nn.Linear(input_size, hidden_size), nn.ReLU(), LayerNorm(hidden_size, eps=1e-12),
                         nn.Dropout(dropout), nn.Linear(hidden_size, output_size))


def layer_repeat(module, N, share_layer=False):
    if share_layer:
        return nn.ModuleList([module] * N)
    return nn.ModuleList([copy.deepcopy(module) for _ in range(N - 1)] + [module])


def init_weights_bert(module, std=0.02):
    """modules/weights.py:3-20."""
    if isinstance(module, nn.Linear):
        module.weight.data.normal_(mean=0.0, std=std)
        if module.bias is not None:
            module.bias.data.zero_()
    elif isinstance(module, nn.Embedding):
        module.weight.data.normal_(mean=0.0, std=std)
        if module.padding_idx is not None:
            module.weight.data[module.padding_idx].zero_()
    elif isinstance(module, nn.LayerNorm):
        module.bias.data.zero_()
        module.weight.data.fill_(1.0)


calc_pairwise_locs = ops.calc_pairwise_locs


class MultiheadAttention(nn.Module):
    """Drop-in for the reference's use of nn.MultiheadAttention(d_model, nhead, dropout, batch_first=True)
    (transformers.py:22-24,69-74,118-120): packed in-projection, key-padding mask, attention-weight dropout.
    Returns (output, None): every reference caller discards the averaged attention map."""

    def __init__(self, embed_dim, num_heads, dropout=0.0, batch_first=True, kdim=None, vdim=None):
        super().__init__()
        assert batch_first and (kdim in (None, embed_dim)) and (vdim in (None, embed_dim))
        self.embed_dim, self.num_heads, self.dropout = embed_dim, num_heads, dropout
        self.in_proj_weight = nn.Parameter(torch.empty(3 * embed_dim, embed_dim))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * embed_dim))
        self.out_proj = nn.Linear(embed_dim, embed_dim)
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.zeros_(self.out_proj.bias)

    def forward(self, query, key, value, attn_mask=None, key_padding_mask=None):
        assert attn_mask is None
        E, H = self.embed_dim, self.num_heads
        w, b = self.in_proj_weight, self.in_proj_bias
        if key is query and value is query:
            # packed projection -> attention on the packed tensor: one dgrad + one wgrad GEMM in the backward
            out = ops.attention_packed(ops.linear(query, w, b), H, key_padding_mask=key_padding_mask,
                                       dropout_p=self.dropout if self.training else 0.0)
            return ops.linear(out, self.out_proj.weight, self.out_proj.bias), None
        else:
            q = ops.linear(query, w[:E], b[:E])
            k, v = ops.linear(key, w[E:], b[E:]).split(E, dim=-1) if key is value else \
                (ops.linear(key, w[E:2 * E], b[E:2 * E]), ops.linear(value, w[2 * E:], b[2 * E:]))
        out = ops.attention(q, k, v, H, key_padding_mask=key_padding_mask,
                            dropout_p=self.dropout if self.training else 0.0)
        return ops.linear(out, self.out_proj.weight, self.out_proj.bias), None


class MultiHeadAttentionSpatial(nn.Module):
    """transformers.py:157-239, `spatial_attn_fusion='cond'` (the only fusion the GPS configs build,
    pcd_openvocab_encoder.py:77-83, unified_encoder.py:23-26,69-72)."""

    def __init__(self, d_model, n_head, dropout=0.1, spatial_multihead=True, spatial_dim=5, spatial_attn_fusion='mul'):
        super().__init__()
        assert d_model % n_head == 0, 'd_model: %d, n_head: %d' % (d_model, n_head)
        if spatial_attn_fusion != 'cond':
            raise NotImplementedError("only spatial_attn_fusion='cond' is on the GPS path")
        self.n_head, self.d_model, self.d_per_head = n_head, d_model, d_model // n_head
        self.spatial_multihead, self.spatial_dim, self.spatial_attn_fusion = spatial_multihead, spatial_dim, spatial_attn_fusion
        self.w_qs = nn.Linear(d_model, d_model)
        self.w_ks = nn.Linear(d_model, d_model)
        self.w_vs = nn.Linear(d_model, d_model)
        self.fc = nn.Linear(d_model, d_model)
        self.spatial_n_head = n_head if spatial_multihead else 1
        self.lang_cond_fc = nn.Linear(d_model, self.spatial_n_head * (spatial_dim + 1))

    def forward(self, q, k, v, pairwise_locs, key_padding_mask=None, txt_embeds=None):
        residual = q
        sw = ops.linear(residual, self.lang_cond_fc.weight, self.lang_cond_fc.bias)  # (b,l,h*(d+1)): [bias,w1..wd] per head
        if k is q and v is q:    # self-attention (every GPS call site): the three projections are one GEMM
            qkv = ops.linear_packed(q, [self.w_qs, self.w_ks, self.w_vs])
            out, attn = ops.spatial_attention_packed(qkv, sw, pairwise_locs, self.n_head, self.spatial_n_head,
                                                     key_padding_mask=key_padding_mask)
            return ops.linear(out, self.fc.weight, self.fc.bias), attn
        qh = ops.linear(q, self.w_qs.weight, self.w_qs.bias)
        kh = ops.linear(k, self.w_ks.weight, self.w_ks.bias)
        vh = ops.linear(v, self.w_vs.weight, self.w_vs.bias)
        out, attn = ops.spatial_attention(qh, kh, vh, sw, pairwise_locs, self.n_head, self.spatial_n_head,
                                          key_padding_mask=key_padding_mask)
        return ops.linear(out, self.fc.weight, self.fc.bias), attn


class TransformerEncoderLayer(nn.Module):
    """transformers.py:115-154."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, batch_first=True, dropout=0.1, activation="relu",
                 prenorm=False):
        super().__init__()
        self.self_attn = MultiheadAttention(d_model, nhead, dropout=dropout, batch_first=batch_first)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1 = LayerNorm(d_model)
        self.norm2 = LayerNorm(d_model)
        self.dropout1 = nn.Dropout(dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.activation_name = activation
        self.activation = get_activation_fn(activation)
        self.prenorm = prenorm

    def _ffn(self, x):
        return ops.ffn(x, self.linear1.weight, self.linear1.bias, self.linear2.weight, self.linear2.bias,
                       activation=self.activation_name, dropout_p=self.dropout.p if self.training else 0.0)

    def forward(self, tgt, tgt_mask=None, tgt_key_padding_mask=None):
        tgt2 = self.norm1(tgt) if self.prenorm else tgt
        tgt2, attn = self.self_attn(tgt2, tgt2, tgt2, attn_mask=tgt_mask, key_padding_mask=tgt_key_padding_mask)
        if self.prenorm:
            tgt = self.norm2(tgt + self.dropout1(tgt2))
            return tgt + self.dropout2(self._ffn(tgt)), attn
        tgt = self.norm1(tgt2, residual=tgt, dropout_p=self._p(self.dropout1))
        tgt = self.norm2(self._ffn(tgt), residual=tgt, dropout_p=self._p(self.dropout2))
        return tgt, attn

    def _p(self, drop):
        return drop.p if self.training else 0.0


class TransformerSpatialEncoderLayer(TransformerEncoderLayer):
    """transformers.py:285-316 (post-norm; the spatial attention ignores its `dropout` argument)."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", spatial_multihead=True,
                 spatial_dim=5, spatial_attn_fusion='mul'):
        super().__init__(d_model, nhead, dim_feedforward=dim_feedforward, dropout=dropout, activation=activation)
        del self.self_attn
        self.self_attn = MultiHeadAttentionSpatial(d_model, nhead, dropout=dropout, spatial_multihead=spatial_multihead,
                                                   spatial_dim=spatial_dim, spatial_attn_fusion=spatial_attn_fusion)

    def forward(self, tgt, tgt_pairwise_locs, tgt_mask=None, tgt_key_padding_mask=None):
        tgt2, attn = self.self_attn(tgt, tgt, tgt, tgt_pairwise_locs, key_padding_mask=tgt_key_padding_mask)
        tgt = self.norm1(tgt2, residual=tgt, dropout_p=self._p(self.dropout1))
        tgt = self.norm2(self._ffn(tgt), residual=tgt, dropout_p=self._p(self.dropout2))
        return tgt, attn


class TransformerDecoderLayer(nn.Module):
    """transformers.py:66-112 (pre-norm self-attention, cross-attention to `memory`, FFN)."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu"):
        super().__init__()
        self.self_attn = MultiheadAttention(d_model, nhead, dropout=dropout, batch_first=True)
        self.multihead_attn = MultiheadAttention(d_model, nhead, dropout=dropout, batch_first=True)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1 = LayerNorm(d_model)
        self.norm2 = LayerNorm(d_model)
        self.norm3 = LayerNorm(d_model)
        self.dropout1 = nn.Dropout(dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.dropout3 = nn.Dropout(dropout)
        self.activation_name = activation
        self.activation = get_activation_fn(activation)

    def _self_attention(self, x, pairwise_locs, key_padding_mask):
        return self.self_attn(x, x, x, key_padding_mask=key_padding_mask)

    def forward(self, tgt, memory, tgt_pairwise_locs=None, tgt_mask=None, memory_mask=None, tgt_key_padding_mask=None,
                memory_key_padding_mask=None):
        tgt2, sa = self._self_attention(self.norm1(tgt), tgt_pairwise_locs, tgt_key_padding_mask)
        tgt = tgt + self.dropout1(tgt2)
        tgt2, ca = self.multihead_attn(self.norm2(tgt), memory, memory, key_padding_mask=memory_key_padding_mask)
        tgt = tgt + self.dropout2(tgt2)
        tgt = tgt + self.dropout3(ops.ffn(self.norm3(tgt), self.linear1.weight, self.linear1.bias, self.linear2.weight,
                                          self.linear2.bias, activation=self.activation_name,
                                          dropout_p=self.dropout.p if self.training else 0.0))
        return tgt, sa, ca


class TransformerSpatialDecoderLayer(TransformerDecoderLayer):
    """transformers.py:242-282."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", spatial_multihead=True,
                 spatial_dim=5, spatial_attn_fusion='mul'):
        super().__init__(d_model, nhead, dim_feedforward=dim_feedforward, dropout=dropout, activation=activation)
        del self.self_attn
        self.self_attn = MultiHeadAttentionSpatial(d_model, nhead, dropout=dropout, spatial_multihead=spatial_multihead,
                                                   spatial_dim=spatial_dim, spatial_attn_fusion=spatial_attn_fusion)

    def _self_attention(self, x, pairwise_locs, key_padding_mask):
        return self.self_attn(x, x, x, pairwise_locs, key_padding_mask=key_padding_mask)
