"""Task heads (reference: modules/heads/grounding_head.py:7-55, modules/heads/pretrain_head.py:8-56)."""
import torch
from torch import nn

from .. import ops
from .layers import LayerNorm, get_mlp_head
from .registry import HEADS_REGISTRY


@HEADS_REGISTRY.register()
class GroundHeadV1(nn.Module):
    def __init__(self, cfg, input_size=768, hidden_size=768, sem_cls_size=607, dropout=0.3, detach_all_aux_loss=False):
        super().__init__()
        self.og3d_head = get_mlp_head(input_size, hidden_size, 1, dropout=dropout)
        self.txt_clf_head = get_mlp_head(input_size, hidden_size, sem_cls_size, dropout=dropout)
        self.obj3d_clf_head = get_mlp_head(input_size, hidden_size, sem_cls_size, dropout=dropout)
        self.obj3d_clf_pre_head = get_mlp_head(input_size, hidden_size, sem_cls_size, dropout=dropout)
        self.detach_all_aux_loss = detach_all_aux_loss

    def forward(self, txt_embeds, obj_embeds, obj_pre_embeds, obj_masks, **kwargs):
        og3d_logits = self.og3d_head(obj_embeds).squeeze(2)
        og3d_logits = og3d_logits.masked_fill_(obj_masks.logical_not(), -float('inf'))
        if self.detach_all_aux_loss:
            txt_embeds, obj_embeds, obj_pre_embeds = txt_embeds.detach(), obj_embeds.detach(), obj_pre_embeds.detach()
        return (self.txt_clf_head(txt_embeds[:, 0]), self.obj3d_clf_head(obj_embeds),
                self.obj3d_clf_pre_head(obj_pre_embeds), og3d_logits)


@HEADS_REGISTRY.register()
class GroundHead(nn.Module):
    def __init__(self, cfg, input_size=768, hidden_size=768, dropout=0.3):
        super().__init__()
        self.og3d_head = get_mlp_head(input_size, hidden_size, 1, dropout=dropout)

    def forward(self, obj_embeds, obj_masks=None, **kwargs):
        og3d_logits = self.og3d_head(obj_embeds).squeeze(2)
        if obj_masks is not None:
            og3d_logits = og3d_logits.masked_fill_(obj_masks.logical_not(), -float('inf'))
        return og3d_logits


class _Transform(nn.Module):
    """dense -> gelu -> LayerNorm; parameter names `dense.*`, `LayerNorm.*` as in pretrain_head.py:8-19."""

    def __init__(self, width):
        super().__init__()
        self.dense, self.LayerNorm = nn.Linear(width, width), LayerNorm(width)


class BertLMPredictionHead(nn.Module):
    """BERT masked-LM head (pretrain_head.py:22-32): logits = decoder(LayerNorm(gelu(dense(h)))) + bias, with the
    state_dict keys `transform.dense.*`, `transform.LayerNorm.*`, `decoder.weight`, `bias`.  The dense+gelu and the
    decoder+bias steps go through `ops.linear` so that they pick up fused epilogues."""

    def __init__(self, hidden_size, vocab_size):
        super().__init__()
        self.transform = _Transform(hidden_size)
        self.decoder = nn.Linear(hidden_size, vocab_size, bias=False)
        self.bias = nn.Parameter(torch.zeros(vocab_size))

    def forward(self, hidden_states):
        t = self.transform
        h = t.LayerNorm(ops.linear(hidden_states, t.dense.weight, t.dense.bias, activation="gelu"))
        return ops.padded_vocab_linear(h, self.decoder.weight, self.bias)


def _lm_heads(owner, hidden_size, **vocabs):
    for name, size in vocabs.items():
        setattr(owner, name, BertLMPredictionHead(hidden_size, size))


@HEADS_REGISTRY.register()
class PretrainHeadV1(nn.Module):
    def __init__(self, cfg, hidden_size=768, vocab_size=30522):
        super().__init__()
        _lm_heads(self, hidden_size, lm_pred_head=vocab_size)

    def forward(self, txt_embeds, **kwargs):
        return self.lm_pred_head(txt_embeds)


@HEADS_REGISTRY.register()
class OVPretrainHead(nn.Module):
    def __init__(self, cfg, hidden_size=768, vocab_size=30522, obj_vocab_size=607):
        super().__init__()
        _lm_heads(self, hidden_size, lm_pred_head=vocab_size, obj_pred_head=obj_vocab_size)

    def forward(self, txt_embeds, obj_embeds, **kwargs):
        return self.lm_pred_head(txt_embeds), self.obj_pred_head(obj_embeds)


class _AttentionPool(nn.Module):
    """Masked soft-attention pooling over a token axis followed by a merge projection (reference: qa_head.py:42-70;
    parameter names `mlp.fc.linear.*`, `mlp.linear.*`, `linear_merge.*` kept for checkpoint compatibility).  One score
    MLP (hidden -> mid -> glimpses, GELU + dropout), scores of masked tokens set to -1e9 before the softmax over tokens;
    the glimpse-weighted sums are one batched contraction instead of the reference's per-glimpse loop + cat (ops.attention_pool:
    one native kernel per direction for one glimpse, reading the padded score rows of the N = 1 linear in place)."""

    def __init__(self, hidden_size, mid_size=512, glimpses=1, out_size=1024, pdrop=0.1):
        super().__init__()
        self.mlp = nn.Module()
        self.mlp.fc = nn.Module()
        self.mlp.fc.linear = nn.Linear(hidden_size, mid_size)
        self.mlp.linear = nn.Linear(mid_size, glimpses)
        self.linear_merge = nn.Linear(hidden_size * glimpses, out_size)
        self.pdrop = pdrop

    def forward(self, x, pad_mask):
        h = ops.linear(x, self.mlp.fc.linear.weight, self.mlp.fc.linear.bias, activation="gelu")
        if self.pdrop > 0:
            h = nn.functional.dropout(h, self.pdrop, self.training)
        att = ops.padded_vocab_linear(h, self.mlp.linear.weight, self.mlp.linear.bias)   # (B, L, G), rows padded to 8
        pooled = ops.attention_pool(att, x, pad_mask)                                   # (B, G*D), glimpse-major like the cat
        return ops.linear(pooled, self.linear_merge.weight, self.linear_merge.bias)


@HEADS_REGISTRY.register()
class QAHeadV1(nn.Module):
    """ScanQA / SQA3D answer head (reference: modules/heads/qa_head.py:72-90): attention-pool the object and the text
    tokens, LayerNorm(sum), 2-layer GELU classifier over the answer vocabulary.  Same constructor, forward contract
    (obj_embeds, obj_masks, txt_embeds, txt_masks; masks True = valid) and state_dict keys.  The classifier's first linear
    carries the (erf) GELU in its epilogue; the answer layer writes rows padded to a multiple of 8 answers (SQA3D: 706 -> 712),
    which ops.bce_with_logits_sum reads in place."""

    def __init__(self, cfg, hidden_size=768, mlp_size=256, glimpse=1, flat_out_size=512, num_answers=8864):
        super().__init__()
        self.attflat_visual = _AttentionPool(hidden_size, mlp_size, glimpse, flat_out_size, 0.1)
        self.attflat_lang = _AttentionPool(hidden_size, mlp_size, glimpse, flat_out_size, 0.1)
        self.answer_cls = nn.Sequential(nn.Linear(flat_out_size, hidden_size), nn.GELU(), nn.Dropout(0.3),
                                        nn.Linear(hidden_size, num_answers))
        self.fusion_norm = LayerNorm(flat_out_size)

    def forward(self, obj_embeds, obj_masks, txt_embeds, txt_masks, **kwargs):
        object_feat = self.attflat_visual(obj_embeds, obj_masks.logical_not())
        lang_feat = self.attflat_lang(txt_embeds, txt_masks.logical_not())
        fuse = self.fusion_norm(lang_feat, residual=object_feat)
        fc0, drop, fc3 = self.answer_cls[0], self.answer_cls[2], self.answer_cls[3]
        h = drop(ops.linear(fuse, fc0.weight, fc0.bias, activation="gelu"))
        return ops.padded_vocab_linear(h, fc3.weight, fc3.bias)
