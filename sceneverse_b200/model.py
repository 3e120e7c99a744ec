"""Model glue of the GPS path (reference: model/openvocab.py:11-126 `OpenVocab`, trainer/openvocab_trainer.py:18-46).

`OpenVocab` consumes the same nested config (cfg.model.{language,vision,grounding,heads,inter}, cfg.data.args)
and fills the same data_dict keys, building its parts through `build_module` under the reference's registry names.
The language encoder is the reference's HuggingFace BERT-4L (modules/language/bert.py:8-26), random-initialised here
because no checkpoint can be downloaded (upstream of the hot path, SURVEY.md §2 row 13).
"""
import torch
from torch import nn

from .modules import grounding, heads, vision  # noqa: F401  (populate the registries)
from . import ops
from .modules.registry import LANGUAGE_REGISTRY, build_module


class _Cfg(dict):
    """dict with attribute access and .get — stands in for the OmegaConf node the reference passes around."""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError as e:
            raise AttributeError(k) from e
        return _Cfg(v) if isinstance(v, dict) and not isinstance(v, _Cfg) else v


def to_cfg(d):
    return _Cfg(d)


@LANGUAGE_REGISTRY.register()
class BERTLanguageEncoder(nn.Module):
    def __init__(self, cfg, weights="bert-base-uncased", hidden_size=768, num_hidden_layers=4, num_attention_heads=12,
                 type_vocab_size=2):
        super().__init__()
        from transformers import BertConfig, BertModel
        self.bert_config = BertConfig(hidden_size=hidden_size, num_hidden_layers=num_hidden_layers,
                                      num_attention_heads=num_attention_heads, type_vocab_size=type_vocab_size)
        self.model = BertModel(self.bert_config)  # no network: random init instead of from_pretrained(weights)
        _fuse_bert_layer_norms(self.model)

    def forward(self, txt_ids, txt_masks, cls_only=False, **kwargs):
        """(B, L, D) last hidden state; cls_only: only its first row (B, D), for which the last layer runs its attention
        output projection, LayerNorms and FFN on that row alone (`_bert_cls_layer_forward`).  The values and dropout
        masks are the same either way."""
        last = self.model.encoder.layer[-1]
        if not hasattr(last, "cls_only"):
            return self.model(txt_ids, txt_masks).last_hidden_state[:, 0] if cls_only else \
                self.model(txt_ids, txt_masks).last_hidden_state
        last.cls_only = cls_only
        try:
            h = self.model(txt_ids, txt_masks).last_hidden_state
        finally:
            last.cls_only = False
        return h[:, 0] if cls_only else h


def _bert_output_forward(self, hidden_states, input_tensor, row_key_stride=1):
    """BertSelfOutput / BertOutput tail LayerNorm(input + dropout(dense(h))) through the fused native kernel."""
    h = ops.linear(hidden_states, self.dense.weight, self.dense.bias)
    return self.LayerNorm(h, residual=input_tensor, dropout_p=self.dropout.p if self.training else 0.0,
                          row_key_stride=row_key_stride)


def _bert_self_attention_forward(self, hidden_states, attention_mask=None, past_key_values=None, query_rows=None, **kwargs):
    """BertSelfAttention through ops.attention (native wgmma forward / backward with in-kernel attention dropout on
    CUDA bf16).  `attention_mask` is the padding mask HF prepared for its SDPA path: None, or (B,1,Lq,Lk) with True /
    0.0 = attend (identical rows), from which the (B,Lk) key-padding mask is read back.  query_rows: only the first rows
    attend (ops.attention_packed)."""
    qkv = ops.linear_packed(hidden_states, [self.query, self.key, self.value])   # one GEMM, [q | k | v]
    kpm = None
    if attention_mask is not None:
        row = attention_mask[:, 0, 0, :]
        kpm = row.logical_not() if row.dtype == torch.bool else row < 0
    out = ops.attention_packed(qkv, self.num_attention_heads, key_padding_mask=kpm,
                               dropout_p=self.dropout.p if self.training else 0.0, query_rows=query_rows)
    return out, None


def _bert_feed_forward_chunk(self, attention_output):
    """BertLayer.feed_forward_chunk (BertIntermediate: dense + gelu; BertOutput: dense, dropout, LayerNorm(+ residual)) as
    one ops.ffn (two native GEMMs, gelu in the first epilogue) + the fused dropout / residual / LayerNorm kernel.  (HF
    counts this method's parameters, so the row-key stride lives in _bert_feed_forward.)"""
    return _bert_feed_forward(self, attention_output)


def _bert_feed_forward(self, attention_output, row_key_stride=1):
    inter, out = self.intermediate.dense, self.output
    h = ops.ffn(attention_output, inter.weight, inter.bias, out.dense.weight, out.dense.bias, activation="gelu")
    return out.LayerNorm(h, residual=attention_output, dropout_p=out.dropout.p if self.training else 0.0,
                         row_key_stride=row_key_stride)


def _bert_cls_layer_forward(self, hidden_states, attention_mask=None, *args, **kwargs):
    """BertLayer.forward of the last layer.  With `cls_only` set (BERTLanguageEncoder(..., cls_only=True)) only row 0 of
    each sequence leaves the layer, so only that row is computed past the packed q | k | v projection, which still runs on
    every row (its gradient stays one dgrad and one wgrad GEMM): 1-query attention over all keys, the output projection
    with residual h[:, :1], and the FFN.  Both LayerNorms key their dropout rows by b * L, so every dropout mask, and
    every value of row 0, is the one of the full layer."""
    if not self.cls_only:
        return type(self).forward(self, hidden_states, attention_mask, *args, **kwargs)
    L = hidden_states.shape[1]
    ctx, _ = self.attention.self(hidden_states, attention_mask, query_rows=1)
    attention_output = self.attention.output(ctx, hidden_states[:, :1], row_key_stride=L)
    return _bert_feed_forward(self, attention_output, row_key_stride=L)


def _fuse_bert_layer_norms(bert):
    """Same modules, parameters and state_dict keys as the HF model; only the forward of the LayerNorms, of the two
    residual tails of every block (-> ops.layer_norm) and of the self-attention core (-> ops.attention) is re-routed."""
    import types
    from .modules.layers import LayerNorm
    for mod in bert.modules():
        if type(mod) is nn.LayerNorm:
            mod.__class__ = LayerNorm
    for layer in bert.encoder.layer:
        for tail in (layer.attention.output, layer.output):
            tail.forward = types.MethodType(_bert_output_forward, tail)
        ffn = getattr(bert.config, "hidden_act", "gelu") == "gelu" and getattr(layer, "chunk_size_feed_forward", 0) == 0
        if ffn:
            layer.feed_forward_chunk = types.MethodType(_bert_feed_forward_chunk, layer)
        if layer.attention.self.attention_head_size == 64:
            layer.attention.self.forward = types.MethodType(_bert_self_attention_forward, layer.attention.self)
            if ffn and layer is bert.encoder.layer[-1]:
                layer.cls_only = False
                layer.forward = types.MethodType(_bert_cls_layer_forward, layer)


def no_decay_param_group(parameters, lr):
    """optim/utils.py:1-18."""
    no_decay = ['bias', 'LayerNorm.bias', 'LayerNorm.weight']
    decay_params, no_decay_params = [], []
    for n, p in parameters:
        if not p.requires_grad:
            continue
        (no_decay_params if any(nd in n for nd in no_decay) else decay_params).append(p)
    return [{'params': decay_params, 'weight_decay': 0.01, 'lr': lr},
            {'params': no_decay_params, 'weight_decay': 0.0, 'lr': lr}]


class OpenVocab(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg = to_cfg(cfg)
        self.lang_encoder = build_module("language", cfg.model.language)
        self.point_encoder = build_module("vision", cfg.model.vision)
        self.unified_encoder = build_module("grounding", cfg.model.grounding)
        self.head_list = list(cfg.model.heads.head_list)
        for head in self.head_list:
            setattr(self, head, build_module("heads", getattr(cfg.model.heads, head)))
        self.use_scene_cap = cfg.data.args.get("use_scene_cap", False)
        from .modules.layers import route_linears
        route_linears(self)

    def forward(self, data_dict):
        if 'cur_step' not in data_dict:
            data_dict['cur_step'], data_dict['total_steps'] = 1, 1
        lang = self.lang_encoder(data_dict['txt_ids'], data_dict['txt_masks'])
        hook = getattr(self, "_lang_grad_hook", None)
        if hook is not None and lang.requires_grad:
            lang.register_hook(hook)       # train.PretrainStep: launch point of the early gradient all-reduce
        if self.use_scene_cap:
            data_dict['scene_text_embed'] = self.lang_encoder(data_dict['scene_txt_ids'], data_dict['scene_txt_masks'],
                                                              cls_only=True)
        obj, obj_pre, obj_cls_raw = self.point_encoder(data_dict['obj_fts'].float(), data_dict['obj_locs'],
                                                       data_dict['obj_masks'], data_dict['obj_sem_masks'],
                                                       data_dict.get('obj_labels'), data_dict['cur_step'],
                                                       data_dict['total_steps'])
        if self.use_scene_cap:
            data_dict["scene_embed"] = obj.mean(dim=1)  # includes padded objects, like openvocab.py:24,52-54
        if self.cfg.model.inter == "before":
            data_dict["inter_text_embed"], data_dict["inter_obj_embeds"] = lang[:, 0], obj
        lang_f, obj_f = self.unified_encoder(lang, data_dict['txt_masks'], obj, data_dict['obj_locs'], data_dict['obj_masks'])
        if self.cfg.model.inter != "before":
            data_dict["inter_text_embed"], data_dict["inter_obj_embeds"] = lang_f[:, 0], obj_f
        data_dict["intra_text_embed"], data_dict["intra_obj_embeds"] = lang_f[:, 0], obj_f
        data_dict['obj_cls_raw_logits'] = obj_cls_raw
        data_dict['og3d_logits'] = torch.einsum("bod,bd->bo", obj_f, lang_f[:, 0])
        if getattr(self, "ground_head", None) is not None:
            txt_cls, obj_cls_post, obj_cls_pre, og3d = self.ground_head(lang_f, obj_f, obj_pre, data_dict['obj_masks'])
            data_dict.update(txt_cls_logits=txt_cls, obj_cls_post_logits=obj_cls_post, obj_cls_pre_logits=obj_cls_pre,
                             og3d_logits=og3d)
        if getattr(self, "qa_head", None) is not None:
            data_dict['answer_scores'] = self.qa_head(obj_f, data_dict['obj_masks'], lang_f, data_dict['txt_masks'])
        if getattr(self, "pretrain_head", None) is not None:
            output = self.pretrain_head(lang_f, obj_f)
            if isinstance(output, tuple):
                data_dict['txt_lm_cls_logits'], data_dict['obj_cls_post_logits'] = output
            else:
                data_dict['txt_lm_cls_logits'] = output
        return data_dict

    def get_opt_params(self):
        def lr_of(c):
            return self.cfg.solver.lr if c.get("lr") is None else c.get("lr")
        groups = []
        groups += no_decay_param_group(self.lang_encoder.named_parameters(), lr_of(self.cfg.model.language))
        groups += no_decay_param_group(self.point_encoder.named_parameters(), lr_of(self.cfg.model.vision))
        groups += no_decay_param_group(self.unified_encoder.named_parameters(), lr_of(self.cfg.model.grounding))
        for head in ("ground_head", "qa_head", "pretrain_head"):
            if head in self.head_list:
                groups += no_decay_param_group(getattr(self, head).named_parameters(),
                                               lr_of(getattr(self.cfg.model.heads, head)))
        return groups


# what the reference's OpenVocabPerScene cannot run on a per-scene batch (model/openvocab.py:141-230), and why
PER_SCENE_UNSUPPORTED = {
    "og3d_loss": "cross-entropy over the (B, U, O) per-scene logits would treat U as the class axis",
    "TextSceneBetweenBatch": "the per-scene model sets no scene_embed / scene_text_embed",
    "answer_loss": "the QA head is given the un-flattened (B, U, T) txt_masks",
    "qa_head": "the QA head is given the un-flattened (B, U, T) txt_masks",
    "og3d_multi_loss": "BCE over the (B, U, O) per-scene logits needs a target of that shape; the per-scene tgt_object_id "
                       "is (B, U)",
    "txt_cls_multi_loss": "no ground head runs per scene, so there are no txt_cls_logits",
    "obj_cls_pre_loss": "no ground head runs per scene, so there are no obj_cls_pre_logits",
    "obj_cls_pre_loss_mask": "no ground head runs per scene, so there are no obj_cls_pre_logits",
    "obj_cls_pre_loss_unmask": "no ground head runs per scene, so there are no obj_cls_pre_logits",
    "obj_cls_post_loss": "the per-scene obj_cls_post_logits has B*U rows of objects against the (B, O) obj_labels",
    "obj_cls_post_loss_mask": "the per-scene obj_cls_post_logits has B*U rows of objects against the (B, O) obj_labels",
    "obj_cls_post_loss_unmask": "the per-scene obj_cls_post_logits has B*U rows of objects against the (B, O) obj_labels",
}


def check_per_scene(cfg):
    """Raises ValueError naming the first loss or head of `cfg` the per-scene model cannot run."""
    cfg = to_cfg(cfg)
    for k in list(cfg.model.get("loss_list", [])) + list(cfg.model.get("vis_loss_list", [])) + \
            list(cfg.model.heads.head_list):
        if k in PER_SCENE_UNSUPPORTED:
            raise ValueError(f"OpenVocabPerScene cannot use {k!r}: {PER_SCENE_UNSUPPORTED[k]}")


class OpenVocabPerScene(OpenVocab):
    """Per-scene grounding (reference: model/openvocab.py:129-255 `OpenVocabPerScene`): the same submodules, parameter names
    and optimizer groups as OpenVocab, so checkpoints move between the two.  A batch is per-scene when txt_ids is (B, U, T):
    U utterances about each of B scenes.  The language encoder, V2 and the heads then run on B*U rows, while PointNet++ and
    the spatial layers run once per scene; their (B, O, D) output (vision dropout applied) is repeated U times by
    ops.scene_broadcast, whose backward sums the U copies.  og3d_logits is (B, U, O).  The ground head is never called and
    no scene-caption embedding is made, in either path; a 2-D batch is OpenVocab without those two."""

    def __init__(self, cfg):
        check_per_scene(cfg)
        super().__init__(cfg)
        self.use_scene_cap = False

    def forward(self, data_dict):
        if data_dict['txt_ids'].dim() != 3:
            return self._forward(data_dict, None)
        return self._forward(data_dict, data_dict['txt_ids'].shape[1])

    def _forward(self, data_dict, U):
        if 'cur_step' not in data_dict:
            data_dict['cur_step'], data_dict['total_steps'] = 1, 1
        txt_ids, txt_masks = data_dict['txt_ids'], data_dict['txt_masks']
        if U is not None:
            txt_ids, txt_masks = txt_ids.reshape(-1, txt_ids.shape[-1]), txt_masks.reshape(-1, txt_masks.shape[-1])
        lang = self.lang_encoder(txt_ids, txt_masks)
        hook = getattr(self, "_lang_grad_hook", None)
        if hook is not None and lang.requires_grad:
            lang.register_hook(hook)
        obj, _, obj_cls_raw = self.point_encoder(data_dict['obj_fts'].float(), data_dict['obj_locs'], data_dict['obj_masks'],
                                                 data_dict['obj_sem_masks'], data_dict.get('obj_labels'),
                                                 data_dict['cur_step'], data_dict['total_steps'])
        obj_locs, obj_masks = data_dict['obj_locs'], data_dict['obj_masks']
        if U is not None:
            B, O = obj_masks.shape
            obj = ops.scene_broadcast(obj, U)      # one tensor into V2 and inter_obj_embeds: one U-sum in the backward
            obj_locs = obj_locs.unsqueeze(1).expand(B, U, O, obj_locs.shape[-1]).reshape(B * U, O, obj_locs.shape[-1])
            obj_masks = obj_masks.unsqueeze(1).expand(B, U, O).reshape(B * U, O)
        if self.cfg.model.inter == "before":
            data_dict["inter_text_embed"], data_dict["inter_obj_embeds"] = lang[:, 0], obj
        lang_f, obj_f = self.unified_encoder(lang, txt_masks, obj, obj_locs, obj_masks)
        if self.cfg.model.inter != "before":
            data_dict["inter_text_embed"], data_dict["inter_obj_embeds"] = lang_f[:, 0], obj_f
        data_dict["intra_text_embed"], data_dict["intra_obj_embeds"] = lang_f[:, 0], obj_f
        data_dict['obj_cls_raw_logits'] = obj_cls_raw
        og3d = torch.einsum("bod,bd->bo", obj_f, lang_f[:, 0])
        data_dict['og3d_logits'] = og3d.reshape(-1, U, og3d.shape[-1]) if U is not None else og3d
        if getattr(self, "pretrain_head", None) is not None:
            output = self.pretrain_head(lang_f, obj_f)
            if isinstance(output, tuple):
                data_dict['txt_lm_cls_logits'], data_dict['obj_cls_post_logits'] = output
            else:
                data_dict['txt_lm_cls_logits'] = output
        return data_dict


MODELS = {"OpenVocab": OpenVocab, "OpenVocabPerScene": OpenVocabPerScene}


def build_model(cfg):
    """model/build.py:16-17: the class named by cfg.model.name (OpenVocab when the config names none)."""
    name = to_cfg(cfg).model.get("name", "OpenVocab")
    if name not in MODELS:
        raise KeyError(f"No model named {name!r}; known: {sorted(MODELS)}")
    return MODELS[name](cfg)


def pretrain_config(num_gpu=1, with_obj_between=True, text_features=None):
    """configs/final/all_pretrain.yaml:205-258 (model/solver part), with TextObjBetweenBatch un-commented as in
    BASELINE.json configs[3] ("obj+scene+ref losses")."""
    losses = ['lm_cls_loss', 'TextObjWithinBatch'] + (['TextObjBetweenBatch'] if with_obj_between else []) + \
        ['TextSceneBetweenBatch']
    return {
        "num_gpu": num_gpu,
        "data": {"args": {"use_scene_cap": True, "max_obj_len": 80, "num_points": 1024, "txt_seq_length": 50,
                          "max_scene_cap_len": 300}},
        "solver": {"lr": 5e-4, "grad_norm": 5.0, "optim": {"name": "AdamW", "args": {"betas": [0.9, 0.98]}},
                   "sched": {"name": "warmup_cosine", "args": {"warmup_steps": 500, "minimum_ratio": 0.1}}},
        "model": {
            "name": "OpenVocab",
            "language": {"name": "BERTLanguageEncoder", "lr": 1e-5,
                         "args": {"weights": "bert-base-uncased", "hidden_size": 768, "num_hidden_layers": 4,
                                  "num_attention_heads": 12, "type_vocab_size": 2}},
            "vision": {"name": "PointOpenVocabEncoder", "lr": 1e-4,
                       "args": {"backbone": "pointnet++", "hidden_size": 768, "freeze": True, "path": None,
                                "num_attention_heads": 12, "spatial_dim": 5, "num_layers": 4, "dim_loc": 6,
                                "dim_feedforward": 2048, "attn_type": "spatial", "pairwise_rel_type": "center",
                                "use_matmul_label": False, "lang_type": "bert", "lang_path": None,
                                "text_features": text_features}},
            "grounding": {"name": "UnifiedSpatialCrossEncoderV2", "lr": 1e-4,
                          "args": {"hidden_size": 768, "num_attention_heads": 12, "num_layers": 4,
                                   "dim_feedforward": 2048, "dim_loc": 6}},
            "inter": "before",
            "heads": {"head_list": ["pretrain_head"],
                      "pretrain_head": {"name": "OVPretrainHead", "args": {"hidden_size": 768, "vocab_size": 30522}}},
            "loss_list": losses, "vis_loss_list": losses,
        },
    }


def pretrain_unfreeze_config(num_gpu=1, text_features=None):
    """configs/final/all_pretrain_unfreeze.yaml (model/solver part): pretrain_config with the object encoder trainable
    (`vision.args.freeze: False`, :214) and 100 warm-up steps (`solver.sched.args.warmup_steps`, :184).  lr 5e-4, grad_norm
    5.0, betas (0.9, 0.98) and minimum_ratio 0.1 (:174-185) and the per-module lrs (language 1e-5, vision and grounding 1e-4,
    :208, :226, :235) are those of all_pretrain.yaml.  PointNet++ then trains with batch-statistic BatchNorm (pn_train.py)
    and its parameters join the vision groups of get_opt_params.  The yaml's `vision.args.path` (:215) is the ObjCls
    checkpoint the backbone starts from: set `model.vision.args.path`, or call PretrainStep.load_pretrain, to continue
    from one; with several GPUs the BatchNorm layers stay plain BatchNorm2d, as in the reference's OpenVocab."""
    cfg = pretrain_config(num_gpu, text_features=text_features)
    cfg["model"]["vision"]["args"]["freeze"] = False
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 100
    return cfg


def per_scene_pretrain_config(num_gpu=1, text_features=None):
    """pretrain_config as OpenVocabPerScene: the losses the reference can run per scene (lm_cls_loss, TextObjWithinBatch,
    TextObjBetweenBatch) and no scene captions.  Batches are synthetic.per_scene_batch-shaped (txt_ids (B, U, T))."""
    cfg = pretrain_config(num_gpu, text_features=text_features)
    cfg["data"]["args"]["use_scene_cap"] = False
    cfg["model"]["name"] = "OpenVocabPerScene"
    losses = ["lm_cls_loss", "TextObjWithinBatch", "TextObjBetweenBatch"]
    cfg["model"]["loss_list"], cfg["model"]["vis_loss_list"] = list(losses), list(losses)
    return cfg


def scanrefer_config(num_gpu=1, text_features=None):
    """configs/final/finetune/scanrefer_finetune.yaml:205-259 — BASELINE.json configs[2]: same encoders, GroundHeadV1
    (hidden 384, detach_all_aux_loss) and `og3d_loss`; the backbone stays frozen, no scene captions."""
    cfg = pretrain_config(num_gpu, text_features=text_features)
    cfg["data"]["args"]["use_scene_cap"] = False
    cfg["solver"]["lr"] = 1e-4
    cfg["model"]["heads"] = {"head_list": ["ground_head"],
                             "ground_head": {"name": "GroundHeadV1",
                                             "args": {"hidden_size": 384, "input_size": 768, "sem_cls_size": 607,
                                                      "dropout": 0.3, "detach_all_aux_loss": True}}}
    cfg["model"]["loss_list"] = ["og3d_loss"]
    cfg["model"]["vis_loss_list"] = ["og3d_loss"]
    return cfg


def _qa_config(num_gpu, text_features, task, num_answers, losses):
    cfg = pretrain_config(num_gpu, text_features=text_features)
    cfg["task"] = task
    cfg["data"]["args"]["use_scene_cap"] = False
    cfg["solver"]["lr"] = 1e-4
    cfg["solver"]["sched"] = {"name": "warmup_cosine", "args": {"warmup_steps": 5000}}
    cfg["model"]["heads"] = {"head_list": ["qa_head"],
                             "qa_head": {"name": "QAHeadV1",
                                         "args": {"hidden_size": 768, "mlp_size": 256, "glimpse": 1, "flat_out_size": 512,
                                                  "num_answers": num_answers}}}
    cfg["model"]["loss_list"] = list(losses)
    cfg["model"]["vis_loss_list"] = list(losses)
    return cfg


def scanqa_config(num_gpu=1, text_features=None):
    """configs/final/finetune/scanqa_finetune.yaml: the pre-training encoders (frozen backbone, inter 'before', no scene
    captions), QAHeadV1 over 8864 answers, `answer_loss` + the masked-BCE TextObjWithinBatch of task 'ScanQA'; lr 1e-4
    (language 1e-5, vision and grounding 1e-4), grad_norm 5.0, betas (0.9, 0.98), 5000 warm-up steps."""
    return _qa_config(num_gpu, text_features, "ScanQA", 8864, ["answer_loss", "TextObjWithinBatch"])


def sqa3d_config(num_gpu=1, text_features=None):
    """configs/final/finetune/sqa3d_finetune.yaml: as scanqa_config with task 'SQA3D', 706 answers and `answer_loss` only."""
    return _qa_config(num_gpu, text_features, "SQA3D", 706, ["answer_loss"])


def warmup_cosine(step, warmup_step, total_step, minimum_ratio=1e-5):
    """optim/scheduler.py warmup_cosine (LambdaLR factor)."""
    import math
    if step <= warmup_step and warmup_step > 0:
        return step / warmup_step
    return max(0.5 * (1 + math.cos((step - warmup_step) / max(total_step - warmup_step, 1) * math.pi)), minimum_ratio)


class ObjCls(nn.Module):
    """Object-level pre-training model (reference: model/objcls.py:16-98), `model_name='pointnet++'`, open-vocabulary
    head against the 607 frozen text embeddings, bert language type (768-d).  PointNet++ is trainable here with
    train-mode BatchNorm (SyncBatchNorm when num_gpu > 1, objcls.py:33-34) on the channels-last native path of pn_train.py;
    SyncBatchNorm exchanges its statistics through pn_train.StatExchange (the generic operator sequence on the native point
    ops remains the fallback)."""

    def __init__(self, cfg, text_embeds=None):
        super().__init__()
        from .modules.pointnet import GPS_SPEC, PointNetPP
        self.cfg = cfg = to_cfg(cfg)
        self.point_feature_extractor = PointNetPP(**GPS_SPEC)
        if cfg.num_gpu > 1:
            self.point_feature_extractor = torch.nn.SyncBatchNorm.convert_sync_batchnorm(self.point_feature_extractor)
        self.register_buffer("text_embeds", text_embeds.float())
        self.dropout = nn.Dropout(0.1)

    def forward(self, data_dict):
        obj_pcds = data_dict["obj_fts"]
        B, O = obj_pcds.shape[:2]
        emb = self.point_feature_extractor(obj_pcds.reshape(B * O, *obj_pcds.shape[2:]).float())
        emb = self.dropout(emb)
        data_dict["obj_logits"] = (emb @ self.text_embeds.t().to(emb.dtype)).view(B, O, -1)
        return data_dict

    def get_opt_params(self):
        return [{"params": list(self.parameters()), "weight_decay": self.cfg.solver.get("weight_decay", 0.0),
                 "lr": self.cfg.solver.lr}]
