"""model.pretrain_unfreeze_config against configs/final/all_pretrain_unfreeze.yaml (model and solver part; the literal values
below are cited by line), and the optimizer groups it gives: the object encoder's PointNet++ joins the vision groups."""
from sceneverse_b200 import model as M, weights

TF = weights.synthetic_tensor("text_features", (607, 768))


def test_config_matches_the_yaml():
    c = M.to_cfg(M.pretrain_unfreeze_config(2, text_features=TF))
    base = M.to_cfg(M.pretrain_config(2, text_features=TF))
    assert c.num_gpu == 2
    assert c.model.vision.args.freeze is False                               # :214 freeze: False
    assert c.solver.sched.name == "warmup_cosine"
    assert c.solver.sched.args.warmup_steps == 100                           # :184
    assert c.solver.sched.args.minimum_ratio == 0.1                          # :185
    assert c.solver.lr == 5e-4 and c.solver.grad_norm == 5.0                 # :174-175
    assert list(c.solver.optim.args.betas) == [0.9, 0.98]                    # :180
    assert (c.model.language.lr, c.model.vision.lr, c.model.grounding.lr) == (1e-5, 1e-4, 1e-4)   # :208, :226, :235
    # everything else is all_pretrain.yaml's model block
    for k in ("language", "grounding", "heads", "inter", "loss_list", "vis_loss_list", "name"):
        assert c.model[k] == base.model[k], k
    assert {k: v for k, v in c.model.vision.args.items() if k != "freeze"} == \
        {k: v for k, v in base.model.vision.args.items() if k != "freeze"}
    assert c.data == base.data
    # the frozen config is untouched
    assert base.model.vision.args.freeze is True and base.solver.sched.args.warmup_steps == 500


def test_backbone_in_the_vision_groups_in_reference_order():
    """get_opt_params (model/openvocab.py:103-126): language decay / no-decay, vision decay / no-decay, grounding, heads.  With
    the encoder unfrozen the PointNet++ parameters are in the vision groups at lr 1e-4, in named_parameters order, conv and
    BatchNorm weights with weight decay 0.01, biases without (optim/utils.py:1-18)."""
    m = M.build_model(M.pretrain_unfreeze_config(1, text_features=TF))
    groups = m.get_opt_params()
    pn = m.point_encoder.point_feature_extractor
    names = {id(p): "point_encoder." + n for n, p in m.point_encoder.named_parameters()}
    backbone = [(n, p) for n, p in pn.named_parameters()]
    assert backbone and all(p.requires_grad for _, p in backbone)
    vis_decay, vis_nodecay = groups[2], groups[3]
    assert vis_decay["lr"] == vis_nodecay["lr"] == 1e-4
    assert (vis_decay["weight_decay"], vis_nodecay["weight_decay"]) == (0.01, 0.0)
    want_decay = [p for n, p in backbone if not n.endswith("bias")]
    want_nodecay = [p for n, p in backbone if n.endswith("bias")]
    got_decay = [p for p in vis_decay["params"] if names[id(p)].startswith("point_encoder.point_feature_extractor.")]
    got_nodecay = [p for p in vis_nodecay["params"] if names[id(p)].startswith("point_encoder.point_feature_extractor.")]
    assert [id(p) for p in got_decay] == [id(p) for p in want_decay]
    assert [id(p) for p in got_nodecay] == [id(p) for p in want_nodecay]
    # the backbone comes first in the vision groups, as it is the encoder's first submodule
    assert vis_decay["params"][:len(want_decay)] == want_decay
    # 9 conv + 9 BatchNorm weights + fc.weight; 9 BatchNorm biases + fc.bias
    assert len(want_decay) == 19 and len(want_nodecay) == 10
    # frozen: no backbone parameter in any group
    f = M.build_model(M.pretrain_config(1, text_features=TF))
    fb = {id(p) for p in f.point_encoder.point_feature_extractor.parameters()}
    assert not any(id(p) in fb for g in f.get_opt_params() for p in g["params"])
