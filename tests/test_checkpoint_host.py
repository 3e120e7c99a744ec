"""Checkpoints on the host (CPU, fp32): the directory is what the reference's modules and torch's AdamW load as they are,
the ObjCls -> GPS hand-off through the vision encoder's `path`, and the data-parallel save / load (gloo, world 2)."""
import os
import socket
import tempfile
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from sceneverse_b200 import checkpoint, model as M, synthetic, train, weights

TF = weights.synthetic_tensor("text_features", (607, 768))


def cpu_step(seed, opt_step=True):
    """A CPU fp32 GPS step; opt_step: one AdamW / schedule step on seeded random gradients, so the optimizer has state."""
    ps = train.PretrainStep(M.pretrain_config(1, text_features=TF), "cpu", dtype=torch.float32, seed=seed)
    if opt_step:
        g = torch.Generator().manual_seed(seed + 1)
        for p in ps.parameters():
            p.grad = torch.randn(p.shape, generator=g) * 1e-2
        ps.optimizer.step()
        ps._advance_lr()
        ps.global_step += 1
    return ps


def close(got, want, tol, what):
    got, want = got.detach().float(), want.detach().float()
    err = ((got - want).abs().max() / (want.abs().max() + 1e-12)).item()
    assert err < tol, f"{what}: max err / max|ref| = {err:.3e} (tol {tol})"


def test_layout_and_eager_round_trip(tmp_path):
    ps = cpu_step(0)
    ps.save_state(tmp_path)
    assert sorted(os.listdir(tmp_path)) == sorted([checkpoint.MODEL, checkpoint.LOSS, checkpoint.OPTIMIZER,
                                                   checkpoint.SCHEDULER, checkpoint.NATIVE, "random_states_0.pkl"])
    want = ps.state_dict()
    q = cpu_step(1, opt_step=False)
    q.load_state(tmp_path)
    got = q.state_dict()
    for k, v in want["model"].items():
        assert torch.equal(got["model"][k], v), k
    assert set(got["optimizer"]["state"]) == set(want["optimizer"]["state"]) and len(want["optimizer"]["state"]) > 100
    for i, s in want["optimizer"]["state"].items():
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(got["optimizer"]["state"][i][k], s[k]), (i, k)
    assert got["scheduler"] == want["scheduler"] and q.global_step == 1 and q.total_steps == ps.total_steps
    assert [g["lr"] for g in q.optimizer.param_groups] == [g["lr"] for g in ps.optimizer.param_groups]
    # the native file is outside the pytorch_model*.bin glob of load_pretrain
    assert set(checkpoint.read_pretrain(tmp_path)) == set(want["model"]) | set(want["loss"])
    with pytest.raises(FileNotFoundError):
        checkpoint.read_pretrain(tmp_path / "missing")
    # the schedule is torch's LambdaLR over the same groups and lambda: the same lrs and the same saved `scheduler` dict,
    # through the warm-up and the cosine
    cfg = M.pretrain_config(1, text_features=TF)
    cfg["solver"]["sched"]["args"]["warmup_steps"] = 3
    r = train.PretrainStep(cfg, "cpu", total_steps=10, dtype=torch.float32, seed=2)
    groups = r.module.model.get_opt_params() + [{"params": list(r.module.loss.parameters()), "weight_decay": 0.0}]
    opt = torch.optim.AdamW(groups, lr=r.cfg.solver.lr)
    lam = torch.optim.lr_scheduler.LambdaLR(opt, r._lr_lambda)
    for i in range(11):
        assert [g["lr"] for g in r.optimizer.param_groups] == lam.get_last_lr(), i
        if i in (0, 10):
            assert r.state_dict()["scheduler"] == lam.state_dict(), i
        r.optimizer.step()
        r._advance_lr()
        opt.step()
        lam.step()


def test_objcls_to_gps_vision_path(tmp_path):
    """ObjClsStep.save_state -> the GPS config's vision.args.path: the frozen backbone (BatchNorm statistics included) is
    the object pre-training's; the optimizer / scheduler files in the same directory are ignored."""
    o = train.ObjClsStep("cpu", TF, dtype=torch.float32, seed=4)
    with torch.no_grad():
        for m in o.model.modules():
            if isinstance(m, torch.nn.BatchNorm2d) or isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.uniform_(-1, 1)
                m.num_batches_tracked.fill_(7)
    o.save_state(tmp_path)
    from sceneverse_b200.modules import vision
    enc = vision.PointOpenVocabEncoder(None, freeze=True, text_features=TF, path=str(tmp_path))
    want = o.model.point_feature_extractor.state_dict()
    got = enc.point_feature_extractor.state_dict()
    assert set(got) == set(want)
    for k in want:
        assert torch.equal(got[k], want[k]), k


def _ref_modules(text_dir):
    from oracle import ref_shims
    ref_shims.install()
    from modules.build import GROUNDING_REGISTRY, HEADS_REGISTRY, VISION_REGISTRY
    import importlib
    import modules.vision.pcd_openvocab_encoder  # noqa: F401
    import modules.grounding.unified_encoder  # noqa: F401
    import modules.heads.pretrain_head  # noqa: F401
    from transformers import BertConfig, BertModel
    ref_shims.write_text_features(text_dir, TF)
    with ref_shims.cpu_cuda_identity():
        mods = {"lang_encoder.model.": BertModel(BertConfig(hidden_size=768, num_hidden_layers=4, num_attention_heads=12,
                                                            type_vocab_size=2)),
                "point_encoder.": VISION_REGISTRY.get("PointOpenVocabEncoder")(None, lang_path=text_dir, freeze=True),
                "unified_encoder.": GROUNDING_REGISTRY.get("UnifiedSpatialCrossEncoderV2")(None),
                "pretrain_head.": HEADS_REGISTRY.get("OVPretrainHead")(None)}
    LL = importlib.import_module("optim.loss.loss")
    c = M.pretrain_config(1)["model"]
    cfg = types.SimpleNamespace(num_gpu=1, task="Pretrain",
                                model=types.SimpleNamespace(loss_list=c["loss_list"], vis_loss_list=c["vis_loss_list"]))
    loss = LL.Loss(cfg)
    no_decay = importlib.import_module("optim.utils").no_decay_param_group
    return mods, loss, no_decay


@pytest.mark.skipif(not __import__("oracle.ref_shims", fromlist=["available"]).available(),
                    reason="needs the reference checkout (oracle/ref_shims.py)")
def test_reference_loads_the_checkpoint(tmp_path):
    """pytorch_model.bin / pytorch_model_1.bin load into the reference's unmodified modules with no missing or unexpected
    key (the language encoder: the HF BertModel the reference wraps), and their fp32 forward on a seeded batch matches this
    model's at 1e-5; a torch AdamW over the reference's get_opt_params() order (+ the loss group) loads optimizer.bin."""
    from oracle import ref_shims
    ps = cpu_step(0)
    ps.save_state(tmp_path / "ckpt")
    mods, ref_loss, no_decay = _ref_modules(str(tmp_path / "text"))
    sd = torch.load(tmp_path / "ckpt" / checkpoint.MODEL, weights_only=True)
    for prefix, m in mods.items():
        part = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
        m.load_state_dict(part, strict=True)
        m.eval()
    assert all(any(k.startswith(p) for p in mods) for k in sd), "keys outside the reference's modules"
    ref_loss.load_state_dict(torch.load(tmp_path / "ckpt" / checkpoint.LOSS, weights_only=True), strict=True)
    # forward parity: the same seeded batch through both
    ours = ps.module.model.eval()
    d = synthetic.scene_batch(5, B=2, O=16, P=1024, L=50, Ls=300, min_obj=6)
    t = {k: torch.from_numpy(v) for k, v in d.items()}
    with torch.no_grad(), ref_shims.cpu_cuda_identity():
        lang_ref = mods["lang_encoder.model."](t["txt_ids"], t["txt_masks"]).last_hidden_state
        pn = {}
        enc = mods["point_encoder."]
        hk = enc.point_feature_extractor.register_forward_hook(lambda m, a, o: pn.__setitem__("out", o))
        obj_ref, pre_ref, sem_ref = enc(t["obj_fts"], t["obj_locs"], t["obj_masks"], t["obj_sem_masks"], t["obj_labels"], 1, 1)
        hk.remove()
        t2_ref, o2_ref = mods["unified_encoder."](lang_ref, t["txt_masks"], obj_ref, t["obj_locs"], t["obj_masks"])
        lm_ref, _ = mods["pretrain_head."](t2_ref, o2_ref)

    class Backbone(torch.nn.Module):          # this model's PointNet++ runs on CUDA only: the reference's features
        def forward(self, x):
            return pn["out"]
    with torch.no_grad():
        lang = ours.lang_encoder(t["txt_ids"], t["txt_masks"])
        ours.point_encoder.point_feature_extractor = Backbone()
        obj, pre, sem = ours.point_encoder(t["obj_fts"], t["obj_locs"], t["obj_masks"], t["obj_sem_masks"], t["obj_labels"],
                                           1, 1)
        t2, o2 = ours.unified_encoder(lang, t["txt_masks"], obj, t["obj_locs"], t["obj_masks"])
        lm, _ = ours.pretrain_head(t2, o2)
    for got, want, what in ((lang, lang_ref, "BERT"), (obj, obj_ref, "object encoder"), (sem, sem_ref, "object classes"),
                            (t2, t2_ref, "unified text"), (o2, o2_ref, "unified objects"), (lm, lm_ref, "LM logits")):
        close(got, want, 1e-5, what)
    # torch AdamW in the reference's group order accepts optimizer.bin as it is
    lr = ps.cfg.solver.lr
    groups = []
    for prefix, key in (("lang_encoder.model.", "language"), ("point_encoder.", "vision"), ("unified_encoder.", "grounding")):
        groups += no_decay(mods[prefix].named_parameters(), ps.cfg.model[key]["lr"])
    groups += no_decay(mods["pretrain_head."].named_parameters(), lr)
    groups.append({"params": list(ref_loss.parameters()), "weight_decay": 0.0, "lr": lr})
    opt = torch.optim.AdamW(groups, lr=lr)
    saved = torch.load(tmp_path / "ckpt" / checkpoint.OPTIMIZER, weights_only=True)
    opt.load_state_dict(saved)
    flat = [p for g in opt.param_groups for p in g["params"]]
    assert len(saved["state"]) > 100
    for i, s in saved["state"].items():
        st = opt.state[flat[i]]
        assert st["exp_avg"].shape == flat[i].shape and torch.equal(st["exp_avg"], s["exp_avg"]), i


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dp_worker(rank, world, port, path, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ps = train.PretrainStep(M.pretrain_config(world, text_features=TF), "cpu", dtype=torch.float32, seed=rank)
        assert ps.use_ddp
        written = []
        real_save = torch.save

        def recording_save(obj, f, *a, **k):
            written.append(os.path.basename(str(f)))
            return real_save(obj, f, *a, **k)
        torch.save = recording_save
        try:
            torch.manual_seed(1000 + rank)
            np.random.seed(rank)
            mine = torch.get_rng_state()
            ps.save_state(path)
        finally:
            torch.save = real_save
        shared = {checkpoint.MODEL, checkpoint.LOSS, checkpoint.OPTIMIZER, checkpoint.SCHEDULER, checkpoint.NATIVE}
        want = (shared if rank == 0 else set()) | {f"random_states_{rank}.pkl"}
        assert set(written) == want, (rank, written)
        rank0 = {n: p.detach().clone() for n, p in ps.module.model.named_parameters()}
        dist.broadcast_object_list(obj := [rank0 if rank == 0 else None], 0)
        rank0 = obj[0]
        fresh = train.PretrainStep(M.pretrain_config(world, text_features=TF), "cpu", dtype=torch.float32, seed=7 + rank)
        torch.manual_seed(55)
        fresh.load_state(path)
        for n, p in fresh.module.model.named_parameters():
            assert torch.equal(p.detach(), rank0[n]), (rank, n)
        assert torch.equal(torch.get_rng_state(), mine), rank
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_data_parallel_save_load_gloo_world2():
    """Rank 0 writes the shared files, every rank its own random states; every rank loads rank 0's parameters and gets
    back its own generator state."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    with tempfile.TemporaryDirectory() as path:
        procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, path, q)) for r in range(2)]
        for p in procs:
            p.start()
        res = [q.get(timeout=600) for _ in range(2)]
        for p in procs:
            p.join(timeout=60)
    assert all(r[1] == "ok" for r in res), res
