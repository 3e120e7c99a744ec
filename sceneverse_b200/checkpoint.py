"""Checkpoints of the training steps (train.PretrainStep, train.ObjClsStep) in the directory layout of accelerate's
`save_state` as the reference trainer calls it (trainer/build.py:131-133,164-172, openvocab_trainer.py:104-109):

    pytorch_model.bin        the model's state_dict, with the reference's keys
    pytorch_model_1.bin      the loss module's state_dict (the contrastive losses' logit_scale)
    optimizer.bin            torch AdamW.state_dict() form: parameters keyed by their index in get_opt_params() order,
                             the loss group last; no dependence on the flat buffers of train.FlatState
    scheduler.bin            torch LambdaLR.state_dict() form
    random_states_<rank>.pkl python / numpy / torch CPU / torch CUDA generator states of each rank
    native_state.pt          what accelerate has no file for: global_step, total_steps, the device dropout counter, the
                             in-kernel dropout seed position and the list of probed unused parameters

With several ranks, rank 0 writes the shared files, every rank its own random state, and a barrier follows; every rank
loads.  `native_state.pt` is deliberately not a `*.bin`, so the `pytorch_model*.bin` glob of load_pretrain and the
`*.bin` glob of the vision encoder's `path` (modules/vision.py) never see it."""
import glob
import os
import random

import numpy as np
import torch
import torch.distributed as dist

MODEL, LOSS, OPTIMIZER, SCHEDULER, NATIVE = "pytorch_model.bin", "pytorch_model_1.bin", "optimizer.bin", "scheduler.bin", \
    "native_state.pt"


def _dist():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def _rank():
    return dist.get_rank() if _dist() else 0


def random_states_name(rank):
    return f"random_states_{rank}.pkl"


def to_cpu(obj):
    """A copy of every tensor in a nested dict / list on the host, each with its own storage (a view of a flat buffer is
    saved as itself, not as the buffer)."""
    if torch.is_tensor(obj):
        return obj.detach().to("cpu", copy=True)
    if isinstance(obj, dict):
        return {k: to_cpu(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(to_cpu(v) for v in obj)
    return obj


def rng_state():
    """accelerate's random_states_<rank>.pkl content."""
    st = {"step": 0, "random_state": random.getstate(), "numpy_random_seed": np.random.get_state(),
          "torch_manual_seed": torch.get_rng_state()}
    if torch.cuda.is_available() and torch.cuda.is_initialized():
        st["torch_cuda_manual_seed"] = torch.cuda.get_rng_state_all()
    return st


def set_rng_state(st):
    random.setstate(st["random_state"])
    np.random.set_state(st["numpy_random_seed"])
    torch.set_rng_state(st["torch_manual_seed"])
    cuda = st.get("torch_cuda_manual_seed")
    if cuda is not None and torch.cuda.is_available():
        for i, s in enumerate(cuda[:torch.cuda.device_count()]):
            torch.cuda.set_rng_state(s, i)


def export_adamw(order, live_groups, lrs, base_lrs, moments):
    """torch AdamW.state_dict() of an optimizer whose groups are `live_groups`, re-indexed over `order` (the parameter groups
    as the reference's get_opt_params() lists them, with the parameters this step froze still in place).
    moments(p) -> (step, exp_avg, exp_avg_sq) or None for a parameter without state."""
    index, n = {}, 0
    for g in order:
        for p in g:
            index[id(p)] = n
            n += 1
    if len(order) != len(live_groups):
        raise RuntimeError(f"{len(live_groups)} optimizer groups for {len(order)} parameter groups")
    groups, state = [], {}
    for ref, live, lr, base in zip(order, live_groups, lrs, base_lrs):
        g = {k: v for k, v in live.items() if k != "params"}
        g.update(lr=float(lr), initial_lr=float(base), capturable=False, fused=None, foreach=None)
        g["params"] = [index[id(p)] for p in ref]
        groups.append(g)
        for p in live["params"]:
            m = moments(p)
            if m is not None:
                step, ea, eas = m
                state[index[id(p)]] = {"step": torch.tensor(float(step), dtype=torch.float32), "exp_avg": ea,
                                       "exp_avg_sq": eas}
    return {"state": state, "param_groups": groups}


def adamw_moments(optimizer):
    """export_adamw's moments(p) for a torch AdamW: its own per-parameter state, copied to the host."""
    def moments(p):
        st = optimizer.state.get(p)
        if not st:
            return None
        return float(st["step"]), to_cpu(st["exp_avg"]), to_cpu(st["exp_avg_sq"])
    return moments


def import_adamw(sd, order, live_groups):
    """Inverse of export_adamw: {parameter: (step, exp_avg, exp_avg_sq) or None} for every parameter of `live_groups`."""
    flat = [p for g in order for p in g]
    if len(sd["param_groups"]) != len(order) or any(len(g["params"]) != len(r) for g, r in zip(sd["param_groups"], order)):
        raise ValueError("optimizer state: the parameter groups differ from this model's get_opt_params()")
    by_id = {}
    for g in sd["param_groups"]:
        for i in g["params"]:
            by_id[id(flat[i])] = sd["state"].get(i, sd["state"].get(str(i)))
    out = {}
    for live in live_groups:
        for p in live["params"]:
            s = by_id[id(p)]
            out[p] = None if s is None else (float(s["step"]), s["exp_avg"], s["exp_avg_sq"])
    return out


def put_adamw_state(optimizer, moments):
    """Write {parameter: (step, exp_avg, exp_avg_sq) or None} into a torch AdamW: in place where the state already exists (a
    captured CUDA graph reads those tensors), created in the form the optimizer's own step makes otherwise."""
    for group in optimizer.param_groups:
        on_dev = bool(group.get("fused")) or bool(group.get("capturable"))
        for p in group["params"]:
            m = moments.get(p)
            st = optimizer.state.get(p)
            if m is None:
                if st and "exp_avg" in st:
                    st["exp_avg"].zero_()
                    st["exp_avg_sq"].zero_()
                    st["step"].fill_(0.0)
                continue
            step, ea, eas = m
            if st and "exp_avg" in st:
                st["exp_avg"].copy_(ea.view_as(p))
                st["exp_avg_sq"].copy_(eas.view_as(p))
                st["step"].fill_(step)
            else:
                optimizer.state[p] = {
                    "step": torch.tensor(step, dtype=torch.float32, device=p.device if on_dev else "cpu"),
                    "exp_avg": ea.to(p.device, p.dtype).view_as(p).clone(),
                    "exp_avg_sq": eas.to(p.device, p.dtype).view_as(p).clone()}


def lambda_lr_state(base_lrs, position, last_lrs):
    """torch LambdaLR.state_dict() of a schedule at `position` (the training steps keep the position as an integer instead
    of a LambdaLR)."""
    return {"base_lrs": [float(b) for b in base_lrs], "last_epoch": int(position), "_step_count": int(position) + 1,
            "_is_initial": False, "_get_lr_called_within_step": False, "_last_lr": [float(x) for x in last_lrs],
            "lr_lambdas": [None] * len(base_lrs)}


def refresh_derived(module):
    """Recompute in place what the forward derives from the parameters once and a captured graph keeps reading: the packed
    set-abstraction weight images of every PointNet++ that has packed them, and the bf16 shadows of ops.register_shadows."""
    from . import ops
    from .modules.pointnet import PointNetPP
    for m in module.modules():
        if isinstance(m, PointNetPP):
            m.refresh_pack_()
    ops.refresh_shadows()


def save_state(step, path):
    """step.state_dict() -> the directory `path` (layout above)."""
    st = step.state_dict()
    rank = _rank()
    os.makedirs(path, exist_ok=True)
    if rank == 0:
        for name, key in ((MODEL, "model"), (LOSS, "loss"), (OPTIMIZER, "optimizer"), (SCHEDULER, "scheduler"),
                          (NATIVE, "native")):
            torch.save(st[key], os.path.join(path, name))
    torch.save(st["random_states"], os.path.join(path, random_states_name(rank)))
    if _dist():
        dist.barrier()


def read_state(path):
    """The state dictionary of a directory written by save_state, with this rank's random states."""
    st = {}
    for name, key in ((MODEL, "model"), (LOSS, "loss"), (OPTIMIZER, "optimizer"), (SCHEDULER, "scheduler"),
                      (NATIVE, "native")):
        st[key] = torch.load(os.path.join(path, name), map_location="cpu", weights_only=True)
    st["random_states"] = torch.load(os.path.join(path, random_states_name(_rank())), map_location="cpu",
                                     weights_only=False)
    return st


def read_pretrain(path):
    """BaseTrainer.load_pretrain (trainer/build.py:174-184): every pytorch_model*.bin of `path`, merged."""
    files = sorted(glob.glob(os.path.join(str(path), "pytorch_model*.bin")))
    if not files:
        raise FileNotFoundError(f"Cannot find pytorch_model.bin in {path}")
    weights = {}
    for f in files:
        weights.update(torch.load(f, map_location="cpu", weights_only=True))
    return weights
