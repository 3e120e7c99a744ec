"""One GPS pre-training step (reference: trainer/openvocab_trainer.py:18-46 `train_step` + `backward`,
trainer/build.py:66-75,121,135-145): forward -> list loss -> backward -> clip_grad_norm_(5.0) -> AdamW -> warm-up/cosine.

Data parallelism (SURVEY.md §8e): one process per GPU, identical replicas, NCCL bucketed gradient all-reduce overlapped
with backward (torch DDP over NVLink) and the embedding all-gather inside the contrastive losses.  Parameters that
never receive a gradient on this path (the reference needs find_unused_parameters=True for them,
trainer/build.py:66) are listed statically and frozen instead of being searched for every step.
"""
import torch
import torch.distributed as dist
from torch import nn

from . import model as M
from . import ops
from .modules import losses as L

# parameters of the reference model that are constructed but never used in OpenVocab.forward
STATIC_UNUSED = ("point_encoder.sem_cls_embed_layer.", "point_encoder.sem_mask_embeddings.", "lang_encoder.model.pooler.")


class StepModule(nn.Module):
    """model + loss in one module so that a single DDP wrapper covers every trainable parameter (incl. logit_scale)."""

    def __init__(self, cfg):
        super().__init__()
        self.model = M.build_model(cfg)
        c = M.to_cfg(cfg)
        self.loss = L.Loss(c.model.loss_list, c.model.vis_loss_list, num_gpu=c.num_gpu,
                           emulate_dist=bool(c.get("emulate_dist", False)), task=c.get("task"))
        # the reference's optimizer groups (get_opt_params before anything is frozen here) + the loss group: the index space
        # of a checkpoint's optimizer state
        self.opt_order = [list(g['params']) for g in self.model.get_opt_params()]
        self.opt_order.append([p for p in self.loss.parameters() if p.requires_grad])
        for n, p in self.model.named_parameters():
            if n.startswith(STATIC_UNUSED):
                p.requires_grad = False
        self.train_log = None      # TrainLog of PretrainStep(train_eval=...): written after the losses, before backward

    def forward(self, data_dict):
        data_dict = self.model(data_dict)
        total, all_losses = self.loss(data_dict)
        if self.train_log is not None:
            self.train_log.write(data_dict, all_losses)
        return total, all_losses


class TrainLog:
    """The per-step train log of trainer/openvocab_trainer.py:26-46 without a host synchronisation per step.  Inside the step
    (captured in the CUDA graph), right after the losses, the evaluator's metric kernels add the batch into a per-step counter
    vector zeroed first, and one native write (sv_train_log_write) copies the device step, every loss-dict value and those
    counters into row (step % slots) of a device ring.  `read` copies the ring to the host once and builds one dictionary per
    step since the previous read with the evaluator's own count -> metric arithmetic (`counts_to_metrics`)."""

    def __init__(self, evaluator, loss_keys, slots, device):
        from . import _lib
        if slots < 1:
            raise ValueError(f"log_every must be at least 1, got {slots}")
        if len(loss_keys) > _lib.TRAIN_LOG_MAX_VALUES:
            raise ValueError(f"at most {_lib.TRAIN_LOG_MAX_VALUES} loss-dict entries can be logged, got {len(loss_keys)}")
        self.evaluator = evaluator
        self.loss_keys = list(loss_keys)
        self.slots = int(slots)
        self.counters = torch.zeros(evaluator.size, dtype=torch.float64, device=device)
        self.ring = torch.zeros((self.slots, 1 + len(self.loss_keys) + evaluator.size), dtype=torch.float64, device=device)
        self.own_step = torch.zeros(1, dtype=torch.int64, device=device)
        self.step_counter, self.advance = self.own_step, True    # eager: the write advances its own counter
        self.seen = 0          # device step of the newest entry already read (or discarded)
        self.pending = []      # (train/step, [lr of each group]) of the steps not read yet, in order

    def write(self, data_dict, all_losses):
        from . import _lib
        import ctypes
        if list(all_losses) != self.loss_keys:
            raise ValueError(f"loss-dict keys {list(all_losses)} differ from the logged {self.loss_keys}")
        with torch.no_grad():
            self.counters.zero_()
            try:
                self.evaluator._launch(data_dict, None, self.counters)
            except KeyError as e:
                raise KeyError(f"{type(self.evaluator).__name__} needs {e.args[0]!r}, which the step's data dict lacks") from None
            vals = [v.detach().reshape(()) if v.dtype == torch.float32 else v.detach().float().reshape(())
                    for v in all_losses.values()]
            ptrs = (ctypes.c_void_p * len(vals))(*[v.data_ptr() for v in vals])
            _lib.call(_lib.gps(), "sv_train_log_write", self.ring.device, len(vals), ptrs, self.counters.data_ptr(),
                      self.counters.numel(), self.step_counter.data_ptr(), int(self.advance), self.ring.data_ptr(), self.slots)

    def begin_step(self):
        if len(self.pending) >= self.slots:
            raise RuntimeError(f"{len(self.pending)} steps since the last logs() call fill the log ring (log_every = "
                               f"{self.slots}): call logs() at least every log_every steps")

    def end_step(self, step, lrs):
        self.pending.append((step, list(lrs)))

    def read(self):
        if not self.pending:
            return []
        ring = self.ring.cpu().tolist()                        # the one device-to-host copy
        rows = sorted((r for r in ring if r[0] > self.seen), key=lambda r: r[0])
        if len(rows) != len(self.pending):
            raise RuntimeError(f"the log ring holds {len(rows)} new entries for {len(self.pending)} steps")
        nl = len(self.loss_keys)
        out = []
        for row, (step, lrs) in zip(rows, self.pending):
            d = {"train/step": step}
            d.update((f"train/{k}", v) for k, v in zip(self.loss_keys, row[1:1 + nl]))
            d.update((f"train/{k}", v) for k, v in self.evaluator.counts_to_metrics(row[1 + nl:]).items())
            d.update((f"train/lr/group_{i}", lr) for i, lr in enumerate(lrs))
            out.append(d)
        self.seen = rows[-1][0]
        self.pending = []
        return out


class CapturedStep:
    """The CUDA-graph path PretrainStep and ObjClsStep share: static input buffers, eager set-up steps on a side stream, the
    capture (one graph, or with several ranks graph A | NCCL mean of flat_grads | graph B), the replay, and a checkpoint
    loaded before the capture applied right after it.  Subclasses set `device` and `graph_mode` and define `_apply_state`."""
    graph = graph_opt = static_batch = static_loss = flat_grads = None
    _pending_state = None             # a checkpoint loaded before the first graph-mode step

    def load_state_dict(self, state):
        """Continue from `state` (state_dict() of this configuration).  Eager, or graph mode after the capture: applied now,
        in place into the memory the graph reads.  Graph mode before the first step: applied right after the set-up steps
        and the capture, before the first replay, so the set-up steps leave no trace."""
        if self.graph_mode and self.graph is None:
            self._pending_state = state
            return
        self._apply_state(state)

    def _apply_pending(self):
        """Apply the checkpoint loaded before the capture, if any (the first replay continues it); True if there was one."""
        if self._pending_state is None:
            return False
        st, self._pending_state = self._pending_state, None
        self._apply_state(st)
        return True

    def save_state(self, path):
        """accelerate.save_state layout (sceneverse_b200/checkpoint.py): rank 0 writes the shared files, every rank its
        random states, then a barrier."""
        from . import checkpoint as C
        C.save_state(self, path)

    def load_state(self, path):
        """Every rank reads the directory written by save_state (its own random states) and load_state_dict()s it."""
        from . import checkpoint as C
        self.load_state_dict(C.read_state(path))

    def _copy_in(self, batch):
        """Put `batch` into the static input buffers the graphs read (the first call makes them); an input that already is
        the static buffer is not copied."""
        if self.static_batch is None:
            self.static_batch = {k: v.clone() for k, v in batch.items() if torch.is_tensor(v)}
            return
        for k, dst in self.static_batch.items():
            if batch[k].data_ptr() != dst.data_ptr():
                dst.copy_(batch[k], non_blocking=True)

    def _side_steps(self, step, n):
        """n calls of step() on a side stream, then a device synchronise: real optimisation steps before a capture, which
        allocate gradient and optimizer state outside the graph pool."""
        cur = torch.cuda.current_stream(self.device)
        side = torch.cuda.Stream(self.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(n):
                step()
        cur.wait_stream(side)
        torch.cuda.synchronize(self.device)

    def _capture_graphs(self, step, opt=None):
        """Capture step() (it returns the loss) as `graph`; with `opt`, step() is forward + backward only and opt() is
        captured as `graph_opt` in the same pool, and _replay all-reduces flat_grads between the two.  Counts the native
        kernel launches one replay makes."""
        from . import _lib
        n0 = _lib.launch_count()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.static_loss = step()
        if opt is not None:
            self.graph_opt = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph_opt, pool=self.graph.pool()):
                opt()
        self.native_launches_per_step = _lib.launch_count() - n0

    def _replay(self):
        self.graph.replay()
        if self.graph_opt is not None:
            self.flat_grads.all_reduce_mean()
            self.graph_opt.replay()
        return self.static_loss


class PretrainStep(CapturedStep):
    def __init__(self, cfg, device, total_steps=100000, dtype=torch.bfloat16, ddp=None, seed=0, cuda_graph=False,
                 overlap_allreduce=False, train_eval=None, log_every=100):
        """cuda_graph=True (single process, CUDA): after a few eager steps the whole step — forward, losses, backward,
        gradient clipping and AdamW — is captured once into a CUDA graph and replayed from static input buffers; the host
        then issues one graph launch per step instead of ~2000 kernel launches.  Dropout stays random: torch's own dropout
        through the graph-registered generator, the in-kernel masks through the device step counter registered with
        sv_dropout_seed_offset.

        train_eval (an evaluator of sceneverse_b200.evaluate: PretrainEval, ScanReferEval, ReferIt3DEval, ScanQAEval or
        SQA3DEval): every step also records its loss dict and the evaluator's counts on the device, inside the graph, and
        `logs()` returns them as the reference trainer's per-step log dictionaries.  log_every: the ring's size; more steps
        than that between two `logs()` calls raise.  None (the default) leaves the step as it is without logs."""
        torch.manual_seed(seed)
        self.cfg = M.to_cfg(cfg)
        if train_eval is not None and self.cfg.model.get("name") == "OpenVocabPerScene":
            raise ValueError("PretrainStep(train_eval=...) does not log per-scene steps: OpenVocabPerScene's outputs are "
                             "B*U rows against (B, U) targets")
        self.device = torch.device(device)
        self.module = StepModule(cfg).to(self.device)
        self.dtype = dtype
        groups = self.module.model.get_opt_params()
        groups.append({'params': [p for p in self.module.loss.parameters() if p.requires_grad], 'weight_decay': 0.0,
                       'lr': self.cfg.solver.lr})
        kw = dict(self.cfg.solver.optim.args)
        kw["betas"] = tuple(kw.get("betas", (0.9, 0.999)))
        self.use_ddp = ddp if ddp is not None else (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1)
        # cuda_graph with several ranks: no DDP wrapper — graph A (forward + losses + backward into one flat gradient
        # buffer), ONE eager NCCL all-reduce (mean) of that buffer, graph B (clipping + AdamW).  No collective is captured;
        # the contrastive exchange inside graph A is the native peer-memory kernel with a device-resident epoch.
        self.graph_mode = bool(cuda_graph) and self.device.type == "cuda"
        self.dp_graph = self.graph_mode and self.use_ddp
        # several ranks, opt-in: the gradient all-reduce of everything BEHIND the text encoder (spatial layers, joint layers,
        # heads, ~57 % of the 491 MB) is launched from an autograd hook as soon as those gradients are final and runs on NCCL's
        # stream under the text encoder's backward; both collectives are captured in the step's CUDA graph.  Parity with the
        # plain path is checked at 2 ranks (scripts/dp_overlap_2rank.py); the long-running bench hung with it on the 2-GPU box
        # (round 2), so the default is the un-overlapped graph | all-reduce | graph path.
        self.overlap_allreduce = bool(overlap_allreduce)
        self.overlapped = False
        self._ar_work = None
        if self.dp_graph:
            self.use_ddp = False
        warm = self.cfg.solver.sched.args.warmup_steps * self.cfg.num_gpu
        mr = self.cfg.solver.sched.args.get("minimum_ratio", 1e-5)
        self.total_steps = total_steps         # read at every evaluation: a loaded checkpoint restores it
        self._lr_lambda = lambda s: M.warmup_cosine(s, warm, self.total_steps, minimum_ratio=mr)
        self._capture_calls = None             # ops._dropout_calls when the replayed graph was captured
        # the warm-up/cosine schedule is its position _sched_step and the base lrs (_set_lrs); in graph mode the torch AdamW
        # holds the parameter groups but never steps: FlatState.optimizer_step does
        self.optimizer = torch.optim.AdamW(groups, lr=self.cfg.solver.lr, fused=self.device.type == "cuda", **kw)
        for g in self.optimizer.param_groups:       # each group's base lr, where torch's lr schedulers keep it
            g['initial_lr'] = g['lr']
        self._base_lrs = [float(g['initial_lr']) for g in self.optimizer.param_groups]
        self._sched_step = 0
        self._set_lrs()
        if self.graph_mode:
            self._step_counter = torch.zeros(1, dtype=torch.int64, device=self.device)
            from . import _lib
            _lib.check(_lib.gps(), _lib.gps().sv_dropout_seed_offset(self._step_counter.data_ptr()), "sv_dropout_seed_offset")
        self.grad_norm = self.cfg.solver.get("grad_norm")
        self.ddp = None
        self.probed = False
        self.module.train()
        self.global_step = 0
        self.train_log = None
        if train_eval is not None:
            self.train_log = TrainLog(train_eval, list(self.module.loss.loss_fn) + ["total_loss"], log_every, self.device)
            if self.graph_mode:    # the graph's own step counter indexes the ring
                self.train_log.step_counter, self.train_log.advance = self._step_counter, False
            self.module.train_log = self.train_log

    def logs(self):
        """One dictionary per step since the previous call, in order, with the reference trainer's keys (`train/step`,
        `train/<loss>` for every loss-dict entry and `train/total_loss`, `train/<metric>` of the evaluator's batch_metrics,
        `train/lr/group_i`), ready for accelerator.log; one device-to-host copy.  Needs train_eval."""
        if self.train_log is None:
            raise RuntimeError("PretrainStep was built without train_eval: there are no logs")
        return self.train_log.read()

    # ---- checkpoints ---------------------------------------------------------------------------------------------------
    def state_dict(self):
        """Everything a resumed run needs, on the host, independent of the flat layout: `model` / `loss` (state_dicts with
        the reference's keys), `optimizer` (torch AdamW.state_dict() form, parameter indices in get_opt_params() order, loss
        group last), `scheduler` (checkpoint.lambda_lr_state), `random_states` (this rank's generators) and `native` (global_step,
        total_steps, the device dropout counter, the in-kernel dropout seed position, the probed unused parameters)."""
        if self._pending_state is not None:          # loaded, not applied yet: that state is this step's state
            return self._pending_state
        from . import checkpoint as C
        flat = self.flat_grads
        if flat is not None:
            step = int(flat.step_t.item())
            host = {name: getattr(flat, name).cpu() for name in ("exp_avg", "exp_avg_sq")}

            def moments(p):
                o, n = flat.offsets[id(p)], p.numel()
                return step, host["exp_avg"][o:o + n].view(p.shape).clone(), host["exp_avg_sq"][o:o + n].view(p.shape).clone()
        else:
            moments = C.adamw_moments(self.optimizer)
        optim = C.export_adamw(self.module.opt_order, self.optimizer.param_groups, self._lrs(), self._base_lrs, moments)
        sched = C.lambda_lr_state(self._base_lrs, self._sched_step, self._lrs())
        counter = getattr(self, "_step_counter", None)
        return {"model": C.to_cpu(self.module.model.state_dict()), "loss": C.to_cpu(self.module.loss.state_dict()),
                "optimizer": optim, "scheduler": sched, "random_states": C.rng_state(),
                "native": {"global_step": self.global_step, "total_steps": self.total_steps,
                           "dropout_counter": int(counter.item()) if counter is not None else None,
                           "dropout_calls": ops._dropout_calls[0], "capture_dropout_calls": self._capture_calls,
                           "unused_parameters": list(self.unused_parameters) if self.probed else None}}

    def _seed_capture(self):
        """The in-kernel dropout seeds are host constants of the captured graph (ops._next_dropout_seed: torch's initial
        seed and a call counter): capture with those of the checkpoint being resumed, and remember them for the next one."""
        st = self._pending_state
        if st is not None and st["native"].get("capture_dropout_calls") is not None:
            torch.set_rng_state(st["random_states"]["torch_manual_seed"])     # torch.initial_seed() of the saved run
            ops._dropout_calls[0] = st["native"]["capture_dropout_calls"]
        self._capture_calls = ops._dropout_calls[0]

    @torch.no_grad()
    def _apply_state(self, state):
        """load_state_dict's work.  After the capture it writes in place into what the graph reads (flat parameters,
        moments, bf16 shadows, step_t, lr_factor, the dropout counter) and recomputes in place everything derived from the
        parameters at capture (PointNet++ packed weights, register_shadows shadows).  A checkpoint loaded before the first
        graph-mode step also gave the capture its in-kernel dropout seeds (_seed_capture), so the run continues exactly as
        the saved one would have."""
        from . import checkpoint as C
        nat = state["native"]
        if not self.probed and nat.get("unused_parameters") is not None:
            self._freeze_unused(nat["unused_parameters"])
        elif self.probed and nat.get("unused_parameters") is not None and \
                sorted(nat["unused_parameters"]) != sorted(self.unused_parameters):
            raise ValueError("the checkpoint's unused parameters differ from this step's: another configuration")
        self.module.model.load_state_dict(state["model"])        # copy_ into the existing (flat-buffer) storage
        self.module.loss.load_state_dict(state["loss"])
        moments = C.import_adamw(state["optimizer"], self.module.opt_order, self.optimizer.param_groups)
        self.total_steps = int(nat["total_steps"])
        flat = self.flat_grads
        if flat is not None:
            steps = {m[0] for m in moments.values() if m is not None}
            if len(steps) > 1:
                raise ValueError(f"per-parameter AdamW steps {sorted(steps)}: the flat optimizer keeps one step for all")
            for p, m in moments.items():
                o, n = flat.offsets[id(p)], p.numel()
                flat.exp_avg[o:o + n].copy_(m[1].reshape(-1) if m is not None else torch.zeros(n))
                flat.exp_avg_sq[o:o + n].copy_(m[2].reshape(-1) if m is not None else torch.zeros(n))
            flat.step_t.fill_(int(steps.pop()) if steps else 0)
            flat.shadow.copy_(flat.flat_p)
        else:
            C.put_adamw_state(self.optimizer, moments)
        C.refresh_derived(self.module)
        if flat is not None:
            self._check_in_place(flat)
        self._sched_step = int(state["scheduler"]["last_epoch"])
        self._set_lrs()
        counter = getattr(self, "_step_counter", None)
        if counter is not None:
            counter.fill_(nat["dropout_counter"] or 0)
        C.set_rng_state(state["random_states"])
        ops._dropout_calls[0] = int(nat["dropout_calls"])
        self.global_step = int(nat["global_step"])
        if self.train_log is not None:          # entries of this object's earlier steps are not steps of the resumed run
            self.train_log.ring.zero_()
            self.train_log.seen = int(self.train_log.step_counter.item())
            self.train_log.pending = []

    def _check_in_place(self, flat):
        """A captured graph reads the flat buffers and the shadows registered at capture: refuse to continue if a parameter
        no longer lives there (its new values would never reach the graph)."""
        from .modules.pointnet import PointNetPP
        base = flat.flat_p.data_ptr()
        for p in flat.params:
            if p.data_ptr() != base + 4 * flat.offsets[id(p)]:
                raise RuntimeError("a parameter was moved out of the flat buffer: the captured graph would train stale weights")
        for s, p in ops._SHADOW.values():
            if s.shape != p.shape:
                raise RuntimeError("a bf16 shadow no longer matches its parameter")
        for m in self.module.modules():
            if isinstance(m, PointNetPP) and m._packed is not None and \
                    m._packed_key != tuple((t.data_ptr(), t._version) for t in list(m.parameters()) + list(m.buffers())):
                raise RuntimeError("the PointNet++ packed weights were not refreshed")

    @torch.no_grad()
    def load_pretrain(self, path):
        """BaseTrainer.load_pretrain (trainer/build.py:174-184): every pytorch_model*.bin of `path` into the model,
        strict=False, before the first step.  Returns (missing_keys, unexpected_keys).  An ObjClsStep checkpoint names its
        backbone `point_feature_extractor.*`; that is the object encoder's PointNet++ here (the stage hand-off that
        all_pretrain_unfreeze.yaml makes through `vision.args.path`), so those keys load into it."""
        if self.probed:
            raise RuntimeError("load_pretrain must run before the first step")
        from . import checkpoint as C
        sd = C.read_pretrain(path)
        obj = "point_feature_extractor."
        sd = {("point_encoder." + k if k.startswith(obj) else k): v for k, v in sd.items()}
        return self.module.model.load_state_dict(sd, strict=False)

    def _lrs(self):
        return [g['lr'] for g in self.optimizer.param_groups]

    def _set_lrs(self):
        """The schedule at _sched_step: base lr * factor into the param groups (the lrs the eager AdamW reads and the logs
        and checkpoints report) and, once the flat state exists, the factor into FlatState.lr_factor (the captured AdamW's)."""
        f = self._lr_lambda(self._sched_step)
        for g, base in zip(self.optimizer.param_groups, self._base_lrs):
            g['lr'] = base * f
        if self.flat_grads is not None:
            self.flat_grads.lr_factor.fill_(f)

    def _advance_lr(self):
        self._sched_step += 1
        self._set_lrs()

    def _probe_unused(self, data_dict):
        """One local forward/backward to find the parameters this configuration never touches (e.g. the object LM head
        when `obj_cls_post_logits` is in no loss, all_pretrain.yaml:246-258).  They are frozen once, so DDP can run with
        find_unused_parameters=False instead of the reference's per-step graph search (trainer/build.py:66)."""
        self.optimizer.zero_grad(set_to_none=True)
        log, self.module.train_log = self.module.train_log, None      # not a training step: nothing to log
        try:
            with torch.autocast(self.device.type, dtype=self.dtype, enabled=self.dtype != torch.float32):
                total, _ = self.module(dict(data_dict))
        finally:
            self.module.train_log = log
        total.backward()
        unused = [n for n, p in self.module.named_parameters() if p.requires_grad and p.grad is None]
        self.optimizer.zero_grad(set_to_none=True)
        self._freeze_unused(unused)

    def _freeze_unused(self, unused):
        """Freeze the parameters named in `unused` (found by _probe_unused, or read from a checkpoint) and wrap in DDP."""
        names = set(unused)
        for n, p in self.module.named_parameters():
            if n in names:
                p.requires_grad = False
        for g in self.optimizer.param_groups:
            g['params'] = [p for p in g['params'] if p.requires_grad]
        self.unused_parameters = unused
        if self.use_ddp:
            self._wrap_ddp()
        self.probed = True

    def _wrap_ddp(self):
        self.ddp = nn.parallel.DistributedDataParallel(
            self.module, device_ids=[self.device.index] if self.device.type == "cuda" else None,
            find_unused_parameters=False, gradient_as_bucket_view=True, bucket_cap_mb=64)

    def parameters(self):
        return [p for p in self.module.parameters() if p.requires_grad]

    def close(self):
        """Unregister the process-wide hooks of graph mode (the dropout seed counter lives in this object's memory, the
        bf16 weight shadows reference its parameters)."""
        if getattr(self, "_step_counter", None) is not None:
            self._step_counter = None
            try:
                from . import _lib
                _lib.gps().sv_dropout_seed_offset(None)
                ops.clear_shadows()
            except Exception:      # interpreter shutdown: modules may already be gone
                pass

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- CUDA-graph path ---------------------------------------------------------------------------------------------
    def _raw_fwd_bwd(self):
        self._step_counter.add_(1)
        self.flat_grads.zero()
        # gradients live in the flat buffer: the wgrad kernels accumulate into it directly (no AccumulateGrad adds)
        prev, ops.DIRECT_GRAD[0] = ops.DIRECT_GRAD[0], True
        self._ar_work = None
        self.module.model._lang_grad_hook = self._early_allreduce if self._overlap_now else None
        try:
            with torch.autocast(self.device.type, dtype=self.dtype, enabled=self.dtype != torch.float32):
                total, _ = self.module(dict(self.static_batch))
            total.backward()
        finally:
            ops.DIRECT_GRAD[0] = prev
            self.module.model._lang_grad_hook = None
        return total.detach()

    _overlap_now = False

    def _early_allreduce(self, grad):
        """autograd hook on the text encoder's output: its gradient is complete, so (the autograd engine runs nodes in reverse
        forward order) every node created after the text encoder's forward has run its backward — the gradients of the
        spatial layers, joint layers, heads and losses are final.  Their slice of the flat buffer goes out now."""
        if self._ar_work is None:
            tail = self.flat_grads.flat[self._lang_end:]
            self._ar_work = dist.all_reduce(tail, op=dist.ReduceOp.AVG, async_op=True)
        return None

    def _finish_allreduce(self):
        head = self.flat_grads.flat[:self._lang_end]
        if self._ar_work is not None:
            self._ar_work.wait()
            dist.all_reduce(head, op=dist.ReduceOp.AVG)
        else:                                   # the hook did not fire (no gradient reached the text encoder's output)
            self.flat_grads.all_reduce_mean()
        self._ar_work = None

    def _raw_step(self):
        """One step of what the graph records, run eagerly on the flat state."""
        loss = self._raw_fwd_bwd()
        if self._overlap_now:
            self._finish_allreduce()
        else:
            self.flat_grads.all_reduce_mean()
        self.flat_grads.optimizer_step()                    # native: clip + AdamW + bf16 shadows, one pass
        return loss

    def _lang_boundary(self):
        """Offset in the flat buffers where the text encoder's parameters end — valid only if they form the head of the layout
        (they do: model.get_opt_params lists the language encoder first)."""
        flat = self.flat_grads
        lang = {id(p) for p in self.module.model.lang_encoder.parameters()}
        end_lang = max((flat.offsets[i] + p.numel() for p in flat.params for i in [id(p)] if i in lang), default=0)
        first_other = min((flat.offsets[id(p)] for p in flat.params if id(p) not in lang), default=flat.n)
        if end_lang == 0 or end_lang > first_other:
            return None
        return (end_lang + 7) // 8 * 8 if (end_lang + 7) // 8 * 8 <= first_other else end_lang

    def _make_flat_state(self):
        """The graph path's optimizer: the trainable parameters, their gradients, AdamW moments and bf16 shadows moved
        into one FlatState (flat_grads) at the schedule's current lr, and the packed sibling projections registered."""
        kw = dict(self.cfg.solver.optim.args)
        self.flat_grads = FlatState(self.optimizer.param_groups, self._base_lrs, betas=tuple(kw.get("betas", (0.9, 0.999))),
                                    eps=float(kw.get("eps", 1e-8)), max_norm=self.grad_norm)
        self._set_lrs()
        register_packs(self.module, self.flat_grads)

    def _set_up_step(self):
        self._raw_step()
        self._advance_lr()

    def _capture(self, data_dict):
        self._copy_in(data_dict)
        if self.dp_graph:
            sync_module_state(self.module)
        ops.clear_shadows()
        self._make_flat_state()
        if self.dtype == torch.bfloat16:
            ops.register_shadows(self.module)       # whatever bf16 linears read outside the flat buffer (frozen parameters)
        self._side_steps(self._set_up_step, 3)
        self._seed_capture()
        if self.dp_graph:
            self._capture_graphs(self._raw_fwd_bwd, self.flat_grads.optimizer_step)
        else:
            self._capture_graphs(self._raw_step)
        if self.dp_graph and self.overlap_allreduce:
            self._lang_end = self._lang_boundary()
            if self._lang_end is not None:
                try:
                    self._overlap_now = True
                    self._side_steps(self._set_up_step, 1)     # one eager step through the hook path (NCCL warm-up)
                    self._seed_capture()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, pool=self.graph.pool()):
                        loss = self._raw_step()       # forward + backward + both all-reduces + clip/AdamW: ONE graph
                    self.graph_overlap, self.static_loss_overlap = g, loss
                    self.overlapped = True
                except Exception as e:                  # NCCL capture unsupported here: keep the two-graph path
                    self._overlap_now = False
                    torch.cuda.synchronize(self.device)
                    if dist.get_rank() == 0:
                        print(f"[sceneverse_b200] overlapped all-reduce unavailable ({type(e).__name__}: {e}); "
                              "using graph | all-reduce | graph")
                finally:
                    self._overlap_now = False
        if self.train_log is not None:          # the eager set-up steps' entries are not steps of the run
            self.train_log.seen = int(self._step_counter.item())

    def _dp_graph_possible(self):
        """Graph A must not contain an NCCL collective: with several ranks the contrastive exchange has to be the native
        peer-memory kernel.  If symmetric memory could not be set up (losses then use NCCL all_gather), run eager DDP."""
        from . import fused_gather
        return all(v is not None for v in fused_gather._state.values())

    def _probe_or_restore(self, data_dict):
        unused = self._pending_state["native"].get("unused_parameters") if self._pending_state is not None else None
        if unused is not None:
            self._freeze_unused(unused)       # the checkpoint's flat layout; no probing pass on the resumed run's batch
        else:
            self._probe_unused(data_dict)

    def _graph_step(self, data_dict):
        if not self.probed:
            self._probe_or_restore(data_dict)
            if self.dp_graph and not self._dp_graph_possible():      # the eager data-parallel step from here on
                self.graph_mode = self.dp_graph = False
                self.use_ddp = True
                self._wrap_ddp()
                if self.train_log is not None:
                    self.train_log.step_counter, self.train_log.advance = self.train_log.own_step, True
                self._apply_pending()
                return self._step(data_dict)
        if self.graph is None:
            self._capture(data_dict)
            self._apply_pending()
        self._copy_in(data_dict)
        if self.overlapped:
            self.graph_overlap.replay()
            self._advance_lr()
            return self.static_loss_overlap
        loss = self._replay()
        self._advance_lr()
        return loss

    def phase_times(self, data_dict, steps=5):
        """(ms_fwd_bwd, ms_allreduce, ms_opt) of the NON-overlapped data-parallel step (graph | NCCL | graph), CUDA events on
        the current stream; the parameters do advance (these are real steps)."""
        assert self.dp_graph and self.graph is not None and self.graph_opt is not None
        warm = 3                      # un-timed: the ranks fall into step (the exchange kernel waits for the slowest peer)
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(warm + steps)]
        self._copy_in(data_dict)
        torch.cuda.synchronize(self.device)
        dist.barrier()
        for e in ev:
            e[0].record()
            self.graph.replay()
            e[1].record()
            self.flat_grads.all_reduce_mean()
            e[2].record()
            self.graph_opt.replay()
            e[3].record()
            self._advance_lr()
        torch.cuda.synchronize(self.device)
        return tuple(sum(e[i].elapsed_time(e[i + 1]) for e in ev[warm:]) / steps for i in range(3))

    def step(self, data_dict):
        """data_dict: tensors already on self.device. Returns the (detached) total loss tensor — no host sync.
        Graph mode: (1) the FIRST call runs the un-timed set-up on its batch — one probing forward/backward, three eager
        optimisation steps (they allocate gradient / optimizer state outside the graph pool), the capture, and the first replay —
        i.e. four parameter updates on that batch, unlike the reference's one step per batch; feed a throw-away batch first if
        that matters.  (2) the returned tensor is the graph's STATIC loss buffer, overwritten by the next replay: read it
        (`.item()` / `.clone()`) before calling step() again if the value has to be kept."""
        if self.train_log is not None:
            self.train_log.begin_step()
        loss = self._step(data_dict)
        self.global_step += 1
        if self.train_log is not None:
            self.train_log.end_step(self.global_step, self._lrs())
        return loss

    def _step(self, data_dict):
        if self.graph_mode:
            return self._graph_step(data_dict)
        if not self.probed:
            self._probe_or_restore(data_dict)
        net = self.ddp if self.ddp is not None else self.module
        self.optimizer.zero_grad(set_to_none=True)
        with torch.autocast(self.device.type, dtype=self.dtype, enabled=self.dtype != torch.float32):
            total, _ = net(data_dict)
        total.backward()
        if self.grad_norm is not None:
            torch.nn.utils.clip_grad_norm_(self.parameters(), self.grad_norm, foreach=True)
        self.optimizer.step()
        self._advance_lr()
        return total.detach()


class FlatGrads:
    """Gradients of `params` as views of ONE flat fp32 buffer, so that the data-parallel mean is a single NCCL call (the
    reference's DDP reduces the same 491 MB in 25 MB buckets, trainer/build.py:66-75)."""

    def __init__(self, params):
        self.params = [p for p in params if p.requires_grad]
        n = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(n, dtype=self.params[0].dtype, device=self.params[0].device)
        o = 0
        for p in self.params:
            p.grad = self.flat[o:o + p.numel()].view_as(p)
            o += p.numel()

    def zero(self):
        self.flat.zero_()

    def all_reduce_mean(self, group=None):
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            if dist.get_backend(group) == "nccl":
                dist.all_reduce(self.flat, op=dist.ReduceOp.AVG, group=group)
            else:
                dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
                self.flat.div_(dist.get_world_size(group))


class FlatState(FlatGrads):
    """Parameters, gradients, AdamW moments and the bf16 weight shadows of the trainable parameters as slices of FIVE flat
    buffers with one layout (parameter-group by parameter-group, every tensor starting on a 16-byte boundary of the bf16
    copy).  What that buys (SURVEY.md §8 f3):
      * clip_grad_norm_ + AdamW + the fp32 -> bf16 shadow refresh are ONE pass over HBM (csrc/train_ops.cu adamw_flat_kernel:
        read p, g, m, v; write p, m, v, bf16 p) after a squared-norm pass over g — instead of torch's multi-tensor AdamW
        (16 launches), 2 clipping launches and a 65-launch shadow copy;
      * the data-parallel mean is one NCCL call on `flat` (as before);
      * sibling projections that read the same input (w_qs | w_ks | w_vs of the spatial attention, query | key | value of
        BERT) are ADJACENT in every buffer, so [3E, E] views of the shadow / gradient buffers let ops.linear_packed run them
        as one GEMM in each direction."""
    ALIGN = 8

    def __init__(self, groups, base_lrs, betas=(0.9, 0.999), eps=1e-8, max_norm=None):
        params, segs, off = [], [], 0
        for g, lr in zip(groups, base_lrs):
            ps = [p for p in g['params'] if p.requires_grad]
            if not ps:
                continue
            begin = off
            for p in ps:
                params.append((p, off))
                off += (p.numel() + self.ALIGN - 1) // self.ALIGN * self.ALIGN
            segs.append((begin, off, float(lr), float(g.get('weight_decay', 0.0))))
        dev = params[0][0].device
        self.params = [p for p, _ in params]
        self.n = off
        self.flat_p = torch.zeros(off, dtype=torch.float32, device=dev)
        self.flat = torch.zeros(off, dtype=torch.float32, device=dev)          # gradients (name kept from FlatGrads)
        self.exp_avg = torch.zeros(off, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(off, dtype=torch.float32, device=dev)
        self.shadow = torch.zeros(off, dtype=torch.bfloat16, device=dev)
        self.offsets = {}
        pairs = []
        for p, o in params:
            n = p.numel()
            self.flat_p[o:o + n].copy_(p.detach().reshape(-1))
            p.data = self.flat_p[o:o + n].view_as(p)
            p.grad = self.flat[o:o + n].view_as(p)
            pairs.append((p, self.shadow[o:o + n].view_as(p)))
            self.offsets[id(p)] = o
        self.shadow.copy_(self.flat_p)
        ops.register_shadow_views(pairs)
        import numpy as np
        seg_dt = np.dtype([("begin", "<i8"), ("end", "<i8"), ("lr_scale", "<f4"), ("weight_decay", "<f4")])
        self.segments = torch.from_numpy(np.array(segs, dtype=seg_dt).view(np.uint8).copy()).to(dev)
        self.nseg = len(segs)
        self.betas, self.eps, self.max_norm = betas, eps, max_norm
        self.lr_factor = torch.ones(1, dtype=torch.float32, device=dev)
        self.step_t = torch.zeros(1, dtype=torch.int64, device=dev)
        self.grad_norm_t = torch.zeros(1, dtype=torch.float32, device=dev)
        from . import _lib
        self.scratch = torch.zeros(_lib.gps().sv_adamw_scratch_floats(), dtype=torch.float32, device=dev)

    def packed_views(self, params):
        """[sum N, K] / [sum N] views of the shadow, gradient and parameter buffers spanning `params` if they are adjacent
        in the flat layout (same trailing shape, no alignment gaps), else None."""
        offs = [self.offsets.get(id(p)) for p in params]
        if any(o is None for o in offs):
            return None
        tail = params[0].shape[1:]
        o = offs[0]
        for p, po in zip(params, offs):
            if po != o or p.shape[1:] != tail:
                return None
            o += p.numel()
        rows = sum(p.shape[0] for p in params)
        sl = slice(offs[0], o)
        return (self.shadow[sl].view(rows, *tail), self.flat[sl].view(rows, *tail), self.flat_p[sl].view(rows, *tail))

    def optimizer_step(self):
        """clip (max_norm) + AdamW + shadow refresh; the step counter lives on the device (CUDA-graph replay safe)."""
        from . import _lib
        self.step_t.add_(1)
        _lib.call(_lib.gps(), "sv_adamw_flat", self.flat.device, self.flat_p.data_ptr(), self.exp_avg.data_ptr(),
                  self.exp_avg_sq.data_ptr(), self.flat.data_ptr(), self.shadow.data_ptr(), self.n, self.segments.data_ptr(),
                  self.nseg, float(self.max_norm) if self.max_norm is not None else 0.0, self.lr_factor.data_ptr(),
                  self.step_t.data_ptr(), 1.0, float(self.betas[0]), float(self.betas[1]), float(self.eps),
                  self.scratch.data_ptr(), self.grad_norm_t.data_ptr())


def register_packs(module, flat):
    """Tell ops.linear_packed which sibling projections are adjacent in the flat buffers."""
    from .modules.layers import MultiHeadAttentionSpatial
    for m in module.modules():
        trip = None
        if isinstance(m, MultiHeadAttentionSpatial):
            trip = (m.w_qs, m.w_ks, m.w_vs)
        elif all(hasattr(m, a) and isinstance(getattr(m, a), nn.Linear) for a in ("query", "key", "value")):
            trip = (m.query, m.key, m.value)       # HF BertSelfAttention
        if trip is None or any(l.bias is None for l in trip):
            continue
        w = flat.packed_views([l.weight for l in trip])
        b = flat.packed_views([l.bias for l in trip])
        if w is not None and b is not None:
            ops.register_pack([l.weight for l in trip], [l.bias for l in trip], w, b)


def sync_module_state(module, src=0):
    """What DDP does at construction: every rank starts from rank `src`'s parameters and buffers."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        for t in list(module.parameters()) + list(module.buffers()):
            dist.broadcast(t.data, src)


def batch_to_device(np_batch, device, pinned=None, non_blocking=True):
    """numpy data_dict (synthetic.scene_batch) -> tensors on device; `pinned` = matching dict of pinned host tensors."""
    out = {}
    for k, v in np_batch.items():
        src = pinned[k] if pinned is not None else torch.from_numpy(v)
        out[k] = src.to(device, non_blocking=non_blocking)
    return out


class ObjClsStep(CapturedStep):
    """Object-level pre-training step (reference: model/objcls.py:64-98 + optim/loss/loss.py:96-102, BASELINE.json configs[1]):
    PointNet++ TRAINABLE with train-mode BatchNorm -> dropout -> 607-way open-vocabulary logits -> label-smoothed CE ->
    AdamW.  The point operators and their gradients (group_points_grad / gather) are the native kernels; conv / BatchNorm
    statistics run on cuDNN / ATen (the fused tensor-core SA-MLP is the eval-BN form).  cuda_graph=True captures the whole
    step after three eager ones.

    num_gpu > 1 (one process per GPU, process group initialised): the backbone's BatchNorm layers are SyncBatchNorm
    (objcls.py:33-34).  Every rank starts from rank 0's parameters and buffers.  With cuda_graph=True and the native statistics
    exchange available (pn_train.exchange_for) a step is graph A (forward + backward into one flat gradient buffer, the 18
    SyncBatchNorm exchanges included) | one NCCL all-reduce (mean) of that buffer | graph B (AdamW), as PretrainStep's
    data-parallel graph path; no collective is captured.  Otherwise the model runs eagerly under DDP."""

    def __init__(self, device, text_embeds, lr=1e-3, dtype=torch.bfloat16, seed=0, cuda_graph=False, num_gpu=1):
        torch.manual_seed(seed)
        self.device, self.dtype = torch.device(device), dtype
        self.model = M.ObjCls({"num_gpu": num_gpu, "solver": {"lr": lr}}, text_embeds=text_embeds).to(self.device).train()
        self.graph_mode = bool(cuda_graph) and self.device.type == "cuda"
        self.ddp = None
        if num_gpu > 1 and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            from . import pn_train
            sync_module_state(self.model)
            if self.graph_mode and pn_train.exchange_for(self.model.point_feature_extractor, self.device):
                self.flat_grads = FlatGrads(self.model.parameters())
            else:
                self.graph_mode = False
                self.ddp = nn.parallel.DistributedDataParallel(
                    self.model, device_ids=[self.device.index] if self.device.type == "cuda" else None)
        self.optimizer = torch.optim.AdamW(self.model.parameters(), lr=torch.tensor(lr, device=self.device) if self.graph_mode else lr,
                                           fused=self.device.type == "cuda", capturable=self.graph_mode)
        self.lr = lr
        self.global_step = 0

    # ---- checkpoints: the layout and forms of PretrainStep's (sceneverse_b200/checkpoint.py) ------------------------------
    def state_dict(self):
        """`model` (PointNet++ with the BatchNorm running statistics, the text embeddings), `loss` (empty: the label-smoothed
        CE has no parameters), `optimizer` (torch AdamW form, one group over model.parameters()), `scheduler` (constant lr,
        LambdaLR form), `random_states`, `native` (global_step)."""
        if self._pending_state is not None:
            return self._pending_state
        from . import checkpoint as C
        order = [list(self.model.parameters())]
        return {"model": C.to_cpu(self.model.state_dict()), "loss": {},
                "optimizer": C.export_adamw(order, self.optimizer.param_groups, [self.lr], [self.lr],
                                            C.adamw_moments(self.optimizer)),
                "scheduler": C.lambda_lr_state([self.lr], self.global_step, [self.lr]), "random_states": C.rng_state(),
                "native": {"global_step": self.global_step, "total_steps": None, "dropout_counter": None,
                           "dropout_calls": None, "capture_dropout_calls": None, "unused_parameters": []}}

    @torch.no_grad()
    def _apply_state(self, state):
        from . import checkpoint as C
        self.model.load_state_dict(state["model"])
        order = [list(self.model.parameters())]
        C.put_adamw_state(self.optimizer, C.import_adamw(state["optimizer"], order, self.optimizer.param_groups))
        C.refresh_derived(self.model)
        C.set_rng_state(state["random_states"])
        self.global_step = int(state["native"]["global_step"])

    def _fwd_bwd(self, batch):
        if self.flat_grads is not None:
            self.flat_grads.zero()
        else:
            self.optimizer.zero_grad(set_to_none=False)
        with torch.autocast(self.device.type, dtype=self.dtype, enabled=self.dtype != torch.float32):
            out = (self.ddp if self.ddp is not None else self.model)(dict(batch))
            loss = L.obj_cls_loss(out)
        loss.backward()
        return loss.detach()

    def _raw(self, batch):
        loss = self._fwd_bwd(batch)
        if self.flat_grads is not None:
            self.flat_grads.all_reduce_mean()
        self.optimizer.step()
        return loss

    def step(self, batch):
        self.global_step += 1
        if not self.graph_mode:
            return self._raw(batch)
        if self.graph is None:
            self._copy_in(batch)
            static = self.static_batch
            self._side_steps(lambda: self._raw(static), 3)
            if self.flat_grads is None:
                self._capture_graphs(lambda: self._raw(static))
            else:
                self._capture_graphs(lambda: self._fwd_bwd(static), self.optimizer.step)
            if self._apply_pending():       # the checkpoint's global_step counts the steps before this one
                self.global_step += 1
        self._copy_in(batch)
        return self._replay()
