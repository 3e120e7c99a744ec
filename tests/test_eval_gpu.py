"""Evaluation on the GPU: the metric kernels (csrc/eval_metrics.cu) against the counters restated in tests/test_eval_host.py
from the golden batches of the unmodified evaluators, graph replay against eager updates, the grounding targets
(csrc/eval_targets.cu) against the numpy-1.26 restatement, and evaluation through the real models."""
import numpy as np
import pytest
import torch

from oracle import make_golden_eval as G
from sceneverse_b200 import evaluate, input_pipeline as IP
from tests.test_eval_host import batch, host_counters, meta

pytestmark = pytest.mark.gpu


def to_dev(d, dtype=None, pad_to=None):
    out = {}
    for k, v in d.items():
        v = v.cuda()
        if k.endswith(("logits", "scores")) and dtype is not None:
            v = v.to(dtype)
            if pad_to is not None:              # padded-vocabulary rows, read in place
                w = torch.full(v.shape[:-1] + (pad_to,), 7.0, dtype=dtype, device="cuda")
                w[..., :v.shape[-1]] = v
                v = w[..., :v.shape[-1]]
        out[k] = v
    return out


@pytest.mark.parametrize("dtype,pad", [(torch.float32, None), (torch.bfloat16, 712)])
@pytest.mark.parametrize("case", list(G.CASES))
def test_counters_match_restatement(case, dtype, pad):
    """Every counter after every batch equals the host restatement exactly (top-10 ties: lower index first); the grading
    values are exact in bf16, so both dtypes give the same counters."""
    M, meta_ = meta()
    m = meta_[case]
    ev = getattr(evaluate, m["evaluator"])()
    want = ev.counters.cpu().tolist()
    for i in range(m["batches"]):
        d = batch(M, case, i)
        host_counters(case, d, want)
        ev.update(to_dev(d, dtype, pad))
        assert ev.counters.cpu().tolist() == want, (case, i)


def test_graph_replay_equals_eager():
    M, meta_ = meta()
    for case in ("scanrefer", "sqa3d"):
        m = meta_[case]
        eager = getattr(evaluate, m["evaluator"])()
        graph = getattr(evaluate, m["evaluator"])()
        batches = [to_dev(batch(M, case, i)) for i in range(m["batches"])]
        for b in batches:
            eager.update(b)
        runner = evaluate.EvalRunner(lambda d: d, [graph], batch_size=batches[0]["obj_masks"].shape[0],
                                     dtype=torch.float32)
        runner.run(batches)
        assert graph.counters.tolist() == eager.counters.tolist(), case
        runner.run(batches)                    # replayed again after reset: same sums
        assert graph.counters.tolist() == eager.counters.tolist(), case


def test_box_iou_and_flags_match_numpy126():
    Z = np.load(G.os.path.join(G.OUT, "eval_boxes.npz"))
    n = len(Z["names"])
    ci = np.concatenate([[0], np.cumsum(Z["cand_len"])])
    gi = np.concatenate([[0], np.cumsum(Z["gt_len"])])
    pts = torch.from_numpy(Z["cand"]).cuda()
    out = IP.grounding_targets(pts, torch.from_numpy(ci).cuda(), np.arange(n + 1), torch.zeros(n, dtype=torch.int64).cuda(),
                               torch.zeros(n, dtype=torch.int64).cuda(), 4, gt_points=torch.from_numpy(Z["gt"]).cuda(),
                               gt_offsets=torch.from_numpy(gi).cuda(), return_iou=True)
    slot_map, tgt, i25, i50, iou = (t.cpu().numpy() for t in out)
    want = Z["iou_np126"]
    assert np.array_equal(iou, want.astype(np.float32))
    assert np.array_equal(i25[:, 0], (want >= 0.25).astype(np.int64))
    assert np.array_equal(i50[:, 0], (want >= 0.5).astype(np.int64))
    assert np.array_equal(tgt[:, 0], np.where(want >= 0.25, 0, 1))
    assert (slot_map[:, 0] == 0).all() and (slot_map[:, 1:] == -1).all()


def crop_items(seed, B=6, O=8):
    rng = np.random.default_rng(seed)
    n = rng.integers(3, 30, size=B)
    gt = [rng.uniform(-1, 1, 3) for _ in range(B)]
    pts, clen, labels = [], [], []
    for b in range(B):
        for c in range(n[b]):
            near = rng.random() < 0.25
            ctr = gt[b] + (rng.normal(0, 0.05, 3) if near else rng.uniform(-5, 5, 3))
            p = ctr + rng.uniform(-0.5, 0.5, (int(rng.integers(1, 40)), 3))
            pts.append(np.concatenate([p, np.zeros_like(p)], 1))
            clen.append(len(p))
            labels.append(int(rng.integers(0, 3)))
    gts = [np.concatenate([g + rng.uniform(-0.5, 0.5, (30, 3)), np.zeros((30, 3))], 1) for g in gt]
    return (np.concatenate(pts).astype(np.float32), np.concatenate([[0], np.cumsum(clen)]), np.concatenate([[0], np.cumsum(n)]),
            np.array(labels), rng.integers(0, 3, size=B), np.concatenate(gts).astype(np.float32), np.arange(B + 1) * 30, O)


def test_crop_priority_and_draw():
    pts, co, io, lab, tl, gpts, go, O = crop_items(3)
    args = [torch.from_numpy(pts).cuda(), torch.from_numpy(co).cuda(), io, torch.from_numpy(lab).cuda(),
            torch.from_numpy(tl).cuda(), O]
    kw = dict(gt_points=torch.from_numpy(gpts).cuda(), gt_offsets=torch.from_numpy(go).cuda(), return_iou=True)
    sm, tgt, i25, i50, iou = (t.cpu().numpy() for t in IP.grounding_targets(*args, seed=11, **kw))
    again = IP.grounding_targets(*args, seed=11, **kw)[0].cpu().numpy()
    other = IP.grounding_targets(*args, seed=12, **kw)[0].cpu().numpy()
    assert np.array_equal(sm, again)
    differs = False
    for b in range(len(io) - 1):
        c0, n = io[b], io[b + 1] - io[b]
        hits = [c for c in range(n) if iou[c0 + c] >= 0.25]
        chosen, need = G.crop_priority([iou[c0 + c] >= 0.25 for c in range(n)], lab[c0:c0 + n].tolist(), int(tl[b]), O)
        kept = [int(c) for c in sm[b] if c >= 0]
        assert len(kept) == min(n, O) and kept == sorted(set(kept))
        assert set(chosen) <= set(kept) and len(set(kept) - set(chosen)) == need
        t = int(tgt[b, 0])
        assert t == (kept.index(hits[-1]) if hits else len(kept))
        for s, c in enumerate(kept):
            assert i25[b, s] == (iou[c0 + c] >= 0.25) and i50[b, s] == (iou[c0 + c] >= 0.5)
        differs |= need > 0 and not np.array_equal(sm[b], other[b])
    assert differs, "a different seed should draw a different remainder"


def test_scanrefer_and_sqa3d_through_the_model():
    """ScanRefer and SQA3D configs: the counters of the graph-captured eval run equal a torch restatement of batch_metrics
    on an eager forward of the same model."""
    from sceneverse_b200 import model as M, synthetic, train, weights
    tf = weights.synthetic_tensor("text_features", (607, 768))
    for name in ("scanrefer", "sqa3d"):
        cfg = M.scanrefer_config(text_features=tf) if name == "scanrefer" else M.sqa3d_config(text_features=tf)
        ps = train.PretrainStep(cfg, "cuda:0", seed=0)
        B = 4
        if name == "scanrefer":
            d = synthetic.scene_batch(5, B=B, O=16, P=1024, L=50, min_obj=6)
            ev = evaluate.ScanReferEval()
            rng = np.random.default_rng(1)
            d["tgt_object_id_iou25"] = (rng.random((B, 16)) < 0.3).astype(np.int64)
            d["tgt_object_id_iou50"] = d["tgt_object_id_iou25"]
            d["is_multiple"] = rng.random(B) < 0.5
            d["tgt_object_label"] = rng.integers(0, 607, (B, 1))
        else:
            d = synthetic.qa_batch(5, "SQA3D", B=B, O=16, P=1024, L=50, num_answers=706, min_obj=6)
            d["sqa_type"] = np.arange(B, dtype=np.int64) % 6
            ev = evaluate.SQA3DEval()
        batch_ = {k: torch.from_numpy(np.asarray(v)).cuda() for k, v in d.items()}
        runner = evaluate.EvalRunner(ps, [ev], batch_size=B)
        runner.run([batch_])
        assert ps.module.model.training
        model = ps.module.model.eval()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(dict(batch_))
        model.train()
        cpu = {k: (v.float().cpu() if v.dtype == torch.bfloat16 else v.cpu()) for k, v in out.items() if torch.is_tensor(v)}
        want = torch.zeros(ev.size, dtype=torch.float64).tolist() if name == "scanrefer" else ev._initial().tolist()
        host_counters("scanrefer" if name == "scanrefer" else "sqa3d", cpu, want)
        assert ev.counters.cpu().tolist() == want, name
        ps.close()


def test_objcls_eval_runs():
    from sceneverse_b200 import synthetic, train, weights
    tf = weights.synthetic_tensor("text_features", (607, 768))
    st = train.ObjClsStep("cuda:0", tf)
    d = synthetic.scene_batch(2, B=2, O=8, P=1024, min_obj=4)
    b = {k: torch.from_numpy(d[k]).cuda() for k in ("obj_fts", "obj_masks", "obj_labels")}
    ev = evaluate.PretrainObjEval()
    (is_best, rec), = evaluate.EvalRunner(st, [ev], batch_size=2).run([b])
    assert st.model.training and 0.0 <= rec["accuracy"] <= 1.0 and ev.counters[1].item() == d["obj_masks"].sum()



def _train_state(ps):
    f = ps.flat_grads
    return {"param": f.flat_p, "exp_avg": f.exp_avg, "exp_avg_sq": f.exp_avg_sq, "grad": f.flat, "shadow": f.shadow,
            "adam_step": f.step_t, "lr_factor": f.lr_factor, "dropout_step": ps._step_counter, "loss": ps.static_loss}


def test_eval_between_steps_changes_no_training_state():
    """An eval run between graph-captured ScanRefer steps leaves every tensor the training step reads or writes bitwise
    unchanged (parameters, gradients, AdamW moments and step, bf16 shadows, lr factor, dropout step counter, loss, buffers,
    torch's CUDA generator), and the next step computes the same loss as a replay from the same state without the eval run.
    Two separate training runs are not compared: the weight-gradient reductions use atomics, so runs differ in the last
    bits whether or not evaluation happens in between."""
    from sceneverse_b200 import model as M, synthetic, train, weights
    tf = weights.synthetic_tensor("text_features", (607, 768))
    d = synthetic.scene_batch(9, B=4, O=16, P=1024, L=50, min_obj=6)
    batch_ = {k: torch.from_numpy(v).cuda() for k, v in d.items()}
    ev_batch = dict(batch_, tgt_object_id_iou25=torch.zeros(4, 16, dtype=torch.int64, device="cuda"),
                    is_multiple=torch.zeros(4, dtype=torch.bool, device="cuda"),
                    tgt_object_label=torch.zeros(4, 1, dtype=torch.int64, device="cuda"))
    ev_batch["tgt_object_id_iou50"] = ev_batch["tgt_object_id_iou25"]
    ps = train.PretrainStep(M.scanrefer_config(text_features=tf), "cuda:0", seed=0, cuda_graph=True)
    try:
        runner = evaluate.EvalRunner(ps, [evaluate.ScanReferEval()], batch_size=4)
        for _ in range(2):
            ps.step(dict(batch_))
        for _ in range(2):
            torch.cuda.synchronize()
            before = {k: v.clone() for k, v in _train_state(ps).items()}
            bufs = [b.clone() for b in ps.module.buffers()]
            rng = torch.cuda.get_rng_state()
            sched = ps._sched_step
            runner.run([ev_batch])
            torch.cuda.synchronize()
            for k, v in _train_state(ps).items():
                assert torch.equal(v, before[k]), k
            assert all(torch.equal(a, b) for a, b in zip(ps.module.buffers(), bufs))
            assert torch.equal(torch.cuda.get_rng_state(), rng) and ps.module.model.training
            loss_after_eval = ps.step(dict(batch_)).clone()
            for k, v in _train_state(ps).items():        # back to the state before the eval run; the same step again
                v.copy_(before[k])
            torch.cuda.set_rng_state(rng)
            ps._sched_step = sched
            assert torch.equal(ps.step(dict(batch_)), loss_after_eval)
    finally:
        ps.close()
