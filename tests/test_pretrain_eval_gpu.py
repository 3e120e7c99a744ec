"""PretrainEval on the GPU: the masked-LM, object-split and grounding counters (csrc/eval_metrics.cu) against the host
restatement of tests/test_pretrain_eval_host.py on the golden batches of the unmodified evaluator, `record()` against the
golden bitwise, the graph runner's padded last batch, and the masked-LM argmax over the full 30,522-wide vocabulary."""
import pytest
import torch

from oracle import make_golden_pretrain_eval as GP
from sceneverse_b200 import _lib, evaluate
from tests.test_pretrain_eval_host import batch, host_counters, meta

pytestmark = pytest.mark.gpu


def to_dev(d, dtype=None, pad=False):
    out = {}
    for k, v in d.items():
        v = v.cuda()
        if k.endswith("logits") and dtype is not None:
            v = v.to(dtype)
            if pad:        # padded rows read in place; the pad columns hold a value above every real logit
                W = (v.shape[-1] + 15) // 8 * 8
                w = torch.full(v.shape[:-1] + (W,), 7.0, dtype=dtype, device="cuda")
                w[..., :v.shape[-1]] = v
                v = w[..., :v.shape[-1]]
        out[k] = v
    return out


@pytest.mark.parametrize("dtype,pad", [(torch.float32, False), (torch.bfloat16, True)])
@pytest.mark.parametrize("case", list(GP.CASES))
def test_counters_match_restatement(case, dtype, pad):
    """Every counter word after every batch equals the host restatement exactly (the grid values are exact in bf16), the
    eager batch_metrics equals the reference's, and record() equals the reference's bitwise."""
    M, m = meta()
    ev = evaluate.PretrainEval()
    want = [0.0] * _lib.EVP_SIZE
    for i in range(m[case]["batches"]):
        d = batch(M, case, i)
        host_counters(d, want)
        ev.update(to_dev(d, dtype, pad))
        assert ev.counters.cpu().tolist() == want, (case, i)
        assert ev.batch_metrics(to_dev(d, dtype, pad)) == m[case]["batch_metrics"][i], (case, i)
    _, rec = ev.record()
    assert rec == m[case]["record"]


def test_eval_runner_partial_batch_counts_no_padding():
    """Batches of 8, 8 and 5 items through the graph runner (batch size 8): the padding of the last batch counts nothing,
    so record() is the reference's over the 21 items."""
    M, m = meta()
    batches = [to_dev(batch(M, "pretrain", i)) for i in range(m["pretrain"]["batches"])]
    ev = evaluate.PretrainEval()
    (_, rec), = evaluate.EvalRunner(lambda d: d, [ev], batch_size=8, dtype=torch.float32).run(batches)
    assert ev.counters[_lib.EVP_ITEMS].item() == 21
    assert rec == m["pretrain"]["record"]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_lm_hits_full_vocabulary(dtype):
    """3200 token rows over V = 30522: bf16 in the LM head's padded (3200, 30528) layout with zero pad columns (16-byte
    loads), f32 unpadded (per-element loads).  About 15 % of the rows are labelled; the grid makes ties for the maximum
    everywhere, one row has NaNs, one row is all negative (a zero pad column would win it).  Hits = torch.argmax over the
    first 30522 columns."""
    V, B, L = 30522, 64, 50
    R = B * L
    W = 30528 if dtype == torch.bfloat16 else V
    g = torch.Generator(device="cuda").manual_seed(0)
    vals = torch.randint(-16, 17, (R, V), device="cuda", generator=g).float() / 4
    labels = torch.where(torch.rand(R, device="cuda", generator=g) < 0.15,
                         torch.randint(0, V, (R,), device="cuda", generator=g), -1)
    labels[:3] = torch.tensor([5, 100, 20], device="cuda")
    vals[0] = -1.0
    vals[0, 5] = -0.5                                    # all negative: column 5 wins
    vals[1, [100, 200]] = float("nan")                   # the first NaN wins
    vals[2, [10, 20]] = 9.0                              # a tie: column 10 wins, a miss
    rows = torch.nonzero(labels[3:] != -1)[:, 0] + 3
    half = rows[::2]
    vals[half, labels[half]] = 4.0                       # ties with the row's other 4.0s: the lowest index wins
    buf = torch.zeros((R, W), dtype=dtype, device="cuda")
    buf[:, :V] = vals.to(dtype)
    ev = evaluate.PretrainEval()
    ev.update({"txt_lm_cls_logits": buf.view(B, L, W)[..., :V], "masked_lm_labels": labels.view(B, L)})
    pred = torch.argmax(buf[:, :V].float().cpu(), 1)
    lab = labels.cpu()
    m = lab != -1
    c = ev.counters.cpu()
    assert pred[1] == 100 and pred[0] == 5
    assert c[_lib.EVP_LM_HIT].item() == int((pred[m] == lab[m]).sum())
    assert c[_lib.EVP_LM_COUNT].item() == int(m.sum()) and c[_lib.EVP_ITEMS].item() == B
    assert 0 < c[_lib.EVP_LM_HIT].item() < c[_lib.EVP_LM_COUNT].item()
