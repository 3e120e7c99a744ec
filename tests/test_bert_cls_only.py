"""BERTLanguageEncoder(..., cls_only=True), the scene-caption path: the last layer computes row 0 only, past its packed
q | k | v projection.  It must return row 0 of the full encoder's output bit for bit, with dropout on, draw the same
number of dropout seeds, and send back the same gradients into layer 2's output and into the embeddings; parameter
gradients, which go through split-K and scatter atomics, agree within the spread of two runs of the full path."""
import pytest
import torch

from sceneverse_b200 import model as M, ops, synthetic
from sceneverse_b200.modules.layers import route_linears


def _captions(device, B=64, Ls=300):
    d = synthetic.scene_batch(5, B=B, O=8, P=16, L=8, Ls=Ls)     # caption lengths 8..Ls
    return torch.from_numpy(d["scene_txt_ids"]).to(device), torch.from_numpy(d["scene_txt_masks"]).to(device)


def test_cls_only_matches_row_zero_fp32_cpu():
    """The fp32 torch formulation (CPU, the fp32 parity path) runs the same CLS-only layer."""
    torch.manual_seed(0)
    enc = route_linears(M.BERTLanguageEncoder(None)).eval()
    ids, masks = _captions("cpu", B=4, Ls=40)
    with torch.no_grad():
        full = enc(ids, masks)
        cls = enc(ids, masks, cls_only=True)
    assert cls.shape == (4, 768) and full.shape == (4, 40, 768)
    torch.testing.assert_close(cls, full[:, 0], rtol=1e-5, atol=1e-5)
    enc.train()
    out = enc(ids, masks, cls_only=True)
    out.sum().backward()
    assert enc.model.encoder.layer[-1].output.dense.weight.grad is not None


def _run(enc, ids, masks, cls_only, proj, rng):
    """One training-mode forward + backward in bf16 from the same dropout state."""
    ops._dropout_calls[0] = 0
    torch.cuda.set_rng_state(rng)                      # the embeddings' nn.Dropout
    enc.zero_grad(set_to_none=True)
    seen = {}

    def keep(name):
        def hook(_m, _i, out):
            out.retain_grad()
            seen[name] = out
        return hook

    hooks = [enc.model.encoder.layer[2].register_forward_hook(keep("layer2")),
             enc.model.embeddings.register_forward_hook(keep("embeddings"))]
    try:
        with torch.autocast("cuda", dtype=torch.bfloat16):
            emb = enc(ids, masks, cls_only=True) if cls_only else enc(ids, masks)[:, 0]
        seeds = ops._dropout_calls[0]
        (emb.float() * proj).sum().backward()
    finally:
        for h in hooks:
            h.remove()
    grads = {n: p.grad.clone() for n, p in enc.named_parameters() if p.grad is not None}
    return emb.detach(), seeds, seen["layer2"].grad, seen["embeddings"].grad, grads


@pytest.mark.gpu
def test_cls_only_matches_full_encoder_bf16_gpu():
    torch.manual_seed(0)
    enc = route_linears(M.BERTLanguageEncoder(None)).cuda().train()
    ids, masks = _captions("cuda")
    proj = torch.randn(64, 768, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    rng = torch.cuda.get_rng_state()
    full = _run(enc, ids, masks, False, proj, rng)
    again = _run(enc, ids, masks, False, proj, rng)
    cls = _run(enc, ids, masks, True, proj, rng)
    assert torch.equal(cls[0], full[0]), "scene_text_embed differs"
    assert cls[1] == full[1] > 0, ("dropout seeds drawn", cls[1], full[1])
    assert torch.equal(cls[2], full[2]), "gradient into layer 2's output differs"
    assert torch.equal(cls[3], full[3]), "gradient into the embeddings differs"
    assert cls[4].keys() == full[4].keys()
    spread = max(((again[4][n] - g).abs().max() / g.abs().max().clamp_min(1e-30)).item() for n, g in full[4].items())
    assert spread > 0, "two full runs gave the same parameter gradients: no spread to compare against"
    tol = max(2 * spread, 1e-5)
    worst = {n: ((cls[4][n] - g).abs().max() / g.abs().max().clamp_min(1e-30)).item() for n, g in full[4].items()}
    print(f"BERT_CLS_ONLY relative spread of two full runs {spread:.3g}, worst CLS-only difference "
          f"{max(worst.values()):.3g} ({max(worst, key=worst.get)})")
    bad = {n: v for n, v in worst.items() if v > tol}
    assert not bad, (tol, bad)
