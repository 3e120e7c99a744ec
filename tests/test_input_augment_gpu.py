"""Augmented object processing on the device (csrc/scene_prep.cu `scene_prep_aug_kernel`, `scene_prep_kernel<true>`):
replay of the reference's own recorded draws (tests/golden/input_aug_*.npz, oracle/make_golden_aug.py), bitwise replay of the
seed mode's own draws, and the distributions of the seeded draws."""
import json
import os

import numpy as np
import pytest
import torch
from scipy import stats

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["shipped_train", "shipped_val", "all_align", "all_free", "post_rot"]
# Measured on an H100 over the five fixtures: obj_locs / obj_boxes differ from the reference by at most 1.6e-6, within the
# rtol = atol = 2e-5 of the input-pipeline tests.  obj_fts differ by at most 1.56e-5, so they get atol = 2.5e-5: the reference
# takes the centre as an f32 mean in torch's / numpy's summation order, the device sums in f64 and rounds once, and the two can
# land on neighbouring f32 values; that one-ulp centre difference (4.8e-7 at |x| ~ 4) is divided by the max norm, which is
# 0.03 for the smallest objects here.
TOL = dict(rtol=2e-5, atol=2e-5)
FTS_TOL = dict(rtol=2e-5, atol=2.5e-5)


def golden(name):
    from sceneverse_b200 import input_pipeline as ip
    z = np.load(os.path.join(GOLDEN, f"input_aug_{name}.npz"))
    cfg = json.loads(str(z["config"]))
    spec = ip.AugSpec.from_config(cfg, bool(z["rot_aug"]), str(z["split"]))
    assert spec.path == str(z["path"])
    return z, spec


def to_cuda(z, keys):
    return {k: torch.from_numpy(np.ascontiguousarray(z[k])).cuda() for k in keys if k in z.files}


@pytest.mark.parametrize("name", CASES)
def test_replay_matches_reference(name):
    from sceneverse_b200 import input_pipeline as ip
    z, spec = golden(name)
    B, O, P = int(z["B"]), int(z["O"]), int(z["P"])
    draws = to_cuda(z, ["item", "obj", "index", "noise", "quarter_turns"])
    fts, locs, masks, boxes = ip.prepare_objects_aug(torch.from_numpy(z["raw"]).cuda(), torch.from_numpy(z["offsets"]).cuda(),
                                                     B, O, P, spec, seed=0, want_boxes=True, draws=draws)
    assert torch.equal(masks.cpu(), torch.from_numpy(z["obj_masks"]))
    # A one-point object without jitter samples P copies of its point.  The device centres them exactly (f64 mean) and outputs
    # zeros; the reference's f32 mean is off by rounding, and it divides that ulp-sized residual by its max norm.  Those slots
    # are compared on their colours and checked to be exactly centred.
    single = (np.diff(z["offsets"]).reshape(B, O) == 1) & (spec.jitter is None)
    keep = ~single
    dev = {k: float(np.abs(v.cpu().numpy().astype(np.float64) - z[k])[keep].max())
           for k, v in (("obj_fts", fts), ("obj_locs", locs), ("obj_boxes", boxes))}
    print(name, "max |device - reference|", dev)
    got = fts.cpu().numpy()
    assert (got[single][..., :3] == 0).all()
    np.testing.assert_array_equal(got[single][..., 3:], z["obj_fts"][single][..., 3:])
    np.testing.assert_allclose(got[keep], z["obj_fts"][keep], **FTS_TOL)
    np.testing.assert_allclose(locs.cpu().numpy(), z["obj_locs"], **TOL)
    np.testing.assert_allclose(boxes.cpu().numpy(), z["obj_boxes"], **TOL)
    if name == "shipped_train":   # a quarter-turned item keeps the unrotated sizes (size taken before the scene rotation)
        th = np.round(np.arctan2(z["item"][:, 14], z["item"][:, 13]) / (np.pi / 2)).astype(int) % 4
        b = int(np.nonzero(th % 2 == 1)[0][0])
        s = b * O
        raw = z["raw"][z["offsets"][s]:z["offsets"][s + 1]]
        samp = raw[z["index"][b, 0], :3]
        np.testing.assert_array_equal(locs[b, 0, 3:].cpu().numpy(), samp.max(0) - samp.min(0))


def ragged(B, O, seed, lo=500, hi=6000, pad=True):
    rng = np.random.default_rng(seed)
    counts = rng.integers(lo, hi + 1, size=(B, O))
    if pad:
        counts[:, -1] = 0
        counts[0, 1], counts[0, 2] = 1, 64
    off = np.concatenate([[0], np.cumsum(counts.reshape(-1))]).astype(np.int64)
    raw = rng.standard_normal((off[-1], 6)).astype(np.float32)
    raw[:, :3] += rng.uniform(-4, 4, size=(1, 3)).astype(np.float32)
    return torch.from_numpy(raw).cuda(), torch.from_numpy(off).cuda(), counts


def specs():
    return {name: golden(name)[1] for name in ("shipped_train", "all_align", "all_free", "post_rot")}


@pytest.mark.parametrize("name", ["shipped_train", "all_align", "all_free", "post_rot"])
def test_seed_mode_equals_replay_of_its_draws(name):
    from sceneverse_b200 import input_pipeline as ip
    spec = specs()[name]
    B, O, P = 4, 6, 1024
    raw, off, _ = ragged(B, O, 5)
    a = ip.prepare_objects_aug(raw, off, B, O, P, spec, seed=123, want_boxes=True, return_draws=True)
    b = ip.prepare_objects_aug(raw, off, B, O, P, spec, seed=999, want_boxes=True, draws=a[4])
    for x, y in zip(a[:4], b[:4]):
        assert torch.equal(x, y)
    c = ip.prepare_objects_aug(raw, off, B, O, P, spec, seed=123, want_boxes=True)
    d = ip.prepare_objects_aug(raw, off, B, O, P, spec, seed=124, want_boxes=True)
    for x, y in zip(a[:4], c):
        assert torch.equal(x, y)
    assert not torch.equal(c[0], d[0])
    idx = a[4]["index"]
    counts = (off[1:] - off[:-1]).view(B, O)
    n = counts[..., None]
    assert (((idx >= 0) & (idx < n)) | ((n == 0) & (idx == -1))).all()


def test_distributions_of_the_seeded_draws():
    from sceneverse_b200 import input_pipeline as ip
    sp = specs()
    B, O, P, n = 2048, 2, 64, 100
    counts = np.full((B, O), n)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(counts.reshape(-1))]).astype(np.int64)).cuda()
    rng = np.random.default_rng(0)
    raw_np = rng.standard_normal((int(off[-1]), 6)).astype(np.float32)
    raw_np[:, :3] += np.repeat(rng.uniform(-4, 4, size=(B * O, 3)), n, axis=0).astype(np.float32)
    raw = torch.from_numpy(raw_np).cuda()
    bound = 5 * np.sqrt(B * 0.25 * 0.75)

    # shipped block: the scene angle is a uniform quarter turn, the same for every object of an item
    fts, locs, masks, d = ip.prepare_objects_aug(raw, off, B, O, P, sp["shipped_train"], seed=1, return_draws=True)
    item, idx = d["item"].cpu().numpy(), d["index"].cpu().numpy()
    th = np.arctan2(item[:, 14], item[:, 13])
    q = np.round(th / (np.pi / 2)).astype(int) % 4
    assert np.allclose(np.abs(th - np.round(th / (np.pi / 2)) * np.pi / 2), 0, atol=1e-12)
    assert (np.abs(np.bincount(q, minlength=4) - B / 4) < bound).all()
    locs = locs.cpu().numpy()
    for s in range(0, B * O, 37):   # each object's centre is its sample mean turned by its item's matrix
        b, o = divmod(s, O)
        m = raw_np[off[s].item() + idx[b, o], :3].astype(np.float64).mean(0)
        np.testing.assert_allclose(locs[b, o, :3], m @ item[b, 13:22].reshape(3, 3), rtol=1e-5, atol=1e-5)

    # every option on, free rotations: flips, translations, scaling, object angles, jitter normals, shuffled position 0
    spec = sp["all_free"]
    _, _, _, d = ip.prepare_objects_aug(raw, off, B, O, P, spec, seed=2, return_draws=True)
    item, obj = d["item"].cpu().numpy(), d["obj"].cpu().numpy().reshape(B * O, 12)
    flip = (item[:, 0] < 0).astype(int) + 2 * (item[:, 4] < 0).astype(int)   # 1: x, 2: y, 3: x and y, 0: none
    assert (np.abs(np.bincount(flip, minlength=4) - B / 4) < bound).all()
    for got, want, m in ((item[:, 10:13], spec.scene_translation, B), (obj[:, 0:3], spec.obj_translation, B * O)):
        z = got / np.asarray(want)
        assert np.abs(z.mean(0)).max() < 5 / np.sqrt(m) and np.abs(z.std(0) - 1).max() < 5 / np.sqrt(2 * m)
    lo, hi = spec.scaling
    assert item[:, 9].min() >= lo and item[:, 9].max() <= hi
    assert stats.kstest(item[:, 9], "uniform", args=(lo, hi - lo)).pvalue > 1e-3
    # object rotation with value [0.1, 0.1, 0.1], axis_align off: each angle uniform on [-0.1 pi, 0.1 pi]
    _, _, _, d = ip.prepare_objects_aug(raw, off, B, O, P, spec.__class__(path="aug", obj_rotation=type(spec.obj_rotation)(
        (0.0, 0.0, 0.1), False, True)), seed=3, return_draws=True)
    r = d["obj"].cpu().numpy().reshape(B * O, 12)[:, 3:]
    tz = np.arctan2(r[:, 1], r[:, 0])
    assert np.abs(tz).max() <= 0.1 * np.pi + 1e-12
    assert stats.kstest(tz, "uniform", args=(-0.1 * np.pi, 0.2 * np.pi)).pvalue > 1e-3
    _, _, _, d = ip.prepare_objects_aug(raw, off, B, O, P, spec, seed=4, return_draws=True)
    g = d["noise"].cpu().numpy().reshape(-1)
    assert abs(g.mean()) < 5 / np.sqrt(g.size) and abs(g.std() - 1) < 5 / np.sqrt(2 * g.size)
    assert stats.kstest(g[::7], "norm").pvalue > 1e-3
    first = d["index"].cpu().numpy()[:, :, 0].reshape(-1)
    assert stats.chisquare(np.bincount(first, minlength=n)).pvalue > 1e-3

    # post path: uniform quarter turns
    _, _, _, d = ip.prepare_objects_aug(raw, off, B, O, P, sp["post_rot"], seed=5, return_draws=True)
    qt = d["quarter_turns"].cpu().numpy()
    assert (np.abs(np.bincount(qt, minlength=4) - B / 4) < bound).all()


def test_no_rotation_post_path_equals_prepare_objects():
    from sceneverse_b200 import input_pipeline as ip
    B, O, P = 3, 5, 1024
    raw, off, _ = ragged(B, O, 9)
    a = ip.prepare_objects(raw, off, B, O, P, seed=17)
    b = ip.prepare_objects_aug(raw, off, B, O, P, ip.AugSpec(), seed=17, want_boxes=True)
    for x, y in zip(a, b[:3]):
        assert torch.equal(x, y)


def test_augmented_data_dict_with_boxes_feeds_the_model():
    from sceneverse_b200 import input_pipeline as ip
    B, O, P = 2, 16, 1024
    raw, off, counts = ragged(B, O, 8, lo=5, hi=4096)
    labels = torch.where(torch.from_numpy(counts) > 0, torch.randint(0, 607, (B, O)), torch.tensor(-100)).cuda()
    ids = torch.randint(1000, 30000, (B, 50)).cuda()
    am = torch.ones(B, 50, dtype=torch.int64).cuda()
    d = ip.build_data_dict(raw, off, labels, ids, am, torch.zeros(B, 1, dtype=torch.int64).cuda(), B, O, P, seed=4,
                           augment=specs()["all_align"], want_boxes=True)
    assert d["obj_boxes"].shape == (B, O, 6) and d["obj_boxes"].dtype == torch.float32
    assert (d["obj_boxes"][~d["obj_masks"]] == 0).all() and (d["obj_fts"][~d["obj_masks"]] == 1).all()
    torch.testing.assert_close(d["obj_boxes"][..., 3:], d["obj_locs"][..., 3:], rtol=0, atol=0)
    plain = ip.build_data_dict(raw, off, labels, ids, am, torch.zeros(B, 1, dtype=torch.int64).cuda(), B, O, P, seed=4)
    assert "obj_boxes" not in plain
    from sceneverse_b200 import weights
    from sceneverse_b200.modules import vision
    enc = vision.PointOpenVocabEncoder(None, freeze=True, text_features=weights.synthetic_tensor("text_features", (607, 768))).cuda().eval()
    with torch.no_grad():
        obj, pre, sem = enc(d["obj_fts"], d["obj_locs"], d["obj_masks"], d["obj_sem_masks"], d["obj_labels"], 1, 1)
    assert torch.isfinite(obj).all() and obj.shape == (B, O, 768)
