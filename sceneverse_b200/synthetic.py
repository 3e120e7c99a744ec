"""Synthetic inputs with the layout of the reference's data_dict (SURVEY.md §8a row D):
object point clouds shaped like data/datasets/base.py:697-741 produces them — surface samples,
subsampled to P points WITH replacement when the raw object has fewer (duplicate points are the
norm, base.py:720-722), centred and scaled to the unit ball (base.py:724-729), rgb in [-1,1];
padded object slots are all-ones (dataset_wrapper.py:62-72).
numpy only, seeded; used by tests/ and bench.py.
"""
import numpy as np


def object_cloud(rng, P=1024, n_raw=None, kind=None):
    """One object: (P,6) float32 = xyz (unit-ball normalised) + rgb."""
    if n_raw is None:
        n_raw = int(rng.integers(64, 4097))
    if kind is None:
        kind = "box" if rng.random() < 0.5 else "ellipsoid"
    ext = rng.uniform(0.1, 2.0, size=3)
    if kind == "box":
        # uniform on the surface of an axis-aligned box
        pts = rng.uniform(-0.5, 0.5, size=(n_raw, 3))
        face = rng.integers(0, 3, size=n_raw)
        sign = rng.integers(0, 2, size=n_raw) * 1.0 - 0.5
        pts[np.arange(n_raw), face] = sign
        pts = pts * ext
    else:
        v = rng.standard_normal((n_raw, 3))
        v /= np.linalg.norm(v, axis=1, keepdims=True) + 1e-12
        pts = v * ext * 0.5
    pts = pts + rng.uniform(-4, 4, size=3)
    sel = rng.choice(n_raw, size=P, replace=n_raw < P)
    xyz = pts[sel]
    xyz = xyz - xyz.mean(0)
    max_dist = np.max(np.sqrt(np.sum(xyz ** 2, 1)))
    if max_dist < 1e-6:
        max_dist = 1.0
    xyz = xyz / max_dist
    rgb = rng.uniform(-1, 1, size=(P, 3))
    return np.concatenate([xyz, rgb], 1).astype(np.float32)


def object_batch(seed, n_clouds, P=1024, pad_fraction=0.0):
    """(n_clouds,P,6) float32; a `pad_fraction` of the clouds are all-ones padding slots."""
    rng = np.random.default_rng(seed)
    out = np.empty((n_clouds, P, 6), np.float32)
    for i in range(n_clouds):
        if rng.random() < pad_fraction:
            out[i] = 1.0
        else:
            out[i] = object_cloud(rng, P)
    return out


def unit_ball_clouds(seed, B, N):
    """(B,N,3) float32 uniform in the unit ball (the C5 sweep distribution, SURVEY.md §8d)."""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((B, N, 3))
    v /= np.linalg.norm(v, axis=2, keepdims=True)
    r = rng.random((B, N, 1)) ** (1.0 / 3.0)
    return (v * r).astype(np.float32)


def adversarial_clouds(seed, N):
    """A few (N,3) clouds that stress FPS tie-breaking and the |p|^2<=1e-3 skip rule."""
    rng = np.random.default_rng(seed)
    out = {}
    out["all_ones"] = np.ones((N, 3), np.float32)
    out["all_zero"] = np.zeros((N, 3), np.float32)
    base = unit_ball_clouds(seed + 1, 1, max(N // 8, 1))[0]
    out["dup8"] = base[rng.integers(0, base.shape[0], size=N)]
    near = unit_ball_clouds(seed + 2, 1, N)[0]
    near[::3] *= 0.02  # |p|^2 <= 4e-4 < 1e-3 -> skipped by the reference
    near[0] = 0.0
    out["near_origin"] = near
    grid = np.stack(np.meshgrid(*[np.arange(-2, 3)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32) * 0.25
    out["lattice"] = grid[rng.integers(0, grid.shape[0], size=N)]  # exact distance ties everywhere
    boundary = unit_ball_clouds(seed + 3, 1, N)[0]
    # |p|^2 straddling the 1e-3 threshold
    boundary[: N // 2] *= (np.sqrt(1e-3) / np.linalg.norm(boundary[: N // 2], axis=1, keepdims=True)) * \
        rng.uniform(0.9999, 1.0001, size=(N // 2, 1)).astype(np.float32)
    out["skip_boundary"] = boundary.astype(np.float32)
    return out


def scene_batch(seed, B=64, O=80, P=1024, L=50, Ls=300, min_obj=8, all_valid=False, max_obj=None):
    """Synthetic `data_dict` with the key set / dtypes of the reference's dataset wrappers
    (data/datasets/dataset_wrapper.py:38-111,147-195; SURVEY.md §8a row D), as numpy arrays:
    txt_ids/txt_masks (B,L) int64, obj_fts (B,O,P,6) f32 (padded objects all 1.0), obj_locs (B,O,6) f32 (pad 0),
    obj_masks/obj_sem_masks (B,O) bool, obj_labels (B,O) int64 (pad -100), tgt_object_id (B,1) int64,
    masked_lm_labels (B,L) int64 (-1 = ignore), scene_txt_ids/scene_txt_masks (B,Ls) int64.
    Each scene has between min_obj and max_obj (default O) valid objects."""
    rng = np.random.default_rng(seed)
    d = {}
    hi = O if max_obj is None else max_obj
    n_obj = np.full(B, O) if all_valid else rng.integers(min(min_obj, hi), hi + 1, size=B)
    obj_fts = np.ones((B, O, P, 6), np.float32)
    obj_locs = np.zeros((B, O, 6), np.float32)
    obj_masks = np.zeros((B, O), bool)
    obj_labels = np.full((B, O), -100, np.int64)
    for b in range(B):
        n = int(n_obj[b])
        for o in range(n):
            obj_fts[b, o] = object_cloud(rng, P)
        obj_locs[b, :n, 0:2] = rng.uniform(-4, 4, size=(n, 2))
        obj_locs[b, :n, 2] = rng.uniform(0, 2.5, size=n)
        obj_locs[b, :n, 3:] = rng.uniform(0.1, 2.0, size=(n, 3))
        obj_masks[b, :n] = True
        obj_labels[b, :n] = rng.integers(0, 607, size=n)
    d["obj_fts"], d["obj_locs"], d["obj_masks"], d["obj_labels"] = obj_fts, obj_locs, obj_masks, obj_labels
    d["obj_sem_masks"] = obj_masks & (rng.random((B, O)) > 0.25)
    d["tgt_object_id"] = np.array([[rng.integers(0, n)] for n in n_obj], np.int64)

    def text(length):
        ids = np.zeros((B, length), np.int64)
        masks = np.zeros((B, length), np.int64)
        for b in range(B):
            ell = int(rng.integers(min(8, length), length + 1))
            ids[b, :ell] = rng.integers(1000, 30000, size=ell)
            ids[b, 0], ids[b, ell - 1] = 101, 102
            masks[b, :ell] = 1
        return ids, masks

    d["txt_ids"], d["txt_masks"] = text(L)
    lm = np.full((B, L), -1, np.int64)
    pick = (rng.random((B, L)) < 0.15) & (d["txt_masks"] == 1)
    pick[:, 1] = True  # at least one supervised position per sample
    lm[pick] = d["txt_ids"][pick]
    d["masked_lm_labels"] = lm
    d["scene_txt_ids"], d["scene_txt_masks"] = text(Ls)
    return d


def qa_batch(seed, task="ScanQA", B=32, O=80, P=1024, L=50, Ls=300, num_answers=8864, min_obj=8, unanswerable=0.1,
             placeholder=0.15, edge_rows=False):
    """scene_batch + the question-answering targets of data/datasets/scannet_old.py:442-459, drawn from a separate RNG
    stream (scene_batch's arrays for the same seed are unchanged):
    answer_label (B, num_answers) int64 multi-hot with 1-3 answers, or all zero for an `unanswerable` fraction of the
    questions (the ones `use_unanswer: True` keeps);
    task 'ScanQA': tgt_object_id (B, O) int64 multi-hot over 1-3 valid objects, or, for a `placeholder` fraction, only the
    'no target' slot n_obj, which obj_masks masks (every scene keeps at least one padded slot for it).
    edge_rows=True: row 0 has no answer and row B-1 only the placeholder target."""
    d = scene_batch(seed, B=B, O=O, P=P, L=L, Ls=Ls, min_obj=min_obj, max_obj=O - 1 if task == "ScanQA" else None)
    rng = np.random.default_rng([seed, 0x51A])
    ans = np.zeros((B, num_answers), np.int64)
    for b in range(B):
        if rng.random() >= unanswerable and not (edge_rows and b == 0):
            ans[b, rng.choice(num_answers, size=int(rng.integers(1, 4)), replace=False)] = 1
    d["answer_label"] = ans
    if task == "ScanQA":
        n_obj = d["obj_masks"].sum(1)
        tgt = np.zeros((B, O), np.int64)
        for b in range(B):
            n = int(n_obj[b])
            if rng.random() < placeholder or (edge_rows and b == B - 1):
                tgt[b, n] = 1
            else:
                tgt[b, rng.choice(n, size=int(rng.integers(1, min(3, n) + 1)), replace=False)] = 1
        d["tgt_object_id"] = tgt
    return d


def per_scene_batch(seed, B=4, U=64, O=80, P=1024, T=50, min_obj=8):
    """A per-scene batch (model.OpenVocabPerScene; reference data/data_utils.py:12 `per_scene_pad`): the object keys of
    scene_batch for B scenes (obj_fts, obj_locs, obj_masks, obj_sem_masks, obj_labels), and U utterances per scene drawn
    from a separate RNG stream: txt_ids / txt_masks / masked_lm_labels (B, U, T) int64; tgt_object_id and
    tgt_object_label (B, U) int64, each target a valid object of its scene; is_multiple / is_hard / is_view_dependent (B, U)
    bool; tgt_object_id_iou25 / tgt_object_id_iou50 (B, U, O) int64 over the valid objects, the target among them, the
    IoU-50 set inside the IoU-25 set."""
    s = scene_batch(seed, B=B, O=O, P=P, L=8, Ls=8, min_obj=min_obj)
    d = {k: s[k] for k in ("obj_fts", "obj_locs", "obj_masks", "obj_sem_masks", "obj_labels")}
    rng = np.random.default_rng([seed, 0x5CE])
    n_obj = d["obj_masks"].sum(1)
    ids = np.zeros((B, U, T), np.int64)
    masks = np.zeros((B, U, T), np.int64)
    ell = rng.integers(min(8, T), T + 1, size=(B, U))
    for b in range(B):
        for u in range(U):
            e = int(ell[b, u])
            ids[b, u, :e] = rng.integers(1000, 30000, size=e)
            ids[b, u, 0], ids[b, u, e - 1] = 101, 102
            masks[b, u, :e] = 1
    d["txt_ids"], d["txt_masks"] = ids, masks
    lm = np.full((B, U, T), -1, np.int64)
    pick = (rng.random((B, U, T)) < 0.15) & (masks == 1)
    pick[:, :, 1] = True  # at least one supervised position per utterance
    lm[pick] = ids[pick]
    d["masked_lm_labels"] = lm
    tgt = np.stack([rng.integers(0, int(n), size=U) for n in n_obj]).astype(np.int64)
    d["tgt_object_id"] = tgt
    d["tgt_object_label"] = np.take_along_axis(d["obj_labels"], tgt, 1)
    valid = d["obj_masks"][:, None, :]
    iou25 = (rng.random((B, U, O)) < 0.2) & valid
    iou50 = iou25 & (rng.random((B, U, O)) < 0.6)
    np.put_along_axis(iou25, tgt[:, :, None], True, 2)
    np.put_along_axis(iou50, tgt[:, :, None], True, 2)
    d["tgt_object_id_iou25"], d["tgt_object_id_iou50"] = iou25.astype(np.int64), iou50.astype(np.int64)
    d["is_multiple"] = rng.random((B, U)) < 0.5
    d["is_hard"] = rng.random((B, U)) < 0.4
    d["is_view_dependent"] = rng.random((B, U)) < 0.3
    return d
