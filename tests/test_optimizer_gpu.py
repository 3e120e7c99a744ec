"""The parameter update of the CUDA-graph training path and the gradient accumulation that feeds it.

* sv_adamw_flat (csrc/train_ops.cu: squared-norm partials, clip_grad_norm_, AdamW and the bf16 shadow refresh in one pass over
  flat buffers) against torch.optim.AdamW + clip_grad_norm_ in float64 over many steps, with an elementwise bound derived
  from fp32 rounding.  Extra float64 runs with one term knocked out show that the bound would catch each term.
* The kernel's contract at its edges: gaps between segments, the n % 4 tail, the bf16 shadow, determinism, non-finite
  gradients, CUDA-graph replay, argument validation.
* train.FlatState on the real GPS parameter groups: its layout (CPU), and five steps against float64 AdamW (GPU).
* ops.DIRECT_GRAD: every backward that adds straight into an existing fp32 .grad instead of returning a gradient.
"""
import functools
import math
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sceneverse_b200 import _lib, model as M, ops, train, weights

U = 2.0 ** -24                          # unit roundoff of fp32 (round to nearest)
SEG_DT = np.dtype([("begin", "<i8"), ("end", "<i8"), ("lr_scale", "<f4"), ("weight_decay", "<f4")])   # as train.FlatState
NORM_BLOCKS, NORM_THREADS = 528, 512    # launch of sqnorm_partial_kernel


def f32(x):
    return float(np.float32(x))


def norm_rel_bound(n):
    """Relative error bound of the kernel's fp32 gradient norm.  Every square reaches the total through at most k rounded
    additions: the fma chain of one thread (4 per float4 it reads, 1 for the n % 4 tail), 5 warp and 4 block shuffle levels,
    and the serial sum of the 528 block partials.  For non-negative terms that bounds the relative error of the sum by
    k u / (1 - k u); the square root halves it and adds one rounding."""
    k = 4 * -(-(n // 4) // (NORM_BLOCKS * NORM_THREADS)) + 1 + 5 + 4 + NORM_BLOCKS
    return k * U / (1 - k * U) / 2 + U


def reference(groups, grads_at, factors, betas, eps, max_norm, n_flat, step0=0, state0=None, knock=None):
    """torch.optim.AdamW(foreach=False) on float64 copies: one param group per entry of `groups` = [(tensors, lr, wd)], lr of
    step i = lr * factors[i], and torch.nn.utils.clip_grad_norm_(max_norm) in float64 before each step (max_norm <= 0: no
    clipping).  grads_at(i) gives the step's gradients in the order of the tensors.  state0 = [(exp_avg, exp_avg_sq)] per
    tensor continues a run at step `step0`.  Yields after every step (norm, params, exp_avgs, exp_avg_sqs, bounds), with
    bounds = (p, m, v) elementwise bounds of |fp32 kernel - this run| (n_flat: elements of the kernel's norm).

    knock removes one term, through the group hyper-parameters torch reads at every step:
      "wd"    no weight decay;
      "bc1"   lr * bc1 and wd / bc1: step size lr instead of lr / bc1, decay 1 - lr wd unchanged;
      "bc2"   lr / s, wd * s, eps / s with s = sqrt(bc2): (lr / s) / bc1 * m / (sqrt(v) / s + eps / s) =
              lr / bc1 * m / (sqrt(v) + eps), decay unchanged;
      "clip"  no clipping;
      "seg0"  every group with group 0's lr and weight decay."""
    b1, b2 = betas
    params = [[t.detach().double().clone().requires_grad_(True) for t in ts] for ts, _, _ in groups]
    flat = [p for ps in params for p in ps]
    opt = torch.optim.AdamW([{"params": ps} for ps in params], betas=betas, eps=eps, foreach=False)
    if state0 is not None:
        for p, (m0, v0) in zip(flat, state0):
            opt.state[p] = {"step": torch.tensor(float(step0)), "exp_avg": m0.double().clone(),
                            "exp_avg_sq": v0.double().clone()}
    hyper = [(lr, wd) for _, lr, wd in groups]
    if knock == "seg0":
        hyper = [hyper[0]] * len(hyper)
    # Elementwise error bound of the fp32 kernel, carried along this run.  The hyper-parameters given here are the fp32
    # values the kernel receives, so only the kernel's fp32 arithmetic differs.  First order in u; the factor 1.01 where the
    # bounds are used covers the second-order terms and the rounding of this float64 run (~1e-16 relative).
    #   clipped g   the norm is within dn = norm_rel_bound(n); c = max_norm / (norm + 1e-6f) rounds twice, g * c once:
    #               dg = dn + 3u relative (0 without clipping, where c is exactly 1)
    #   m = fma(b1, m, (1 - b1) g)        1 - b1 is exact (Sterbenz), 2 roundings:
    #               Em' = b1 Em + (1 - b1) |g| (dg + u) + u |m'|
    #   v = fma(b2, v, (1 - b2) g g)      3 roundings, g^2 carries 2 dg:
    #               Ev' = b2 Ev + (1 - b2) g^2 (2 dg + 2u) + u v'
    #   den = sqrt(v) / sqrt(bc2) + eps   sqrt, the fp32 sqrt(bc2), division, addition: dD = Ev / 2v + 4u relative
    #   step = lr / bc1                   lr = base * scale * factor (2 roundings), fp32 bc1 (1), division (1): 4u relative
    #   upd = step m / den                2 more roundings: Eu = |upd| (6u + dD) + step Em / den
    #   p' = p (1 - lr wd) - upd          fp32 1 - lr wd is off by half an ulp of 1.0 (u) plus 4u lr wd; the product and the
    #                                     difference round once each:
    #               Ep' = Ep + |p| (2u + 4u lr wd) + Eu + u |p'|
    dg = norm_rel_bound(n_flat) + 3 * U if max_norm > 0 else 0.0
    em, ev, ep = ([torch.zeros_like(p) for p in flat] for _ in range(3))
    for i, f in enumerate(factors):
        t = step0 + i + 1
        for p, g in zip(flat, grads_at(i)):
            p.grad = g.detach().double()
        if max_norm > 0 and knock != "clip":
            norm = torch.nn.utils.clip_grad_norm_(flat, max_norm, foreach=False)
        else:
            norm = torch.nn.utils.get_total_norm([p.grad for p in flat], foreach=False)
        bc1, bc2s = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
        for grp, (lr, wd) in zip(opt.param_groups, hyper):
            lr, wd, e = lr * f, (0.0 if knock == "wd" else wd), eps
            if knock == "bc1":
                lr, wd = lr * bc1, wd / bc1
            elif knock == "bc2":
                lr, wd, e = lr / bc2s, wd * bc2s, eps / bc2s
            grp.update(lr=lr, weight_decay=wd, eps=e)
        prev = [p.detach().abs() for p in flat] if knock is None else None
        opt.step()
        ms = [opt.state[p]["exp_avg"] for p in flat]
        vs = [opt.state[p]["exp_avg_sq"] for p in flat]
        if knock is None:
            k = 0
            for grp, ps in zip(opt.param_groups, params):
                lr, wd = grp["lr"], grp["weight_decay"]
                step = lr / bc1
                for p in ps:
                    g, m, v = p.grad.abs(), ms[k], vs[k]
                    em[k].mul_(b1).add_((1 - b1) * (dg + U) * g).add_(U * m.abs())
                    ev[k].mul_(b2).add_((1 - b2) * (2 * dg + 2 * U) * g * g).add_(U * v)
                    den = v.sqrt() / bc2s + eps
                    d_den = ev[k] / (2 * v).clamp_min(1e-300) + 4 * U
                    eu = (step * m / den).abs() * (6 * U + d_den) + step * em[k] / den
                    ep[k].add_(prev[k] * (2 * U + 4 * U * lr * wd)).add_(eu).add_(U * p.detach().abs())
                    k += 1
        yield float(norm), [p.detach() for p in flat], ms, vs, (ep, em, ev)


def within(got, want, bound, what):
    """|got - want| <= 1.01 bound wherever the reference is finite, non-finite exactly where it is not.  Returns the worst
    |got - want| / bound."""
    got = got.detach().double().to(want.device)
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(got), fin), f"{what}: non-finite elements differ"
    err, b = (got - want).abs()[fin], 1.01 * bound[fin]
    bad = err > b
    assert not bad.any(), f"{what}: {int(bad.sum())} elements outside the bound, worst |err| / bound " \
                          f"{float((err / b.clamp_min(1e-300)).max()):.3g}"
    return float((err / b.clamp_min(1e-300)).max()) if err.numel() else 0.0


class FlatBuffers:
    """Device buffers of a sequence of sv_adamw_flat calls on one flat layout."""

    def __init__(self, p0, segs, m0=None, v0=None, step0=0, shadow=True):
        self.p = p0.float().cuda().contiguous()
        self.m = m0.float().cuda().contiguous() if m0 is not None else torch.zeros_like(self.p)
        self.v = v0.float().cuda().contiguous() if v0 is not None else torch.zeros_like(self.p)
        self.g = torch.zeros_like(self.p)
        self.shadow = self.p.bfloat16() if shadow else None
        self.segs = torch.from_numpy(segs.view(np.uint8).copy()).cuda()
        self.nseg = len(segs)
        self.lr_factor = torch.ones(1, device="cuda")
        self.step_t = torch.full((1,), step0, dtype=torch.int64, device="cuda")
        self.scratch = torch.zeros(_lib.gps().sv_adamw_scratch_floats(), device="cuda")
        self.norm = torch.zeros(1, device="cuda")

    def step(self, g, factor, max_norm, betas, eps, base_lr):
        lib = _lib.gps()
        self.g.copy_(g)
        self.lr_factor.fill_(factor)
        self.step_t.add_(1)
        st = lib.sv_adamw_flat(self.p.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.g.data_ptr(),
                               self.shadow.data_ptr() if self.shadow is not None else None, self.p.numel(),
                               self.segs.data_ptr(), self.nseg, max_norm, self.lr_factor.data_ptr(), self.step_t.data_ptr(),
                               base_lr, betas[0], betas[1], eps, self.scratch.data_ptr(), self.norm.data_ptr(),
                               torch.cuda.current_stream().cuda_stream)
        _lib.check(lib, st, "sv_adamw_flat")


# ---- 1a: many steps against float64 torch.optim.AdamW ---------------------------------------------------------------------
# 11 segments: more than the 8 grid rows of the update, so the segment loop wraps.  The 8-element one is a single float4 of
# work; the 1,126,400-element one takes several passes of the 264-CTA x 256-thread x float4 update loop; n = 2,270,624 makes
# the 528-block x 512-thread x float4 squared-norm loop run three passes.
SIZES = [8, 1_126_400, 4096, 36, 300_000, 64, 520_000, 12, 200_000, 120_004, 4]
LR_SCALES = [1.0, 0.5, 2.0, 1.5, 0.25, 3.0, 1.0, 0.75, 2.5, 0.1, 1.25]
WDS = [0.1, 0.05, 0.0, 0.2, 0.1, 0.0, 0.3, 0.02, 0.0, 0.1, 0.05]
BASE_LR = 4e-3          # lr * wd >= 4e-6 = 67 u where wd > 0: weight decay stands well above the rounding of 1 - lr wd
STEPS = 24
CASES = {"betas0.98_eps1e-8": dict(betas=(0.9, 0.98), eps=1e-8, clip=True, step0=0),
         "betas0.999_eps1e-6": dict(betas=(0.9, 0.999), eps=1e-6, clip=True, step0=0),
         "no_clip": dict(betas=(0.9, 0.98), eps=1e-8, clip=False, step0=0),
         "from_step10000": dict(betas=(0.9, 0.999), eps=1e-8, clip=True, step0=10000)}   # bc2 = 1 - 4.5e-5


@functools.lru_cache(maxsize=1)
def make_case(name):
    c = CASES[name]
    rng = np.random.default_rng(1234)
    edges = np.cumsum([0] + SIZES)
    n = int(edges[-1])
    segs = np.array([(edges[s], edges[s + 1], f32(LR_SCALES[s]), f32(WDS[s])) for s in range(len(SIZES))], dtype=SEG_DT)
    gen = torch.Generator().manual_seed(7)
    p0 = torch.randn(n, generator=gen) * 0.5
    # gradient magnitude per (step, segment) from 1e-4 to 1e2
    mag = 10.0 ** rng.uniform(-4, 2, size=(STEPS, len(SIZES)))
    grads = []
    for i in range(STEPS):
        g = torch.randn(n, generator=gen)
        for s in range(len(SIZES)):
            g[edges[s]:edges[s + 1]] *= f32(mag[i, s])
        grads.append(g)
    norms = np.array([float(torch.linalg.vector_norm(g.double())) for g in grads])
    max_norm = f32(np.median(norms)) if c["clip"] else 0.0
    if c["clip"]:
        assert 0 < int((norms > max_norm).sum()) < STEPS      # clipping active on some steps, inactive on others
    state0 = None
    if c["step0"]:
        s = torch.from_numpy(10.0 ** rng.uniform(-3, 1, size=n)).float()
        m0 = torch.randn(n, generator=gen) * s
        state0 = (m0, m0 * m0 + (torch.randn(n, generator=gen) * s) ** 2)
    factors = [f32(M.warmup_cosine(i + 1, 4, 30, minimum_ratio=0.1)) for i in range(STEPS)]   # changes at every step
    groups = [([p], f32(BASE_LR) * float(seg["lr_scale"]), float(seg["weight_decay"]))
              for p, seg in zip(p0.split(SIZES), segs)]
    return types.SimpleNamespace(n=n, segs=segs, p0=p0, grads=grads, norms=norms, max_norm=max_norm, state0=state0,
                                 factors=factors, groups=groups, betas=tuple(f32(b) for b in c["betas"]), eps=f32(c["eps"]),
                                 step0=c["step0"])


def case_reference(c, knock=None):
    state0 = list(zip(c.state0[0].split(SIZES), c.state0[1].split(SIZES))) if c.state0 is not None else None
    return reference(c.groups, lambda i: c.grads[i].split(SIZES), c.factors, c.betas, c.eps, c.max_norm, c.n,
                     step0=c.step0, state0=state0, knock=knock)


def run_against_reference(buf, ref, grads, factors, max_norm, betas, eps, base_lr, what):
    """Step the kernel and the float64 reference in lockstep and compare p, m, v and the norm after every step."""
    worst = dict.fromkeys(("p", "m", "v", "norm"), 0.0)
    for i, (norm, ps, ms, vs, bounds) in enumerate(ref):
        buf.step(grads[i].cuda(), factors[i], max_norm, betas, eps, base_lr)
        got = buf.norm.item()
        if math.isfinite(norm):
            err = abs(got - norm) / norm
            assert err <= norm_rel_bound(buf.p.numel()), f"{what} step {i}: norm {got} vs {norm}"
            worst["norm"] = max(worst["norm"], err / norm_rel_bound(buf.p.numel()))
        else:
            assert math.isnan(got) if math.isnan(norm) else got == norm, f"{what} step {i}: norm {got} vs {norm}"
        for key, t, want, bound in (("p", buf.p, ps, bounds[0]), ("m", buf.m, ms, bounds[1]), ("v", buf.v, vs, bounds[2])):
            worst[key] = max(worst[key], within(t, torch.cat(want), torch.cat(bound), f"{what} step {i} {key}"))
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_adamw_flat_matches_float64_torch_adamw_over_many_steps(name):
    c = make_case(name)
    buf = FlatBuffers(c.p0, c.segs, *(c.state0 or ()), step0=c.step0)
    worst = run_against_reference(buf, case_reference(c), c.grads, c.factors, c.max_norm, c.betas, c.eps, f32(BASE_LR), name)
    assert int(buf.step_t) == c.step0 + STEPS
    print(f"ADAMW_FLAT {name}: worst |err| / bound", {k: f"{v:.3g}" for k, v in worst.items()},
          f"clipped steps {int((c.norms > c.max_norm).sum()) if c.max_norm else 0}/{STEPS}")


@pytest.mark.parametrize("name", ["betas0.98_eps1e-8", "betas0.999_eps1e-6"])
def test_reference_bound_detects_each_knocked_out_term(name):
    """The bound used above is tight enough to matter: removing any one term of the update moves the float64 result by at
    least 20 x the bound somewhere in p, m or v."""
    c = make_case(name)
    knocks = ("wd", "bc1", "bc2", "clip", "seg0")
    runs = {k: case_reference(c, knock=k) for k in knocks}
    margin = dict.fromkeys(knocks, 0.0)
    for _, ps, ms, vs, bounds in case_reference(c):
        want = [torch.cat(x) for x in (ps, ms, vs)]
        tol = [1.01 * torch.cat(b) for b in bounds]
        for k, run in runs.items():
            _, kp, km, kv, _ = next(run)
            for w, t, x in zip(want, tol, (kp, km, kv)):
                margin[k] = max(margin[k], float(((torch.cat(x) - w).abs() / t).max()))
    print(f"KNOCKOUT {name}: max |knocked - full| / bound", {k: f"{v:.3g}" for k, v in margin.items()})
    assert all(m >= 20 for m in margin.values()), margin


# ---- 1b: contract edges ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_adamw_flat_leaves_gaps_untouched_and_counts_the_tail():
    """Elements outside every segment keep p, m, v and the shadow bitwise; the n % 4 tail still counts in the norm; inside
    the segments the shadow is p rounded to bf16 after every step."""
    n = 4099
    segs = np.array([(8, 1000, 1.0, 0.1), (1024, 2048, 2.0, 0.0), (3000, 4000, 0.5, 0.05)], dtype=SEG_DT)
    gen = torch.Generator().manual_seed(3)
    buf = FlatBuffers(torch.randn(n, generator=gen), segs, torch.randn(n, generator=gen) * 0.1,
                      torch.rand(n, generator=gen) * 0.01)
    buf.shadow = torch.randn(n, generator=gen).bfloat16().cuda()       # not p's rounding: a stray write would show
    inside = torch.zeros(n, dtype=torch.bool, device="cuda")
    for b, e, _, _ in segs:
        inside[b:e] = True
    before = [t.clone() for t in (buf.p, buf.m, buf.v, buf.shadow)]
    for i in range(3):
        g = torch.randn(n, generator=gen)
        g[-3:] = 1e3 * (i + 1)          # the scalar tail of sqnorm_partial_kernel dominates the norm
        buf.step(g.cuda(), 1.0, 1.0, (0.9, 0.98), 1e-8, 1e-3)
        for t, t0, what in zip((buf.p, buf.m, buf.v, buf.shadow), before, ("p", "m", "v", "shadow")):
            assert torch.equal(t[~inside], t0[~inside]), (i, what)
        assert torch.equal(buf.shadow[inside], buf.p[inside].bfloat16()), i
        want = float(torch.linalg.vector_norm(g.double()))
        assert abs(buf.norm.item() - want) <= norm_rel_bound(n) * want, (i, buf.norm.item(), want)
    assert not torch.equal(buf.p[inside], before[0][inside])


def three_steps(shadow):
    c = make_case("betas0.98_eps1e-8")
    buf = FlatBuffers(c.p0, c.segs, shadow=shadow)
    norms = []
    for i in range(3):
        buf.step(c.grads[i].cuda(), c.factors[i], c.max_norm, c.betas, c.eps, f32(BASE_LR))
        norms.append(buf.norm.clone())
    return buf, torch.cat(norms)


@pytest.mark.gpu
def test_adamw_flat_is_deterministic():
    (a, na), (b, nb) = three_steps(True), three_steps(True)
    for x, y, what in ((a.p, b.p, "p"), (a.m, b.m, "m"), (a.v, b.v, "v"), (na, nb, "norm"), (a.shadow, b.shadow, "shadow")):
        assert torch.equal(x, y), what


@pytest.mark.gpu
def test_adamw_flat_without_shadow_updates_the_same():
    (a, na), (b, nb) = three_steps(True), three_steps(False)
    for x, y, what in ((a.p, b.p, "p"), (a.m, b.m, "m"), (a.v, b.v, "v"), (na, nb, "norm")):
        assert torch.equal(x, y), what


def small_case(n=8192, seed=4):
    segs = np.array([(0, 4096, 1.0, 0.1), (4096, n, 0.5, 0.0)], dtype=SEG_DT)
    gen = torch.Generator().manual_seed(seed)
    p0 = torch.randn(n, generator=gen)
    groups = [([p], f32(1e-3) * float(s["lr_scale"]), float(s["weight_decay"])) for p, s in zip(p0.split(4096), segs)]
    return segs, p0, groups, gen


@pytest.mark.gpu
def test_adamw_flat_nan_gradient_poisons_every_parameter_like_torch():
    """One NaN gradient: clip_grad_norm_ multiplies every gradient by a NaN coefficient, so torch's AdamW makes every
    parameter NaN.  The kernel must not read the NaN norm as 'no clipping needed'."""
    segs, p0, groups, gen = small_case()
    g = torch.randn(p0.numel(), generator=gen)
    g[1234] = float("nan")
    betas, eps = (f32(0.9), f32(0.98)), f32(1e-8)
    norm, ps, ms, vs, _ = next(reference(groups, lambda i: g.split(4096), [1.0], betas, eps, 1.0, p0.numel()))
    assert math.isnan(norm) and all(torch.isnan(torch.cat(x)).all() for x in (ps, ms, vs))    # torch's behaviour
    buf = FlatBuffers(p0, segs)
    buf.step(g.cuda(), 1.0, 1.0, betas, eps, f32(1e-3))
    assert math.isnan(buf.norm.item())
    for t, what in ((buf.p, "p"), (buf.m, "m"), (buf.v, "v")):
        assert torch.isnan(t).all(), f"{what}: {int((~torch.isnan(t)).sum())} of {t.numel()} elements are not NaN"


@pytest.mark.gpu
def test_adamw_flat_inf_gradient_zeroes_the_clip_factor_like_torch():
    """One inf gradient on step 3: the norm is inf, the clip factor 0, the inf coordinate becomes NaN and every other one
    takes the step of a zero gradient (weight decay plus the momentum of steps 1 and 2)."""
    segs, p0, groups, gen = small_case(seed=5)
    grads = [torch.randn(p0.numel(), generator=gen) for _ in range(3)]
    grads[2][777] = float("inf")
    betas, eps, factors = (f32(0.9), f32(0.98)), f32(1e-8), [1.0, 0.5, 0.75]
    ref = reference(groups, lambda i: grads[i].split(4096), factors, betas, eps, 1.0, p0.numel())
    buf = FlatBuffers(p0, segs)
    run_against_reference(buf, ref, grads, factors, 1.0, betas, eps, f32(1e-3), "inf gradient")
    assert buf.norm.item() == math.inf
    assert torch.isnan(buf.p[777]) and int(torch.isnan(buf.p).sum()) == 1


@pytest.mark.gpu
def test_flat_state_step_replays_in_a_cuda_graph():
    """FlatState.optimizer_step() captured once and replayed k times, with new gradients and a new lr factor before each
    replay, equals k eager steps bitwise: the step count and the lr factor are read from the device at replay time."""
    K = 6

    def make():
        torch.manual_seed(5)
        ps = [torch.nn.Parameter(torch.randn(s, device="cuda")) for s in ((64, 40), (40,), (7, 3), (1000,), (33,))]
        groups = [{"params": ps[:2], "weight_decay": 0.1}, {"params": ps[2:4], "weight_decay": 0.0},
                  {"params": ps[4:], "weight_decay": 0.01}]
        return train.FlatState(groups, [1e-3, 5e-4, 2e-3], betas=(0.9, 0.98), eps=1e-8, max_norm=1.0), ps

    (eager, _), (graphed, _) = make(), make()
    gen = torch.Generator(device="cuda").manual_seed(11)
    grads = [torch.randn(eager.n, device="cuda", generator=gen) * 10.0 ** (i % 3 - 2) for i in range(K)]
    factors = [M.warmup_cosine(i + 1, 2, K) for i in range(K)]
    for g, f in zip(grads, factors):
        eager.flat.copy_(g)
        eager.lr_factor.fill_(f)
        eager.optimizer_step()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graphed.optimizer_step()
    for g, f in zip(grads, factors):
        graphed.flat.copy_(g)
        graphed.lr_factor.fill_(f)
        graph.replay()
    torch.cuda.synchronize()
    assert int(graphed.step_t) == K
    for name in ("flat_p", "exp_avg", "exp_avg_sq", "shadow", "grad_norm_t", "step_t"):
        assert torch.equal(getattr(eager, name), getattr(graphed, name)), name


# ---- 1c: without a GPU ----------------------------------------------------------------------------------------------------
_VALIDATION = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from sceneverse_b200 import _lib
lib = _lib.gps()
a = 0x1000      # 16-byte aligned fake address


def call(p=a, m=a, v=a, g=a, shadow=a, n=1024, segs=a, nseg=2, lr=a, step=a, scratch=a):
    return lib.sv_adamw_flat(p, m, v, g, shadow, n, segs, nseg, 1.0, lr, step, 1.0, 0.9, 0.999, 1e-8, scratch, None, None)


out = {"misaligned " + w: call(**{w: a + 8}) for w in ("p", "m", "v", "g")}       # float4 access needs 16 bytes
out["misaligned shadow"] = call(shadow=a + 4)                                        # written as uint2
out["misaligned segs"] = call(segs=a + 4)                                            # read as 8-byte fields
out["n < 0"], out["nseg < 0"] = call(n=-1), call(nseg=-1)
out.update({"NULL " + w: call(**{w: None}) for w in ("p", "m", "v", "g", "segs", "lr", "step", "scratch")})
out["n == 0"], out["nseg == 0"] = call(n=0), call(nseg=0)
print(json.dumps(out))
"""


def test_adamw_flat_argument_validation_without_gpu():
    """sv_adamw_flat rejects malformed calls before touching the device (1 = SV_ERR_INVALID_ARG, 0 for empty work).  The
    calls run in a process that sees no CUDA device: if a check were missing, the launch on the fake pointers fails there
    with status 2 instead of running."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", _VALIDATION, root], capture_output=True, text=True, timeout=120,
                         env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    want = {k: 0 if k in ("n == 0", "nseg == 0") else 1 for k in got}
    assert len(got) == 18 and got == want, {k: v for k, v in got.items() if v != want[k]}


def gps_groups(device):
    """The GPS pre-training parameter groups as PretrainStep builds them: model.get_opt_params() plus the loss group, passed
    through torch.optim.AdamW (which fills in its defaults); the LambdaLR schedule keeps each group's base lr as
    'initial_lr'."""
    tf = weights.synthetic_tensor("text_features", (607, 768))
    ps = train.PretrainStep(M.pretrain_config(1, text_features=tf), device, dtype=torch.bfloat16, seed=0)
    groups = ps.optimizer.param_groups
    return ps, groups, [g["initial_lr"] for g in groups]


def round8(n):
    return (n + 7) // 8 * 8


def test_flat_state_layout_of_the_gps_parameter_groups():
    ps, groups, base = gps_groups("cpu")
    before = {id(p): p.detach().clone() for g in groups for p in g["params"]}
    flat = train.FlatState(groups, base, betas=(0.9, 0.98), eps=1e-8, max_norm=5.0)
    seg = np.frombuffer(flat.segments.numpy().tobytes(), dtype=SEG_DT)
    live = [(g, lr) for g, lr in zip(groups, base) if any(p.requires_grad for p in g["params"])]
    print("GPS_SEGMENTS", flat.nseg, "segments,", flat.n, "elements")
    assert flat.nseg == len(seg) == len(live) > 8     # more segments than grid rows: the kernel's segment loop wraps
    used = torch.zeros(flat.n, dtype=torch.bool)
    off = 0
    for s, (g, lr) in zip(seg, live):
        assert s["begin"] == off
        for p in (p for p in g["params"] if p.requires_grad):
            o, n = flat.offsets[id(p)], p.numel()
            assert o == off and o % 8 == 0
            assert p.data.untyped_storage().data_ptr() == flat.flat_p.untyped_storage().data_ptr()
            assert p.data.data_ptr() == flat.flat_p.data_ptr() + 4 * o and p.data.is_contiguous()
            assert p.grad.data_ptr() == flat.flat.data_ptr() + 4 * o and p.grad.shape == p.shape
            assert torch.equal(p.detach(), before[id(p)])
            used[o:o + n] = True
            off = o + round8(n)
        assert s["end"] == off
        assert s["lr_scale"] == np.float32(lr) and s["weight_decay"] == np.float32(g["weight_decay"])
    assert off == flat.n
    for name in ("flat_p", "flat", "exp_avg", "exp_avg_sq", "shadow"):
        assert not getattr(flat, name)[~used].any(), name          # alignment padding is zero
    assert torch.equal(flat.shadow, flat.flat_p.bfloat16())
    trips = [(m.query, m.key, m.value) for m in ps.module.modules() if all(hasattr(m, a) for a in ("query", "key", "value"))]
    trips += [(m.w_qs, m.w_ks, m.w_vs) for m in ps.module.modules() if hasattr(m, "w_qs")]
    assert len(trips) >= 2
    for trip in trips:
        for attr in ("weight", "bias"):
            ts = [getattr(l, attr) for l in trip]
            views = flat.packed_views(ts)
            assert views is not None
            sh, gr, pv = views
            assert torch.equal(pv, torch.cat([t.detach() for t in ts])) and pv.data_ptr() == ts[0].data_ptr()
            assert torch.equal(sh, pv.bfloat16()) and gr.data_ptr() == ts[0].grad.data_ptr()
            assert gr.shape == pv.shape == (sum(t.shape[0] for t in ts), *ts[0].shape[1:])


# ---- 1d: FlatState on the real model -------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_flat_state_on_the_gps_model_matches_float64_adamw():
    """Five FlatState.optimizer_step() calls over every trainable GPS parameter (~123M, 491 MB) against float64 AdamW +
    clip_grad_norm_ built from the parameter groups themselves, not from FlatState's segment table."""
    ps, groups, base = gps_groups("cuda")
    flat = train.FlatState(groups, base, betas=(0.9, 0.98), eps=1e-8, max_norm=5.0)
    live = [([p for p in g["params"] if p.requires_grad], lr, g["weight_decay"]) for g, lr in zip(groups, base)]
    live = [(ts, f32(lr), f32(wd)) for ts, lr, wd in live if ts]
    params = [p for ts, _, _ in live for p in ts]
    gen = torch.Generator(device="cuda").manual_seed(21)
    pscale = [f32(10.0 ** u) for u in torch.empty(len(params)).uniform_(-2, 0, generator=torch.Generator().manual_seed(2))]
    step_scale = [1e-2, 1e-4, 3e-3, 3e-5, 1e-2]
    factors = [f32(M.warmup_cosine(i + 1, 3, 10)) for i in range(5)]

    def grads_at(i):
        return [p.grad for p in params]

    ref = reference(live, grads_at, factors, (f32(0.9), f32(0.98)), f32(1e-8), 5.0, flat.n)
    worst = dict.fromkeys(("p", "m", "v", "norm"), 0.0)
    clipped = 0
    for i in range(5):
        for p, s in zip(params, pscale):
            p.grad.copy_(torch.randn(p.shape, device="cuda", generator=gen) * (s * step_scale[i]))
        norm, rp, rm, rv, (bp, bm, bv) = next(ref)
        flat.lr_factor.fill_(factors[i])
        flat.optimizer_step()
        clipped += norm > 5.0
        err = abs(flat.grad_norm_t.item() - norm) / norm
        assert err <= norm_rel_bound(flat.n), (i, flat.grad_norm_t.item(), norm)
        worst["norm"] = max(worst["norm"], err / norm_rel_bound(flat.n))
        for k, p in enumerate(params):
            o = flat.offsets[id(p)]
            sl = slice(o, o + p.numel())
            worst["p"] = max(worst["p"], within(p.detach().reshape(-1), rp[k].reshape(-1), bp[k].reshape(-1), f"step {i} p"))
            worst["m"] = max(worst["m"], within(flat.exp_avg[sl], rm[k].reshape(-1), bm[k].reshape(-1), f"step {i} m"))
            worst["v"] = max(worst["v"], within(flat.exp_avg_sq[sl], rv[k].reshape(-1), bv[k].reshape(-1), f"step {i} v"))
    for p in params:            # what every ops linear reads as its bf16 weight
        sh = ops._bf16_of(p)
        assert sh.data_ptr() == flat.shadow.data_ptr() + 2 * flat.offsets[id(p)]
        assert torch.equal(sh, p.detach().bfloat16())
    assert 0 < clipped < 5
    print(f"FLATSTATE_GPS {len(params)} parameters, {flat.nseg} segments, clipped steps {clipped}/5: worst |err| / bound",
          {k: f"{v:.3g}" for k, v in worst.items()})


# ---- 1e: direct accumulation into .grad ----------------------------------------------------------------------------------
def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed + sum(s))
    return torch.randn(*s, device="cuda", generator=g) * scale


def rel(got, want):
    return (got.float() - want.float()).abs().max().item() / (want.float().abs().max().item() + 1e-9)


def check_direct_accumulation(params, incs, run, tol, what):
    """Pre-fill every p.grad with values of the size of its increment, run forward + backward with ops.DIRECT_GRAD set, and
    check that autograd delivered no parameter gradient and that p.grad, same storage, equals pre + increment."""
    gen = torch.Generator(device="cuda").manual_seed(99)
    for p, inc in zip(params, incs):
        if p.grad is None:
            p.grad = torch.empty_like(p)
        p.grad.copy_(torch.randn(p.shape, device="cuda", generator=gen) * inc.abs().mean())
    pre = [p.grad.clone() for p in params]
    ptrs = [p.grad.data_ptr() for p in params]
    seen = []
    # the hook also runs, with None, for an input whose backward returned no gradient
    hooks = [p.register_hook(lambda g, k=k: seen.append(k) if g is not None else None) for k, p in enumerate(params)]
    ops.DIRECT_GRAD[0] = True
    try:
        run()
    finally:
        ops.DIRECT_GRAD[0] = False
        for h in hooks:
            h.remove()
    assert not seen, f"{what}: autograd returned gradients for parameters {seen}"
    for k, (p, p0, inc) in enumerate(zip(params, pre, incs)):
        assert p.grad.data_ptr() == ptrs[k], (what, k)
        err = rel(p.grad, p0 + inc)
        assert err < tol, f"{what} parameter {k}: max |err| / max |ref| = {err:.3g} (tol {tol})"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "residual", "applied_twice"])
def test_direct_grad_layer_norm(mode):
    """ops.layer_norm with DIRECT_GRAD: sv_layer_norm_bwd_acc adds d(gamma), d(beta) into the existing gradients."""
    R, D = 600, 768
    x, r, x2 = rnd(R, D).bfloat16(), rnd(R, D, seed=1).bfloat16(), rnd(R, D, seed=2).bfloat16()
    go = rnd(R, D, seed=3).bfloat16()
    gamma = (1 + rnd(D, seed=4, scale=0.1)).requires_grad_(True)
    beta = rnd(D, seed=5, scale=0.1).requires_grad_(True)
    calls = {"plain": [(x, None)], "residual": [(x, r)], "applied_twice": [(x, r), (x2, None)]}[mode]
    gr, br = gamma.detach().clone().requires_grad_(True), beta.detach().clone().requires_grad_(True)
    for a, res in calls:        # the kernel normalises residual + x as stored in bf16
        s = (a.float() + res.float()).bfloat16().float() if res is not None else a.float()
        F.layer_norm(s, (D,), gr, br, 1e-5).backward(go.float())

    def run():
        sum(ops.layer_norm(a, gamma, beta, residual=res).float() for a, res in calls).backward(go.float())

    check_direct_accumulation([gamma, beta], [gr.grad, br.grad], run, 2e-3, f"layer_norm {mode}")


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["relu", "gelu"])
def test_direct_grad_ffn(act):
    """ops.ffn with DIRECT_GRAD: both wgrad GEMMs add W1, b1, W2, b2 gradients into the existing ones."""
    Mr, D, H = 1000, 768, 2048
    x, go = rnd(Mr, D).bfloat16(), rnd(Mr, D, seed=3).bfloat16()
    ps = [rnd(H, D, seed=1, scale=D ** -0.5), rnd(H, seed=2), rnd(D, H, seed=4, scale=H ** -0.5), rnd(D, seed=5)]
    ps = [p.requires_grad_(True) for p in ps]
    rs = [p.detach().clone().requires_grad_(True) for p in ps]
    pre = F.linear(x.float(), rs[0].bfloat16().float(), rs[1])
    h = torch.relu(pre) if act == "relu" else F.gelu(pre)
    h = h + (h.detach().bfloat16().float() - h.detach())          # the kernel stores h in bf16
    F.linear(h, rs[2].bfloat16().float(), rs[3]).backward(go.float())

    def run():
        ops.ffn(x, *ps, activation=act).backward(go)

    check_direct_accumulation(ps, [r.grad for r in rs], run, 2.5e-2, f"ffn {act}")


class QKV(torch.nn.Module):
    def __init__(self, E):
        super().__init__()
        self.query, self.key, self.value = (torch.nn.Linear(E, E) for _ in range(3))


@pytest.mark.gpu
def test_direct_grad_linear_packed_writes_the_flat_state_pack_views():
    """ops.linear_packed on a q | k | v module whose parameters live in a FlatState: the single wgrad GEMM adds into the
    [3E, E] / [3E] gradient views that train.register_packs registered."""
    torch.manual_seed(0)
    E = 384
    mod = QKV(E).cuda()
    groups = M.no_decay_param_group(mod.named_parameters(), 1e-3)     # weights adjacent in one group, biases in the other
    flat = train.FlatState(groups, [1e-3, 1e-3])
    train.register_packs(mod, flat)
    lins = [mod.query, mod.key, mod.value]
    assert tuple(id(l.weight) for l in lins) in ops._PACKS
    params = [l.weight for l in lins] + [l.bias for l in lins]
    x, go = rnd(8, 130, E).bfloat16(), rnd(8, 130, 3 * E, seed=1).bfloat16()
    rs = [p.detach().clone().requires_grad_(True) for p in params]
    torch.cat([F.linear(x.float(), w.bfloat16().float(), b) for w, b in zip(rs[:3], rs[3:])], -1).backward(go.float())

    def run():
        ops.linear_packed(x, lins).backward(go)

    check_direct_accumulation(params, [r.grad for r in rs], run, 1e-2, "linear_packed")


@pytest.mark.gpu
@pytest.mark.parametrize("V,pad", [(1000, None), (1000, 3), (5, 0), (4, None), (4, 0), (3, 2)])
def test_direct_grad_embedding(V, pad):
    """ops.embedding with DIRECT_GRAD on both backward paths: the scatter kernel (V >= 5) and masked column sums (V <= 4)."""
    ids = torch.randint(0, V, (64, 50), device="cuda", generator=torch.Generator(device="cuda").manual_seed(V))
    w = rnd(V, 768).requires_grad_(True)
    go = rnd(64, 50, 768, seed=3)
    wr = w.detach().clone().requires_grad_(True)
    F.embedding(ids, wr, pad).backward(go)

    def run():
        ops.embedding(ids, w, pad).backward(go)

    check_direct_accumulation([w], [wr.grad], run, 1e-5, f"embedding V={V} padding_idx={pad}")
