"""Native SyncBatchNorm for the trainable PointNet++ (csrc/pn_train.cu sv_pn_bn_sync_*, pn_train.StatExchange; reference:
model/objcls.py:33-34 convert_sync_batchnorm, torch.nn.SyncBatchNorm semantics).

* world 1 (a `local=True` exchange) reproduces the plain BatchNorm2d path bit for bit;
* k ranks emulated on one GPU (every push launched before any finish, so no kernel waits) against float64 statistics of the
  concatenated bf16 Y and against the full-batch single-rank call, with elementwise bounds derived from fp32 / bf16 rounding;
* a float64 knock-out check: local statistics in the forward or the local 1/R in the backward break those bounds by far;
* CUDA-graph replay with an odd number of exchanges per replay; routing; argument validation without a GPU;
* two real ranks (scripts/objcls_syncbn_2rank.py, skipped with fewer than 2 GPUs)."""
import copy
import json
import os
import subprocess
import sys

import pytest
import torch

from sceneverse_b200 import synthetic, weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32, UBF = 2.0 ** -24, 2.0 ** -8          # unit roundoff of fp32 and of bf16 (8 significant bits)
TX_TY = 8                                 # rows per thread stripe step in col_sums_kernel (TY)


def gamma_n(n):
    return n * U32 / (1 - n * U32)


def chain(R, cap_slabs):
    """Longest fp32 addition chain of col_sums_kernel for R rows: a thread's stripe of its slab, then the TY-way sum in
    shared memory (the slab sums are added in fp64)."""
    slabs = max(1, min(-(-R // 256), cap_slabs))
    per = -(-R // slabs) if R else 0
    return -(-per // TX_TY) + TX_TY + 2


def make_pn(seed=0):
    from sceneverse_b200.modules.pointnet import GPS_SPEC, PointNetPP
    torch.manual_seed(seed)
    net = PointNetPP(**GPS_SPEC)
    net.load_state_dict(weights.synthetic_state_dict(net, seed))
    return net


# ---- routing (CPU) ----------------------------------------------------------------------------------------------------------
def test_bn_all_eval_sees_sync_batchnorm():
    net = torch.nn.SyncBatchNorm.convert_sync_batchnorm(make_pn()).train()
    assert any(isinstance(m, torch.nn.SyncBatchNorm) for m in net.modules())
    assert not net._bn_all_eval()
    assert net.eval()._bn_all_eval()


# ---- argument validation (no GPU) -------------------------------------------------------------------------------------------
_VALIDATION = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from sceneverse_b200 import _lib
lib = _lib.gps()
a = 0x1000      # 16-byte aligned fake address


def push(mode=0, y=a, dout=a, R=256, C=64, g=a, b=a, mean=a, rstd=a, scratch=a, peers=a, cap=768, done=a, world=2, rank=0, ep=a):
    return lib.sv_pn_bn_sync_push(mode, y, dout, R, C, g, b, mean, rstd, scratch, peers, cap, done, world, rank, ep, None)


def ffwd(y=a, R=256, C=64, g=a, b=a, mean=a, rstd=a, var=a, out=a, peers=a, cap=768, world=2, rank=0, ep=a):
    return lib.sv_pn_bn_sync_finish_fwd(y, R, C, g, b, 1e-5, mean, rstd, var, out, peers, cap, world, rank, ep, None)


def fbwd(y=a, dout=a, R=256, C=64, g=a, b=a, mean=a, rstd=a, dy=a, dg=a, db=a, gsum=a, peers=a, cap=768, world=2, rank=0, ep=a):
    return lib.sv_pn_bn_sync_finish_bwd(y, dout, R, C, g, b, mean, rstd, dy, dg, db, 0, gsum, peers, cap, world, rank, ep, None)


common = {"C < 8": dict(C=0), "C % 8": dict(C=12), "C > cap": dict(C=776), "world 0": dict(world=0), "world 65": dict(world=65),
          "rank < 0": dict(rank=-1), "rank == world": dict(rank=2), "R < 0": dict(R=-1), "NULL peers": dict(peers=None),
          "misaligned peers": dict(peers=a + 4), "NULL epoch": dict(ep=None), "misaligned epoch": dict(ep=a + 2),
          "misaligned y": dict(y=a + 8), "NULL y": dict(y=None)}
out = {}
for k, kw in common.items():
    out["push " + k], out["finish_fwd " + k], out["finish_bwd " + k] = push(**kw), ffwd(**kw), fbwd(**kw)
out["push mode 2"], out["push NULL scratch"], out["push NULL done"] = push(mode=2), push(scratch=None), push(done=None)
out["push misaligned done"] = push(done=a + 2)
out.update({"push mode 1 NULL " + w: push(mode=1, **{w: None}) for w in ("dout", "g", "b", "mean", "rstd")})
out["push mode 1 misaligned dout"] = push(mode=1, dout=a + 8)
out.update({"finish_fwd NULL " + w: ffwd(**{w: None}) for w in ("g", "b", "mean", "rstd", "out")})
out["finish_fwd misaligned out"] = ffwd(out=a + 8)
out.update({"finish_bwd NULL " + w: fbwd(**{w: None}) for w in ("dout", "g", "b", "mean", "rstd", "dy", "dg", "db", "gsum")})
out["finish_bwd misaligned dy"] = fbwd(dy=a + 8)
sizes = {"floats C=8 world=1": lib.sv_pn_sync_floats(8, 1), "floats C=768 world=2": lib.sv_pn_sync_floats(768, 2),
         "floats C=12": lib.sv_pn_sync_floats(12, 2), "floats world 0": lib.sv_pn_sync_floats(64, 0)}
print(json.dumps({"status": out, "sizes": sizes}))
"""


def test_sync_entry_points_validate_arguments_without_gpu():
    """The push / finish entry points reject malformed calls before any launch (1 = SV_ERR_INVALID_ARG).  The calls run in a
    process that sees no CUDA device: a missing check would reach the launch on fake pointers and return 2 instead."""
    res = subprocess.run([sys.executable, "-c", _VALIDATION, ROOT], capture_output=True, text=True, timeout=120,
                         env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    bad = {k: v for k, v in got["status"].items() if v != 1}
    assert len(got["status"]) == 3 * 14 + 4 + 6 + 6 + 10 and not bad, bad
    # [2][world][2C+1] doubles as float pairs, then `world` flags rounded up to 8 bytes; 0 for an invalid C or world
    assert got["sizes"] == {"floats C=8 world=1": 4 * 17 + 2, "floats C=768 world=2": 8 * 1537 + 2, "floats C=12": 0,
                            "floats world 0": 0}


# ---- GPU ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_world1_exchange_reproduces_plain_batchnorm_bitwise(monkeypatch):
    """Output, every BatchNorm / fc gradient, running statistics and num_batches_tracked are bitwise equal.  The 1x1-conv
    weight gradients come from the split-K weight-gradient GEMM, whose fp32 atomics make their bits order-dependent even
    between two runs of one path: for them the operands (dy, X) of that GEMM are checked bitwise instead, and the results
    within the ordering bound."""
    from sceneverse_b200 import pn_train
    Fn = pn_train._ConvBNReLUFn
    dev = torch.device("cuda", 0)
    plain = make_pn().to(dev).train()
    sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    assert sum(isinstance(m, torch.nn.SyncBatchNorm) for m in sync.modules()) == 9
    ex = pn_train.StatExchange(dev, local=True)
    x = torch.from_numpy(synthetic.object_batch(3, 48, 1024, pad_fraction=0.1)).to(dev)
    go = torch.randn(48, 768, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    conv_bwd = Fn.conv_bwd
    seen = []

    def recording_conv_bwd(X, wb, dy, cin, need_dx=True):
        seen[-1].append((X, dy, cin))
        return conv_bwd(X, wb, dy, cin, need_dx)
    monkeypatch.setattr(Fn, "conv_bwd", staticmethod(recording_conv_bwd))
    for step in range(2):                     # the second step runs on the running statistics / parity of the first
        with torch.autocast("cuda", dtype=torch.bfloat16):
            assert pn_train.available(x, plain) and pn_train.available(x, sync)
            yp = plain(x)
            ys = pn_train.forward(sync, x, exchange=ex)
        seen.append([])
        yp.float().backward(go)
        seen.append([])
        ys.float().backward(go)
        torch.cuda.synchronize()
        assert torch.equal(yp, ys)
        wgrad_ops = [list(reversed(s)) for s in seen[-2:]]            # backward visits the 9 layers last to first
        assert len(wgrad_ops[0]) == len(wgrad_ops[1]) == 9
        conv = [n for n, _ in plain.named_parameters() if n.endswith("conv.weight")]
        for (n, p), (_, q) in zip(plain.named_parameters(), sync.named_parameters()):
            assert p.grad is not None, n
            if n in conv:
                (Xp, dyp, cin), (Xs, dys, _) = wgrad_ops[0][conv.index(n)], wgrad_ops[1][conv.index(n)]
                assert torch.equal(Xp, Xs) and torch.equal(dyp, dys), n
                diff = (p.grad - q.grad).abs().reshape(p.shape[0], cin).double()
                assert (diff <= wgrad_order_bound(dyp, Xp, cin)).all(), n
            else:
                assert torch.equal(p.grad, q.grad), n
        for (n, s), (_, t) in zip(plain.named_buffers(), sync.named_buffers()):
            assert torch.equal(s, t), n
        assert int(ex.epoch_dev) == 18 * (step + 1)
        for n in (plain, sync):
            n.zero_grad(set_to_none=True)


class Layer:
    """One conv1x1 + BN + ReLU layer (Cin -> C) with its operands: k shards of the rows, parameters, output gradients."""

    def __init__(self, sizes, cin, C, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        kp = (cin + 7) // 8 * 8
        R = sum(sizes)
        X = torch.zeros(R, kp, device="cuda", dtype=torch.bfloat16)
        # every shard draws from its own distribution, as objects on different GPUs do: local statistics are visibly wrong
        scale = torch.cat([torch.full((n, 1), 1 + 0.3 * r) for r, n in enumerate(sizes)]).cuda()
        X[:, :cin] = (torch.randn(R, cin, device="cuda", generator=g) * scale + 0.5 * scale).bfloat16()
        self.X = X
        self.Xs = list(X.split(sizes))
        self.sizes, self.cin, self.C = sizes, cin, C
        self.W = torch.randn(C, cin, 1, 1, device="cuda", generator=g) * 0.2
        self.g32 = (1 + 0.2 * torch.randn(C, device="cuda", generator=g)).contiguous()
        self.b32 = (0.2 * torch.randn(C, device="cuda", generator=g)).contiguous()
        self.dout = torch.randn(R, C, device="cuda", generator=g).bfloat16()
        self.douts = [d.contiguous() for d in self.dout.split(sizes)]
        self.Xs = [x.contiguous() for x in self.Xs]


def sync_layer(exs, L, eps=1e-5):
    """The layer over the k emulated ranks through _ConvBNReLUFn's phases: push on every rank, then finish on every rank, in
    each direction.  Returns per rank (y, out, stats, dX, dW, dgb)."""
    from sceneverse_b200.pn_train import _ConvBNReLUFn as Fn
    conv = [Fn.conv_fwd(X, L.W) for X in L.Xs]
    for ex, (_, y) in zip(exs, conv):
        ex.push(0, y)
    fwd = [ex.finish_fwd(y, L.g32, L.b32, eps) for ex, (_, y) in zip(exs, conv)]
    for ex, (_, y), (_, st), d in zip(exs, conv, fwd, L.douts):
        ex.push(1, y, d, st, L.g32, L.b32)
    bwd = [ex.finish_bwd(y, d, st, L.g32, L.b32) for ex, (_, y), (_, st), d in zip(exs, conv, fwd, L.douts)]
    res = []
    for X, (wb, y), (out, st), (dy, dgb) in zip(L.Xs, conv, fwd, bwd):
        dX, dW = Fn.conv_bwd(X, wb, dy, L.cin)
        res.append(dict(X=X, y=y, out=out, stats=st, dy=dy, dX=dX, dW=dW, dgb=dgb))
    return res


def wgrad_order_bound(dy, X, cin):
    """The weight-gradient GEMM adds its split-K partial tiles (at most 32) with fp32 atomics, so its bits depend on their
    arrival order: two runs on identical operands differ by at most 2 * gamma_32 * (|dy|^T |X|) elementwise."""
    return 2 * gamma_n(32) * (dy.double().abs().t() @ X.double().abs())[:, :cin]


def full_layer(L, eps=1e-5):
    """The same layer as ONE rank over all rows on the plain BatchNorm2d path (sv_pn_bn_relu_fwd / _bwd)."""
    from sceneverse_b200.pn_train import _ConvBNReLUFn as Fn
    X = L.X.clone().requires_grad_(True)
    W = L.W.clone().requires_grad_(True)
    g, b = L.g32.clone().requires_grad_(True), L.b32.clone().requires_grad_(True)
    out, st = Fn.apply(X, W, g, b, eps)
    out.backward(L.dout)
    y = Fn.conv_fwd(L.X, L.W)[1]
    return dict(y=y, out=out.detach(), stats=st, dX=X.grad, dW=W.grad, dgb=torch.stack([g.grad, b.grad]))


def reference(L, y, mask, rows, eps=1e-5):
    """float64 SyncBatchNorm over the concatenated bf16 Y (rows `rows` of it for the local sums) and the elementwise
    bound of each kernel result, from fp32 / bf16 rounding: m = the longest fp32 addition chain of the column sums.
    `mask` = where the path's forward output is positive (its own ReLU decision)."""
    d = torch.float64
    y, g, b = y.to(d), L.g32.to(d), L.b32.to(d)
    N = y.shape[0]
    m = max(chain(n, 127) for n in list(L.sizes) + [N])
    mean = y.mean(0)
    var = (y * y).mean(0) - mean * mean                          # the kernels' formula (E[y^2] - mean^2), evaluated exactly
    rstd = (var + eps).rsqrt()
    e_s0, e_s1 = gamma_n(m) * y.abs().sum(0), gamma_n(m + 1) * (y * y).sum(0)
    e_mean = e_s0 / N + U32 * mean.abs()
    e_var = e_s1 / N + (2 * mean.abs() + e_s0 / N) * e_s0 / N
    e_rstd = ((var + eps - e_var).clamp_min(1e-300).rsqrt() - rstd).abs() + U32 * rstd
    var_u = var * N / (N - 1)
    e_var_u = e_var * N / (N - 1) + U32 * var_u
    xh = (y - mean) * rstd
    e_xh = e_mean * rstd + (y - mean).abs() * e_rstd + 3 * U32 * xh.abs()
    pre = xh * g + b
    e_pre = g.abs() * e_xh + 2 * U32 * (xh * g).abs() + U32 * pre.abs()
    out = pre.clamp_min(0)
    e_out = e_pre + UBF * (out + e_pre)
    gg = L.dout.to(d) * mask
    Sb, Sg = gg.sum(0), (gg * xh).sum(0)
    e_Sb = gamma_n(m) * gg.abs().sum(0) + U32 * Sb.abs()
    e_Sg = (gg.abs() * e_xh).sum(0) + gamma_n(m + 1) * (gg * xh).abs().sum(0) + U32 * Sg.abs()
    inner = gg - Sb / N - xh * Sg / N
    e_inner = (e_Sb + 2 * U32 * Sb.abs()) / N + (e_xh * Sg.abs() + xh.abs() * (e_Sg + 2 * U32 * Sg.abs())) / N \
        + 4 * U32 * (gg.abs() + Sb.abs() / N + (xh * Sg).abs() / N)
    dy = g * rstd * inner
    e_dy = g.abs() * (e_rstd * inner.abs() + (rstd + e_rstd) * e_inner) + 3 * U32 * dy.abs()
    e_dy = e_dy + UBF * (dy.abs() + e_dy)                                     # stored in bf16
    Wb = torch.nn.functional.pad(L.W.reshape(L.C, L.cin).bfloat16(), (0, L.X.shape[1] - L.cin)).to(d)
    dX = dy @ Wb
    e_dX = e_dy @ Wb.abs() + gamma_n(L.C) * ((dy.abs() + e_dy) @ Wb.abs())
    e_dX = e_dX + UBF * (dX.abs() + e_dX)
    lgg, lxh, le = gg[rows], xh[rows], e_xh[rows]
    ldb, ldg = lgg.sum(0), (lgg * lxh).sum(0)
    ml = chain(lgg.shape[0], 127)
    e_ldb = gamma_n(ml) * lgg.abs().sum(0) + U32 * ldb.abs()
    e_ldg = (lgg.abs() * le).sum(0) + gamma_n(ml + 1) * (lgg * lxh).abs().sum(0) + U32 * ldg.abs()
    return dict(mean=(mean, e_mean), rstd=(rstd, e_rstd), var_u=(var_u, e_var_u), out=(out, e_out), dy=(dy, e_dy),
                dX=(dX, e_dX), dgamma=(ldg, e_ldg), dbeta=(ldb, e_ldb), xh=xh, gg=gg, Sb=Sb, Sg=Sg, g=g, b=b, N=N)


def ratio(got, ref_err):
    ref, err = ref_err
    return ((got.double() - ref).abs() / (err + 1e-300)).max().item()


CASES = [(2, (4096, 2500), 67, 128), (3, (1000, 0, 7000), 131, 256), (4, (2048, 4096, 333, 9000), 259, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("k,sizes,cin,C", CASES, ids=["k2", "k3-empty-shard", "k4"])
def test_emulated_ranks_match_float64_and_the_full_batch(k, sizes, cin, C):
    from sceneverse_b200 import pn_train
    L = Layer(sizes, cin, C, seed=k)
    exs = pn_train.StatExchange.emulated(k, torch.device("cuda", 0))
    res = sync_layer(exs, L)
    full = full_layer(L)
    torch.cuda.synchronize()
    assert [int(ex.epoch_dev) for ex in exs] == [2] * k
    # the statistics are bit-identical on every rank (rank-ordered fp64 sums of the same slots)
    for r in res[1:]:
        assert torch.equal(r["stats"], res[0]["stats"])
    Y = torch.cat([r["y"] for r in res])
    worst = {}
    offs = [0]
    for n in sizes:
        offs.append(offs[-1] + n)
    mask_s = (torch.cat([r["out"] for r in res]) > 0).double()
    for name, path, mask in (("sync", res, mask_s), ("full", None, (full["out"] > 0).double())):
        ref = reference(L, Y if path is not None else full["y"], mask, slice(0, Y.shape[0]))
        st = res[0]["stats"] if path is not None else full["stats"]
        for i, key in enumerate(("mean", "rstd", "var_u")):
            worst[f"{name} {key}"] = ratio(st[i], ref[key])
        out = torch.cat([r["out"] for r in res]) if path is not None else full["out"]
        dX = torch.cat([r["dX"] for r in res]) if path is not None else full["dX"]
        worst[f"{name} out"] = ratio(out, ref["out"])
        worst[f"{name} dX"] = ratio(dX, ref["dX"])
        if path is None:
            worst["full dgamma"], worst["full dbeta"] = ratio(full["dgb"][0], ref["dgamma"]), ratio(full["dgb"][1], ref["dbeta"])
    # d gamma / d beta stay the shard's LOCAL sums (torch SyncBatchNorm); only dX uses the global sums.  Their sum (taken in
    # fp64 here) is the full-batch value within the sum of the shards' bounds.
    e_sum = torch.zeros(2, C, dtype=torch.float64, device="cuda")
    for r, (a, z) in enumerate(zip(offs[:-1], offs[1:])):
        ref = reference(L, Y, mask_s, slice(a, z))
        worst[f"rank {r} dgamma"] = ratio(res[r]["dgb"][0], ref["dgamma"])
        worst[f"rank {r} dbeta"] = ratio(res[r]["dgb"][1], ref["dbeta"])
        e_sum += torch.stack([ref["dgamma"][1], ref["dbeta"][1]])
    ref = reference(L, Y, mask_s, slice(0, Y.shape[0]))
    dgb_sum = torch.stack([r["dgb"] for r in res]).double().sum(0)
    worst["sum of shard dgamma"] = ratio(dgb_sum[0], (ref["dgamma"][0], e_sum[0]))
    worst["sum of shard dbeta"] = ratio(dgb_sum[1], (ref["dbeta"][0], e_sum[1]))
    print("SYNCBN worst error / bound", k, {n: round(v, 4) for n, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst

    # knock-out, in float64: the same quantities without the exchange are far outside the bounds
    ref = reference(L, Y, mask_s, slice(0, Y.shape[0]))
    live = [(a, z) for a, z in zip(offs[:-1], offs[1:]) if z > a]
    ko_fwd, ko_bwd = [], []
    for a, z in live:
        y = Y[a:z].double()
        local = ((y - y.mean(0)) * (y.var(0, unbiased=False) + 1e-5).rsqrt() * ref["g"] + ref["b"]).clamp_min(0)
        ko_fwd.append(ratio(local, (ref["out"][0][a:z], ref["out"][1][a:z])))
        n = z - a
        dy = ref["g"] * ref["rstd"][0] * (ref["gg"][a:z] - ref["Sb"] / n - ref["xh"][a:z] * ref["Sg"] / n)
        ko_bwd.append(ratio(dy, (ref["dy"][0][a:z], ref["dy"][1][a:z])))
    print("SYNCBN knock-out error / bound", k, "local stats", round(max(ko_fwd), 1), "local 1/R", round(max(ko_bwd), 1))
    assert max(ko_fwd) > 20 and max(ko_bwd) > 20


def _replay_case(exs, L1, L2, steps=5):
    """L1 forward, then L2 forward + backward: 3 exchanges per step, so the parity of every replay differs from the last."""
    gen = torch.Generator(device="cuda").manual_seed(9)

    def refresh():
        for x in L1.Xs:
            x[:, :L1.cin].copy_((torch.randn(x.shape[0], L1.cin, device="cuda", generator=gen)).bfloat16())
        for d in L2.douts:
            d.copy_(torch.randn(d.shape, device="cuda", generator=gen).bfloat16())

    def step():
        from sceneverse_b200.pn_train import _ConvBNReLUFn as Fn
        conv = [Fn.conv_fwd(X, L1.W) for X in L1.Xs]
        for ex, (_, y) in zip(exs, conv):
            ex.push(0, y)
        outs = [ex.finish_fwd(y, L1.g32, L1.b32, 1e-5)[0] for ex, (_, y) in zip(exs, conv)]
        for x, o in zip(L2.Xs, outs):
            x[:, :L2.cin].copy_(o[:, :L2.cin])
        return sync_layer(exs, L2)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    e0 = [int(ex.epoch_dev) for ex in exs]
    for it in range(steps):
        refresh()
        graph.replay()
        torch.cuda.synchronize()
        assert [int(ex.epoch_dev) for ex in exs] == [e + 6 * it + 3 for e in e0], it
        got = [{k: v.clone() for k, v in r.items()} for r in static]
        want = step()                                             # eager, same inputs
        torch.cuda.synchronize()
        for g_, w_ in zip(got, want):
            for key in ("out", "stats", "dX", "dgb"):             # (dW: split-K fp32 atomics, order-dependent bits)
                assert torch.equal(g_[key], w_[key]), (it, key)
            assert torch.equal(g_["dy"], w_["dy"]), (it, "dy")
            diff = (g_["dW"] - w_["dW"]).abs().reshape(L2.C, L2.cin).double()
            assert (diff <= wgrad_order_bound(w_["dy"], w_["X"], L2.cin)).all(), (it, "dW")
        assert [int(ex.epoch_dev) for ex in exs] == [e + 6 * (it + 1) for e in e0], it


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3])
def test_graph_replay_with_an_odd_number_of_exchanges(k):
    from sceneverse_b200 import pn_train
    dev = torch.device("cuda", 0)
    exs = [pn_train.StatExchange(dev, local=True)] if k == 1 else pn_train.StatExchange.emulated(k, dev)
    sizes = (3000,) if k == 1 else (1500, 800, 2100)
    L1 = Layer(sizes, 13, 64, seed=20 + k)
    L2 = Layer(sizes, 64, 128, seed=30 + k)
    _replay_case(exs, L1, L2)


@pytest.mark.gpu
def test_sync_batchnorm_net_routing_on_gpu(monkeypatch):
    """A train-mode SyncBatchNorm net is not an eval-BN net: under no_grad it must not take the fused eval-BN kernels (they
    normalise with running statistics), and the native train-mode path accepts it."""
    from sceneverse_b200 import pn_train
    from sceneverse_b200.modules.pointnet import PointNetPP
    net = torch.nn.SyncBatchNorm.convert_sync_batchnorm(make_pn()).cuda().train()
    x = torch.from_numpy(synthetic.object_batch(4, 16, 1024)).cuda()

    def boom(*a, **k):
        raise AssertionError("forward_fused taken by a train-mode SyncBatchNorm net")
    monkeypatch.setattr(PointNetPP, "forward_fused", boom)
    with torch.no_grad():
        assert not net.fused_available(x)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            assert pn_train.available(x, net)
            y = net(x)
    assert y.shape == (16, 768) and torch.isfinite(y.float()).all()
    assert all(int(m.num_batches_tracked) == 1 for m in net.modules() if isinstance(m, torch.nn.SyncBatchNorm))


@pytest.mark.gpu
def test_objcls_syncbn_two_ranks():
    """PointNet++ and ObjClsStep at 2 ranks x 32 objects against one process x 64 objects and torch SyncBatchNorm."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", "29579",
                          os.path.join(ROOT, "scripts", "objcls_syncbn_2rank.py")], capture_output=True, text=True,
                         timeout=900, cwd=ROOT)
    assert "OBJCLS_SYNCBN_OK=True" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
