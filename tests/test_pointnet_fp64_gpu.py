"""The frozen PointNet++ encoder (PointNetPP.forward_fused: csrc/sa_mlp.cu for SA1 / SA2, four GEMMs for SA3 + fc) and the
train-mode BatchNorm kernels of csrc/pn_train.cu against float64, element by element.

* A float64 reference of the encoder, written from the reference operator sequence rather than the kernels' layout:
  QueryAndGroup (pointnet2_utils.py:314-363: neighbour xyz minus the centre, cat([xyz, features]) at :354-356), SharedMLP =
  3 x (Conv2d 1x1 -> BatchNorm2d -> ReLU) (pytorch_utils.py:11-36, :67-120), max over nsample (pointnet2_modules.py:65-71);
  then GroupAll with UNCENTRED xyz (pointnet2_utils.py:389-419), SA3, the max over the 16 points and fc
  (modules/layers/pointnet.py:55-63).  It reads the module's fp32 parameters and running statistics, so fold_bn,
  pack_sa_params, the SA2 / SA3 column permutations and the SA3 [feat | xyz | 0] padding are under test too.  Only the
  sampled centres and ball indices come from the kernels (sampling is index work, tested bit-exact elsewhere).
* A bound on |kernel - float64| for every element of feat1, feat2 and out, first order in the unit roundoffs, each term next
  to the kernel line it comes from.  The factor TOL covers the second-order terms.
* GPU cases: 1, 4 (exactly 128 SA1 centres), 37 and 5,120 clouds (the step's batch: the persistent loop over super-tiles),
  32 and 1,024 points, all-ones padded clouds, nsample 1 and 17 through the C entry points, and BatchNorm statistics with
  negative gamma, tiny running variances and running means several standard deviations off.
* A CPU knock-out test: each plausible kernel or packing slip, applied to the float64 reference, moves some element by at
  least 4 x the bound.
* The train-mode BatchNorm + ReLU kernels (sv_pn_bn_relu_fwd / _bwd) at the step's row counts against the per-column part of
  tests/test_syncbn_gpu.py::reference(), with a float64 knock-out, and bitwise checks of the exact grouping and row-group max
  kernels at the step's shapes.
"""
import math
import types

import pytest
import torch

from sceneverse_b200 import _lib, synthetic
from tests.test_syncbn_gpu import U32, UBF, chain, gamma_n, make_pn

UB = 2.0 ** -8              # unit roundoff of bf16 (8 significand bits, round to nearest: pack_bf16, __float2bfloat16_rn)
UF = 2.0 ** -24             # unit roundoff of fp32
TC = 2 * UF                 # per addition of the tensor core's fp32 accumulation (2u also covers a truncating accumulator)
# fold_bn (modules/pointnet.py:74-79) in fp32: running_var + eps, sqrt and the division leave <= 2.5 u on the scale (3 u with
# eps given as a double), W * scale one more; to_umma_sw128 / .to(bf16) then round the folded weight to bf16
S_REL = 3 * UF
W_ROUND = UB + S_REL + UF
K_SA1, K_SA2, K_SA3, K_FC = (16, 64, 64), (144, 128, 128), (272, 256, 512), 768   # K of every layer as the kernels run it
TOL = 1.01
CHUNK = 128                 # clouds per float64 reference chunk: <= ~1 GB of device memory at SA1


# ---- float64 reference ------------------------------------------------------------------------------------------------
KNOCKS = ("sa2_unpermuted", "z_col_shift", "z_not_centred", "max_ns_minus_1", "sa2_half_shift", "shift_without_mean",
          "fold_without_eps", "sa3_centred", "rowmax_off_by_one")


def _layer(net, lvl, j, knock=None):
    """Layer j of SA level lvl (0, 1, 2) in float64: the conv weight, the BatchNorm2d in eval mode and the bound terms of
    its fp32 fold.  knock: shift_without_mean (shift = beta), fold_without_eps (scale = gamma / sqrt(running_var))."""
    layer = getattr(net.encoder[lvl].mlps[0], f"layer{j}")
    bn = layer.bn.bn
    W = layer.conv.weight.detach().reshape(layer.conv.weight.shape[0], -1).double()
    g, b, rm, rv = (t.detach().double() for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))
    eps = 0.0 if knock == "fold_without_eps" else bn.eps
    if knock == "shift_without_mean":
        rm = torch.zeros_like(rm)
    s = g / torch.sqrt(rv + eps)
    shift = b - rm * s
    L = types.SimpleNamespace(W=W, s=s, shift=shift, aWs=(W * s[:, None]).abs().t().contiguous())
    L.bn = lambda y: (y - rm) / torch.sqrt(rv + eps) * g + b              # BatchNorm2d.eval, as the reference runs it
    # shift = beta - running_mean * scale in fp32: the scale's error and the product, then the subtraction
    L.e_shift = (S_REL + UF) * (rm * s).abs() + UF * shift.abs()
    return L


def _conv_bn(x, ex, net, lvl, j, K, knock=None, calib=None):
    """Layer j (conv 1x1 -> eval BN) of SA level lvl over rows x (..., Cin) in the reference channel order, ex the bound of
    the kernel's operand -> the pre-activation, the raw accumulator (the BN scale folded into the weight: what the kernels
    take the maximum of), its bound and the layer.  calib(lvl, j, y), if given, sees the conv output before the layer's
    BatchNorm statistics are read."""
    y = x @ getattr(net.encoder[lvl].mlps[0], f"layer{j}").conv.weight.detach().flatten(1).double().t()
    if calib is not None:
        calib(lvl, j, y)
    L = _layer(net, lvl, j, knock)
    # the K-sum of the layer (sa_mlp.cu layer(), gemm.cu mainloop): bf16 x bf16 products, exact in fp32, summed by the
    # tensor core in fp32; the operand's own error and the bf16 folded weight's through |W scale|
    e_acc = ex @ L.aWs + (W_ROUND + K * TC) * (x.abs() @ L.aWs)
    pre = L.bn(y)
    if knock == "sa2_half_shift" and (lvl, j) == (1, 2):     # the second column half adds the first half's shift
        n = L.shift.shape[0] // 2
        pre = y * L.s + torch.cat([L.shift[:n], L.shift[:n]])
    return pre, y * L.s, e_acc, L


def _relu_store(pre, e_acc, L):
    """relu(acc + shift) in fp32, stored as bf16 to the A tile (sa_mlp.cu:107) or the output (gemm.cu:394-405)."""
    return pre.clamp_min(0), _relu_bf16(pre, e_acc + L.e_shift + UF * pre.abs())


def _mlp(x, ex, net, lvl, ks, knock=None, calib=None):
    """The three layers of a fused SA level: layers 1 and 2 feed the next through bf16; returns _conv_bn of layer 3."""
    for j in (0, 1):
        pre, _, e_acc, L = _conv_bn(x, ex, net, lvl, j, ks[j], knock, calib)
        x, ex = _relu_store(pre, e_acc, L)
    return _conv_bn(x, ex, net, lvl, 2, ks[2], knock, calib)


def _relu_bf16(pre, e_pre):
    """Bound of bf16(relu(p)) for a kernel pre-activation p within e_pre of pre: ReLU is 1-Lipschitz, and where
    pre <= -e_pre the kernel's value is negative too and its ReLU exactly 0."""
    e = torch.where(pre >= 0, e_pre, (pre + TOL * e_pre).clamp_min(0))
    return e + UB * (pre.clamp_min(0) + e)


def _max_rows(pre, acc, e_acc, L, dim, packed):
    """The neighbourhood max of relu(pre) over `dim` (the reference: ReLU, then max_pool2d), its bound and the share of
    the packed-max term in the bound of the pre-activation.  The kernels take the max of the raw accumulators
    (relu(acc + shift) is monotone in acc) and add the shift once; the kernel's max lies between the largest lower and
    the largest upper end of its group's intervals."""
    out = pre.clamp_min(0).amax(dim)
    m = acc.amax(dim)
    e_m = torch.maximum((acc + e_acc).amax(dim) - m, m - (acc - e_acc).amax(dim))
    # SA2 only: the running max is packed bf16, so the raw accumulator is rounded BEFORE the shift is added (sa_mlp.cu:233,
    # :251).  Where the shift cancels most of the accumulator this term is far larger than u |out|.
    e_pk = UB * m.abs() if packed else torch.zeros_like(m)
    pre_m = m + L.shift
    e_pre = e_m + e_pk + L.e_shift + UF * pre_m.abs()           # m + shift in fp32 (sa_mlp.cu:254, gemm.cu:394-417)
    return out, _relu_bf16(pre_m, e_pre), e_pk / e_pre          # ReLU, bf16 store (sa_mlp.cu:254, gemm.cu:486)


def _gather(t, idx):
    """t (B, N, C), idx (B, M, ns) -> (B, M, ns, C)."""
    B = t.shape[0]
    return t[torch.arange(B, device=t.device)[:, None, None], idx.long()]


def sa1_reference(net, pts, nx1, bi1, knock=None, calib=None):
    """SA1 of clouds pts (B, P, 6) f32 around centres nx1 (B, 32, 3) with neighbours bi1 (B, 32, ns) -> (feat1, bound, -)."""
    g = _gather(pts.double(), bi1)
    c = nx1.double()[:, :, None, :]
    dxyz = g[..., :3] - c
    if knock == "z_not_centred":
        dxyz[..., 2] = g[..., 2]
    x = torch.cat([dxyz, g[..., 3:6]], -1)
    # sa_mlp.cu:182-184: xyz - centre in fp32, then every operand rounded to bf16
    ex = torch.cat([(UB + UF) * dxyz.abs(), UB * g[..., 3:6].abs()], -1)
    if knock == "z_col_shift":                                  # dz lands in column 3, r in column 2
        x, ex = x[..., [0, 1, 3, 2, 4, 5]], ex[..., [0, 1, 3, 2, 4, 5]]
    pre, acc, e_acc, L = _mlp(x, ex, net, 0, K_SA1, knock, calib)
    if knock == "max_ns_minus_1" and pre.shape[2] > 1:
        pre, acc, e_acc = pre[:, :, :-1], acc[:, :, :-1], e_acc[:, :, :-1]
    return _max_rows(pre, acc, e_acc, L, 2, packed=False)


def sa2_reference(net, nx1, feat1, nx2, bi2, knock=None, calib=None):
    """SA2 of the SA1 points nx1 (B, 32, 3) with features feat1 (B, 32, 128) (the kernel's bf16 feat1: an exact operand)
    around centres nx2 (B, 16, 3) with neighbours bi2 (B, 16, ns) -> (feat2, bound, share of the packed-max term in it)."""
    dxyz = _gather(nx1.double(), bi2) - nx2.double()[:, :, None, :]
    f = _gather(feat1.double(), bi2)
    x = torch.cat([dxyz, f], -1)                                # reference channel order [xyz | feat]
    ex = torch.cat([(UB + UF) * dxyz.abs(), torch.zeros_like(f)], -1)     # sa_mlp.cu:195 (feat1 as stored), :201-202
    if knock == "sa2_unpermuted":                               # weights packed in the reference order, operand [feat | xyz]
        x = torch.cat([f, dxyz], -1)
    pre, acc, e_acc, L = _mlp(x, ex, net, 1, K_SA2, knock, calib)
    if knock == "max_ns_minus_1" and pre.shape[2] > 1:
        pre, acc, e_acc = pre[:, :, :-1], acc[:, :, :-1], e_acc[:, :, :-1]
    return _max_rows(pre, acc, e_acc, L, 2, packed=True)


def head_reference(net, nx2, feat2, xs=None, knock=None, calib=None):
    """SA3 (GroupAll over the 16 SA2 centres nx2 with features feat2 (B, 16, 256), the kernel's bf16 feat2: an exact
    operand; xyz not centred) and fc, one GEMM at a time: each layer reads xs = the kernel's bf16 outputs (x1 (B, 16, 256),
    x2 (B, 16, 512), g (B, 768)) of the layer below, or, without them (calibration), the float64 values.  Returns
    {sa3_1, sa3_2, sa3_max, out: (value, bound)}."""
    xyz = nx2.double()
    if knock == "sa3_centred":
        xyz = xyz - xyz.mean(1, keepdim=True)
    f2 = feat2.double()
    x = torch.cat([xyz, f2], -1)
    ex = torch.cat([UB * nx2.double().abs(), torch.zeros_like(f2)], -1)   # forward_fused: nx2.to(bf16)
    res = {}
    for j in (0, 1):
        pre, _, e_acc, L = _conv_bn(x, ex, net, 2, j, K_SA3[j], knock, calib)
        res[f"sa3_{j + 1}"] = _relu_store(pre, e_acc, L)
        x, ex = (xs[j].double(), torch.zeros_like(pre)) if xs is not None else res[f"sa3_{j + 1}"]
    pre, acc, e_acc, L = _conv_bn(x, ex, net, 2, 2, K_SA3[2], knock, calib)
    if knock == "rowmax_off_by_one":                            # groups of rows [16 b + 1, 16 b + 17)
        B = pre.shape[0]
        pre, acc, e_acc = (t.reshape(B * 16, -1).roll(-1, 0).reshape(B, 16, -1) for t in (pre, acc, e_acc))
    g, eg, _ = _max_rows(pre, acc, e_acc, L, 1, packed=False)
    res["sa3_max"] = (g, eg)
    if xs is not None:
        g, eg = xs[2].double(), torch.zeros_like(g)
    Wfc, bfc = net.fc.weight.detach().double(), net.fc.bias.detach().double()
    out = g @ Wfc.t() + bfc
    # bf16 fc weight, K = 768 tensor-core sum, fp32 bias add, fp32 output (gemm.cu:394-396, :456)
    aW = Wfc.abs().t()
    res["out"] = (out, eg @ aW + (UB + K_FC * TC) * (g.abs() @ aW) + UF * out.abs())
    return res


OUTPUTS = ("feat1", "feat2", "sa3_1", "sa3_2", "sa3_max", "out")


def encoder_reference(net, pts, inter, knock=None, chunk=CHUNK, calib=None):
    """float64 outputs of every kernel of PointNetPP.forward_fused (OUTPUTS) with their bounds, computed `chunk` clouds at a
    time.  Each kernel reads the kernels' output of the level below (inter["feat1"], inter["feat2"], inter["head"]), so
    each comparison tests one kernel and the bounds do not compound over ten layers; without them (calibration) the levels
    chain in float64."""
    res = {k: ([], []) for k in OUTPUTS}
    pk = []
    for a in range(0, pts.shape[0], chunk):
        z = a + chunk
        nx1, nx2 = inter["new_xyz"][a:z], inter["new_xyz2"][a:z]
        f1, e1, _ = sa1_reference(net, pts[a:z], nx1, inter["ball_idx"][a:z], knock, calib)
        f2, e2, p2 = sa2_reference(net, nx1, inter["feat1"][a:z] if "feat1" in inter else f1, nx2, inter["ball_idx2"][a:z],
                                   knock, calib)
        head = head_reference(net, nx2, inter["feat2"][a:z] if "feat2" in inter else f2,
                              [t[a:z] for t in inter["head"]] if "head" in inter else None, knock, calib)
        for k, v in (("feat1", (f1, e1)), ("feat2", (f2, e2)), *head.items()):
            res[k][0].append(v[0])
            res[k][1].append(TOL * v[1])
        pk.append(p2.amax())
    res = {k: (torch.cat(v), torch.cat(e)) for k, (v, e) in res.items()}
    res["packed_share"] = float(torch.stack(pk).max())
    return res


def ratio(got, ref_err):
    """Largest |got - ref| / bound: 0 where they agree exactly, inf where got is NaN or infinite."""
    ref, err = ref_err
    d = (got.double() - ref).abs()
    return float(torch.where(d == 0, torch.zeros_like(d), d / err).nan_to_num(nan=math.inf, posinf=math.inf).max())




def test_ratio_fails_on_nan_and_inf():
    """A kernel output that is NaN or infinite breaks every bound; exact agreement under a zero bound does not."""
    ref = (torch.zeros(3, dtype=torch.float64), torch.tensor([1.0, 1.0, 0.0], dtype=torch.float64))
    assert ratio(torch.tensor([math.nan, 0.1, 0.0]), ref) == math.inf
    assert ratio(torch.tensor([0.1, -math.inf, 0.0]), ref) == math.inf
    assert ratio(torch.tensor([0.1, 0.5, 0.0]), ref) == 0.5


# ---- the two encoders under test -----------------------------------------------------------------------------------------
KINDS = ("edges", "conditioned")


def _edges_calib(net):
    """BatchNorm statistics from the conv outputs, with channels moved to the edges by their index: running means 3 or 6
    standard deviations off (channels mostly dead or always on, and the shift cancelling most of the accumulator, where the
    SA2 packed-max term dominates); near-constant channels, whose conv weight row is scaled so that their running variance
    is 1e-5, as large as eps (a folded scale of ~200); negative gamma (a negative scale folded into W while the max is taken
    on raw accumulators)."""
    def calib(lvl, j, y):
        layer = getattr(net.encoder[lvl].mlps[0], f"layer{j}")
        bn = layer.bn.bn
        y = y.reshape(-1, y.shape[-1])
        mu, sd = y.mean(0), y.std(0)
        c = torch.arange(y.shape[-1], device=y.device)
        tiny = c % 16 == 2
        f = torch.where(tiny, 1e-5 ** 0.5 / sd, 1.0)
        layer.conv.weight.mul_(f.to(layer.conv.weight)[:, None, None, None])
        y.mul_(f)                                           # the conv output under the scaled weight, in place
        mu, sd = mu * f, sd * f
        # periods 13 and 5 do not divide the 128-column halves of SA2, so the two halves' shifts differ
        k = torch.tensor([0, 3, 0, 0, -3, 0, 0, 6, 0, 0, -6, 0, 0], dtype=y.dtype, device=y.device)[c % 13]
        bn.running_mean.copy_(mu + k * sd)
        bn.running_var.copy_(sd * sd)
        bn.weight.copy_(torch.where(c % 5 == 3, -bn.weight.abs(), bn.weight.abs()))
    return calib


def _conditioned_calib(net):
    """BatchNorm statistics of a well-conditioned encoder: running means a quarter of the batch mean and gamma > 0, so that
    with nonnegative weights |W| |x| stays close to |W x| at every layer and the bound a few per cent of the values; the
    same near-constant channels as _edges_calib; two dominant SA1 output channels, so that SA2 weights applied to the
    wrong columns show."""
    def calib(lvl, j, y):
        layer = getattr(net.encoder[lvl].mlps[0], f"layer{j}")
        bn = layer.bn.bn
        y = y.reshape(-1, y.shape[-1])
        mu, sd = y.mean(0), y.std(0)
        tiny = torch.arange(y.shape[-1], device=y.device) % 16 == 2
        f = torch.where(tiny, 1e-5 ** 0.5 / sd, 1.0)
        layer.conv.weight.mul_(f.to(layer.conv.weight)[:, None, None, None])
        y.mul_(f)
        bn.running_mean.copy_(torch.where(tiny, mu * f, 0.25 * mu))
        bn.running_var.copy_(torch.where(tiny, sd * f, mu) ** 2)
        bn.weight.abs_()
        if (lvl, j) == (0, 2):
            bn.weight[[0, 64]] *= 20
    return calib


def prepare(net, kind, pts, inter):
    """Turn the synthetic-weight encoder `net` into one of KINDS and calibrate its BatchNorm statistics on the clouds `pts`
    with the sampled centres / neighbours of `inter`; the levels chain in float64 (kernel outputs in `inter` are ignored).
    edges: the synthetic weights, statistics at the edges (_edges_calib).  conditioned: nonnegative conv / fc weights, z
    weighing 5 x more than r at SA1 and xyz 5 x more than the features at SA2 (column mix-ups show), and
    _conditioned_calib."""
    inter = {k: inter[k] for k in ("new_xyz", "ball_idx", "new_xyz2", "ball_idx2")}
    with torch.no_grad():
        if kind == "conditioned":
            for p_ in net.parameters():
                if p_.dim() > 1:
                    p_.abs_()
            net.encoder[0].mlps[0].layer0.conv.weight[:, 2] *= 5
            net.encoder[1].mlps[0].layer0.conv.weight[:, :3] *= 5
        calib = _edges_calib(net) if kind == "edges" else _conditioned_calib(net)
        encoder_reference(net, pts, inter, chunk=pts.shape[0], calib=calib)
    return net


# ---- CPU: the bound catches every plausible slip ------------------------------------------------------------------------
KNOCK_CLOUDS = 8
def _knock_inputs(B=KNOCK_CLOUDS):
    """B clouds of 64 points far from the origin, so that centring matters at SA1 and GroupAll's missing centring at
    SA3, growing brighter from cloud to cloud, so that a row-group max one row off takes the next cloud's larger first row.
    Each cloud has a bright point (rgb 6) and a dark one (rgb 0) that only the LAST ball-query sample of alternate SA1
    centres reaches (the one stands out where the weights add colour, the other where they subtract it), and SA1 point 31
    is only the last sample of every SA2 centre."""
    gen = torch.Generator().manual_seed(0)
    P = 64
    off = 5 + 15 * torch.rand(B, 3, generator=gen)
    xyz = 0.3 * torch.randn(B, P, 3, generator=gen) + off[:, None]
    rgb = torch.rand(B, P, 3, generator=gen) * torch.linspace(1.0, 3.0, B)[:, None, None]
    rgb[:, -1], rgb[:, -2] = 6.0, 0.0
    bi1 = torch.randint(0, P - 2, (B, 32, 32), generator=gen, dtype=torch.int32)
    bi1[..., -1] = P - 1 - torch.arange(32, dtype=torch.int32) % 2
    bi2 = torch.randint(0, 31, (B, 16, 32), generator=gen, dtype=torch.int32)
    bi2[..., -1] = 31
    nx1 = xyz[:, :32].contiguous()
    return torch.cat([xyz, rgb], -1), dict(new_xyz=nx1, ball_idx=bi1, new_xyz2=nx1[:, :16].contiguous(), ball_idx2=bi2)


def test_knockouts_break_the_bound():
    """Every slip in KNOCKS, applied to the float64 reference, moves some kernel output by >= 4 x its bound on at least one
    of the two encoders the GPU tests run, so the GPU tests catch each of them.  On the edges encoder the fused SA levels'
    bounds cover three layers of random-sign weights and extreme statistics and are loose by construction; the
    conditioned encoder is there so that the subtler slips still show."""
    got = {}
    for kind in KINDS:
        pts, inter = _knock_inputs()
        net = prepare(make_pn(0).eval(), kind, pts, inter)
        with torch.no_grad():
            ref = encoder_reference(net, pts, inter)
            # the kernels' bf16 outputs, as the kernel of the level above reads them, emulated from the unknocked reference
            bf = {k: ref[k][0].bfloat16() for k in OUTPUTS}
            inter.update(feat1=bf["feat1"], feat2=bf["feat2"], head=(bf["sa3_1"], bf["sa3_2"], bf["sa3_max"]))
            ref = encoder_reference(net, pts, inter)
            for k in KNOCKS:
                kr = encoder_reference(net, pts, inter, knock=k)
                got[k, kind] = max(ratio(kr[o][0], ref[o]) for o in OUTPUTS)
        print(f"PN FP64 knock-out error / bound ({kind})", {k: round(got[k, kind], 1) for k in KNOCKS})
    caught = {k: max(got[k, kind] for kind in KINDS) for k in KNOCKS}
    assert min(caught.values()) >= 4, caught


# ---- GPU: the frozen encoder --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=KINDS)
def net(request):
    """The GPS encoder with synthetic weights, prepared as `kind` on 64 clouds."""
    dev = torch.device("cuda", 0)
    n = make_pn(0).to(dev).eval().requires_grad_(False)
    pts = torch.from_numpy(synthetic.object_batch(5, 64, 1024, pad_fraction=0.1)).to(dev)
    _, inter = n.forward_fused(pts, return_intermediates=True)
    return prepare(n, request.param, pts, inter)


def head_kernels(net, feat2, nx2):
    """SA3 and fc as forward_fused runs them (four GEMMs on the packed weights), keeping every GEMM's output."""
    from sceneverse_b200 import native
    B = feat2.shape[0]
    (w1, s1), (w2, s2), (w3, s3) = net._pack()["sa3"]
    x = torch.zeros((B * 16, 272), dtype=torch.bfloat16, device=feat2.device)
    x[:, :256] = feat2.reshape(B * 16, 256)
    x[:, 256:259] = nx2.reshape(B * 16, 3).to(torch.bfloat16)
    x1 = native.gemm(x, w1, s1, "relu")
    x2 = native.gemm(x1, w2, s2, "relu")
    g = native.gemm(x2, w3, s3, "relu", rowmax=16)
    out = native.gemm(g, *net._pack()["fc"], out_dtype=torch.float32)
    return (x1.view(B, 16, -1), x2.view(B, 16, -1), g), out


MODULE_CASES = [(1, 32, 0.0), (1, 1024, 0.0), (4, 1024, 0.0), (37, 32, 0.5), (37, 1024, 0.5), (5120, 1024, 0.1)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,P,pad", MODULE_CASES, ids=[f"B{b}-P{p}-pad{f}" for b, p, f in MODULE_CASES])
def test_frozen_encoder_against_float64(net, B, P, pad):
    """B = 1: one partial super-tile per level; B = 4: exactly 128 SA1 centres; B = 5,120: 1,280 SA1 super-tiles over at most
    132 CTAs.  pad > 0: all-ones clouds, whose ball indices repeat and whose maxima tie.  SA3 and fc are checked GEMM by
    GEMM; their chain reproduces forward_fused's output bit for bit."""
    pts = torch.from_numpy(synthetic.object_batch(B + P, B, P, pad_fraction=pad)).cuda()
    out, inter = net.forward_fused(pts, return_intermediates=True)
    head, out_chain = head_kernels(net, inter["feat2"], inter["new_xyz2"])
    assert torch.equal(out_chain, out)
    inter["head"] = head
    with torch.no_grad():
        ref = encoder_reference(net, pts, inter)
    got = dict(feat1=inter["feat1"], feat2=inter["feat2"], sa3_1=head[0], sa3_2=head[1], sa3_max=head[2], out=out)
    worst = {k: ratio(got[k], ref[k]) for k in OUTPUTS}
    print(f"PN FP64 worst error / bound B={B} P={P} pad={pad}", {k: round(v, 4) for k, v in worst.items()},
          "largest share of the SA2 packed-max term in a feat2 bound", round(ref["packed_share"], 3))
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.gpu
@pytest.mark.parametrize("ns", [1, 17])
def test_sa_entry_points_at_other_nsample(net, ns):
    """sv_sa1_mlp_bf16 / sv_sa2_mlp_bf16 with hand-built centres and ball indices at an nsample the module never uses."""
    dev = torch.device("cuda", 0)
    B, P = 37, 1024
    gen = torch.Generator(device=dev).manual_seed(ns)
    pts = torch.from_numpy(synthetic.object_batch(ns, B, P, pad_fraction=0.25)).to(dev)
    nx1 = _gather(pts[..., :3], torch.randint(0, P, (B, 32, 1), device=dev, generator=gen))[:, :, 0].contiguous()
    bi1 = torch.randint(0, P, (B, 32, ns), device=dev, generator=gen, dtype=torch.int32)
    nx2 = nx1[:, 16:].contiguous()
    bi2 = torch.randint(0, 32, (B, 16, ns), device=dev, generator=gen, dtype=torch.int32)
    pk = net._pack()
    lib = _lib.gps()
    feat1 = torch.empty((B, 32, 128), dtype=torch.bfloat16, device=dev)
    _lib.call(lib, "sv_sa1_mlp_bf16", dev, pts.data_ptr(), nx1.data_ptr(), bi1.data_ptr(), pk["sa1"].data_ptr(), B, P, ns,
              feat1.data_ptr())
    feat2 = torch.empty((B, 16, 256), dtype=torch.bfloat16, device=dev)
    _lib.call(lib, "sv_sa2_mlp_bf16", dev, nx1.data_ptr(), feat1.data_ptr(), nx2.data_ptr(), bi2.data_ptr(),
              pk["sa2"].data_ptr(), B, 32, ns, feat2.data_ptr())
    with torch.no_grad():
        f1, e1, _ = sa1_reference(net, pts, nx1, bi1)
        f2, e2, _ = sa2_reference(net, nx1, feat1, nx2, bi2)
    worst = {"feat1": ratio(feat1, (f1, TOL * e1)), "feat2": ratio(feat2, (f2, TOL * e2))}
    print(f"PN FP64 worst error / bound nsample={ns}", {k: round(v, 4) for k, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst


# ---- GPU: the train-mode layers at the step's row counts ----------------------------------------------------------------
def bn_train_reference(y, dout, mask, g, b, eps, m_f, m_b):
    """The per-column part of tests/test_syncbn_gpu.py::reference() for one rank holding all R rows of y (R, c) bf16: float64
    mean, rstd, unbiased variance, output, dY, d gamma and d beta with their bounds, m_f / m_b the longest fp32 addition
    chain of the forward / backward column sums (col_sums_kernel<0> over up to 128 slabs, col_sums_kernel<1> over 127)."""
    d = torch.float64
    y, g, b = y.to(d), g.to(d), b.to(d)
    N = y.shape[0]
    mean = y.mean(0)
    var = (y * y).mean(0) - mean * mean
    rstd = (var + eps).rsqrt()
    e_s0, e_s1 = gamma_n(m_f) * y.abs().sum(0), gamma_n(m_f + 1) * (y * y).sum(0)
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
    gg = dout.to(d) * mask
    Sb, Sg = gg.sum(0), (gg * xh).sum(0)
    e_Sb = gamma_n(m_b) * gg.abs().sum(0) + U32 * Sb.abs()
    e_Sg = (gg.abs() * e_xh).sum(0) + gamma_n(m_b + 1) * (gg * xh).abs().sum(0) + U32 * Sg.abs()
    inner = gg - Sb / N - xh * Sg / N
    e_inner = (e_Sb + 2 * U32 * Sb.abs()) / N + (e_xh * Sg.abs() + xh.abs() * (e_Sg + 2 * U32 * Sg.abs())) / N \
        + 4 * U32 * (gg.abs() + Sb.abs() / N + (xh * Sg).abs() / N)
    dy = g * rstd * inner
    e_dy = g.abs() * (e_rstd * inner.abs() + (rstd + e_rstd) * e_inner) + 3 * U32 * dy.abs()
    e_dy = e_dy + UBF * (dy.abs() + e_dy)
    return dict(mean=(mean, e_mean), rstd=(rstd, e_rstd), var_u=(var_u, e_var_u), out=(out, e_out), dy=(dy, e_dy),
                dgamma=(Sg, e_Sg), dbeta=(Sb, e_Sb))


BN_CASES = [(100_003, 64), (81_920, 512), (81_920, 768), (5_242_880, 64), (5_242_880, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("R,C", BN_CASES, ids=[f"R{r}-C{c}" for r, c in BN_CASES])
def test_train_bn_relu_at_step_rows(R, C):
    """sv_pn_bn_relu_fwd / _bwd at the step's row counts (SA1: 5,242,880 rows at C = 64 / 128; SA3: 81,920 at 512 / 768) and
    at R = 100,003 (128 capped slabs, a ragged last one).  Columns 8..15 sit ~10 standard deviations off zero, where the
    one-pass variance E[y^2] - mean^2 loses the most.  dX is the dgrad GEMM's, tested with the GEMMs."""
    dev = torch.device("cuda", 0)
    eps = 1e-5
    gen = torch.Generator(device=dev).manual_seed(C)
    sd = 0.5 + 1.5 * torch.rand(C, device=dev, generator=gen)
    mu = (2 * torch.rand(C, device=dev, generator=gen) - 1) * sd
    mu[8:16] = 10 * sd[8:16]
    slabs = min(-(-R // 256), 128)
    last = (slabs - 1) * -(-R // slabs)             # first row of the forward's last slab
    y = torch.empty((R, C), dtype=torch.bfloat16, device=dev)
    dout = torch.empty_like(y)
    for c0 in range(0, C, 16):
        blk = torch.randn(R, 16, device=dev, generator=gen) * sd[c0:c0 + 16] + mu[c0:c0 + 16]
        blk[last:] += 2 * sd[c0:c0 + 16]            # a distinct offset on the rows of the last slab
        y[:, c0:c0 + 16] = blk
        dout[:, c0:c0 + 16] = torch.randn(R, 16, device=dev, generator=gen)
        del blk
    g32 = 1 + 0.3 * torch.randn(C, device=dev, generator=gen)
    g32[3::4] *= -1
    b32 = 0.2 * torch.randn(C, device=dev, generator=gen)

    lib = _lib.gps()
    stats = torch.empty((3, C), dtype=torch.float32, device=dev)
    out, dy = torch.empty_like(y), torch.empty_like(y)
    dgb = torch.empty((2, C), dtype=torch.float32, device=dev)
    scratch = torch.empty(lib.sv_pn_scratch_floats(C), dtype=torch.float32, device=dev)
    _lib.call(lib, "sv_pn_bn_relu_fwd", dev, y.data_ptr(), R, C, g32.data_ptr(), b32.data_ptr(), eps, stats[0].data_ptr(),
              stats[1].data_ptr(), stats[2].data_ptr(), out.data_ptr(), scratch.data_ptr())
    _lib.call(lib, "sv_pn_bn_relu_bwd", dev, y.data_ptr(), dout.data_ptr(), R, C, g32.data_ptr(), b32.data_ptr(),
              stats[0].data_ptr(), stats[1].data_ptr(), dy.data_ptr(), dgb[0].data_ptr(), dgb[1].data_ptr(), 0,
              scratch.data_ptr())

    m_f, m_b = chain(R, 128), chain(R, 127)
    w = min(C, 1 << ((2 ** 23 // R).bit_length() - 1))     # columns per float64 block: <= 8 M elements per tensor
    keys = ("mean", "rstd", "var_u", "out", "dy", "dgamma", "dbeta")
    worst, knock = dict.fromkeys(keys, 0.0), 0.0
    for c0 in range(0, C, w):
        sl = slice(c0, c0 + w)
        ref = bn_train_reference(y[:, sl], dout[:, sl], out[:, sl] > 0, g32[sl], b32[sl], eps, m_f, m_b)
        got = dict(mean=stats[0, sl], rstd=stats[1, sl], var_u=stats[2, sl], out=out[:, sl], dy=dy[:, sl],
                   dgamma=dgb[0, sl], dbeta=dgb[1, sl])
        for k in keys:
            worst[k] = max(worst[k], ratio(got[k], ref[k]))
        # knock-out in float64: the forward's column sums without the last slab's rows
        knock = max(knock, ratio(y[:last, sl].double().mean(0), ref["mean"]))
        del ref, got
    print(f"PN TRAIN-BN worst error / bound R={R} C={C}", {k: round(v, 4) for k, v in worst.items()},
          "knock-out (last slab dropped)", round(knock, 1))
    assert max(worst.values()) <= 1.0, worst
    assert knock >= 4, knock


@pytest.mark.gpu
def test_group_rows_groupall_bitwise_at_sa3_shape():
    """sv_pn_group_rows as SA3 calls it (GroupAll: centre and idx NULL, bf16 features) over 5,120 clouds: raw xyz rounded
    to bf16, the features copied, the padding columns 259..263 zero."""
    from sceneverse_b200.pn_train import _GroupRowsFn
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(3)
    B = 5120
    xyz = 2 * torch.randn(B, 16, 3, device=dev, generator=gen)
    feat = torch.randn(B, 16, 256, device=dev, generator=gen).bfloat16()
    X = _GroupRowsFn.apply(xyz, None, feat, None, 1, 16)
    want = torch.zeros((B * 16, 264), dtype=torch.bfloat16, device=dev)
    want[:, :3] = xyz.reshape(-1, 3).bfloat16()
    want[:, 3:259] = feat.reshape(-1, 256)
    assert torch.equal(X.view(torch.int16), want.view(torch.int16))


ROWMAX_CASES = [(5120, 16, 768), (5120 * 16, 32, 256), (5120 * 32, 32, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("G,ns,C", ROWMAX_CASES, ids=["sa3", "sa2", "sa1"])
def test_rowgroup_max_and_gradient_bitwise_at_step_shapes(G, ns, C):
    """sv_pn_rowgroup_max (max and FIRST maximal sample) and its gradient at the step's shapes, on values in quarter steps
    so that ties at the maximum are common."""
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(ns + C)
    x = torch.empty((G * ns, C), dtype=torch.bfloat16, device=dev)
    step = max(1, 2 ** 24 // C)
    for a in range(0, G * ns, step):
        # + 0.0 turns -0.0 into +0.0: a group whose maximum is a tie of -0.0 and +0.0 has no bitwise-defined max
        x[a:a + step] = (4 * torch.randn(min(step, G * ns - a), C, device=dev, generator=gen)).round() / 4 + 0.0
    g = torch.randn(G, C, device=dev, generator=gen).bfloat16()
    lib = _lib.gps()
    out = torch.empty((G, C), dtype=torch.bfloat16, device=dev)
    arg = torch.empty((G, C), dtype=torch.uint8, device=dev)
    gx = torch.empty_like(x)
    _lib.call(lib, "sv_pn_rowgroup_max", dev, x.data_ptr(), G, ns, C, out.data_ptr(), arg.data_ptr())
    _lib.call(lib, "sv_pn_rowgroup_max_grad", dev, g.data_ptr(), arg.data_ptr(), G, ns, C, gx.data_ptr())
    s = torch.arange(ns, device=dev, dtype=torch.int32)[None, :, None]
    ties = 0
    gs = max(1, step // ns)
    for a in range(0, G, gs):
        z = min(G, a + gs)
        xv = x[a * ns:z * ns].view(-1, ns, C)
        m = xv.amax(1)
        hit = xv == m[:, None]
        first = torch.where(hit, s, ns).amin(1)
        ties += int((hit.sum(1) > 1).sum())
        assert torch.equal(out[a:z].view(torch.int16), m.view(torch.int16)), a
        assert torch.equal(arg[a:z].int(), first), a
        want = torch.where(s == first[:, None], g[a:z, None], torch.zeros((), dtype=g.dtype, device=dev))
        assert torch.equal(gx[a * ns:z * ns].view(torch.int16), want.reshape(-1, C).view(torch.int16)), a
    assert ties > 0
