"""Fused attention forward and backward (csrc/attention.cu, csrc/attention_bwd.cu) against float64, element by element.

* A float64 reference of the forward (plain masked softmax, the spatial gate log(clamp(sigmoid(z), 1e-6)) of
  ops._spatial_attention_torch, attention-weight dropout) and its backward, written out so that every intermediate the
  bound needs is at hand.  A CPU test checks it against torch autograd of ops._spatial_attention_torch and of the plain
  masked softmax.
* A bound on |kernel - float64| for every element of out, lse, dvec (D = rowsum(dO o O)), dq, dk, dv and the gate-weight
  gradient, derived from the arithmetic the kernels perform: first order in the unit roundoffs, each term next to the
  kernel line it comes from.  The factor 1.01 in within() covers the second-order terms.
* GPU cases: plain, gated and dropout attention at the tail shapes of the 64-row units and the 16-column last key block,
  strided operands, a gate shared across heads, and the contract edges (masked keys, a scene with every key masked, scene
  independence, argument validation).
* A CPU knock-out test: each plausible kernel slip, applied to the float64 reference, moves some output element by at
  least 4 x the bound, so the bound is tight enough to catch it.
"""
import math
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sceneverse_b200 import ops
from tests.test_attention_gpu import _dropout_keep

UB = 2.0 ** -8              # unit roundoff of bf16 (8 significand bits, round to nearest)
UF = 2.0 ** -24             # unit roundoff of fp32
TC = 2 * UF                 # per addition of the tensor core's fp32 accumulation (not specified as round to nearest:
                            # 2u also covers a truncating accumulator)
EX2 = 2.0 ** -22            # ex2.approx.ftz.f32: 2 ulp relative error
LG2 = 2.0 ** -22            # lg2.approx.ftz.f32: 2^-22 absolute in [0.5, 2], 2 ulp relative elsewhere
LOG2E, LN2 = 1.0 / math.log(2.0), math.log(2.0)
SCALE = 0.125               # 1 / sqrt(64), exact
C2 = SCALE * LOG2E          # the kernels' logit scale in the log2 domain
CLAMP = 1e-6
LOG2_CLAMP = math.log2(CLAMP)
P_DROP, SEED = 0.1, 123456789
INV_KEEP = 1.0 / (1.0 - float(np.float32(P_DROP)))   # the kernels receive dropout_p as fp32


# ---- float64 reference ------------------------------------------------------------------------------------------------
def _heads(x, H):
    """(B, L, H * 64) -> float64 (B, H, L, 64)."""
    B, L, _ = x.shape
    return x.double().reshape(B, L, H, 64).transpose(1, 2)


def _flat(x):
    B, H, L, _ = x.shape
    return x.transpose(1, 2).reshape(B, L, H * 64)


KNOCKS = ("drop_last_key", "drop_block_key", "first_masked_live", "drop_last_query", "drop_query_64", "gate_next_head",
          "no_clamp", "grad_through_clamp", "next_row_D", "no_rescale")


def reference(x, knock=None):
    """float64 forward and backward of the attention of inputs `x` (see inputs()), in the (B, H, Lq, Lk) layout.

    A query row without a live key gets P = 0, out = 0 and lse = +inf: the kernels' contract (attention.cu:131, :197).
    `knock` applies one kernel slip:
      drop_last_key        key Lk - 1 is treated as masked
      drop_block_key       key 64 (nblk - 1), the first of the last 64-key block, is treated as masked
      first_masked_live    the first masked key of each scene is live
      drop_last_query      query row Lq - 1 is left out of the dk / dv sums
      drop_query_64        query row 64 is left out of the dk / dv sums
      gate_next_head       head h reads the gate weights of head h + 1
      no_clamp             log(sigmoid(z)) without the clamp at 1e-6
      grad_through_clamp   the gate-weight gradient also flows through the clamped pairs
      next_row_D           dS of row i uses D of row i + 1
      no_rescale           kept attention weights are not scaled by 1 / (1 - p)"""
    B, Lq, _ = x.q.shape
    Lk, H = x.k.shape[1], x.H
    qh, kh, vh, gh = (_heads(t, H) for t in (x.q, x.k, x.v, x.go))
    live = ~x.mask.clone()
    if knock == "drop_last_key":
        live[:, Lk - 1] = False
    elif knock == "drop_block_key":
        live[:, 64 * ((Lk - 1) // 64)] = False
    elif knock == "first_masked_live":
        for b in range(B):
            idx = torch.nonzero(x.mask[b])
            if len(idx):
                live[b, idx[0, 0]] = True
    s = qh @ kh.transpose(-1, -2)
    logit = s * SCALE
    r = types.SimpleNamespace(s=s, live=live, sig=None, lg=None, z=None, unclamped=None)
    if x.sw is not None:
        SH = x.sw.shape[-1] // 6
        w = x.sw.double().reshape(B, Lq, SH, 6).transpose(1, 2)                       # (B, SH, Lq, 6)
        if knock == "gate_next_head":
            w = w.roll(-1, dims=1)
        z = w[..., :1] + torch.einsum("bhik,bijk->bhij", w[..., 1:], x.locs.double())
        r.z = z.expand(B, H, Lq, Lk)
        r.sig = torch.sigmoid(r.z)
        r.lg = F.logsigmoid(r.z) if knock == "no_clamp" else torch.log(r.sig.clamp_min(CLAMP))
        r.unclamped = torch.ones_like(r.sig, dtype=torch.bool) if knock in ("no_clamp", "grad_through_clamp") \
            else r.sig > CLAMP
        logit = logit + r.lg
    logit = logit.masked_fill(~live[:, None, None, :], -math.inf)
    mx = logit.amax(-1, keepdim=True)
    rowlive = torch.isfinite(mx)
    mx = torch.where(rowlive, mx, torch.zeros_like(mx))
    e = torch.exp(logit - mx)
    tot = e.sum(-1, keepdim=True)
    r.P = torch.where(rowlive, e / tot.clamp_min(1e-300), torch.zeros_like(e))
    r.lse = torch.where(rowlive, mx + torch.log(tot.clamp_min(1e-300)), torch.full_like(mx, math.inf)).squeeze(-1)
    r.M = 1.0
    if x.keep is not None:
        r.M = x.keep.double() * (1.0 if knock == "no_rescale" else INV_KEEP)
    r.Pd = r.P * r.M
    r.O = r.Pd @ vh
    r.dP = (gh @ vh.transpose(-1, -2)) * r.M
    r.D = (gh * r.O).sum(-1)
    D = r.D.roll(-1, dims=-1) if knock == "next_row_D" else r.D
    r.dS = r.P * (r.dP - D[..., None])                 # gradient of the natural-log logits
    dSk, Pdk = r.dS, r.Pd
    if knock in ("drop_last_query", "drop_query_64"):
        row = Lq - 1 if knock == "drop_last_query" else 64
        dSk, Pdk = r.dS.clone(), r.Pd.clone()
        dSk[:, :, row] = 0
        Pdk[:, :, row] = 0
    r.dq = SCALE * r.dS @ kh
    r.dk = SCALE * dSk.transpose(-1, -2) @ qh
    r.dv = Pdk.transpose(-1, -2) @ gh
    out = dict(out=_flat(r.O), lse=r.lse, dq=_flat(r.dq), dk=_flat(r.dk), dv=_flat(r.dv))
    if x.sw is not None:
        r.dz = r.dS * (1 - r.sig) * r.unclamped          # d log(sigmoid(z)) / dz = 1 - sigmoid(z), 0 under the clamp
        g = torch.einsum("bhij,bijk->bhik", r.dz, _loc_terms(x.locs.double()))       # (B, H, Lq, 6)
        if SH == 1:
            g = g.sum(1, keepdim=True)
        out["dsw"] = g.transpose(1, 2).reshape(B, Lq, SH * 6)
    r.outputs = out
    return r


def _loc_terms(locs):
    """(B, Lq, Lk, 6): the factor of each gate weight in z = bias + w . loc."""
    return torch.cat([torch.ones_like(locs[..., :1]), locs], -1)


# ---- error bound ------------------------------------------------------------------------------------------------------
def bounds(x, r):
    """Elementwise bounds of |kernel - float64 reference| for the reference `r` of inputs `x`.  Every term is first order in
    UB / UF and is computed from absolute values with float64 matmuls; p_ij below is the normalised probability."""
    B, Lq, _ = x.q.shape
    Lk, H = x.k.shape[1], x.H
    aq, ak, av, ag = (_heads(t, H).abs() for t in (x.q, x.k, x.v, x.go))
    livep = r.live[:, None, None, :]
    drop = x.keep is not None
    P, Pd, aO = r.P, r.Pd, r.O.abs()

    # -- forward (attention.cu) --
    # S = Q K^T: 64 bf16 products (exact in fp32) summed by the tensor core in fp32 (mma_kk, line 103)
    eS = 64 * TC * (aq @ ak.transpose(-1, -2))
    s2 = r.s * C2
    m2 = s2.masked_fill(~livep, -math.inf).amax(-1, keepdim=True)                    # pass 1 row maximum (line 120)
    m2 = torch.where(torch.isfinite(m2), m2, torch.zeros_like(m2))
    # x = fmaf(s, c2, kb) - m2 (line 154): c2 = scale * LOG2E rounded to fp32, the fma and the subtraction round once each
    dx = C2 * eS + 2 * UF * s2.abs() + UF * (s2 - m2).abs()
    g2 = 0.0
    dg = amb = None
    if x.sw is not None:
        SH = x.sw.shape[-1] // 6
        g2 = r.lg * LOG2E
        aw = x.sw.double().abs().reshape(B, Lq, SH, 6).transpose(1, 2)
        zabs = LOG2E * (aw[..., :1] + torch.einsum("bhik,bijk->bhij", aw[..., 1:], x.locs.double().abs()))
        g2raw = F.logsigmoid(r.z) * LOG2E
        # GateW (attn_common.cuh:76-82): the weights -LOG2E * w round twice (fp32 LOG2E, the product) and the chain
        # of five fmas once per step: 7u of |bias| + sum |w l| in the log2 domain.  d(-log2(1 + t)) / da = -(1 - sigmoid):
        # that error and ex2's scale by 1 - sigmoid; 1 + t rounds once (u / ln 2 after lg2), lg2 adds its own error
        g_un = (1 - r.sig) * (7 * UF * zabs + EX2 / LN2) + UF / LN2 + LG2 * g2raw.abs().clamp_min(1.0)
        g_cl = UF * abs(LOG2_CLAMP)                                                     # LOG2_CLAMP as an fp32 constant
        # pairs whose exact gate lies within the error of the clamp: the kernel's `gli > LOG2_CLAMP` may go either way
        amb = (g2raw - LOG2_CLAMP).abs() <= g_un + g_cl
        dg = torch.where(amb, torch.maximum(g_un, torch.full_like(g_un, g_cl)),
                         torch.where(r.unclamped, g_un, torch.full_like(g_un, g_cl)))
        dx = dx + UF * (s2 + g2 - m2).abs() + dg                                        # x0 += log2gate (line 158)
    lx = (s2 + g2 - m2).masked_fill(~livep, 0.0)
    assert float(lx.min()) > -100, "an exponent below -126 would be flushed to zero by ex2.approx.ftz"
    rho = LN2 * dx + EX2                                                                # p = ex2(x), relative (line 165)
    # sum[r] += p0 + p1 and the two shuffles: at most Lk roundings of the row sum, relative to it (line 166, 188)
    dtot = (P * rho).sum(-1, keepdim=True) + Lk * UF
    # p * inv_keep (inv_keep = 1 / (1 - p): two fp32 roundings) then bf16 P (line 169, 173)
    pr = UB + (3 * UF if drop else 0.0)
    # O += P V over Lk keys (tensor core, line 181); o * (1 / tot): two roundings, bf16 store (line 195, 201)
    e_out = (Pd * (rho + pr)) @ av + Lk * TC * (Pd @ av) + aO * (dtot + 2 * UF + UB)
    lse = torch.where(torch.isfinite(r.lse), r.lse, torch.zeros_like(r.lse))[..., None]
    # lse = (m2 + lg2(tot)) * LN2 (line 197): the row sum's error, lg2's, the addition, fp32 LN2 and the product
    e_lse = dtot + LN2 * LG2 * (lse * LOG2E - m2).abs().clamp_min(1.0) + 3 * UF * lse.abs()
    b = dict(out=_flat(e_out), lse=e_lse.squeeze(-1))

    # -- backward (attention_bwd.cu); SIDE 1 rounds the exponent less often than SIDE 0, so SIDE 0's terms cover both --
    lse2 = lse * LOG2E
    dlse2 = LOG2E * e_lse + 2 * UF * lse2.abs()                     # the forward's lse, times LOG2E in fp32 (line 151, 111)
    # p = ex2(fmaf(s, c2, kb) - lse2 + gli) (line 223): four roundings of the exponent, the gate's and lse's errors
    dxb = C2 * eS + 2 * UF * s2.abs() + UF * (s2 - lse2).abs() + dlse2
    if x.sw is not None:
        dxb = dxb + UF * (s2 + g2 - lse2).abs() + dg
    rho_b = LN2 * dxb + EX2
    # D = rowsum(dO o O) over the kernel's bf16 O (line 152-166): O's own error plus the 64-term fp32 fma chain
    eD = (ag * e_out).sum(-1, keepdim=True) + 64 * UF * (aO * ag).sum(-1, keepdim=True)
    edP = 64 * TC * (ag @ av.transpose(-1, -2))                     # dP = dO V^T (tensor core)
    Dm = (r.dP - r.D[..., None]).abs()
    # dsi = p * (dpi * m - D) in fp32 (line 226-229): p's error, dP's and D's, the subtraction and the product; the dropout
    # factor m = inv_keep and dpi * m round once more
    eds = P * (rho_b * Dm + r.M * edP + eD + 2 * UF * Dm + (3 * UF * r.dP.abs() if drop else 0.0))
    ads = SCALE * r.dS.abs()
    # scale * dsi rounded to bf16 (line 236, 257), dQ = dS K / dK = dS^T Q over the tensor core, bf16 stores (line 286, 293)
    e_dq = (SCALE * eds + (UB + Lk * TC) * ads) @ ak + UB * r.dq.abs()
    e_dk = (SCALE * eds + (UB + Lq * TC) * ads).transpose(-1, -2) @ aq + UB * r.dk.abs()
    # P^T: p * m (exact without dropout) rounded to bf16 (line 253, 258), dV = P^T dO (tensor core), bf16 store (line 294)
    e_dv = (Pd * (rho_b + pr + Lq * TC)).transpose(-1, -2) @ ag + UB * r.dv.abs()
    b.update(dq=_flat(e_dq), dk=_flat(e_dk), dv=_flat(e_dv))
    if x.sw is not None:
        incl = r.unclamped | amb
        om = 1 - r.sig
        ads_n = r.dS.abs()
        # dz = dsi * (1 - ex2(gli)) from the fp32 dsi before rounding (line 231): gli's error moves sigmoid by
        # sigmoid (ln2 dg + ex2's error); 1 - sigmoid and the product round once each; an ambiguous pair may be left out
        edz = (eds * om + ads_n * (r.sig * (LN2 * dg + EX2) + 2 * UF * om)) * incl + ads_n * om * amb
        lt = _loc_terms(x.locs.double().abs())
        # gg += dz, fmaf(dz, l, gg) over the keys, then two shuffle levels (line 232-234, 280-281)
        e = torch.einsum("bhij,bijk->bhik", edz, lt) + (Lk + 2) * UF * torch.einsum("bhij,bijk->bhik", r.dz.abs(), lt)
        if SH == 1:
            e = e.sum(1, keepdim=True)
        b["dsw"] = e.transpose(1, 2).reshape(B, Lq, SH * 6)
        b["gate_silent_rows"] = ~(incl & livep).any(-1)                # (B, H, Lq): no pair passes the clamp
    return b


def dvec_bound(out_kernel, go, H):
    """D = rowsum(dO o O) in float64 from the kernel's own bf16 O, and the bound of the kernel's fp32 fma chain of 64."""
    o, g = _heads(out_kernel, H), _heads(go, H)
    return (o * g).sum(-1), 64 * UF * (o.abs() * g.abs()).sum(-1)


def within(got, want, bound, what):
    """|got - want| <= 1.01 bound wherever the reference is finite; non-finite exactly where, and as, it is.  Returns the
    worst |got - want| / bound; on failure names the worst element."""
    got = got.detach().double().to(want.device)
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(got), fin), f"{what}: non-finite elements differ"
    assert torch.equal(got[~fin], want[~fin]), f"{what}: non-finite elements differ in value"
    err = torch.where(fin, (got - want).abs(), torch.zeros_like(want))
    b = 1.01 * torch.where(fin, bound, torch.ones_like(bound))
    ratio = err / b.clamp_min(1e-300)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if worst > 1.0:
        idx = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
        raise AssertionError(f"{what}: {int((err > b).sum())} elements outside the bound; worst at index {tuple(int(i) for i in idx)}: "
                             f"got {float(got[idx]):.6g}, want {float(want[idx]):.6g}, bound {float(bound[idx]):.3g}, "
                             f"|err| / bound {worst:.3g}")
    return worst


# ---- inputs -----------------------------------------------------------------------------------------------------------
def gate_weights(B, L, SH, g):
    """(B, L, SH * 6) fp32 gate weights [bias, w1..w5].  The (query, head) rows cycle through four classes so that pairs sit
    in every region of the gate: z < -14 for every key (under the clamp), z > 90 for every key (t = exp(-z) underflows to 0
    in fp32), z spread around 0, and rows that straddle the clamp (the distance weight moves z across it)."""
    w = torch.randn(B, L, SH, 6, generator=g)
    clamp, sat, mid, straddle = w.clone(), w.clone(), w.clone(), w.clone()
    clamp[..., 0], clamp[..., 1:] = -35 + w[..., 0], 0.5 * w[..., 1:]
    sat[..., 0], sat[..., 1:] = 105 + w[..., 0], 0.5 * w[..., 1:]
    mid[..., 0], mid[..., 1:] = 3 * w[..., 0], 2 * w[..., 1:]
    straddle[..., 0], straddle[..., 1], straddle[..., 2:] = -12.0, -4.0, 0.5 * w[..., 2:]
    cls = ((torch.arange(L)[:, None] + torch.arange(SH)[None, :]) % 4)[None, :, :, None]
    out = torch.where(cls == 0, clamp, torch.where(cls == 1, sat, torch.where(cls == 2, mid, straddle)))
    return out.reshape(B, L, SH * 6)


def inputs(Lq, Lk, H, seed=1, gate=None, dropout=False, device="cuda", B=2):
    """bf16 q, k, v, dO with unit variance (logits of unit variance); scene 1 masks the second half of its keys.
    gate: None, "per_head" or "shared"."""
    g = torch.Generator().manual_seed(seed)
    q, k, v, go = (torch.randn(B, L, H * 64, generator=g).bfloat16() for L in (Lq, Lk, Lk, Lq))
    mask = torch.zeros(B, Lk, dtype=torch.bool)
    if B > 1:
        mask[1, (Lk + 1) // 2:] = True
    sw = locs = keep = None
    if gate is not None:
        assert Lq == Lk
        sw = gate_weights(B, Lq, H if gate == "per_head" else 1, g)
        locs = ops.calc_pairwise_locs(torch.randn(B, Lq, 3, generator=g) * 2.0, None)
    if dropout:
        keep = torch.from_numpy(_dropout_keep(SEED, B, H, Lq, Lk, P_DROP))
    x = types.SimpleNamespace(q=q, k=k, v=v, go=go, mask=mask, sw=sw, locs=locs, keep=keep, H=H)
    for name in ("q", "k", "v", "go", "mask", "sw", "locs", "keep"):
        t = getattr(x, name)
        if t is not None:
            setattr(x, name, t.to(device).contiguous())
    return x


# ---- the kernels --------------------------------------------------------------------------------------------------------
def forward(x, q=None, k=None, v=None):
    from sceneverse_b200 import native
    sh = 0 if x.sw is None else x.sw.shape[-1] // 6
    return native.attention(x.q if q is None else q, x.k if k is None else k, x.v if v is None else v, x.H,
                            key_padding_mask=x.mask, spatial_w=x.sw, spatial_heads=sh, pairwise_locs=x.locs,
                            return_lse=True, dropout_p=P_DROP if x.keep is not None else 0.0, seed=SEED)


def backward(x, out, lse):
    """sv_attention_bwd_strided_bf16 called directly, so that D (dvec) is returned too.  Outputs start as NaN: an element
    the kernels do not write shows."""
    from sceneverse_b200 import _lib, native
    B, Lq, E = x.q.shape
    Lk = x.k.shape[1]
    nan = dict(dtype=torch.bfloat16, device=x.q.device)
    dq, dk, dv = torch.full((B, Lq, E), math.nan, **nan), torch.full((B, Lk, E), math.nan, **nan), \
        torch.full((B, Lk, E), math.nan, **nan)
    dvec = torch.full((B, x.H, Lq), math.nan, device=x.q.device)
    dsw = torch.full_like(x.sw, math.nan) if x.sw is not None else None
    kpm = native._mask_bytes(x.mask)
    lib = _lib.gps()
    st = lib.sv_attention_bwd_strided_bf16(
        x.q.data_ptr(), x.q.stride(0), x.q.stride(1), x.k.data_ptr(), x.k.stride(0), x.k.stride(1), x.v.data_ptr(),
        x.v.stride(0), x.v.stride(1), out.data_ptr(), x.go.data_ptr(), _lib.ptr(kpm), _lib.ptr(x.sw), _lib.ptr(x.locs),
        lse.data_ptr(), B, x.H, Lq, Lk, SCALE, dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), E, _lib.ptr(dsw), dvec.data_ptr(),
        P_DROP if x.keep is not None else 0.0, SEED, torch.cuda.current_stream().cuda_stream)
    _lib.check(lib, st, "sv_attention_bwd_strided_bf16")
    got = dict(dq=dq, dk=dk, dv=dv, dvec=dvec)
    if dsw is not None:
        got["dsw"] = dsw
    return got


def run(x, with_backward=True):
    out, lse = forward(x)
    got = dict(out=out, lse=lse)
    if with_backward:
        got.update(backward(x, out, lse))
    return got


def check(x, got, what):
    """Every output the kernels returned against the float64 reference and its bound; prints the worst |err| / bound."""
    r = reference(x)
    b = bounds(x, r)
    worst = {}
    for name in ("out", "lse", "dq", "dk", "dv", "dsw"):
        if name in got:
            worst[name] = within(got[name], r.outputs[name], b[name], f"{what} {name}")
    if "dvec" in got:
        want, bd = dvec_bound(got["out"], x.go, x.H)
        worst["dvec"] = within(got["dvec"], want, bd, f"{what} dvec")
    print(f"ATTN_FP64 {what}: worst |err| / bound", {k: f"{v:.3g}" for k, v in worst.items()})
    if "dk" in got:   # masked keys: exactly zero dk / dv rows
        for name in ("dk", "dv"):
            assert not got[name][x.mask].any(), f"{what} {name}: masked keys have non-zero rows"
    return r, b


def check_scenes_alone(x, got, what):
    """Each scene run on its own gives the same bits as in the batch: the work units are independent."""
    for s in range(x.q.shape[0]):
        xs = types.SimpleNamespace(**vars(x))
        for name in ("q", "k", "v", "go", "mask", "sw", "locs"):
            t = getattr(x, name)
            setattr(xs, name, None if t is None else t[s:s + 1].contiguous())
        alone = run(xs, with_backward="dq" in got)
        for name, t in alone.items():
            assert torch.equal(t, got[name][s:s + 1]), f"{what} scene {s} {name}: differs from the batched run"


PLAIN = [(64, 1), (65, 17), (80, 80), (50, 80), (129, 65), (130, 130), (193, 304), (384, 384)]
GATED = [1, 17, 63, 64, 65, 80, 129, 130, 193, 384]


@pytest.mark.gpu
@pytest.mark.parametrize("H", [12, 5])
@pytest.mark.parametrize("Lq,Lk", PLAIN)
def test_plain_attention_within_fp64_bound(Lq, Lk, H):
    x = inputs(Lq, Lk, H)
    got = run(x)
    check(x, got, f"plain Lq={Lq} Lk={Lk} H={H}")
    check_scenes_alone(x, got, f"plain Lq={Lq} Lk={Lk} H={H}")


@pytest.mark.gpu
@pytest.mark.parametrize("H", [12, 5])
@pytest.mark.parametrize("L", GATED)
def test_gated_attention_within_fp64_bound(L, H):
    x = inputs(L, L, H, gate="per_head")
    got = run(x)
    r, b = check(x, got, f"gated L={L} H={H}")
    live = r.live[:, None, None, :].expand_as(r.z) & torch.isfinite(r.lse)[..., None]
    z = r.z[live]
    regions = {"clamped": int((z < -14).sum()), "saturated": int((z > 90).sum()),
               "between": int(((z >= -14) & (z <= 90)).sum())}
    assert all(regions.values()), regions
    # under the clamp the gate-weight gradient is zero: rows in which no live pair passes the clamp get exact zeros
    silent = b["gate_silent_rows"].transpose(1, 2)                                    # (B, Lq, H)
    assert silent.any()
    assert not got["dsw"].view(*silent.shape, 6)[silent].any(), "gate-weight gradient through clamped pairs"
    check_scenes_alone(x, got, f"gated L={L} H={H}")


@pytest.mark.gpu
@pytest.mark.parametrize("L", [65, 130])
def test_gate_shared_across_heads_within_fp64_bound(L):
    """spatial_heads = 1: the native forward, and ops.spatial_attention, whose backward recomputes the same formulas with
    torch in fp32.  The kernel bound covers that backward too: each of its roundings is fp32 where the kernels round P and
    dS to bf16."""
    H = 12
    x = inputs(L, L, H, gate="shared")
    got = run(x, with_backward=False)
    check(x, got, f"shared gate L={L}")
    q, k, v = (t.clone().requires_grad_(True) for t in (x.q, x.k, x.v))
    sw = x.sw.clone().requires_grad_(True)
    out, _ = ops.spatial_attention(q, k, v, sw, x.locs, H, 1, key_padding_mask=x.mask)
    assert isinstance(out.grad_fn, ops._SpatialAttentionRecomputeFn._backward_cls)
    assert torch.equal(out, got["out"])
    out.backward(x.go)
    r = reference(x)
    b = bounds(x, r)
    worst = {name: within(t.grad, r.outputs[name], b[name], f"shared gate L={L} recompute {name}")
             for name, t in (("dq", q), ("dk", k), ("dv", v), ("dsw", sw))}
    print(f"ATTN_FP64 shared gate L={L} recompute backward: worst |err| / bound", {k: f"{v:.3g}" for k, v in worst.items()})


@pytest.mark.gpu
@pytest.mark.parametrize("H", [12, 5])
@pytest.mark.parametrize("Lq,Lk", [(80, 50), (130, 130), (384, 384)])
def test_dropout_attention_within_fp64_bound(Lq, Lk, H):
    x = inputs(Lq, Lk, H, dropout=True)
    assert abs(x.keep.double().mean().item() - (1 - P_DROP)) < 0.01
    check(x, run(x), f"dropout Lq={Lq} Lk={Lk} H={H}")


@pytest.mark.gpu
@pytest.mark.parametrize("gate", [None, "per_head"])
def test_strided_operands_within_fp64_bound(gate):
    """q, k, v as column views of one packed (B, L, 3E) projection, and the backward writing into one packed gradient: the
    same bits as with contiguous operands, and within the bound."""
    from sceneverse_b200 import native
    L, H = 130, 12
    x = inputs(L, L, H, gate=gate)
    E = H * 64
    qkv = torch.cat([x.q, x.k, x.v], -1)
    qv, kv, vv = qkv[..., :E], qkv[..., E:2 * E], qkv[..., 2 * E:]
    assert qv.stride(1) == 3 * E
    got = run(x)
    out, lse = forward(x, qv, kv, vv)
    assert torch.equal(out, got["out"]) and torch.equal(lse, got["lse"])
    packed = torch.full((2, L, 3 * E), math.nan, dtype=torch.bfloat16, device="cuda")
    dq, dk, dv, dsw = native.attention_backward(qv, kv, vv, out, x.go, lse, H, key_padding_mask=x.mask, spatial_w=x.sw,
                                                pairwise_locs=x.locs, packed_grad=packed)
    for name, t in (("dq", dq), ("dk", dk), ("dv", dv)):
        assert torch.equal(t, got[name]), f"packed {name} differs from the contiguous run"
    if gate is not None:
        assert torch.equal(dsw, got["dsw"])
    check(x, dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv, **({"dsw": dsw} if gate else {})), f"strided gate={gate}")


@pytest.mark.gpu
@pytest.mark.parametrize("Lq,Lk,gate", [(65, 17, None), (130, 130, None), (130, 130, "per_head")])
def test_scene_with_every_key_masked(Lq, Lk, gate):
    """attention.cu:131, :197: a row without a live key gets output 0 and lse = +inf, and the backward gives zero
    gradients for it, not NaN."""
    x = inputs(Lq, Lk, 12, gate=gate)
    x.mask[1] = True
    got = run(x)
    for name, t in got.items():
        assert not torch.isnan(t).any(), f"{name}: NaN"
    assert not got["out"][1].any() and torch.equal(got["lse"][1], torch.full_like(got["lse"][1], math.inf))
    for name in ("dq", "dk", "dv", "dvec") + (("dsw",) if gate else ()):
        assert not got[name][1].any(), f"{name}: non-zero for the scene without a live key"
    check(x, got, f"scene fully masked Lq={Lq} Lk={Lk} gate={gate}")


# ---- without a GPU ----------------------------------------------------------------------------------------------------
def _autograd_reference(x):
    """torch autograd of ops._spatial_attention_torch (gated) or of the plain masked softmax, in float64."""
    B, Lq, E = x.q.shape
    Lk, H = x.k.shape[1], x.H
    q, k, v = (t.double().requires_grad_(True) for t in (x.q, x.k, x.v))
    sw = x.sw.double().requires_grad_(True) if x.sw is not None else None
    if sw is not None:
        out, _ = ops._spatial_attention_torch(q, k, v, sw, x.locs.double(), H, sw.shape[-1] // 6, key_padding_mask=x.mask)
    else:
        qh, kh, vh = (t.view(B, -1, H, 64).transpose(1, 2) for t in (q, k, v))
        att = ((qh @ kh.transpose(-1, -2)) * SCALE).masked_fill(x.mask[:, None, None, :], -math.inf).softmax(-1)
        if x.keep is not None:
            att = att * x.keep / (1 - float(np.float32(P_DROP)))
        out = (att @ vh).transpose(1, 2).reshape(B, Lq, E)
    out.backward(x.go.double())
    got = dict(out=out.detach(), dq=q.grad, dk=k.grad, dv=v.grad)
    if sw is not None:
        got["dsw"] = sw.grad
    return got


@pytest.mark.parametrize("Lq,Lk,gate,dropout", [(65, 17, None, False), (50, 80, None, True), (40, 40, "per_head", False),
                                                (40, 40, "shared", False)])
def test_reference_matches_torch_autograd(Lq, Lk, gate, dropout):
    """The written-out float64 reference equals torch autograd of the formulas the model uses."""
    x = inputs(Lq, Lk, 4, gate=gate, dropout=dropout, device="cpu")
    r = reference(x)
    want = _autograd_reference(x)
    for name, w in want.items():
        err = float((r.outputs[name] - w).abs().max()) / float(w.abs().max())
        assert err < 1e-12, (name, err)
    logits = _heads(x.q, 4) @ _heads(x.k, 4).transpose(-1, -2) * SCALE + (r.lg if gate else 0)
    lse = torch.logsumexp(logits.masked_fill(x.mask[:, None, None, :], -math.inf), -1)
    assert float((r.lse - lse).abs().max()) < 1e-12


KNOCK_CASES = {"plain Lq=Lk=384": dict(Lq=384, Lk=384), "gated L=130": dict(Lq=130, Lk=130, gate="per_head"),
               "dropout Lq=Lk=130": dict(Lq=130, Lk=130, dropout=True)}


def _applies(knock, x):
    if knock in ("gate_next_head", "no_clamp", "grad_through_clamp"):
        return x.sw is not None
    return x.keep is not None if knock == "no_rescale" else True


@pytest.mark.parametrize("case", list(KNOCK_CASES))
def test_bound_detects_each_kernel_slip(case):
    """Each slip moves some element of an output it affects by at least 4 x the bound (1.01 x bounds()) that the GPU tests
    hold the kernels to."""
    x = inputs(H=4, device="cpu", **KNOCK_CASES[case])
    full = reference(x)
    b = bounds(x, full)
    margins = {}
    for knock in (k for k in KNOCKS if _applies(k, x)):
        kn = reference(x, knock).outputs
        per = {}
        for name, want in full.outputs.items():
            fin = torch.isfinite(want) & torch.isfinite(kn[name])
            moved = (kn[name] - want).abs()[fin] / (1.01 * b[name][fin]).clamp_min(1e-300)
            per[name] = float(moved.max())
        margins[knock] = per
        print(f"KNOCKOUT {case} {knock}: max |knocked - full| / bound",
              {k: (f"{v:.3g}" if v < 1e6 else "inf") for k, v in per.items()})
    low = {k: max(v.values()) for k, v in margins.items() if max(v.values()) < 4}
    assert not low, low


_VALIDATION = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from sceneverse_b200 import _lib
lib = _lib.gps()
a = 0x1000      # 16-byte aligned fake address


def fwd(Lk=64, sw=None, sh=0, locs=None, p=0.0):
    return lib.sv_attention_fwd_dropout_bf16(a, 8, 768, a, 8, 768, a, 8, 768, a, 8, 768, None, sw, sh, locs, 1, 12, 4, Lk,
                                             0.125, None, p, 0, None)


def bwd(Lq=64, Lk=64, sw=None, locs=None, dsw=None, p=0.0):
    return lib.sv_attention_bwd_strided_bf16(a, 8, 768, a, 8, 768, a, 8, 768, a, a, None, sw, locs, a, 1, 12, Lq, Lk, 0.125,
                                             a, a, a, 768, dsw, a, p, 0, None)


out = {"fwd Lk 385": fwd(Lk=385), "fwd spatial_heads 0": fwd(sw=a, locs=a, sh=0),
       "fwd spatial_heads 2": fwd(sw=a, locs=a, sh=2), "fwd spatial_heads 13": fwd(sw=a, locs=a, sh=13),
       "fwd gate without locs": fwd(sw=a, sh=12), "fwd gate with dropout": fwd(sw=a, locs=a, sh=12, p=0.1),
       "bwd Lk 385": bwd(Lk=385), "bwd Lq 385": bwd(Lq=385), "bwd gate with dropout": bwd(sw=a, locs=a, dsw=a, p=0.1),
       "bwd gate without d_spatial_w": bwd(sw=a, locs=a),
       # accepted by the validation: they get as far as the device, which this process does not see
       "fwd Lk 384": fwd(Lk=384), "fwd spatial_heads 1": fwd(sw=a, locs=a, sh=1), "fwd spatial_heads 12": fwd(sw=a, locs=a, sh=12),
       "bwd Lq Lk 384": bwd(Lq=384, Lk=384), "bwd gate": bwd(sw=a, locs=a, dsw=a)}
print(json.dumps(out))
"""


def test_attention_argument_validation_without_gpu():
    """The attention entry points reject what the kernels cannot run (1 = SV_ERR_INVALID_ARG) before touching the device.
    The calls run in a process that sees no CUDA device, so a missing check shows as a CUDA error (2) instead of a launch
    on the fake pointers; the accepted calls show that the checks reject no more than they should."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", _VALIDATION, root], capture_output=True, text=True, timeout=120,
                         env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    accepted = ("fwd Lk 384", "fwd spatial_heads 1", "fwd spatial_heads 12", "bwd Lq Lk 384", "bwd gate")
    want = {k: 2 if k in accepted else 1 for k in got}
    assert len(got) == 15 and got == want, {k: v for k, v in got.items() if v != want[k]}
