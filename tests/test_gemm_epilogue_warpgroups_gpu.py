"""The epilogue-warpgroup schedule of the staged GEMM (csrc/gemm.cu, GemmCfg::EW): at 64- and 128-column tiles the forward and
dgrad epilogues run in two warpgroups of their own, fed each tile's fp32 accumulators through a shared-memory hand-off, while
the MMA warpgroups go on to the next tile.  Every output element gets the same accumulator and the same arithmetic, so the
outputs must equal the per-element epilogue (an output pitch that cannot take TMA boxes, cooperative schedule) bit for bit:
at step shapes with many tiles per CTA (the hand-off and the aux ring reused across the persistent loop), with fewer tiles
than SMs, ragged M, the N = 607 / 30522 tails, and every epilogue the GPS step uses.  sv_gemm_profile slot 8 names the
schedule each CTA ran (1 = epilogue warpgroups), slot 7 the epilogue (1 = staged)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
SENT = 1232.0   # exact in bf16 and fp32


def gamma_n(n):
    return n * U32 / (1 - n * U32)


def rnd(*s, seed=0, scale=0.5):
    g = torch.Generator(device="cuda").manual_seed(seed + sum(s))
    return torch.randn(*s, device="cuda", generator=g) * scale


EW = 16   # sv_gemm_force_ctas: the staged forward / dgrad on epilogue warpgroups
COOP = 8  # ... on the cooperative schedule


@pytest.fixture(params=[1, 2], ids=["bn64", "bn128"])
def tile(request):
    """64 / 128 output columns and the epilogue-warpgroup schedule forced."""
    from sceneverse_b200 import native
    native.gemm_force_ctas(request.param | EW)
    yield request.param
    native.gemm_force_ctas(0)


class Schedule:
    """Collects the (epilogue, schedule) pair of every CTA that issued k-steps in the GEMM launches inside the block."""

    def __enter__(self):
        from sceneverse_b200 import _lib
        self.lib = _lib.gps()
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        self.prof = torch.zeros(self.sms * 16, dtype=torch.int64, device="cuda")
        assert self.lib.sv_gemm_profile(self.prof.data_ptr()) == 0
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.lib.sv_gemm_profile(None)

    def runs(self):
        torch.cuda.synchronize()
        p = self.prof.view(self.sms, 16)
        live = p[p[:, 3] > 0]
        return {(int(a), int(b)) for a, b in zip(live[:, 7].tolist(), live[:, 8].tolist())}


def odd_pitch(n, esz):
    p = n + 1
    while (p * esz) % 16 == 0:
        p += 1
    return p


def tma_pitch(n, esz):
    step = 16 // esz
    return (n // step + 1) * step


# (M, N, K): BERT-300 ffn1 (3600 tiles at 128 columns: many per CTA), BERT-50 qkv, joint-130 out, fewer tiles than SMs
# (130 x 768), ragged M (1000), the 607-class head (N = 607 in a 608 pitch), the LM head (N = 30522)
FWD_SHAPES = [(19200, 3072, 768), (3200, 2304, 768), (8320, 768, 768), (130, 768, 768), (1000, 607, 768), (3200, 30522, 768)]
# (act, dropout p, want_pre): bias only, ReLU + dropout (joint / spatial ffn1), GELU with its pre-activation copy (BERT ffn1),
# GELU + dropout with the copy, dropout alone
FWD_EPILOGUES = [(None, 0.0, False), ("relu", 0.1, False), ("gelu", 0.0, True), ("gelu", 0.1, True), (None, 0.1, False)]


@pytest.mark.parametrize("M,N,K", FWD_SHAPES)
@pytest.mark.parametrize("act,p,want_pre", FWD_EPILOGUES)
def test_fwd_epilogue_warpgroups_bitwise(M, N, K, act, p, want_pre, tile):
    from sceneverse_b200 import native
    Np = (N + 7) // 8 * 8
    x, w, b = rnd(M, K).bfloat16(), rnd(Np, K, scale=K ** -0.5).bfloat16(), rnd(N, seed=1)
    kw = dict(dropout_p=p, seed=1357911, want_pre=want_pre, n_out=N)
    ref_buf = torch.zeros(M, odd_pitch(N, 2), dtype=torch.bfloat16, device="cuda")
    with Schedule() as s:
        ref = native.linear_fwd(x, w, b, act, out=ref_buf, **kw)
        assert s.runs() == {(0, 0)}
    buf = torch.full((M + 64, tma_pitch(N, 2)), SENT, dtype=torch.bfloat16, device="cuda")
    with Schedule() as s:
        got = native.linear_fwd(x, w, b, act, out=buf[:M], **kw)
        assert s.runs() == {(1, 1)}
    if want_pre:
        (ref, ref_pre), (got, got_pre) = ref, got
        assert torch.equal(got_pre[:, :N], ref_pre[:, :N])
    assert torch.equal(buf[:M, :N], ref_buf[:, :N])
    assert (buf[:, N:] == SENT).all() and (buf[M:] == SENT).all()


def _dgrad(g, w, M, N, Kin, act, aux, p, dx):
    from sceneverse_b200 import _lib
    lib = _lib.gps()
    st = lib.sv_linear_dgrad_bf16(g.data_ptr(), g.stride(0), w.data_ptr(), w.stride(0), M, N, Kin, {None: 0, "relu": 1, "gelu": 2}[act],
                                  aux.data_ptr() if aux is not None else None, aux.stride(0) if aux is not None else 0,
                                  float(p), 24680, dx.data_ptr(), dx.stride(0), 0, torch.cuda.current_stream().cuda_stream)
    _lib.check(lib, st, "sv_linear_dgrad_bf16")


# (M, N reduced over, Kin written): BERT-300 ffn2 (GELU'), joint-130 ffn2 (ReLU'), spatial-80 qkv, fewer tiles than SMs,
# ragged M with Kin = 607 and its per-element tail
DGRAD_SHAPES = [(19200, 768, 3072), (8320, 768, 2048), (5120, 2304, 768), (130, 768, 768), (1000, 768, 607)]


@pytest.mark.parametrize("M,N,Kin", DGRAD_SHAPES)
@pytest.mark.parametrize("act,p", [(None, 0.0), ("relu", 0.1), ("gelu", 0.0), ("gelu", 0.1)])
def test_dgrad_epilogue_warpgroups_bitwise(M, N, Kin, act, p, tile):
    """The plain dgrad and the activation-derivative dgrads, whose saved activation the epilogue warpgroups load by TMA into
    their output ring while the MMA warpgroups run the tile's main loop."""
    Kp = (Kin + 7) // 8 * 8
    g, w = rnd(M, N).bfloat16(), rnd(N, Kp, scale=N ** -0.5).bfloat16()
    aux = None
    if act:
        aux = rnd(M, Kp, seed=3, scale=1.5).bfloat16()
        if act == "relu":
            aux = torch.relu(aux)
    ref = torch.zeros(M, odd_pitch(Kin, 2), dtype=torch.bfloat16, device="cuda")
    with Schedule() as s:
        _dgrad(g, w, M, N, Kin, act, aux, p, ref)
        assert s.runs() == {(0, 0)}
    buf = torch.full((M + 64, tma_pitch(Kin, 2)), SENT, dtype=torch.bfloat16, device="cuda")
    with Schedule() as s:
        _dgrad(g, w, M, N, Kin, act, aux, p, buf[:M])
        assert s.runs() == {(1, 1)}
    assert torch.equal(buf[:M, :Kin], ref[:, :Kin])
    assert (buf[:, Kin:] == SENT).all() and (buf[M:] == SENT).all()


@pytest.mark.parametrize("M,N,K,want", [
    (19200, 2304, 768, 1), (19200, 3072, 768, 1), (8320, 2304, 768, 1), (5120, 2048, 768, 1), (3200, 30522, 768, 1),
    (5120, 768, 2048, 0), (3200, 768, 3072, 0), (130, 768, 768, 0)])
def test_heuristic_schedule(M, N, K, want):
    """With width and schedule left to the heuristic, the step's forwards with at least three tiles per CTA run the epilogue
    warpgroups (the LM head writes N = 30522 into its 30528-wide buffer, as in the step); the spatial-80 / BERT-50 ffn2
    forwards (two tiles per CTA) and a launch with fewer tiles than SMs keep the cooperative schedule."""
    from sceneverse_b200 import native
    native.gemm_force_ctas(0)
    Np = (N + 7) // 8 * 8
    x, w, b = rnd(M, K).bfloat16(), rnd(Np, K, scale=K ** -0.5).bfloat16(), rnd(N, seed=1)
    out = torch.empty(M, Np, dtype=torch.bfloat16, device="cuda")
    with Schedule() as s:
        native.linear_fwd(x, w, b, "relu", out=out, n_out=N)
        assert s.runs() == {(1, want)}


@pytest.mark.parametrize("M,N,K", [(19200, 2304, 768), (5120, 768, 2048), (1000, 607, 768)])
@pytest.mark.parametrize("bn", [1, 2])
def test_forced_schedules_agree(M, N, K, bn):
    """The two staged schedules at the same width give the same bits (GELU with pre-activation copy and dropout)."""
    from sceneverse_b200 import native
    Np = (N + 7) // 8 * 8
    x, w, b = rnd(M, K).bfloat16(), rnd(Np, K, scale=K ** -0.5).bfloat16(), rnd(N, seed=1)
    outs = []
    try:
        for sched, want in ((COOP, 0), (EW, 1)):
            native.gemm_force_ctas(bn | sched)
            buf = torch.full((M, Np), SENT, dtype=torch.bfloat16, device="cuda")
            with Schedule() as s:
                _, pre = native.linear_fwd(x, w, b, "gelu", dropout_p=0.1, seed=77, want_pre=True, out=buf, n_out=N)
                assert s.runs() == {(1, want)}
            outs.append((buf, pre))
    finally:
        native.gemm_force_ctas(0)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1][:, :N], outs[1][1][:, :N])


@pytest.mark.parametrize("M,N,Kin", [(19200, 768, 3072), (3200, 30522, 768), (8320, 607, 768)])
def test_wgrad_against_fp64(M, N, Kin, tile):
    """The weight gradients of the same launches (split-K reduce-add, cooperative schedule) stay within the summation bound."""
    from sceneverse_b200 import native
    Np = (N + 7) // 8 * 8
    g, x = rnd(M, Np).bfloat16(), rnd(M, Kin, seed=5).bfloat16()
    dw, db = native.linear_wgrad(g, x, n_out=N, want_db=True)
    torch.cuda.synchronize()
    g64, x64 = g[:, :N].double(), x.double()
    exact, mag = g64.t() @ x64, g64.abs().t() @ x64.abs()
    assert ((dw.double() - exact).abs() <= gamma_n(M + 33) * mag).all()
    assert ((db.double() - g64.sum(0)).abs() <= gamma_n(M + 33) * g64.abs().sum(0)).all()
