"""The staged GEMM epilogue (csrc/gemm.cu): outputs whose rows take 16-byte-aligned boxes go out through shared memory by TMA
store (forward, dgrad) or TMA reduce-add (split-K weight gradient); every other pitch keeps the per-element stores.  The
register arithmetic is shared, so the two paths must agree bit for bit, and neither may write outside [M, N].  A TMA store
clips a row only at whole 16-byte units, so for widths like 607 (in a 608-wide buffer), 30522 or Kin = 607 the last columns
are copied out of the staged box per element: the pad columns around them are checked like every other.  Every launch is
checked to have taken the path it is compared as (sv_gemm_profile records the epilogue of each CTA)."""
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


@pytest.fixture(params=[0, 1, 2, 4], ids=["auto", "bn64", "bn128", "bn192"])
def tile(request):
    """Heuristic tile width, then 64 / 128 / 192 output columns forced."""
    from sceneverse_b200 import native
    native.gemm_force_ctas(request.param)
    yield request.param
    native.gemm_force_ctas(0)


def tma_pitch(n, esz):
    """A row pitch >= n whose bytes are a multiple of 16 (the TMA path), with at least one pad column."""
    step = 16 // esz
    return (n // step + 1) * step


def odd_pitch(n, esz):
    """A row pitch >= n whose bytes are not a multiple of 16 (the per-element path)."""
    p = n + 1
    while (p * esz) % 16 == 0:
        p += 1
    return p


class EpiloguePath:
    """Records which epilogue the GEMM launches inside the block ran: slot 7 of the sv_gemm_profile record of every CTA
    that issued k-steps is 1 for the staged TMA epilogue, 0 for per-element stores."""

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

    def staged(self):
        """True if every CTA staged its output, False if every CTA stored per element (anything else fails)."""
        torch.cuda.synchronize()
        p = self.prof.view(self.sms, 16)
        flags = set(p[p[:, 3] > 0, 7].tolist())
        assert flags in ({0}, {1}), flags
        return flags == {1}


def sentinel_buf(rows, cols, dtype):
    return torch.full((rows, cols), SENT, dtype=dtype, device="cuda")


def assert_untouched(region):
    assert (region == SENT).all()


# (M, N, K): step shapes, ragged M (3, 130, 1000), a narrow N (72), the padded 607 -> 608 and 30522 -> 30528 (LM head)
FWD_SHAPES = [(19200, 2304, 768), (3200, 3072, 768), (8320, 768, 2048), (3, 768, 768), (130, 72, 768), (1000, 607, 768),
              (3200, 30528, 768), (3200, 30522, 768)]
# (act, dropout p, out dtype, want_pre)
FWD_VARIANTS = [(None, 0.0, torch.bfloat16, False), ("relu", 0.1, torch.bfloat16, False), ("gelu", 0.0, torch.bfloat16, True),
                ("gelu", 0.1, torch.bfloat16, True), ("gelu", 0.1, torch.float32, False), ("relu", 0.0, torch.float32, False)]


@pytest.mark.parametrize("M,N,K", FWD_SHAPES)
@pytest.mark.parametrize("act,p,dtype,want_pre", FWD_VARIANTS)
def test_fwd_tma_store_matches_per_element(M, N, K, act, p, dtype, want_pre, tile):
    from sceneverse_b200 import native
    Np = (N + 7) // 8 * 8
    x, w, b = rnd(M, K).bfloat16(), rnd(Np, K, scale=K ** -0.5).bfloat16(), rnd(N, seed=1)
    esz = 4 if dtype == torch.float32 else 2
    kw = dict(dropout_p=p, seed=987654321, want_pre=want_pre, n_out=N)

    ref_buf = torch.zeros(M, odd_pitch(N, esz), dtype=dtype, device="cuda")
    with EpiloguePath() as path:
        ref = native.linear_fwd(x, w, b, act, out=ref_buf, **kw)
        assert not path.staged()
    buf = sentinel_buf(M + 64, tma_pitch(N, esz), dtype)
    with EpiloguePath() as path:
        got = native.linear_fwd(x, w, b, act, out=buf[:M], **kw)
        assert path.staged()
    if want_pre:
        (ref, ref_pre), (got, got_pre) = ref, got
        assert torch.equal(got_pre[:, :N], ref_pre[:, :N])
    assert torch.equal(buf[:M, :N], ref_buf[:, :N])
    assert_untouched(buf[:, N:])
    assert_untouched(buf[M:])


def test_fwd_tma_store_into_column_slice(tile):
    """The BERT qkv layout: a projection written at column 768 of a packed (M, 2304) buffer."""
    from sceneverse_b200 import native
    M, K, N = 1000, 768, 768
    x, w, b = rnd(M, K).bfloat16(), rnd(N, K, scale=K ** -0.5).bfloat16(), rnd(N, seed=1)
    ref_buf = torch.zeros(M, odd_pitch(N, 2), dtype=torch.bfloat16, device="cuda")
    native.linear_fwd(x, w, b, "gelu", out=ref_buf, n_out=N)
    buf = sentinel_buf(M, 2304, torch.bfloat16)
    with EpiloguePath() as path:
        native.linear_fwd(x, w, b, "gelu", out=buf[:, 768:1536], n_out=N)
        assert path.staged()
    assert torch.equal(buf[:, 768:1536], ref_buf[:, :N])
    assert_untouched(buf[:, :768])
    assert_untouched(buf[:, 1536:])


def _dgrad(g, w, M, N, Kin, act, aux, p, dx, out_f32):
    from sceneverse_b200 import _lib
    lib = _lib.gps()
    st = lib.sv_linear_dgrad_bf16(g.data_ptr(), g.stride(0), w.data_ptr(), w.stride(0), M, N, Kin, {None: 0, "relu": 1, "gelu": 2}[act],
                                  aux.data_ptr() if aux is not None else None, aux.stride(0) if aux is not None else 0,
                                  float(p), 424242, dx.data_ptr(), dx.stride(0), 1 if out_f32 else 0,
                                  torch.cuda.current_stream().cuda_stream)
    _lib.check(lib, st, "sv_linear_dgrad_bf16")


# (M, N reduced over, Kin written)
DGRAD_SHAPES = [(19200, 768, 3072), (8320, 768, 2048), (3, 768, 768), (130, 2304, 768), (1000, 768, 72), (1000, 768, 607)]


@pytest.mark.parametrize("M,N,Kin", DGRAD_SHAPES)
@pytest.mark.parametrize("act,p,dtype", [(None, 0.0, torch.bfloat16), (None, 0.0, torch.float32), ("relu", 0.1, torch.bfloat16),
                                         ("gelu", 0.0, torch.bfloat16), ("gelu", 0.1, torch.float32)])
def test_dgrad_tma_store_matches_per_element(M, N, Kin, act, p, dtype, tile):
    Kp = (Kin + 7) // 8 * 8
    g, w = rnd(M, N).bfloat16(), rnd(N, Kp, scale=N ** -0.5).bfloat16()
    aux = rnd(M, Kp, seed=3, scale=1.5).bfloat16() if act else None
    if act == "relu":
        aux = torch.relu(aux)
    esz = 4 if dtype == torch.float32 else 2
    ref = torch.zeros(M, odd_pitch(Kin, esz), dtype=dtype, device="cuda")
    with EpiloguePath() as path:
        _dgrad(g, w, M, N, Kin, act, aux, p, ref, dtype == torch.float32)
        assert not path.staged()
    buf = sentinel_buf(M + 64, tma_pitch(Kin, esz), dtype)
    with EpiloguePath() as path:
        _dgrad(g, w, M, N, Kin, act, aux, p, buf[:M], dtype == torch.float32)
        assert path.staged()
    torch.cuda.synchronize()
    assert torch.equal(buf[:M, :Kin], ref[:, :Kin])
    assert_untouched(buf[:, Kin:])
    assert_untouched(buf[M:])


@pytest.mark.parametrize("M,N,Kin", [(19200, 1, 768), (8320, 607, 768), (3200, 30522, 768), (19200, 768, 3072), (130, 72, 136),
                                     (130, 72, 134)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_wgrad_tma_reduce_add(M, N, Kin, accumulate, tile):
    """Split-K reduce-add into a dw whose pitch is wider than Kin: against fp64, and against the per-element atomics of an odd
    pitch.  Each split's partial tile comes out of the same MMAs in both paths; only the order in which the (at most 32)
    partials and the prior dw are added differs, so the two agree within 2 gamma_33 (|dw0| + |g|^T |x|)."""
    from sceneverse_b200 import native
    Np = (N + 7) // 8 * 8
    g, x = rnd(M, Np).bfloat16(), rnd(M, (Kin + 7) // 8 * 8, seed=5).bfloat16()[:, :Kin]
    dw0 = rnd(N, Kin, seed=7) if accumulate else torch.zeros(N, Kin, device="cuda")
    db0 = rnd(N, seed=9) if accumulate else torch.zeros(N, device="cuda")

    buf = sentinel_buf(N + 8, tma_pitch(Kin, 4), torch.float32)
    buf[:N, :Kin] = dw0
    dw, db = buf[:N, :Kin], db0.clone()
    with EpiloguePath() as path:
        native.linear_wgrad(g, x, n_out=N, dw=dw, db=db, accumulate=accumulate)
        assert path.staged()
    ref_buf = torch.zeros(N, odd_pitch(Kin, 4), device="cuda")
    ref_buf[:, :Kin] = dw0
    ref_dw, ref_db = ref_buf[:, :Kin], db0.clone()
    with EpiloguePath() as path:
        native.linear_wgrad(g, x, n_out=N, dw=ref_dw, db=ref_db, accumulate=accumulate)
        assert not path.staged()
    torch.cuda.synchronize()

    g64, x64 = g[:, :N].double(), x.double()
    mag = dw0.double().abs() + g64.abs().t() @ x64.abs()
    exact = dw0.double() + g64.t() @ x64
    assert ((dw.double() - exact).abs() <= gamma_n(M + 33) * mag).all()
    assert ((dw.double() - ref_dw.double()).abs() <= 2 * gamma_n(33) * mag).all()
    assert torch.equal(db, ref_db) or ((db.double() - ref_db.double()).abs()
                                       <= 2 * gamma_n(33) * (db0.double().abs() + g64.abs().sum(0))).all()
    assert_untouched(buf[N:])
    if accumulate:   # accumulate = 0 zero-fills the whole pitch before the reduction
        assert_untouched(buf[:N, Kin:])
