"""The dgrad's saved activation by TMA (csrc/gemm.cu): when its rows take 16-byte-aligned boxes and the output is bf16, each
64-row x 64-column aux box is loaded by TMA into the shared-memory box its output columns go out through, and read back with
ldmatrix in the accumulator's fragment layout.  That path must agree bit for bit with the per-element loads of an aux pitch that
cannot take a TMA map, write nothing outside [M, Kin] (N = 607 with its per-element tail included), and stay close to an fp64
product of the same bf16 operands, on every tile width."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SENT = 1232.0   # exact in bf16 and fp32
U32 = 2.0 ** -24


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


def _dgrad(g, w, act, aux, p, dx):
    from sceneverse_b200 import _lib
    lib = _lib.gps()
    M, N = g.shape
    st = lib.sv_linear_dgrad_bf16(g.data_ptr(), g.stride(0), w.data_ptr(), w.stride(0), M, N, dx.shape[1],
                                  {"relu": 1, "gelu": 2}[act], aux.data_ptr(), aux.stride(0), float(p), 424242, dx.data_ptr(),
                                  dx.stride(0), 0, torch.cuda.current_stream().cuda_stream)
    _lib.check(lib, st, "sv_linear_dgrad_bf16")


# (M, N reduced over, Kin written): the 607 tail, ragged M and Kin around 64 / 128 / 192, the BERT-300 ffn2 shape, one box
@pytest.mark.parametrize("M,N,Kin", [(1000, 768, 607), (130, 384, 136), (257, 256, 200), (19200, 768, 3072), (64, 96, 8)])
@pytest.mark.parametrize("act,p", [("relu", 0.1), ("gelu", 0.0), ("gelu", 0.1)])
def test_dgrad_aux_by_tma(M, N, Kin, act, p, tile):
    """The saved activation at a 16-byte-aligned pitch (loaded by TMA into the output box) against the same aux at a pitch
    that cannot take a TMA map (per-element loads): bitwise equal, no write outside [M, Kin], and close to fp64."""
    Kp = (Kin + 7) // 8 * 8
    g, w = rnd(M, N).bfloat16(), rnd(N, Kp, scale=N ** -0.5).bfloat16()[:, :Kin]
    aux = rnd(M, Kin, seed=3, scale=1.5).bfloat16()
    if act == "relu":
        aux = torch.relu(aux)
    aux_al = torch.zeros(M, Kp + 8, dtype=torch.bfloat16, device="cuda")
    aux_al[:, :Kin] = aux
    aux_odd = torch.zeros(M, Kin + 1 if (Kin + 1) % 8 else Kin + 3, dtype=torch.bfloat16, device="cuda")
    aux_odd[:, :Kin] = aux
    out_pitch = Kp + 8
    got = torch.full((M + 64, out_pitch), SENT, dtype=torch.bfloat16, device="cuda")
    ref = torch.full((M + 64, out_pitch), SENT, dtype=torch.bfloat16, device="cuda")
    _dgrad(g, w, act, aux_al[:, :Kin], p, got[:M, :Kin])
    _dgrad(g, w, act, aux_odd[:, :Kin], p, ref[:M, :Kin])
    torch.cuda.synchronize()
    assert torch.equal(got, ref)
    assert (got[:, Kin:] == SENT).all() and (got[M:] == SENT).all()
    if p == 0.0:
        a = aux.double()
        deriv = (a > 0).double() if act == "relu" else \
            0.5 * (1 + torch.erf(a / 2 ** 0.5)) + a * torch.exp(-a * a / 2) / (2 * torch.pi) ** 0.5
        prod = g.double() @ w.double()
        mag = g.double().abs() @ w.double().abs()
        exact = prod * deriv
        # accumulation, the derivative's erf / exp approximations (< 1e-6 absolute), the bf16 store
        tol = gamma_n(N + 1) * mag * deriv.abs() + 1e-6 * prod.abs() + 2.0 ** -8 * exact.abs()
        assert ((got[:M, :Kin].double() - exact).abs() <= tol).all()
