"""wgmma dense layer (dpvo_linear_f16) vs an fp32 torch reference of the same op."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ref(x, w, b, epi, res=None, gate=None, gather=None):
    x = x.float()
    if gather is not None:
        x = torch.where(gather[:, None] >= 0, x[gather.clamp(min=0)], torch.zeros((), device=x.device))
    y = x @ w.float().t() + (b if b is not None else 0)
    if epi == 1:
        y = F.relu(y)
    elif epi == 2:
        y = torch.sigmoid(y)
    elif epi == 3:
        y = res.float() + y
    elif epi == 4:
        y = res.float() + gate.float() * y
    return y


@pytest.mark.parametrize("rows,N,K", [(128, 192, 64), (1000, 384, 384), (4097, 384, 896), (300, 768, 384), (47712, 384, 384), (5, 32, 64)])
@pytest.mark.parametrize("epi", [0, 1, 2])
def test_linear_plain(ext, rows, N, K, epi):
    g = torch.Generator(device=DEV).manual_seed(rows + N + K + epi)
    x = (torch.randn(rows, K, generator=g, device=DEV) * 0.5).half()
    w = (torch.randn(N, K, generator=g, device=DEV) / K ** 0.5).half()
    b = torch.randn(N, generator=g, device=DEV)
    y = ext[3].linear_f16(x, w, b, epi)
    ref = _ref(x, w, b, epi)
    assert y.shape == (1, rows, N) and y.dtype == torch.half
    err = (y[0].float() - ref).abs().max().item()
    assert err <= 2e-3 * max(1.0, ref.abs().max().item()), err
    y32 = ext[3].linear_f16(x, w, b, epi, out_f32=True)
    assert (y32[0] - ref).abs().max().item() <= 2e-4 * max(1.0, ref.abs().max().item())


def test_linear_gather_residual_gate(ext):
    g = torch.Generator(device=DEV).manual_seed(5)
    rows, N, K = 3000, 384, 384
    x = (torch.randn(rows, K, generator=g, device=DEV) * 0.5).half()
    w = (torch.randn(N, K, generator=g, device=DEV) / K ** 0.5).half()
    b = torch.randn(N, generator=g, device=DEV)
    idx = torch.randint(-1, rows, (rows,), generator=g, device=DEV)
    y = ext[3].linear_f16(x, w, b, 1, gather=idx, out_f32=True)
    assert (y[0] - _ref(x, w, b, 1, gather=idx)).abs().max().item() < 1e-3
    res = torch.randn(1, rows, N, generator=g, device=DEV)
    gate = torch.rand(1, rows, N, generator=g, device=DEV).half()
    ref3 = _ref(x, w, b, 3, res=res[0])
    ref4 = _ref(x, w, b, 4, res=res[0], gate=gate[0])
    out = res.clone()
    out16 = torch.empty(1, rows, N, device=DEV, dtype=torch.half)
    r = ext[3].linear_f16(x, w, b, 3, res=out, out_f32=True, out=out, out16=out16)     # in place on the residual
    assert r.data_ptr() == out.data_ptr()
    assert (out[0] - ref3).abs().max().item() < 1e-3
    assert torch.equal(out16, out.half())
    y4 = ext[3].linear_f16(x, w, b, 4, res=res, gate=gate, out_f32=True)
    assert (y4[0] - ref4).abs().max().item() < 1e-3


def test_linear_stacked_gate_and_strided_operands(ext):
    """the GatedResidual block as the update operator runs it: gate and first residual layer stacked in one GEMM
    (sigmoid | relu halves), whose two halves then feed the gated layer as STRIDED operand views"""
    g = torch.Generator(device=DEV).manual_seed(9)
    rows, D = 5000, 384
    x = (torch.randn(rows, D, generator=g, device=DEV) * 0.5).half()
    wg, wa, wb = [(torch.randn(D, D, generator=g, device=DEV) / D ** 0.5).half() for _ in range(3)]
    bg, ba, bb = [torch.randn(D, generator=g, device=DEV) for _ in range(3)]
    res = torch.randn(1, rows, D, generator=g, device=DEV)
    ga = ext[3].linear_f16(x, torch.cat([wg, wa], 0).contiguous(), torch.cat([bg, ba], 0), 5)
    assert ga.shape == (1, rows, 2 * D)
    ref_gate, ref_r1 = _ref(x, wg, bg, 2), _ref(x, wa, ba, 1)
    assert (ga[0, :, :D].float() - ref_gate).abs().max().item() < 2e-3
    assert (ga[0, :, D:].float() - ref_r1).abs().max().item() <= 2e-3 * ref_r1.abs().max().item()
    out = ext[3].linear_f16(ga[..., D:], wb, bb, 4, res=res, gate=ga[..., :D], out_f32=True)
    ref = _ref(ga[0, :, D:], wb, bb, 4, res=res[0], gate=ga[0, :, :D])
    assert (out[0] - ref).abs().max().item() < 1e-3


def test_linear_no_bias_and_bad_shapes(ext):
    x = torch.randn(64, 128, device=DEV).half()
    w = torch.randn(64, 128, device=DEV).half()
    y = ext[3].linear_f16(x, w, None, 0)
    assert (y[0].float() - x.float() @ w.float().t()).abs().max().item() < 5e-2
    with pytest.raises(RuntimeError):
        ext[3].linear_f16(torch.randn(8, 100, device=DEV).half(), torch.randn(16, 100, device=DEV).half(), None, 0)   # K % 64
