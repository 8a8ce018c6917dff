"""BIT-EXACT checks of the wgmma network kernels on integer-valued operands.

bf16 tensor-core kernels cannot meet a 1e-4 tolerance against an fp32 network on generic data (the operands are
rounded to 8 mantissa bits), so closeness tests alone cannot tell "right up to rounding" from "slightly wrong".  Here
every operand is a small integer — exactly representable in bf16, every product exact, every fp32 partial sum exact
(< 2^24) and every result a small integer again (|v| <= 256, exact in bf16) — so the kernels must reproduce a float32
torch reference of the same layer EXACTLY: any wrong tap shift, channel permutation, swizzle phase, mask or
accumulator mix-up shows up as an integer-sized error.  Covers the three layer shapes of the Atari actor-critic
(benchmark/torch/a2c/atari_model.py:26-44) for forward, data gradient and weight gradient, and the linear layers."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F = torch.nn.functional


def _ints(shape, lo, hi, g, density=1.0):
    x = torch.randint(lo, hi + 1, shape, device=DEV, generator=g).float()
    if density < 1.0:
        x = x * (torch.rand(shape, device=DEV, generator=g) < density).float()
    return x


LAYERS = [(33, 21, 64, 32, 2), (200, 21, 64, 32, 2), (17, 12, 128, 64, 2), (130, 12, 128, 64, 2), (9, 11, 64, 64, 3),
          (260, 11, 64, 64, 3)]


@pytest.fixture(params=[0, 1], ids=['per_tap', 'coltaps_fused'])
def conv_form(request):
    """Both tile forms of the TMA-window conv (rl_debug_set_shiftconv_form); the default is restored afterwards."""
    from parl_b200 import kernels as K
    K.set_shiftconv_form(request.param)
    yield request.param
    K.set_shiftconv_form(0)


@pytest.mark.parametrize('N,H,Cin,Cout,k', LAYERS)
def test_conv_forward_exact_on_integers(N, H, Cin, Cout, k, conv_form):
    from parl_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(N * 7 + H)
    x = _ints((N, H, H, Cin), -2, 2, g)
    w = _ints((Cout, Cin, k, k), -1, 1, g, density=0.08)
    b = _ints((Cout, ), -3, 3, g)
    ref = torch.relu(F.conv2d(x.permute(0, 3, 1, 2), w, b)).permute(0, 2, 3, 1)
    assert ref.abs().max().item() <= 256
    w_krsc = w.permute(0, 2, 3, 1).reshape(Cout, k * k * Cin).contiguous().to(torch.bfloat16)
    out = K.conv2d_s1_nhwc_bf16_fwd(x.to(torch.bfloat16), w_krsc, b, k, k, relu=True)
    torch.cuda.synchronize()
    assert torch.equal(out.float(), ref)


@pytest.mark.parametrize('N', [5, 150])
def test_conv1_block_layout_output_exact_on_integers(N, conv_form):
    """out_mode 1: conv1's 20x20x32 map written as conv2's zero-padded 2x2 space-to-depth input [N,12,12,128]."""
    from parl_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(N)
    x = _ints((N, 21, 21, 64), -2, 2, g)
    w = _ints((32, 64, 2, 2), -1, 1, g, density=0.08)
    b = _ints((32, ), -3, 3, g)
    ref = torch.relu(F.conv2d(x.permute(0, 3, 1, 2), w, b)).permute(0, 2, 3, 1)            # [N,20,20,32]
    pad = torch.zeros(N, 24, 24, 32, device=DEV)
    pad[:, 2:22, 2:22] = ref
    blocks = pad.view(N, 12, 2, 12, 2, 32).permute(0, 1, 3, 2, 4, 5).reshape(N, 12, 12, 128)
    w_krsc = w.permute(0, 2, 3, 1).reshape(32, 256).contiguous().to(torch.bfloat16)
    out = torch.zeros(N, 12, 12, 128, device=DEV, dtype=torch.bfloat16)
    K.conv2d_s1_nhwc_bf16_fwd(x.to(torch.bfloat16), w_krsc, b, 2, 2, relu=True, out=out, out_mode=1)
    torch.cuda.synchronize()
    assert torch.equal(out.float(), blocks)


@pytest.mark.parametrize('N,H,Cin,Cout,k', [(9, 11, 64, 64, 3), (160, 11, 64, 64, 3), (11, 12, 128, 64, 2),
                                            (90, 12, 128, 64, 2)])
def test_conv_dgrad_exact_on_integers(N, H, Cin, Cout, k, conv_form):
    from parl_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(N * 3 + H)
    Ho = H - k + 1
    x = _ints((N, H, H, Cin), -1, 2, g)                                   # saved activation: mask = x > 0
    w = _ints((Cout, Cin, k, k), -1, 1, g, density=0.08)
    dout = _ints((N, Ho, Ho, Cout), -2, 2, g)
    xin = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    F.conv2d(xin, w).backward(dout.permute(0, 3, 1, 2))
    ref = xin.grad.permute(0, 2, 3, 1) * (x > 0)
    assert ref.abs().max().item() <= 256
    dgrid = torch.zeros(N, H, H, Cout, device=DEV, dtype=torch.bfloat16)
    dgrid[:, :Ho, :Ho] = dout.to(torch.bfloat16)
    wt = w.permute(1, 2, 3, 0).reshape(Cin, k * k * Cout).contiguous().to(torch.bfloat16)
    out = torch.zeros(N, H, H, Cin, device=DEV, dtype=torch.bfloat16)
    K.conv2d_s1_nhwc_bf16_dgrad(dgrid, wt, k, k, out, act_mask=x.to(torch.bfloat16))
    torch.cuda.synchronize()
    assert torch.equal(out.float(), ref)


@pytest.mark.parametrize('N,H,Cin,Cout,k', LAYERS)
def test_conv_wgrad_and_bias_grad_exact_on_integers(N, H, Cin, Cout, k):
    from parl_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(N + H * 5)
    Ho = H - k + 1
    x = _ints((N, H, H, Cin), -2, 2, g)
    dout = _ints((N, Ho, Ho, Cout), -2, 2, g, density=0.3)
    w = torch.zeros(Cout, Cin, k, k, device=DEV, requires_grad=True)
    F.conv2d(x.permute(0, 3, 1, 2), w).backward(dout.permute(0, 3, 1, 2))
    ref = w.grad.permute(0, 2, 3, 1).reshape(Cout, -1)
    assert ref.abs().max().item() < 2 ** 24                               # float32 sums of integers stay exact
    dgrid = torch.zeros(N, H, H, Cout, device=DEV, dtype=torch.bfloat16)
    dgrid[:, :Ho, :Ho] = dout.to(torch.bfloat16)
    db = torch.empty(Cout, device=DEV)
    dw = K.conv2d_s1_nhwc_bf16_wgrad(dgrid, x.to(torch.bfloat16), k, k, db=db)
    torch.cuda.synchronize()
    assert torch.equal(dw, ref)
    assert torch.equal(db, dout.sum((0, 1, 2)))


@pytest.mark.parametrize('M,N,K_', [(300, 512, 5184), (4096, 19, 512), (129, 130, 72), (2048, 512, 5184)])
def test_gemm_exact_on_integers(M, N, K_):
    from parl_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(M + N)
    a = _ints((M, K_), -2, 2, g, density=0.5)
    b = _ints((N, K_), -1, 1, g, density=0.02)
    bias = _ints((N, ), -4, 4, g)
    ref = torch.relu(a @ b.t() + bias)
    assert ref.abs().max().item() <= 256
    for dt in (torch.float32, torch.bfloat16):
        out = K.gemm_bf16_tn(a.to(torch.bfloat16), b.to(torch.bfloat16), bias, relu=True, out_dtype=dt)
        torch.cuda.synchronize()
        assert torch.equal(out.float(), ref), dt


def test_masked_gemm_exact_on_integers():
    """dX = (dY . W) * (act > 0): the fc data gradient with the ReLU mask fused in the epilogue."""
    from parl_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(9)
    M, N, K_ = 700, 576, 512
    dy = _ints((M, K_), -2, 2, g, density=0.4)
    wT = _ints((N, K_), -1, 1, g, density=0.03)                           # rows = output features of the product
    act = _ints((M, N), -1, 1, g)
    ref = (dy @ wT.t()) * (act > 0)
    assert ref.abs().max().item() <= 256
    out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    K.gemm_bf16_tn_masked(dy.to(torch.bfloat16), wT.to(torch.bfloat16), act.to(torch.bfloat16), out)
    torch.cuda.synchronize()
    assert torch.equal(out.float(), ref)
