"""Bit-exact checks of the learner's bf16 glue kernels (csrc/elementwise.cu), which run on the library fc path the
learner batch takes (AtariTrainNet with N > 16384): the fc bias + ReLU after the library GEMM, and the fc data
gradient's ReLU mask + move from the compact [N,9,9,64] product onto conv3's 11x11 gradient grid.  Both kernels
compute in fp32 and round to nearest even once, as torch's float32 -> bfloat16 conversion does, so they must match a
torch reference bit for bit.  The larger sizes make the grid-stride loops (at most 148 * 16 blocks) run twice.
Worst error on an H100 80GB HBM3 (700 W): 0, every case bit-exact."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SENTINEL = 0x7FC1                                                         # a bf16 NaN no kernel writes


@pytest.mark.parametrize('relu', [True, False], ids=['relu', 'linear'])
@pytest.mark.parametrize('M', [7, 16385])
def test_bias_act_bf16_bit_exact(M, relu):
    from parl_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(M)
    x = (2 * torch.randn((M, 512), device=DEV, generator=g)).to(torch.bfloat16)
    bias = torch.randn(512, device=DEV, generator=g)                      # a different bias in every column
    ref = x.float() + bias
    if relu:
        ref.relu_()
    got = K.bias_act_bf16(x.clone(), bias, relu=relu)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), ref.to(torch.bfloat16).view(torch.int16))


@pytest.mark.parametrize('N', [3, 977])
def test_mask_scatter_grid_bf16_bit_exact(N):
    """dst[:, :9, :9] = src * (act > 0) with masked elements +0; every other cell of the 11x11 grid untouched.  The
    saved activations include +0 and -0, which must be masked."""
    from parl_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(N)
    src = torch.randn((N, 5184), device=DEV, generator=g).to(torch.bfloat16)
    act = torch.randn((N, 9, 9, 64), device=DEV, generator=g)
    zero = torch.rand(act.shape, device=DEV, generator=g)
    act = torch.where(zero < 0.1, 0.0, torch.where(zero < 0.2, -0.0, act)).to(torch.bfloat16)
    dst = torch.full((N, 11, 11, 64), SENTINEL, device=DEV, dtype=torch.int16).view(torch.bfloat16)
    K.mask_scatter_grid_bf16(src, act, dst, N, 9, 9, 11, 11, 64)
    torch.cuda.synchronize()
    ref = torch.where(act > 0, src.view(N, 9, 9, 64), torch.zeros((), device=DEV, dtype=torch.bfloat16))
    assert torch.equal(dst[:, :9, :9].view(torch.int16), ref.view(torch.int16))
    outside = torch.ones(11, 11, dtype=torch.bool, device=DEV)
    outside[:9, :9] = False
    assert (dst.view(torch.int16)[:, outside] == SENTINEL).all()
