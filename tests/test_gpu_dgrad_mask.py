"""The ReLU-backward mask of the window-conv data gradient on generic bf16 data, at the two learner layers.

The masked data gradient must equal the unmasked one with every element whose saved activation is <= 0 set to zero,
bit for bit: the mask is applied to the rounded bf16 result, so nothing but the mask may differ.  The epilogue
requests the mask words of a row in groups before it stores them; a ragged last tile (positions past the end of the
batch) and both output layouts (conv3 onto the 12x12 grid, conv2 onto the 21x21 image of 32 channels) are covered."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _dgrad_pair(dgrid, wt, k, out_shape, act, out_mode):
    from parl_b200 import kernels as K
    masked = torch.zeros(out_shape, device=DEV, dtype=torch.bfloat16)
    plain = torch.zeros(out_shape, device=DEV, dtype=torch.bfloat16)
    K.conv2d_s1_nhwc_bf16_dgrad(dgrid, wt, k, k, masked, act_mask=act, out_mode=out_mode)
    K.conv2d_s1_nhwc_bf16_dgrad(dgrid, wt, k, k, plain, out_mode=out_mode)
    torch.cuda.synchronize()
    return masked, plain


@pytest.mark.parametrize('N', [977, 4096])
def test_conv3_dgrad_mask_matches_unmasked(N):
    """conv3: da3g [N,11,11,64] -> da2g [N,12,12,64], mask a2 [N,11,11,64]."""
    g = torch.Generator(device=DEV).manual_seed(N)
    dgrid = torch.randn((N, 11, 11, 64), device=DEV, generator=g).to(torch.bfloat16)
    wt = (0.05 * torch.randn((64, 576), device=DEV, generator=g)).to(torch.bfloat16)
    act = torch.randn((N, 11, 11, 64), device=DEV, generator=g).to(torch.bfloat16)
    masked, plain = _dgrad_pair(dgrid, wt, 3, (N, 12, 12, 64), act, 0)
    keep = torch.zeros((N, 12, 12, 64), device=DEV, dtype=torch.bool)
    keep[:, :11, :11] = act > 0
    assert plain.abs().amax().item() > 0
    assert torch.equal(masked, torch.where(keep, plain, torch.zeros_like(plain)))


@pytest.mark.parametrize('N', [977, 4096])
def test_conv2_dgrad_mask_matches_unmasked(N):
    """conv2 (2x2 block form): da2g [N,12,12,64] -> da1g [N,21,21,32] (out_mode 2), mask a1 [N,12,12,128]."""
    g = torch.Generator(device=DEV).manual_seed(N + 1)
    dgrid = torch.randn((N, 12, 12, 64), device=DEV, generator=g).to(torch.bfloat16)
    wt = (0.05 * torch.randn((128, 256), device=DEV, generator=g)).to(torch.bfloat16)
    act = torch.randn((N, 12, 12, 128), device=DEV, generator=g).to(torch.bfloat16)
    masked, plain = _dgrad_pair(dgrid, wt, 2, (N, 21, 21, 32), act, 2)
    # channel block (dy,dx) of block position (Y,X) is pixel (2Y+dy-2, 2X+dx-2) of the image
    keep = (act > 0).view(N, 12, 12, 2, 2, 32).permute(0, 1, 3, 2, 4, 5).reshape(N, 24, 24, 32)[:, 2:23, 2:23]
    assert plain.abs().amax().item() > 0
    assert torch.equal(masked, torch.where(keep, plain, torch.zeros_like(plain)))
