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


# bf16 bit patterns: +0, -0, the smallest subnormals, the largest subnormals, the smallest normals, +-inf, NaNs, the
# largest finite values and +-1
SPECIAL = [0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x807F, 0x0080, 0x8080, 0x7F80, 0xFF80, 0x7FC0, 0xFFC0, 0x7F7F, 0xFF7F,
           0x3F80, 0xBF80]


def test_relu_backward_masks_agree_on_special_values():
    """The learner's three ReLU-backward masks are one function, "keep where act > 0" as torch evaluates it:
    the window-conv data-gradient epilogue (packed bf16x2 compare), the masked GEMM (fp32 compare) and
    rl_mask_scatter_grid_bf16 (fp32 compare), on saved activations holding signed zeros, subnormals, infinities and
    NaNs.  Gradients are negative everywhere, so a masked element must come out as +0 (no sign of a product).
    On an H100 80GB HBM3 (700 W) all three keep exactly the elements torch's act > 0 keeps, subnormals included."""
    from parl_b200 import kernels as K
    N = 64
    g = torch.Generator(device=DEV).manual_seed(7)
    codes = torch.tensor([v - 65536 if v >= 32768 else v for v in SPECIAL], dtype=torch.int16, device=DEV)
    act = codes[torch.randint(0, len(SPECIAL), (N, 11, 11, 64), device=DEV, generator=g)].view(torch.bfloat16)
    keep = act.double() > 0
    assert torch.equal(keep, act.cpu().double().gt(0).to(DEV)) and torch.equal(keep, act > 0)
    assert bool(keep[act.view(torch.int16) == 0x0001].all()) and not bool(keep[act.view(torch.int16) == 0x7FC0].any())

    def check(masked, plain):
        assert bool((plain.float() < 0).all())
        want = torch.where(keep, plain, torch.zeros_like(plain))
        assert torch.equal(masked.view(torch.int16), want.view(torch.int16))

    # 1) conv3's data gradient: every position of the 11x11 grid receives a negative sum
    dgrid = torch.zeros((N, 11, 11, 64), device=DEV, dtype=torch.bfloat16)
    dgrid[:, :9, :9] = -torch.randint(1, 3, (N, 9, 9, 64), device=DEV, generator=g).to(torch.bfloat16)
    wt = torch.full((64, 576), 1.0 / 64, device=DEV, dtype=torch.bfloat16)
    masked, plain = _dgrad_pair(dgrid, wt, 3, (N, 11, 11, 64), act, 0)
    check(masked, plain)
    # 2) the masked GEMM: rows = positions, columns = channels
    dy = -torch.randint(1, 3, (N * 121, 64), device=DEV, generator=g).to(torch.bfloat16)
    w = torch.full((64, 64), 1.0 / 64, device=DEV, dtype=torch.bfloat16)
    out = torch.empty((N * 121, 64), device=DEV, dtype=torch.bfloat16)
    K.gemm_bf16_tn_masked(dy, w, act.view(N * 121, 64), out)
    plain = (dy.float() @ w.float().t()).to(torch.bfloat16)
    torch.cuda.synchronize()
    check(out.view(N, 11, 11, 64), plain.view(N, 11, 11, 64))
    # 3) the compact-to-grid mask
    src = -torch.randint(1, 4, (N, 11, 11, 64), device=DEV, generator=g).to(torch.bfloat16)
    dst = torch.empty((N, 11, 11, 64), device=DEV, dtype=torch.bfloat16)
    K.mask_scatter_grid_bf16(src, act, dst, N, 11, 11, 11, 11, 64)
    torch.cuda.synchronize()
    check(dst, src)
