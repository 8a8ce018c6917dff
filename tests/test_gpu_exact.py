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
# shapes large enough to wrap every ring under a cap of 1 or 2 CTAs; tiles of 128 positions: 114 ragged, 441 exact,
# 690 ragged, 45 exact, 147 ragged, 35 ragged, 246 ragged
WRAP_LAYERS = [(33, 21, 64, 32, 2), (128, 21, 64, 32, 2), (200, 21, 64, 32, 2), (40, 12, 128, 64, 2),
               (130, 12, 128, 64, 2), (37, 11, 64, 64, 3), (260, 11, 64, 64, 3)]
SM_LIMITS = [0, 1, 2, 57, 75]
SENTINEL = 0x7FC1                                                         # a bf16 NaN no kernel writes


@pytest.fixture(params=[0, 1], ids=['per_tap', 'coltaps_fused'])
def conv_form(request):
    """Both tile forms of the TMA-window conv (rl_debug_set_shiftconv_form); the default is restored afterwards."""
    from parl_b200 import kernels as K
    K.set_shiftconv_form(request.param)
    try:
        yield request.param
    finally:
        K.set_shiftconv_form(0)


@pytest.fixture
def sm_limit(request):
    """CTA caps of the persistent kernels (rl_set_sm_limit): 0 = one per SM; 1 and 2 make every CTA walk its TMA ring
    many times round (stage reuse, parity flips, both consumer warpgroups on each slot of an odd ring); 57 and 75 are
    the actor and learner caps of the pipelined engine, which also change the GEMM's tile width and split-K."""
    from parl_b200 import kernels as K
    K.set_sm_limit(request.param)
    try:
        yield request.param
    finally:
        K.set_sm_limit(0)


def _id(v):
    return ('mask' if v else 'nomask') if isinstance(v, bool) else str(v)


def _cases(base, wrap, base_id_len):
    """Parameters (..., sm_limit): each base case on the whole GPU under its original id, then every wrap case under
    every CTA cap (ids end in -sms<k>)."""
    out = [pytest.param(*c, 0, id='-'.join(_id(v) for v in c[:base_id_len])) for c in base]
    out += [pytest.param(*c, k, id='-'.join(_id(v) for v in c) + '-sms%d' % k)
            for c in wrap for k in SM_LIMITS if not (k == 0 and c in base)]
    return out


def _assert_ring_wraps(positions, sm_limit, min_tiles_per_cta=17):
    """Under a cap of 1 or 2 CTAs, each CTA must take enough 128-position tiles to wrap the deepest ring (8) twice."""
    tiles = -(-positions // 128)
    if sm_limit in (1, 2):
        assert tiles / min(tiles, sm_limit) >= min_tiles_per_cta, (positions, sm_limit)


def _sentinel(shape):
    return torch.full(shape, SENTINEL, device=DEV, dtype=torch.int16).view(torch.bfloat16)


@pytest.mark.parametrize('N,H,Cin,Cout,k,sm_limit', _cases(LAYERS, WRAP_LAYERS, 5), indirect=['sm_limit'])
def test_conv_forward_exact_on_integers(N, H, Cin, Cout, k, conv_form, sm_limit):
    from parl_b200 import kernels as K
    _assert_ring_wraps(N * H * H, sm_limit)
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


# OG: the output grid.  conv3's production call writes the 11x11 input grid onto the 12x12 grid conv2's weight gradient
# reads, whose row and column 11 must stay as they are (zero there).
@pytest.mark.parametrize('N,H,Cin,Cout,k,OG,masked,sm_limit', _cases(
    [(9, 11, 64, 64, 3, 11, True), (160, 11, 64, 64, 3, 11, True), (11, 12, 128, 64, 2, 12, True),
     (90, 12, 128, 64, 2, 12, True)],
    [(N, H, Ci, Co, k, OG, m) for (N, H, Ci, Co, k, OG) in [(37, 11, 64, 64, 3, 11), (160, 11, 64, 64, 3, 12),
                                                            (128, 11, 64, 64, 3, 12), (40, 12, 128, 64, 2, 12),
                                                            (90, 12, 128, 64, 2, 12)] for m in (True, False)], 5),
    indirect=['sm_limit'])
def test_conv_dgrad_exact_on_integers(N, H, Cin, Cout, k, OG, masked, conv_form, sm_limit):
    from parl_b200 import kernels as K
    _assert_ring_wraps(N * H * H, sm_limit)
    g = torch.Generator(device=DEV).manual_seed(N * 3 + H)
    Ho = H - k + 1
    x = _ints((N, H, H, Cin), -1, 2, g)                                   # saved activation: mask = x > 0
    w = _ints((Cout, Cin, k, k), -1, 1, g, density=0.08)
    dout = _ints((N, Ho, Ho, Cout), -2, 2, g)
    xin = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    F.conv2d(xin, w).backward(dout.permute(0, 3, 1, 2))
    ref = xin.grad.permute(0, 2, 3, 1) * (x > 0) if masked else xin.grad.permute(0, 2, 3, 1)
    assert ref.abs().max().item() <= 256
    dgrid = torch.zeros(N, H, H, Cout, device=DEV, dtype=torch.bfloat16)
    dgrid[:, :Ho, :Ho] = dout.to(torch.bfloat16)
    wt = w.permute(1, 2, 3, 0).reshape(Cin, k * k * Cout).contiguous().to(torch.bfloat16)
    out = _sentinel((N, OG, OG, Cin))
    K.conv2d_s1_nhwc_bf16_dgrad(dgrid, wt, k, k, out, act_mask=x.to(torch.bfloat16) if masked else None)
    torch.cuda.synchronize()
    assert torch.equal(out[:, :H, :H].float(), ref)
    untouched = torch.ones(OG, OG, dtype=torch.bool, device=DEV)
    untouched[:H, :H] = False
    assert (out.view(torch.int16)[:, untouched] == SENTINEL).all()


@pytest.mark.parametrize('N', [40, 90])
@pytest.mark.parametrize('masked', [True, False], ids=['mask', 'nomask'])
@pytest.mark.parametrize('sm_limit', SM_LIMITS, ids=lambda k: 'sms%d' % k, indirect=True)
def test_conv2_dgrad_block_layout_exact_against_strided_conv(N, masked, conv_form, sm_limit):
    """out_mode 2: conv2's data gradient in the network's own form (2x2 filter over the 2x2 space-to-depth blocks of
    da2g [N,12,12,64]) written as the 20x20 image of 32 channels on conv1's 21x21 gradient grid, against the original
    4x4 / stride-2 / pad-2 layer.  Operands are laid out as the engine lays them out (train_net.py); the mask's padding
    cells are positive, so only the image bounds of the copy-out keep padding-position gradients out of da1g, whose
    row and column 20 must stay as they are.  Worst error on an H100 80GB HBM3 (700 W): 0, every case bit-exact."""
    from parl_b200 import kernels as K
    _assert_ring_wraps(N * 144, sm_limit)
    g = torch.Generator(device=DEV).manual_seed(N + 17)
    img = _ints((N, 32, 20, 20), -1, 2, g)                                 # conv2's input (saved a1): mask = img > 0
    w = _ints((64, 32, 4, 4), -1, 1, g, density=0.08)
    dout = _ints((N, 64, 11, 11), -2, 2, g)
    xin = img.clone().requires_grad_(True)
    F.conv2d(xin, w, stride=2, padding=2).backward(dout)
    ref = (xin.grad * (img > 0) if masked else xin.grad).permute(0, 2, 3, 1)   # [N,20,20,32]
    assert ref.abs().max().item() <= 256
    dgrid = torch.zeros(N, 12, 12, 64, device=DEV, dtype=torch.bfloat16)
    dgrid[:, :11, :11] = dout.permute(0, 2, 3, 1).to(torch.bfloat16)
    w2p = w.view(64, 32, 2, 2, 2, 2).permute(0, 2, 4, 3, 5, 1)                  # (o, a, b, dy, dx, c)
    w2T = w2p.permute(3, 4, 5, 1, 2, 0).reshape(128, 256).contiguous().to(torch.bfloat16)
    pad = torch.ones(N, 24, 24, 32, device=DEV)                               # positive padding: would pass the mask
    pad[:, 2:22, 2:22] = img.permute(0, 2, 3, 1)
    act = pad.view(N, 12, 2, 12, 2, 32).permute(0, 1, 3, 2, 4, 5).reshape(N, 12, 12, 128).to(torch.bfloat16)
    out = _sentinel((N, 21, 21, 32))
    K.conv2d_s1_nhwc_bf16_dgrad(dgrid, w2T, 2, 2, out, act_mask=act if masked else None, out_mode=2)
    torch.cuda.synchronize()
    assert torch.equal(out[:, :20, :20].float(), ref)
    assert (out.view(torch.int16)[:, 20] == SENTINEL).all() and (out.view(torch.int16)[:, :, 20] == SENTINEL).all()


@pytest.mark.parametrize('N,H,Cin,Cout,k,sm_limit', _cases(LAYERS, WRAP_LAYERS, 5), indirect=['sm_limit'])
def test_conv_wgrad_and_bias_grad_exact_on_integers(N, H, Cin, Cout, k, sm_limit):
    from parl_b200 import kernels as K
    _assert_ring_wraps(N * H * H, sm_limit)
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


GEMMS = [(300, 512, 5184), (4096, 19, 512), (129, 130, 72), (2048, 512, 5184)]


@pytest.mark.parametrize('M,N,K_,sm_limit', _cases(GEMMS, GEMMS, 3), indirect=['sm_limit'])
def test_gemm_exact_on_integers(M, N, K_, sm_limit):
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
    _masked_gemm_exact()


@pytest.mark.parametrize('sm_limit', SM_LIMITS[1:], ids=lambda k: 'sms%d' % k, indirect=True)
def test_masked_gemm_exact_on_integers_under_sm_limit(sm_limit):
    """The masked GEMM under the CTA caps, which change its tile width."""
    _masked_gemm_exact()


def _masked_gemm_exact():
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
