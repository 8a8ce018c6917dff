"""GPU parity: the wgmma/TMA bf16 GEMM against a float32 torch matmul of the same bf16 inputs."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.mark.parametrize('M,N,K', [(128, 64, 64), (256, 512, 5184), (1000, 512, 576), (4096, 32, 256), (300, 19, 512),
                                   (128, 256, 128), (129, 130, 72)])
@pytest.mark.parametrize('relu', [False, True])
def test_gemm_bf16_tn(M, N, K, relu):
    from parl_b200 import kernels as K_
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    b = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV, generator=g)
    ref = a.float() @ b.float().t() + bias
    if relu:
        ref = torch.relu(ref)
    for dt, tol in ((torch.float32, 2e-3), (torch.bfloat16, 1.5e-2)):
        out = K_.gemm_bf16_tn(a, b, bias, relu=relu, out_dtype=dt)
        torch.cuda.synchronize()
        err = (out.float() - ref).abs().max().item()
        assert err < tol * max(1.0, ref.abs().max().item()), (dt, err)


@pytest.mark.parametrize('N,H,Cin,Cout,k,stride,pad', [(3, 21, 64, 32, 2, 1, 0), (5, 20, 32, 64, 4, 2, 2),
                                                        (7, 11, 64, 64, 3, 1, 0), (300, 11, 64, 64, 3, 1, 0),
                                                        (64, 20, 32, 64, 4, 2, 2)])
def test_conv2d_nhwc_bf16_fwd(N, H, Cin, Cout, k, stride, pad):
    """wgmma implicit-GEMM conv vs torch conv2d in float32 on the same bf16 operands (the three layer shapes of
    the Atari actor-critic: s2d conv1, conv2 with padding, conv3)."""
    from parl_b200 import kernels as K_
    g = torch.Generator(device=DEV).manual_seed(N + H + Cin)
    x = torch.randn(N, H, H, Cin, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, k, k, device=DEV, generator=g) / (Cin * k * k) ** 0.5).to(torch.bfloat16)
    b = torch.randn(Cout, device=DEV, generator=g)
    w_krsc = w.permute(0, 2, 3, 1).reshape(Cout, k * k * Cin).contiguous()
    out = K_.conv2d_nhwc_bf16_fwd(x, w_krsc, b, k, k, stride, pad, relu=True)
    torch.cuda.synchronize()
    ref = torch.relu(torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, stride=stride, padding=pad))
    ref = ref.permute(0, 2, 3, 1)
    err = (out.float() - ref).abs().max().item()
    assert out.shape == ref.shape and err < 2e-2 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize('window_form', [True, False])
def test_native_actor_net_matches_torch_model(window_form):
    """The wgmma inference path (s2d conv1 -> conv2 -> conv3 -> fc -> policy head) against the torch model
    (bf16 autocast) on real observations from the device env pool."""
    from parl_b200 import kernels as K_
    from parl_b200.engine.nets import AtariActorCritic
    from parl_b200.engine.actor_net import AtariActorNet
    torch.manual_seed(0)
    B = 300
    model = AtariActorCritic(18).to(DEV)
    net = AtariActorNet(model, B, DEV, window_form=window_form)
    planes = torch.zeros(5, B, 84 * 84, dtype=torch.uint8, device=DEV)
    ages = torch.zeros(2, B, dtype=torch.uint8, device=DEV)
    st = K_.EpisodeStats(B, DEV)
    for p in range(4):
        K_.env_atari_synth_step(planes[p], None, None, None, ages[0], st, 7, p, reset=True)
    ages[0] = 3
    obs = torch.empty(B, 21, 21, 64, dtype=torch.bfloat16, device=DEV)
    K_.obs_stack_gather(planes, ages, 0, 1, obs, scale=1.0 / 255.0, s2d=True)
    logits = torch.empty(B, 18, dtype=torch.float32, device=DEV)
    net.policy(obs, logits)
    val = torch.empty(B, 1, dtype=torch.float32, device=DEV)
    net.value(val)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref_l, ref_v = model.policy_and_value(obs)
    scale = max(1.0, ref_l.abs().max().item())
    assert (logits - ref_l).abs().max().item() < 3e-2 * scale
    assert (val.squeeze(1) - ref_v).abs().max().item() < 3e-2 * max(1.0, ref_v.abs().max().item())
    # fp32 reference of the same function (reference-form network on uint8 NCHW obs)
    u8 = torch.empty(B, 4, 84, 84, dtype=torch.uint8, device=DEV)
    K_.obs_stack_gather(planes, ages, 0, 1, u8)
    m32 = AtariActorCritic(18, compute_dtype=torch.float32).to(DEV)
    m32.load_state_dict(model.state_dict())
    with torch.no_grad():
        l32 = m32.policy(u8)
    assert (logits - l32).abs().max().item() < 5e-2 * scale


@pytest.mark.parametrize('N,H,Cin,Cout,k', [(3, 21, 64, 32, 2), (300, 21, 64, 32, 2), (5, 12, 128, 64, 2),
                                            (200, 12, 128, 64, 2), (7, 11, 64, 64, 3), (300, 11, 64, 64, 3)])
def test_conv2d_s1_tma_window_form(N, H, Cin, Cout, k):
    """The TMA-window (shifted-descriptor) conv against torch conv2d in float32 on the same bf16 operands."""
    from parl_b200 import kernels as K_
    g = torch.Generator(device=DEV).manual_seed(N + H + Cin)
    x = torch.randn(N, H, H, Cin, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, k, k, device=DEV, generator=g) / (Cin * k * k) ** 0.5).to(torch.bfloat16)
    b = torch.randn(Cout, device=DEV, generator=g)
    w_krsc = w.permute(0, 2, 3, 1).reshape(Cout, k * k * Cin).contiguous()
    out = K_.conv2d_s1_nhwc_bf16_fwd(x, w_krsc, b, k, k, relu=True)
    torch.cuda.synchronize()
    ref = torch.relu(torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b)).permute(0, 2, 3, 1)
    err = (out.float() - ref).abs().max().item()
    assert out.shape == ref.shape and err < 2e-2 * max(1.0, ref.abs().max().item()), err


def test_conv1_to_conv2_space_to_depth_chain():
    """conv1 (s2d form) writing conv2's padded 2x2-block input, then conv2 as a 2x2/1 conv: equals the
    reference pair conv(8x8/4/p1) -> relu -> conv(4x4/2/p2) -> relu."""
    from parl_b200 import kernels as K_
    torch.manual_seed(1)
    N = 37
    x = torch.rand(N, 4, 84, 84, device=DEV)
    w1 = (torch.randn(32, 4, 8, 8, device=DEV) / 16).to(torch.bfloat16)
    w2 = (torch.randn(64, 32, 4, 4, device=DEV) / 22).to(torch.bfloat16)
    b1, b2 = torch.randn(32, device=DEV) * 0.1, torch.randn(64, device=DEV) * 0.1
    F = torch.nn.functional
    xb = x.to(torch.bfloat16)
    r1 = torch.relu(F.conv2d(xb.float(), w1.float(), b1, stride=4, padding=1)).to(torch.bfloat16)
    ref = torch.relu(F.conv2d(r1.float(), w2.float(), b2, stride=2, padding=2)).permute(0, 2, 3, 1)
    pad = torch.zeros(N, 4, 85, 85, device=DEV, dtype=torch.bfloat16)
    pad[:, :, 1:, 1:] = xb
    s2d = pad[:, :, :84, :84].reshape(N, 4, 21, 4, 21, 4).permute(0, 2, 4, 3, 5, 1).reshape(N, 21, 21, 64).contiguous()
    w1p = w1.view(32, 4, 2, 4, 2, 4).permute(0, 2, 4, 3, 5, 1).reshape(32, 256).contiguous()      # (o,a,b,dy,dx,c)
    w2p = w2.view(64, 32, 2, 2, 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(64, 512).contiguous()     # (o,a,b,dy,dx,c)
    a1 = torch.zeros(N, 12, 12, 128, device=DEV, dtype=torch.bfloat16)
    K_.conv2d_s1_nhwc_bf16_fwd(s2d, w1p, b1, 2, 2, relu=True, out=a1, out_mode=1)
    out = K_.conv2d_s1_nhwc_bf16_fwd(a1, w2p, b2, 2, 2, relu=True)
    torch.cuda.synchronize()
    err = (out.float() - ref).abs().max().item()
    assert out.shape == ref.shape and err < 3e-2 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize('N,H,Cin,Cout,k', [(5, 11, 64, 64, 3), (150, 11, 64, 64, 3), (40, 12, 128, 64, 2)])
def test_conv2d_s1_dgrad_tma_window_form(N, H, Cin, Cout, k):
    """dgrad of the window-form conv (+ ReLU mask) against torch autograd on the same bf16 operands."""
    from parl_b200 import kernels as K_
    g = torch.Generator(device=DEV).manual_seed(N + H)
    Ho = H - k + 1
    x = torch.randn(N, H, H, Cin, device=DEV, generator=g).to(torch.bfloat16)          # saved (post-ReLU-like) input
    w = (torch.randn(Cout, Cin, k, k, device=DEV, generator=g) / (Cin * k * k) ** 0.5).to(torch.bfloat16)
    dout = torch.randn(N, Ho, Ho, Cout, device=DEV, generator=g).to(torch.bfloat16)
    xin = x.float().permute(0, 3, 1, 2).requires_grad_(True)
    torch.nn.functional.conv2d(xin, w.float()).backward(dout.float().permute(0, 3, 1, 2))
    ref = (xin.grad.permute(0, 2, 3, 1) * (x.float() > 0))
    dgrid = torch.zeros(N, H, H, Cout, device=DEV, dtype=torch.bfloat16)
    dgrid[:, :Ho, :Ho] = dout
    wt = w.permute(1, 2, 3, 0).reshape(Cin, k * k * Cout).contiguous()                 # [ci][(r,s,co)]
    out = torch.zeros(N, H, H, Cin, device=DEV, dtype=torch.bfloat16)
    K_.conv2d_s1_nhwc_bf16_dgrad(dgrid, wt, k, k, out, act_mask=x)
    torch.cuda.synchronize()
    err = (out.float() - ref).abs().max().item()
    assert err < 3e-2 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize('N,H,Cin,Cout,k', [(5, 11, 64, 64, 3), (150, 11, 64, 64, 3), (9, 12, 128, 64, 2),
                                            (7, 21, 64, 32, 2), (160, 21, 64, 32, 2)])
@pytest.mark.parametrize('legacy', [0, 2])
def test_conv2d_s1_wgrad_tma_window_form(N, H, Cin, Cout, k, legacy):
    """Window-form weight gradient (positions as the GEMM K dimension, MN-major wgmma operands) against torch
    autograd on the same bf16 operands.  legacy=0: A = input window, B = dout (Cout=32: SWIZZLE_64B), bias gradient
    in the same pass; legacy=2: operand roles swapped for Cout=64, bias gradient by a column-sum pass."""
    from parl_b200 import kernels as K_, _lib
    _lib.load().rl_debug_set_wgrad_lane_map(legacy)
    try:
        _wgrad_case(K_, N, H, Cin, Cout, k)
    finally:
        _lib.load().rl_debug_set_wgrad_lane_map(0)


def _wgrad_case(K_, N, H, Cin, Cout, k):
    g = torch.Generator(device=DEV).manual_seed(N + H + Cout)
    Ho = H - k + 1
    x = torch.randn(N, H, H, Cin, device=DEV, generator=g).to(torch.bfloat16)
    dout = torch.randn(N, Ho, Ho, Cout, device=DEV, generator=g).to(torch.bfloat16)
    w = torch.zeros(Cout, Cin, k, k, device=DEV, requires_grad=True)
    torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w).backward(dout.float().permute(0, 3, 1, 2))
    ref = w.grad.permute(0, 2, 3, 1).reshape(Cout, -1)
    dgrid = torch.zeros(N, H, H, Cout, device=DEV, dtype=torch.bfloat16)
    dgrid[:, :Ho, :Ho] = dout
    dbf = torch.empty(Cout, device=DEV)
    dw = K_.conv2d_s1_nhwc_bf16_wgrad(dgrid, x, k, k, db=dbf)
    torch.cuda.synchronize()
    assert (dw - ref).abs().max().item() < 1e-3 * max(1.0, ref.abs().max().item())
    db = K_.colsum_bf16(dgrid)
    ref_db = dgrid.float().sum((0, 1, 2))
    assert (db - ref_db).abs().max().item() < 1e-2
    assert (dbf - ref_db).abs().max().item() < 1e-3 * max(1.0, ref_db.abs().max().item())   # fused bias gradient


@pytest.mark.parametrize('N,H,Cin,Cout,k', [(160, 12, 128, 64, 2), (160, 11, 64, 64, 3), (160, 21, 64, 32, 2)])
@pytest.mark.parametrize('legacy', [0, 2])
def test_conv2d_s1_wgrad_without_bias_gradient(N, H, Cin, Cout, k, legacy):
    """db=None changes how the accumulator slots are grouped: the workspace the library reports must still cover a
    full grid of CTAs (more position tiles than SMs), in both weight-gradient forms."""
    from parl_b200 import kernels as K_, _lib
    g = torch.Generator(device=DEV).manual_seed(N + H + Cin)
    Ho = H - k + 1
    x = torch.randn(N, H, H, Cin, device=DEV, generator=g).to(torch.bfloat16)
    dout = torch.randn(N, Ho, Ho, Cout, device=DEV, generator=g).to(torch.bfloat16)
    w = torch.zeros(Cout, Cin, k, k, device=DEV, requires_grad=True)
    torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w).backward(dout.float().permute(0, 3, 1, 2))
    ref = w.grad.permute(0, 2, 3, 1).reshape(Cout, -1)
    dgrid = torch.zeros(N, H, H, Cout, device=DEV, dtype=torch.bfloat16)
    dgrid[:, :Ho, :Ho] = dout
    _lib.load().rl_debug_set_wgrad_lane_map(legacy)
    try:
        dw = K_.conv2d_s1_nhwc_bf16_wgrad(dgrid, x, k, k)
        torch.cuda.synchronize()
    finally:
        _lib.load().rl_debug_set_wgrad_lane_map(0)
    assert (dw - ref).abs().max().item() < 1e-3 * max(1.0, ref.abs().max().item())


def test_conv2d_s1_wgrad_accumulate_and_bias():
    """accumulate=1 adds the weight AND the fused bias gradient to what is already there (paired-tap form)."""
    from parl_b200 import kernels as K_
    g = torch.Generator(device=DEV).manual_seed(11)
    N, H, Cin, Cout, k = 20, 12, 128, 64, 2
    x = torch.randn(N, H, H, Cin, device=DEV, generator=g).to(torch.bfloat16)
    dgrid = torch.zeros(N, H, H, Cout, device=DEV, dtype=torch.bfloat16)
    dgrid[:, :H - k + 1, :H - k + 1] = torch.randn(N, H - k + 1, H - k + 1, Cout, device=DEV, generator=g).to(torch.bfloat16)
    db1 = torch.empty(Cout, device=DEV)
    dw1 = K_.conv2d_s1_nhwc_bf16_wgrad(dgrid, x, k, k, db=db1).clone()
    dw2, db2 = dw1.clone(), db1.clone()
    K_.conv2d_s1_nhwc_bf16_wgrad(dgrid, x, k, k, dw_krsc=dw2, accumulate=True, db=db2)
    torch.cuda.synchronize()
    assert torch.equal(dw2, dw1 + dw1) and torch.equal(db2, db1 + db1)       # deterministic: exactly twice
    assert (db1 - dgrid.float().sum((0, 1, 2))).abs().max().item() < 1e-3 * max(1.0, db1.abs().max().item())


def test_obs_gather_s2d_matches_reference_layout():
    """rl_obs_stack_gather out_dtype 3 (smem-staged, magic-number u8->float) against a torch restatement:
    out[n,Y,X,(dy*4+dx)*4+c] = bf16(frame_c[4Y+dy-1, 4X+dx-1] / 255), zero outside the image."""
    from parl_b200 import kernels as K_
    g = torch.Generator(device=DEV).manual_seed(5)
    n = 37
    obs = torch.randint(0, 256, (n, 4, 84, 84), device=DEV, generator=g, dtype=torch.uint8)
    out = torch.empty((n, 21, 21, 64), device=DEV, dtype=torch.bfloat16)
    K_.obs_stack_gather(obs, None, 0, 1, out, scale=1.0 / 255.0, s2d=True)
    pad = torch.zeros((n, 4, 88, 88), device=DEV)
    pad[:, :, 1:85, 1:85] = obs.float()
    ref = (pad[:, :, :84, :84] * (1.0 / 255.0)).view(n, 4, 21, 4, 21, 4).permute(0, 2, 4, 3, 5, 1).reshape(n, 21, 21, 64)
    torch.cuda.synchronize()
    assert torch.equal(out, ref.to(torch.bfloat16))


@pytest.fixture
def sm_limit(request):
    """CTA caps (rl_set_sm_limit) that change the GEMM's tile width and split-K choice; 57 is the pipelined engine's
    actor cap.  0 (one CTA per SM) is restored afterwards."""
    from parl_b200 import kernels as K_
    K_.set_sm_limit(request.param)
    try:
        yield request.param
    finally:
        K_.set_sm_limit(0)


@pytest.mark.parametrize('heads_mma', [1, 0])
@pytest.mark.parametrize('M,sm_limit', [pytest.param(M, k, id=str(M) if k == 0 else '%d-sms%d' % (M, k))
                                        for M in (96, 512, 4096) for k in (0, 1, 2, 57, 75)], indirect=['sm_limit'])
def test_gemm_heads_fused_matches_separate_calls(M, heads_mma, sm_limit):
    """rl_gemm_bf16_tn_heads (actor fc + policy head; split-K reduce and heads in one kernel at small M) against the
    two separate wgmma GEMMs for H (bit-identical) and an fp32 product of the stored bf16 H for the heads, both under
    the same CTA cap."""
    from parl_b200 import kernels as K_
    torch.manual_seed(M)
    N, Kd, N2 = 512, 5184, 18
    a = (torch.randn(M, Kd, device=DEV) * 0.05).to(torch.bfloat16)
    b = (torch.randn(N, Kd, device=DEV) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV) * 0.1
    w2 = (torch.randn(N2, N, device=DEV) * 0.1).to(torch.bfloat16)
    b2 = torch.randn(N2, device=DEV)
    h = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    out2 = torch.empty(M, N2, device=DEV)
    from parl_b200 import _lib
    _lib.load().rl_debug_set_heads_mma(heads_mma)
    try:
        K_.gemm_bf16_tn_heads(a, b, bias, h, w2, b2, out2)
    finally:
        _lib.load().rl_debug_set_heads_mma(1)
    h_ref = K_.gemm_bf16_tn(a, b, bias, relu=True)
    torch.cuda.synchronize()
    assert torch.equal(h, h_ref)
    ref2 = h.float() @ w2.float().t() + b2
    assert (out2 - ref2).abs().max().item() < 1e-3 * max(1.0, ref2.abs().max().item())
