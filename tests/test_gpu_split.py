"""fp32-level verification of the wgmma kernels with float32 outputs (VERDICT r1 "pin network parity properly").

bf16 operands cannot meet 1e-4 against an fp32 network on generic data, which leaves the question whether the kernels
are RIGHT or merely as noisy as autocast.  Here every fp32 operand is split into two bf16 pieces, x = hi + lo with
hi = bf16(x), lo = bf16(x - hi) (|x - hi - lo| <= 2^-17 |x|), the kernel is run on the four piece products and the
float32 results are summed: (a_hi + a_lo)(b_hi + b_lo) reproduces the fp32 product to ~2^-16 relative, so the sum must
agree with a float64 torch reference to ~1e-5 of the output scale (asserted: 1e-4) — far inside bf16
rounding (4e-3).  Any mis-accumulation (dropped K step, wrong tap shift, lost split-K partial, fp16-ish accumulate)
would show at the 1e-3 level and up.  Covers the GEMM (plain and split-K paths, the learner's fc shape included) and
the TMA-window weight gradient at the three conv layer shapes; the conv forward / data gradient write bf16 activations
and are pinned bit-exactly on integer operands in test_gpu_exact.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def split(x):
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize('M,N,K', [(256, 512, 5184), (4096, 512, 5184), (1000, 512, 576), (300, 19, 512), (129, 130, 72)])
def test_gemm_split_operands_reach_fp32(M, N, K):
    from parl_b200 import kernels as K_
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a = torch.randn(M, K, device=DEV, generator=g)
    b = torch.randn(N, K, device=DEV, generator=g) / K ** 0.5
    ref = (a.double() @ b.double().t()).float()
    out = torch.zeros(M, N, device=DEV)
    for pa in split(a):
        for pb in split(b):
            out += K_.gemm_bf16_tn(pa, pb, None, relu=False, out_dtype=torch.float32)
    torch.cuda.synchronize()
    err = (out - ref).abs().max().item() / ref.abs().max().item()
    one = K_.gemm_bf16_tn(a.to(torch.bfloat16), b.to(torch.bfloat16), None, relu=False, out_dtype=torch.float32)
    err_bf16 = (one - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-4, (err, err_bf16)
    assert err < 0.1 * err_bf16, (err, err_bf16)        # and far inside what one bf16 pass gives


@pytest.mark.parametrize('N,H,Cin,Cout,k', [(150, 11, 64, 64, 3), (40, 12, 128, 64, 2), (160, 21, 64, 32, 2)])
def test_conv_wgrad_split_operands_reach_fp32(N, H, Cin, Cout, k):
    """conv3 / conv2' / conv1' weight-gradient shapes (positions as the GEMM K dimension, up to 70 560 positions)."""
    from parl_b200 import kernels as K_
    g = torch.Generator(device=DEV).manual_seed(N + H + Cout)
    Ho = H - k + 1
    x = torch.randn(N, H, H, Cin, device=DEV, generator=g)
    dout = torch.randn(N, Ho, Ho, Cout, device=DEV, generator=g)
    # reference: dW[co, (r, s, ci)] = sum over samples and positions of dout[n, y, x, co] * x[n, y + r, x + s, ci], as k*k
    # float64 matrix products (cuDNN's float64 convolution backward takes a minute at these shapes)
    ref = torch.empty(Cout, k, k, Cin, device=DEV, dtype=torch.float64)
    dflat = dout.double().reshape(-1, Cout)
    for r in range(k):
        for c in range(k):
            ref[:, r, c, :] = dflat.t() @ x[:, r:r + Ho, c:c + Ho, :].double().reshape(-1, Cin)
    ref = ref.reshape(Cout, -1).float()
    dw = torch.zeros(Cout, k * k * Cin, device=DEV)
    for px in split(x):
        for pd in split(dout):
            dgrid = torch.zeros(N, H, H, Cout, device=DEV, dtype=torch.bfloat16)
            dgrid[:, :Ho, :Ho] = pd
            K_.conv2d_s1_nhwc_bf16_wgrad(dgrid, px.contiguous(), k, k, dw_krsc=dw, accumulate=True)
    torch.cuda.synchronize()
    scale = ref.abs().max().item()
    err = (dw - ref).abs().max().item() / scale
    dgrid = torch.zeros(N, H, H, Cout, device=DEV, dtype=torch.bfloat16)
    dgrid[:, :Ho, :Ho] = dout.to(torch.bfloat16)
    one = K_.conv2d_s1_nhwc_bf16_wgrad(dgrid, x.to(torch.bfloat16), k, k)
    err_bf16 = (one - ref).abs().max().item() / scale
    assert err < 1e-4, (err, err_bf16)
    assert err < 0.1 * err_bf16, (err, err_bf16)
