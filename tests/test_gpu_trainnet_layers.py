"""Layer-by-layer check of the learner network (AtariTrainNet): every kernel call of one forward_from_x0() + backward()
against a float64 reference of the original layer, in the model's NCHW layout and parameters.

Each reference takes the net's own saved bf16 tensors as its inputs (x0, a1, a2, a3, h, dheads, dh, da3g, da2g,
da1g), so one comparison isolates one call and its layout glue, and the bounds can be tight:
  * bf16 activations and data gradients: |got - ref| <= R * 2^-8 |ref| + 2^-16 S, where S is the same reference run on
    |operands| (the sum of |terms|) and R counts the bf16 roundings (1; 2 where the library fc path rounds the product
    and then bias_act rounds again, the second rounding also relative to the product).  Masked elements are exactly
    zero, and grid cells outside each valid region (a1's zero padding, da3g outside 9x9, row and column 11 of da2g,
    row and column 20 of da1g) are zero.
  * logits and values (float32 from bf16 h): |got - ref| <= 2^-16 S.
  * every model parameter's .grad: |got - ref| <= 2^-8 |ref| + 2^-16 S for the bf16-output library products (fc
    weight; heads weights above 4096 samples), |got - ref| <= 2^-19 S for the fp32 sums (conv weights, all biases,
    heads weights up to 4096 samples).
A wrong operand, a wrong permutation into a .grad or one slightly wrong layer moves some element by a sizeable
fraction of |ref|, far outside these bounds.

Worst |got - ref| / bound over the five cases, one run on an H100 80GB HBM3 (700 W): 0.992 for the bf16 activations
and data gradients (one rounding uses up to 2^-8 |ref|: bf16 keeps 8 significant bits), 0.93 for h on the library
path, 0.009 for logits and values, 0.992 for the bf16-output weight gradients, 0.11 for the fp32 weight and bias
gradients (0.0139 of 2^-16 S, at N = 20000).  Peak device memory: 6.7 GB allocated by torch at N = 20000.

References are float64 matrix products over F.unfold / F.fold columns, chunked over samples (weight gradients
accumulate across chunks in float64), which keeps the device memory of the largest case to a few GB."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F = torch.nn.functional
CHUNK = 512
EPS = 2.0 ** -8          # one bf16 rounding, relative
ACC = 2.0 ** -16         # fp32 accumulation, relative to the sum of |terms|
ACC_W = 2.0 ** -19       # fp32 weight-gradient sums of the wgmma kernels and colsum (no bf16 rounding)


def _conv(x, w, b, stride, pad):
    """float64 conv as unfold + matmul: returns (y, S) with S the same conv of |x|, |w|, |b|."""
    n, _, H, W = x.shape
    O, _, k, _ = w.shape
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    cols = F.unfold(x, k, padding=pad, stride=stride)
    wm = w.reshape(O, -1)
    y = (wm @ cols + b.view(1, O, 1)).view(n, O, Ho, Wo)
    s = (wm.abs() @ cols.abs() + b.abs().view(1, O, 1)).view(n, O, Ho, Wo)
    return y, s


def _conv_dgrad(dy, w, hw, stride, pad):
    """Data gradient of a conv (w [O,C,k,k]) with respect to an input of size hw, and its sum of |terms|."""
    n, O = dy.shape[:2]
    k = w.shape[-1]
    wm = w.reshape(O, -1).t()
    d = dy.reshape(n, O, -1)
    dx = F.fold(wm @ d, hw, k, padding=pad, stride=stride)
    s = F.fold(wm.abs() @ d.abs(), hw, k, padding=pad, stride=stride)
    return dx, s


def _conv_wgrad(dy, x, k, stride, pad):
    """Weight and bias gradient sums of one chunk (float64) and their sums of |terms|."""
    n, O = dy.shape[:2]
    cols = F.unfold(x, k, padding=pad, stride=stride)                   # [n, C*k*k, L]
    d = dy.reshape(n, O, -1).transpose(0, 1).reshape(O, -1)             # [O, n*L]
    c = cols.transpose(0, 1).reshape(cols.shape[1], -1).t()             # [n*L, C*k*k]
    return d @ c, d.abs() @ c.abs(), d.sum(1), d.abs().sum(1)


class _Ratios(object):
    """Worst |got - ref| / bound per checked tensor."""

    def __init__(self):
        self.r = {}

    def add(self, name, got, ref, bound):
        r = ((got.double() - ref).abs() / bound.clamp_min(1e-30)).max().item()
        self.r[name] = max(self.r.get(name, 0.0), r)


def _blocks_to_image(a1):
    """a1 [n,12,12,128] (zero-padded 2x2-block layout) -> the padded image [n,24,24,32]."""
    n = a1.shape[0]
    return a1.view(n, 12, 12, 2, 2, 32).permute(0, 1, 3, 2, 4, 5).reshape(n, 24, 24, 32)


def layer_ratios(N, fc_backend, sm_limit=0, seed=0, A=18):
    """Run the net once and return ({tensor: worst error / bound}, list of structural failures)."""
    from parl_b200 import kernels as K
    from parl_b200.engine.nets import AtariActorCritic
    from parl_b200.engine.train_net import AtariTrainNet
    torch.manual_seed(seed)
    model = AtariActorCritic(A).to(DEV)
    with torch.no_grad():            # non-zero biases so that every path is exercised
        for p in model.parameters():
            if p.dim() == 1:
                p.normal_(0, 0.1)
    for p in model.parameters():
        p.grad = torch.zeros_like(p)
    net = AtariTrainNet(model, N, DEV, fc_backend=fc_backend)
    obs = torch.randint(0, 256, (N, 4, 84, 84), dtype=torch.uint8, device=DEV)
    d_logits = torch.randn(N, A, device=DEV) * 0.1
    d_values = torch.randn(N, device=DEV) * 0.1
    K.set_sm_limit(sm_limit)
    try:
        K.obs_stack_gather(obs, None, 0, 1, net.x0, scale=1.0 / 255.0, s2d=True)
        net.forward_from_x0()
        net.backward(d_logits, d_values)
        torch.cuda.synchronize()
    finally:
        K.set_sm_limit(0)
    lib = net.fc_library
    bf = lambda t: t.detach().to(torch.bfloat16).double()                # the operand copies the kernels read
    W1, W2, W3, Wfc, Wpi, Wv = (bf(getattr(model, m).weight) for m in ('conv1', 'conv2', 'conv3', 'fc', 'fc_pi', 'fc_v'))
    b1, b2, b3, bfc, bpi, bv = (getattr(model, m).bias.detach().double()
                                for m in ('conv1', 'conv2', 'conv3', 'fc', 'fc_pi', 'fc_v'))
    R, bad = _Ratios(), []
    wsum = {k: 0.0 for k in ('w1', 'w2', 'w3', 'wfc', 'wh', 'b1', 'b2', 'b3', 'bfc', 'bh')}
    wabs = dict(wsum)
    for i in range(0, N, CHUNK):
        j = min(N, i + CHUNK)
        n = j - i
        # ---- saved tensors, in NCHW
        xb = (obs[i:j].float() * (1.0 / 255.0)).to(torch.bfloat16)
        pad = torch.zeros((n, 4, 88, 88), device=DEV, dtype=torch.bfloat16)
        pad[:, :, 1:85, 1:85] = xb
        x0_want = pad[:, :, :84, :84].reshape(n, 4, 21, 4, 21, 4).permute(0, 2, 4, 3, 5, 1).reshape(n, 21, 21, 64)
        if not torch.equal(net.x0[i:j], x0_want):
            bad.append('x0')
        x = xb.double()
        a1p = _blocks_to_image(net.a1[i:j])
        if a1p[:, :2].any() or a1p[:, 22:].any() or a1p[:, :, :2].any() or a1p[:, :, 22:].any():
            bad.append('a1 padding')
        a1 = a1p[:, 2:22, 2:22].permute(0, 3, 1, 2).double()              # [n,32,20,20]
        a2 = net.a2[i:j].permute(0, 3, 1, 2).double()                     # [n,64,11,11]
        a3 = net.a3[i:j].permute(0, 3, 1, 2).double()                     # [n,64,9,9]
        h = net.h[i:j].double()
        dheads = net.dheads[i:j, :A + 1].double()
        dh = net.dh[i:j].double()
        da3 = net.da3g[i:j, :9, :9].permute(0, 3, 1, 2).double()
        da2 = net.da2g[i:j, :11, :11].permute(0, 3, 1, 2).double()
        da1 = net.da1g[i:j, :20, :20].permute(0, 3, 1, 2).double()
        # ---- forward
        y, s = _conv(x, W1, b1, 4, 1)
        R.add('a1', a1, y.relu(), EPS * y.abs() + ACC * s)
        y, s = _conv(a1, W2, b2, 2, 2)
        R.add('a2', a2, y.relu(), EPS * y.abs() + ACC * s)
        y, s = _conv(a2, W3, b3, 1, 0)
        R.add('a3', a3, y.relu(), EPS * y.abs() + ACC * s)
        f = a3.reshape(n, 5184)                                           # (c,h,w) order, as nn.Flatten
        acc = f @ Wfc.t()
        y, s = acc + bfc, f.abs() @ Wfc.abs().t() + bfc.abs()
        R.add('h', h, y.relu(), EPS * y.abs() + ACC * s + (EPS * acc.abs() if lib else 0))
        for name, out, w, b in (('logits', net.logits[i:j], Wpi, bpi), ('values', net.values[i:j], Wv, bv)):
            R.add(name, out, h @ w.t() + b, ACC * (h.abs() @ w.abs().t() + b.abs()))
        # ---- backward: data gradients
        dl = torch.cat([Wpi, Wv])                                         # [A+1, 512]
        y = (dheads @ dl) * (h > 0)
        R.add('dh', dh, y, EPS * y.abs() + ACC * (dheads.abs() @ dl.abs()))
        if (dh[h <= 0] != 0).any():
            bad.append('dh mask')
        y = (dh @ Wfc).view(n, 64, 9, 9) * (a3 > 0)
        R.add('da3', da3, y, EPS * y.abs() + ACC * (dh.abs() @ Wfc.abs()).view(n, 64, 9, 9))
        g3 = net.da3g[i:j]
        if (da3[a3 <= 0] != 0).any() or g3[:, 9:].any() or g3[:, :, 9:].any():
            bad.append('da3g mask / grid')
        y, s = _conv_dgrad(da3, W3, (11, 11), 1, 0)
        y = y * (a2 > 0)
        R.add('da2', da2, y, EPS * y.abs() + ACC * s)
        g2 = net.da2g[i:j]
        if (da2[a2 <= 0] != 0).any() or g2[:, 11:].any() or g2[:, :, 11:].any():
            bad.append('da2g mask / grid')
        y, s = _conv_dgrad(da2, W2, (20, 20), 2, 2)
        y = y * (a1 > 0)
        R.add('da1', da1, y, EPS * y.abs() + ACC * s)
        g1 = net.da1g[i:j]
        if (da1[a1 <= 0] != 0).any() or g1[:, 20:].any() or g1[:, :, 20:].any():
            bad.append('da1g mask / grid')
        # ---- backward: conv weight and bias gradients (sums over chunks)
        for key, dy, xin, k, st, pd in (('1', da1, x, 8, 4, 1), ('2', da2, a1, 4, 2, 2), ('3', da3, a2, 3, 1, 0)):
            dw, sw, db, sb = _conv_wgrad(dy, xin, k, st, pd)
            wsum['w' + key] = wsum['w' + key] + dw
            wabs['w' + key] = wabs['w' + key] + sw
            wsum['b' + key] = wsum['b' + key] + db
            wabs['b' + key] = wabs['b' + key] + sb
        # ---- fc and head weight / bias gradients (the heads' from the bf16 copy of the loss gradients the net keeps)
        for key, dy, xin in (('fc', dh, f), ('h', dheads, h)):
            wsum['w' + key] = wsum['w' + key] + dy.t() @ xin
            wabs['w' + key] = wabs['w' + key] + dy.abs().t() @ xin.abs()
            wsum['b' + key] = wsum['b' + key] + dy.sum(0)
            wabs['b' + key] = wabs['b' + key] + dy.abs().sum(0)
    refs = {'fc.weight': (wsum['wfc'].view(512, 5184), wabs['wfc'].view(512, 5184), 1),
            'fc.bias': (wsum['bfc'], wabs['bfc'], 0),
            'fc_pi.weight': (wsum['wh'][:A], wabs['wh'][:A], int(N > 4096)),
            'fc_v.weight': (wsum['wh'][A:], wabs['wh'][A:], int(N > 4096)),
            'fc_pi.bias': (d_logits.double().sum(0), d_logits.double().abs().sum(0), 0),
            'fc_v.bias': (d_values.double().sum().view(1), d_values.double().abs().sum().view(1), 0)}
    for key in ('1', '2', '3'):
        shape = getattr(model, 'conv' + key).weight.shape
        refs['conv%s.weight' % key] = (wsum['w' + key].view(shape), wabs['w' + key].view(shape), 0)
        refs['conv%s.bias' % key] = (wsum['b' + key], wabs['b' + key], 0)
    params = dict(model.named_parameters())
    for name, (ref, s, rounds) in refs.items():
        R.add(name, params[name].grad, ref, EPS * ref.abs() + ACC * s if rounds else ACC_W * s)
    return R.r, bad


@pytest.mark.parametrize('N,fc_backend,sm_limit', [(977, 'native', 0), (977, 'library', 0), (5000, 'native', 0),
                                                   (20000, 'auto', 0), (977, 'native', 75)])
def test_train_net_every_call_matches_float64_layer(N, fc_backend, sm_limit):
    ratios, bad = layer_ratios(N, fc_backend, sm_limit)
    assert not bad, bad
    worst = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not worst, worst
