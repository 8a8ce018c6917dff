"""Exact and near-exact checks of the fused fp32 MLP kernels (csrc/mlp.cu: rl_mlp_fwd, rl_mlp_bwd and its grad-reduce
kernel) against float64 references written here.

Exact regime (ReLU and identity nets).  x, W and b are small integers and d_out is an integer times 2^-6, so every
fp32 product and partial sum the kernels form is exact in any order as long as the sum of |terms| of every
accumulated quantity stays below 2^24 grid units.  The reference computes those magnitudes next to the float64 result
(|W| |h| + |b| for each pre-activation, |d| |W| for each delta, sum_n |d| |h| and sum_n |d| for each weight and bias
gradient, plus |old| when accumulating) and asserts that precondition, so the kernels must then match bit for bit:
an indexing, padding, segment or tile-walk bug is a hard mismatch, whatever its magnitude.  The nets run every
template instantiation (forward JT = 1, 2, 4, 8; delta KT = 1, 2, 4, 8; weight gradient with G = in_p / 4 odd and
not a power of two), depths 1 to 4, hidden layers split into row segments (one without a bias), all 8 segments,
every split point of a 7-output net, and batches that put a ragged tile on a CTA's second and third pass of the
grid-stride loop.  Hidden units that are dead on every sample must get weight and bias gradients of exactly +0.

Tanh regime (the production nets: PPO MuJoCo 17-64-64 with heads 6+1, A2C CartPole 4-64 and 4-64-64 with heads 2+1,
the policy-gradient CartPole 4-20-2).  Random fp32 data; every output and gradient must lie within a per-element
float64 bound, with u = 2^-24 and gamma(k) = k u / (1 - k u):
  * forward   e_l = |W_l| e_{l-1} + gamma(k_l) (|W_l| |h_{l-1}| + |b_l|), k_l = padded input width + 1 (the bias); a
              hidden tanh adds 2 ulp of its output (2^-22 (|h| + e));
  * backward  the delta error goes back through |W_l^T| the same way (k = padded output width) and through the
              derivative 1 - h^2 with 2 |h| e_h + e_h^2 + 3u, plus one rounding of the product;
  * gradients sum_n (e_d |h| + |d| e_h + e_d e_h) + gamma(k_w) sum_n (|d| + e_d)(|h| + e_h) with
              k_w = 64 (one tile's fma chain) + tiles per CTA + ceil(grid / 32) + 5 (the reduce's shuffle tree).
Worst measured |got - ref| / bound on an H100 80GB HBM3 (700 W), over all 16 tanh cases: forward outputs 0.063
(PG CartPole, n = 131 109), weight gradients 0.066, bias gradients 0.024 (both at n = 1, where the bound has the
least slack).

Argument checks: every rejection the library documents raises RuntimeError with its message before any launch.
The largest exact-regime nets keep rl_mlp_bwd's shared memory (parameters, saved activations, two delta tiles) under
its 220 KB limit; test_mlp_rejects_bad_plans checks that a net over it is refused."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
RELU, TANH, NONE = 0, 1, 2
KD = 6                       # d_out (and so every delta and gradient) lives on the integer grid times 2^-KD
LIM = 2.0 ** 24
TS = 68                      # shared-memory row stride of one feature row of a tile (floats)


def _pad(d):
    return 16 if d <= 16 else 32 if d <= 32 else 64 if d <= 64 else 128


def _layout(dims):
    """(padded widths, padded parameter count, backward shared memory bytes) as csrc/mlp.cu lays the net out."""
    L = len(dims) - 1
    pd = [(dims[0] + 3) // 4 * 4] + [_pad(d) for d in dims[1:]]
    np_pad = sum(pd[l + 1] * pd[l] + pd[l + 1] for l in range(L))
    smem_bwd = (np_pad + 3) // 4 * 4 * 4 + sum(pd[:L]) * TS * 4 + 2 * 128 * TS * 4
    return pd, np_pad, smem_bwd


def _nsm():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _bwd_grid(dims, n):
    """CTAs rl_mlp_bwd launches: 2 per SM when the backward's shared memory fits twice (<= 110 KB), else 1."""
    per_sm = 2 if _layout(dims)[2] <= 110 * 1024 else 1
    return min((n + 63) // 64, per_sm * _nsm()), per_sm


def _ints(shape, lo, hi, density, gen, dev):
    v = torch.randint(lo, hi + 1, shape, generator=gen, device=dev).double()
    if density < 1:
        v = v * (torch.rand(shape, generator=gen, device=dev, dtype=torch.float64) < density)
    return v


class Net(object):
    """An integer-grid net: W[l], b[l] float64 (exact small integers), split into row segments per layer."""

    def __init__(self, dims, act, segs=None, nobias=(), dead=0, w_density=1.0, seed=0, dev=DEV):
        gen = torch.Generator(device=dev).manual_seed(seed)
        self.dims, self.act, self.L = tuple(dims), act, len(dims) - 1
        self.segs = segs if segs is not None else [[d] for d in dims[1:]]
        self.nobias = set(nobias)
        self.W, self.b, self.dead = [], [], []
        bound = torch.full((dims[0], ), 2.0, dtype=torch.float64, device=dev)       # max |x|
        for l in range(self.L):
            W = _ints((dims[l + 1], dims[l]), -1, 1, w_density, gen, dev)
            b = _ints((dims[l + 1], ), -2, 2, 1.0, gen, dev)
            has_b = torch.ones(dims[l + 1], dtype=torch.bool)
            for g, rows in enumerate(self.segs[l]):   # a segment without a bias has b = 0 on its rows
                if (l, g) in self.nobias:
                    r0 = sum(self.segs[l][:g])
                    b[r0:r0 + rows] = 0
                    has_b[r0:r0 + rows] = False
            dl = []
            if dead and act == RELU and l + 1 < self.L:
                # units whose pre-activation is negative on every sample: W row kept, bias below -sum |W| max|h|
                dl = [j for j in range(1, dims[l + 1], max(1, dims[l + 1] // dead)) if has_b[j]][:dead]
                for j in dl:
                    b[j] = -(W[j].abs() @ bound).item() - 1
            self.W.append(W)
            self.b.append(b)
            self.dead.append(dl)
            bound = W.abs() @ bound + b.abs()
            if act == RELU:
                bound = bound.clone()
                bound[dl] = 0

    def plan(self):
        from parl_b200 import kernels
        self.dev_segs = []
        layers = []
        for l in range(self.L):
            r0, lay = 0, []
            for g, rows in enumerate(self.segs[l]):
                w = self.W[l][r0:r0 + rows].float().contiguous().to(DEV)
                b = None if (l, g) in self.nobias else self.b[l][r0:r0 + rows].float().contiguous().to(DEV)
                lay.append((w, b))
                self.dev_segs.append((l, r0, rows, b is not None))
                r0 += rows
            layers.append(lay)
        return kernels.MlpPlan(layers, self.act)

    def grads_like(self, fill=float('nan')):
        return [(torch.full((rows, self.dims[l]), fill, device=DEV),
                 torch.full((rows, ), fill, device=DEV) if hb else None) for (l, r0, rows, hb) in self.dev_segs]

    def data(self, n, x_range=2, d_range=2, d_density=1.0, seed=1, dev=DEV):
        gen = torch.Generator(device=dev).manual_seed(seed)
        x = _ints((n, self.dims[0]), -x_range, x_range, 1.0, gen, dev)
        d = _ints((n, self.dims[-1]), -d_range, d_range, d_density, gen, dev) * 2.0 ** -KD
        return x, d

    def reference(self, x, d_out):
        """float64 forward and backward, plus the largest sum of |terms| (in grid units) of any accumulation."""
        hs, worst = [x], 0.0
        for l in range(self.L):
            z = hs[-1] @ self.W[l].t() + self.b[l]
            worst = max(worst, (hs[-1].abs() @ self.W[l].abs().t() + self.b[l].abs()).max().item())
            hs.append(z.clamp_min(0) if (self.act == RELU and l + 1 < self.L) else z)
        d, dW, db = d_out, [None] * self.L, [None] * self.L
        for l in reversed(range(self.L)):
            dW[l], db[l] = d.t() @ hs[l], d.sum(0)
            worst = max(worst, (d.abs().t() @ hs[l].abs()).max().item() * 2 ** KD,
                        d.abs().sum(0).max().item() * 2 ** KD)
            if l > 0:
                worst = max(worst, (d.abs() @ self.W[l].abs()).max().item() * 2 ** KD)
                d = d @ self.W[l]
                if self.act == RELU:
                    d = d * (hs[l] > 0)
        return hs[-1], dW, db, worst


def _check_grads(net, grads, dW, db, plus=None):
    for s, (l, r0, rows, hb) in enumerate(net.dev_segs):
        rw, rb = dW[l][r0:r0 + rows], db[l][r0:r0 + rows]
        if plus is not None:
            rw, rb = rw + plus[s][0].double(), (rb + plus[s][1].double() if hb else None)
        assert torch.equal(grads[s][0].double(), rw), ('dW', s, (grads[s][0].double() - rw).abs().max().item())
        if hb:
            assert torch.equal(grads[s][1].double(), rb), ('db', s, (grads[s][1].double() - rb).abs().max().item())


def _dead_are_plus_zero(net, grads):
    for s, (l, r0, rows, hb) in enumerate(net.dev_segs):
        for j in net.dead[l]:
            if r0 <= j < r0 + rows:
                row = grads[s][0][j - r0]
                assert torch.equal(row, torch.zeros_like(row)) and not torch.signbit(row).any(), ('dead dW', l, j)
                if hb:
                    assert grads[s][1][j - r0].item() == 0 and not torch.signbit(grads[s][1][j - r0]).item()


def _run_exact(net, n, x_range=2, d_range=2, d_density=1.0, seed=1):
    """Forward, backward, accumulate and a repeat of one net at batch n, all against the float64 reference."""
    plan = net.plan()
    x, d = net.data(n, x_range, d_range, d_density, seed)
    out_ref, dW, db, worst = net.reference(x, d)
    on_grid = lambda t: None if t is None else torch.randint(-3, 4, t.shape, device=DEV) * 2.0 ** -KD
    old = [(on_grid(a), on_grid(b)) for a, b in net.grads_like()]      # |old| <= 3 grid units
    assert worst + 3 < LIM, 'exactness precondition: %g grid units' % worst
    xf, df = x.float(), d.float()
    out = plan.forward(xf)
    assert torch.equal(out.double(), out_ref), (out.double() - out_ref).abs().max().item()
    grads = net.grads_like()
    plan.backward(xf, df, grads=grads)
    _check_grads(net, grads, dW, db)
    _dead_are_plus_zero(net, grads)
    acc = [(a.clone(), None if b is None else b.clone()) for a, b in old]
    plan.backward(xf, df, grads=acc, accumulate=True)
    _check_grads(net, acc, dW, db, plus=old)
    again = net.grads_like()
    plan.backward(xf, df, grads=again)
    for (a, b), (c, e) in zip(grads, again):
        assert torch.equal(a, c) and (b is None or torch.equal(b, e))
    torch.cuda.synchronize()
    return plan, x, d


# dims, act, n: the forward's out widths cover JT = 1, 2, 4, 8 (<=16, 17..32, 33..64, 65..128), hidden widths
# KT = 1, 2, 4, 8, input widths 1, 3, 5, 9, 17, 100, 128 give G = in_p / 4 = 1, 1, 2, 3, 5, 25, 32
EXACT_NETS = [
    ('L1-1x7', (1, 7), NONE, 777),
    ('L1-17x128', (17, 128), RELU, 300),
    ('L1-9x20', (9, 20), NONE, 129),
    ('L2-5x16x3', (5, 16, 3), RELU, 1000),
    ('L3-9x17x33x2', (9, 17, 33, 2), RELU, 1500),
    ('L2-17x65x128', (17, 65, 128), RELU, 2000),
    ('L2-100x128x7-none', (100, 128, 7), NONE, 700),
    ('L2-128x48x16', (128, 48, 16), RELU, 600),
    ('L4-5x32x16x64x7', (5, 32, 16, 64, 7), RELU, 3000),
    ('L4-3x8x24x8x40-none', (3, 8, 24, 8, 40), NONE, 900),
    ('L3-dqn-4x128x128x2', (4, 128, 128, 2), RELU, 4096),
]


@pytest.mark.parametrize('dims,act,n', [c[1:] for c in EXACT_NETS], ids=[c[0] for c in EXACT_NETS])
def test_mlp_exact_every_instantiation(dims, act, n):
    net = Net(dims, act, dead=2, seed=len(dims) * 1000 + dims[-1])
    _run_exact(net, n)


# hidden layer 1 in three row segments (the middle one without a bias), heads in four (one without a bias): 8 in all
SEG_NET = dict(dims=(6, 40, 24, 7), segs=[[40], [5, 11, 8], [1, 2, 1, 3]], nobias=[(1, 1), (2, 2)])


@pytest.mark.parametrize('act', [RELU, NONE], ids=['relu', 'none'])
@pytest.mark.parametrize('n', [1, 65, 1000])
def test_mlp_exact_segments(act, n):
    net = Net(SEG_NET['dims'], act, segs=SEG_NET['segs'], nobias=SEG_NET['nobias'], dead=2, seed=7)
    assert sum(len(s) for s in net.segs) == 8
    plan, x, d = _run_exact(net, n)
    # the same net given as one segment per layer (the missing biases as zeros) is bit-identical
    one = Net(SEG_NET['dims'], act, dead=2, seed=7)
    one.W, one.b = net.W, net.b
    plan1 = one.plan()
    assert torch.equal(plan.forward(x.float()), plan1.forward(x.float()))
    g8, g1 = net.grads_like(), one.grads_like()
    plan.backward(x.float(), d.float(), grads=g8)
    plan1.backward(x.float(), d.float(), grads=g1)
    for s, (l, r0, rows, hb) in enumerate(net.dev_segs):
        assert torch.equal(g8[s][0], g1[l][0][r0:r0 + rows])
        if hb:
            assert torch.equal(g8[s][1], g1[l][1][r0:r0 + rows])


@pytest.mark.parametrize('act', [RELU, NONE], ids=['relu', 'none'])
def test_mlp_exact_every_split_point(act):
    """forward(split=s) and backward(d_out, d_out2, split=s) equal the unsplit call on the concatenated tensors."""
    net = Net((11, 48, 7), act, segs=[[48], [6, 1]], dead=2, seed=3)
    plan, x, d = _run_exact(net, 333)
    xf, df = x.float(), d.float()
    out = plan.forward(xf)
    ref = net.grads_like()
    plan.backward(xf, df, grads=ref)
    for s in range(1, 7):
        o1, o2 = plan.forward(xf, split=s)
        assert o1.shape == (333, s) and o2.shape == (333, 7 - s)
        assert torch.equal(torch.cat([o1, o2], 1), out), s
        got = net.grads_like()
        plan.backward(xf, df[:, :s].contiguous(), grads=got, d_out2=df[:, s:].contiguous(), split=s)
        for (a, b), (c, e) in zip(got, ref):
            assert torch.equal(a, c) and torch.equal(b, e), s


EDGE_NETS = {'dqn': ((4, 128, 128, 2), 1), 'cartpole': ((4, 20, 2), 2)}


@pytest.mark.parametrize('which', sorted(EDGE_NETS))
@pytest.mark.parametrize('nk', ['1', '63', '64', '65', '64g+1', '128g+37', '131109'])
def test_mlp_exact_batch_edges(which, nk):
    """n = 64 g + 1 puts a one-sample tile on CTA 0's second pass, n = 64 * 2g + 37 a 37-sample tile on its third."""
    dims, per_sm = EDGE_NETS[which]
    g, got_per_sm = _bwd_grid(dims, 1 << 30)
    assert got_per_sm == per_sm and g == per_sm * _nsm()
    n = {'64g+1': 64 * g + 1, '128g+37': 64 * 2 * g + 37}.get(nk) or int(nk)
    net = Net(dims, RELU, dead=2, w_density=0.5, seed=11)
    _run_exact(net, n, x_range=1, d_range=1, d_density=min(1.0, 2048.0 / n), seed=n)


# --------------------------------------------------------------------------- tanh regime: the production nets
def _gamma(k):
    u = 2.0 ** -24
    return k * u / (1 - k * u)


TANH_NETS = {
    'ppo-17x64x64+6+1': ((17, 64, 64), (6, 1)),
    'a2c-4x64+2+1': ((4, 64), (2, 1)),
    'a2c-4x64x64+2+1': ((4, 64, 64), (2, 1)),
    'pg-4x20x2': ((4, 20), (2, )),
}


@pytest.mark.parametrize('n', [1, 777, 2048, 131072 + 37])
@pytest.mark.parametrize('which', sorted(TANH_NETS))
def test_mlp_tanh_within_fp32_bound(which, n):
    from parl_b200 import kernels
    trunk, heads = TANH_NETS[which]
    torch.manual_seed(n + len(which))
    dims = trunk + (sum(heads), )
    L, O = len(dims) - 1, dims[-1]
    lin = [torch.nn.Linear(trunk[i], trunk[i + 1]) for i in range(len(trunk) - 1)]
    hd = [torch.nn.Linear(trunk[-1], h) for h in heads]
    for m in lin + hd:
        m.to(DEV)
    plan = kernels.MlpPlan([[(m.weight.detach(), m.bias.detach())] for m in lin] +
                           [[(m.weight.detach(), m.bias.detach()) for m in hd]], kernels.ACT_TANH)
    W = [m.weight.detach().double() for m in lin] + [torch.cat([m.weight.detach().double() for m in hd])]
    B = [m.bias.detach().double() for m in lin] + [torch.cat([m.bias.detach().double() for m in hd])]
    x = torch.randn(n, dims[0], device=DEV)
    d_out = torch.randn(n, O, device=DEV)
    split = heads[0] if len(heads) > 1 else 0
    if split:
        o1, o2 = plan.forward(x, split=split)
        out = torch.cat([o1, o2], 1)
        dW = [torch.empty_like(w, dtype=torch.float32) for w in W[:-1]] + [m.weight.detach().clone() for m in hd]
        dB = [torch.empty_like(b, dtype=torch.float32) for b in B[:-1]] + [m.bias.detach().clone() for m in hd]
        grads = list(zip(dW, dB))
        plan.backward(x, d_out[:, :split].contiguous(), grads=grads, d_out2=d_out[:, split:].contiguous(),
                      split=split)
        gw = [g[0] for g in grads[:L - 1]] + [torch.cat([g[0] for g in grads[L - 1:]])]
        gb = [g[1] for g in grads[:L - 1]] + [torch.cat([g[1] for g in grads[L - 1:]])]
    else:
        out = plan.forward(x)
        grads = [(torch.empty_like(w, dtype=torch.float32), torch.empty_like(b, dtype=torch.float32))
                 for w, b in zip(W, B)]
        plan.backward(x, d_out, grads=grads)
        gw, gb = [g[0] for g in grads], [g[1] for g in grads]
    pd = _layout(dims)[0]
    u = 2.0 ** -24
    # forward reference and its error bound
    hs, es = [x.double()], [torch.zeros_like(x, dtype=torch.float64)]
    for l in range(L):
        A = hs[-1].abs() @ W[l].abs().t() + B[l].abs()
        z = hs[-1] @ W[l].t() + B[l]
        e = es[-1] @ W[l].abs().t() + _gamma(pd[l] + 1) * A
        if l + 1 < L:
            z = torch.tanh(z)
            e = e + 2.0 ** -22 * (z.abs() + e)
        hs.append(z)
        es.append(e)
    ratios = {'out': ((out.double() - hs[-1]).abs() / es[-1]).max().item()}
    assert ((out.double() - hs[-1]).abs() <= es[-1]).all(), ('out', ratios['out'])
    # backward
    grid, _ = _bwd_grid(dims, n)
    tiles = (n + 63) // 64
    kw = 64 + (tiles + grid - 1) // grid + (grid + 31) // 32 + 5
    d, ed = d_out.double(), torch.zeros(n, O, dtype=torch.float64, device=DEV)
    ratios['dW'] = ratios['db'] = 0.0
    for l in reversed(range(L)):
        h, eh = hs[l], es[l]
        rw, rb = d.t() @ h, d.sum(0)
        bw = ed.t() @ h.abs() + d.abs().t() @ eh + ed.t() @ eh + _gamma(kw) * ((d.abs() + ed).t() @ (h.abs() + eh))
        bb = ed.sum(0) + _gamma(kw) * (d.abs() + ed).sum(0)
        ew, eb = (gw[l].double() - rw).abs(), (gb[l].double() - rb).abs()
        ratios['dW'] = max(ratios['dW'], (ew / bw).max().item())
        ratios['db'] = max(ratios['db'], (eb / bb).max().item())
        assert (ew <= bw).all(), ('dW', l, (ew / bw).max().item())
        assert (eb <= bb).all(), ('db', l, (eb / bb).max().item())
        if l > 0:
            acc = d @ W[l]
            eacc = ed @ W[l].abs() + _gamma(pd[l + 1]) * (d.abs() @ W[l].abs())
            der = 1 - h * h
            eder = 2 * h.abs() * eh + eh * eh + 3 * u
            ed = eacc * (der.abs() + eder) + acc.abs() * eder + u * (acc.abs() + eacc) * (der.abs() + eder)
            d = acc * der
    print('mlp tanh %s n=%d worst ratio: %s' % (which, n, ' '.join('%s %.3g' % kv for kv in sorted(ratios.items()))))


# --------------------------------------------------------------------------- argument checks
def _lin(rows, cols):
    return torch.zeros(rows, cols, device=DEV), torch.zeros(rows, device=DEV)


def _still_works():
    """A rejected call launched nothing and left no error behind: a valid call runs and is right."""
    from parl_b200 import kernels
    torch.cuda.synchronize()
    w = torch.ones(3, 2, device=DEV)
    out = kernels.MlpPlan([[(w, None)]], kernels.ACT_NONE).forward(torch.ones(5, 2, device=DEV))
    assert torch.equal(out, torch.full((5, 3), 2.0, device=DEV))


@pytest.mark.parametrize('case', ['5-layers', 'width-129', '9-segments', 'bwd-smem'])
def test_mlp_rejects_bad_plans(case):
    from parl_b200 import kernels
    if case == '5-layers':
        plan, msg = kernels.MlpPlan([[_lin(8, 4)]] + [[_lin(8, 8)] for _ in range(4)], RELU), r'layers=5 \(1\.\.4\)'
    elif case == 'width-129':
        plan, msg = kernels.MlpPlan([[_lin(129, 4)], [_lin(2, 129)]], RELU), 'width 129 of layer 1 outside 1..128'
    elif case == '9-segments':
        plan, msg = kernels.MlpPlan([[_lin(4, 4)], [_lin(1, 4) for _ in range(8)]], RELU), '9 parameter segments'
    else:
        # (128, 128, 64, 4): the forward fits in 220 KB of shared memory, the backward (saved activations) does not
        plan = kernels.MlpPlan([[_lin(128, 128)], [_lin(64, 128)], [_lin(4, 64)]], RELU)
        xx = torch.randn(100, 128, device=DEV)
        assert _layout((128, 128, 64, 4))[2] > 220 * 1024
        out = plan.forward(xx)
        assert torch.equal(out, torch.zeros_like(out))
        grads = [(torch.empty(r, c, device=DEV), torch.empty(r, device=DEV)) for r, c in ((128, 128), (64, 128), (4, 64))]
        with pytest.raises(RuntimeError, match='mlp_bwd: network too large for shared memory'):
            plan.backward(xx, torch.zeros(100, 4, device=DEV), grads=grads)
        _still_works()
        return
    xx = torch.zeros(10, 4, device=DEV)
    if plan.ws.numel() == 0:                 # rl_mlp_workspace_bytes has no size for 5 layers: the check must still fire
        plan.ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    with pytest.raises(RuntimeError, match=msg):
        plan.forward(xx)
    grads = [(torch.empty_like(w), torch.empty_like(b)) for (_, w, b) in plan.segs]
    with pytest.raises(RuntimeError, match=msg):
        plan.backward(xx, torch.zeros(10, plan.out_dim, device=DEV), grads=grads)
    _still_works()


def test_mlp_rejects_bad_rows_and_splits():
    """Checks MlpPlan cannot reach (it derives the widths from the segments and treats split 0 as no split): the C
    entry points are called directly.  Every buffer is large enough for the unchecked launch, should a check fail."""
    from parl_b200 import _lib, kernels
    from parl_b200._lib import ptr, stream
    lib = _lib.load()
    w1, b1 = torch.randn(10, 6, device=DEV), torch.randn(10, device=DEV)
    w2, b2 = torch.randn(7, 10, device=DEV), torch.randn(7, device=DEV)
    plan = kernels.MlpPlan([[(w1, b1)], [(w2, b2)]], RELU)
    n = 50
    x = torch.randn(n, 6, device=DEV)
    big = [torch.randn(n * 12, device=DEV) for _ in range(2)]       # d_out, d_out2 / out, out2
    gw = [torch.empty_like(w1), torch.empty_like(w2)]
    gb = [torch.empty_like(b1), torch.empty_like(b2)]
    c_dw = (ctypes.c_void_p * 2)(gw[0].data_ptr(), gw[1].data_ptr())
    c_db = (ctypes.c_void_p * 2)(gb[0].data_ptr(), gb[1].data_ptr())

    def fwd(dims, out2, split):
        return lib.rl_mlp_fwd(ptr(x), n, 2, dims, 2, plan.c_layer, plan.c_rows, plan.c_w, plan.c_b, RELU, ptr(big[0]),
                              ptr(out2), split, stream())

    def bwd(dims, d2, split, ws_bytes=None):
        return lib.rl_mlp_bwd(ptr(x), n, 2, dims, 2, plan.c_layer, plan.c_rows, plan.c_w, plan.c_b, RELU, ptr(big[0]),
                              ptr(d2), split, c_dw, c_db, 0, ptr(plan.ws),
                              plan.ws.numel() if ws_bytes is None else ws_bytes, stream())

    def err():
        return lib.rl_last_error().decode()

    bad_dims = (ctypes.c_int * 3)(6, 12, 7)                 # the segments of layer 0 cover 10 of 12 rows
    assert fwd(bad_dims, None, 0) == -1 and 'segments of layer 0 cover 10 of 12 rows' in err()
    assert bwd(bad_dims, None, 0) == -1 and 'segments of layer 0 cover 10 of 12 rows' in err()
    for split in (7, 0, -1):                                # split = O and split 0 with a second output
        assert fwd(plan.c_dims, big[1], split) == -1 and 'mlp_fwd: split %d outside 1..6' % split in err()
        assert bwd(plan.c_dims, big[1], split) == -1 and 'mlp_bwd: split %d outside 1..6' % split in err()
    # a workspace one float short of grid * np_pad floats
    grid, _ = _bwd_grid((6, 10, 7), n)
    need = grid * _layout((6, 10, 7))[1] * 4
    assert bwd(plan.c_dims, None, 0, need - 4) == -5 and 'workspace too small' in err()
    assert bwd(plan.c_dims, None, 0, need) == 0
    _still_works()
    ref = torch.relu(x @ w1.t() + b1)
    dref = big[0][:n * 7].view(n, 7)
    assert torch.allclose(gb[1], dref.sum(0), rtol=1e-5, atol=1e-6)
    assert torch.allclose(gw[1], dref.t() @ ref, rtol=1e-5, atol=1e-5)


def test_mlp_plan_workspace_short_raises():
    from parl_b200 import kernels
    dims = (4, 128, 128, 2)
    plan = kernels.MlpPlan([[_lin(128, 4)], [_lin(128, 128)], [_lin(2, 128)]], RELU)
    n = 64 * 1000
    grid, _ = _bwd_grid(dims, n)
    need = grid * _layout(dims)[1] * 4
    full = plan.ws
    plan.ws = full[:need - 4]
    grads = [(torch.empty_like(w), torch.empty_like(b)) for (_, w, b) in plan.segs]
    x, d = torch.zeros(n, 4, device=DEV), torch.zeros(n, 2, device=DEV)
    with pytest.raises(RuntimeError, match=r'code -5\).*workspace too small'):
        plan.backward(x, d, grads=grads)
    plan.ws = full[:need]
    plan.backward(x, d, grads=grads)
    torch.cuda.synchronize()


@pytest.mark.parametrize('dims', [(4, 128, 128, 2), (4, 20, 2), (17, 64, 64, 7), (128, 128, 128, 128, 128)])
def test_mlp_workspace_covers_two_ctas_per_sm(dims):
    from parl_b200 import _lib
    L = len(dims) - 1
    got = _lib.load().rl_mlp_workspace_bytes(L, (ctypes.c_int * (L + 1))(*dims))
    assert got >= 2 * _nsm() * _layout(dims)[1] * 4
