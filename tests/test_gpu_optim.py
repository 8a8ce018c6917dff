"""The learner update's optimiser kernels (csrc/optim.cu: rl_grad_global_norm, rl_adam_step), FlatAdam around them,
and the PPO minibatch update they end, checked against float64 restatements written here.  u = 2^-24,
gamma(k) = k u / (1 - k u).

grad_global_norm
  * integer gradients with sum g^2 < 2^24: every partial sum is exact, so the result must be
    float32(sqrt(float64 sum g^2)) bit for bit.  The last n % 4 elements are nonzero, so the scalar tail counts.
  * random gradients: |got / ref - 1| <= gamma(k) + u, with k = float4 passes per thread + 18 (4 in one float4
    group, the tail element, 5 shuffle levels, 8 warp partials): all terms are positive, so the bound is rigorous.
  * n reaches 3 * 148 * 8 * 256 * 4 + r, where every thread's float4 loop strides three times.
  * the grid-reduce ticket is back at 0 after each call: calls of different grid sizes and an a2c_loss_fwd_bwd
    sharing the same workspace leave the norm bit-identical.
adam_step, against torch.optim.Adam (foreach off) after the clip, restated in float64 with the float32
hyperparameters the kernel receives and the float32 norm it consumed:
  * m within 8u (b1 |m| + (1 - b1) |g s|), v within 8u b2 v + 8u (1 - b2) (g s)^2 (12u on the second term when a
    clip factor scales g: its two roundings enter g^2 twice);
  * p within 2^-20 lr / bc1 (b1 |m| + (1 - b1) |g s|) / (sqrt(v / bc2) + eps), plus one ulp of p;
  * clip modes 0, 1 and 2 with the norm below and above max_norm, mode 1 near 1e-3 where its 1e-6 matters,
    grad_div 1 and 4 (applied to g and to the norm), zero_grad on (grad exactly 0 after) and off (grad untouched),
    n on both sides of the 148 * 8 * 256 grid-stride threshold;
  * the device-resident step / learning rate give bit-identical results to the host scalars over steps 1..20.
Worst measured ratio to these bounds on an H100 80GB HBM3 (700 W): norm 0.028, m 0.27, v 0.39, p 0.50 (the one ulp
of p: the update is often below it).
FlatAdam: five steps of parameters whose sizes are not multiples of 4, each step against the one-step restatement
from the kernel's previous state and the whole run against float64 torch.optim.Adam; padding lanes stay exactly 0.
PPOEngine.learn_minibatch: CUDA-graph replay is bit-identical to the eager body, minibatch by minibatch."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
GRID_CAP = 148 * 8             # CTA cap of both optimiser kernels
NT = 256


def _gamma(k):
    return k * U / (1 - k * U)


def _f32(v):
    return float(np.float32(v))


def _norm(g):
    from parl_b200 import kernels
    out = torch.full((1, ), float('nan'), device=DEV)
    kernels.grad_global_norm(g, out)
    return out


NORM_N = [1, 2, 3, 5, 4096 + 3] + [3 * GRID_CAP * NT * 4 + r for r in (1, 2, 3)]


@pytest.mark.parametrize('n', NORM_N)
def test_grad_global_norm_exact_integers(n):
    gen = torch.Generator(device=DEV).manual_seed(n)
    g = torch.randint(-2, 3, (n, ), generator=gen, device=DEV).float()
    if n & 3:
        g[n - (n & 3):] = 3.0                         # the scalar tail is nonzero
    s = (g.double() ** 2).sum().item()
    assert s < 2 ** 24
    got = _norm(g).cpu().numpy()[0]
    assert got == np.float32(math.sqrt(s)), (got, math.sqrt(s))


@pytest.mark.parametrize('n', NORM_N)
def test_grad_global_norm_random_within_bound(n):
    gen = torch.Generator(device=DEV).manual_seed(n + 1)
    g = torch.randn(n, generator=gen, device=DEV) * torch.exp(torch.randn(n, generator=gen, device=DEV))
    ref = math.sqrt((g.double() ** 2).sum().item())
    blocks = min(max(((n >> 2) + NT - 1) // NT, 1), GRID_CAP)
    passes = ((n >> 2) + blocks * NT - 1) // (blocks * NT)
    bound = _gamma(passes + 18) + U
    err = abs(_norm(g).item() / ref - 1)
    print('grad_global_norm n=%d passes=%d ratio %.3g' % (n, passes, err / bound))
    assert err <= bound, (err, bound)


def test_grad_global_norm_ticket_reset_between_calls():
    from parl_b200 import kernels
    gen = torch.Generator(device=DEV).manual_seed(3)
    big = torch.randn(2 * GRID_CAP * NT * 4 + 3, generator=gen, device=DEV)
    small = torch.randn(4101, generator=gen, device=DEV)
    ws = kernels._flat_ws(big.device, 1)
    first = _norm(big).clone()
    seq = [_norm(small).clone(), _norm(big).clone(), _norm(small).clone()]
    N, A = 3000, 5                                    # a2c loss over the same workspace (its own ticket use)
    logits = torch.randn(N, A, generator=gen, device=DEV)
    vals, adv, tv = (torch.randn(N, generator=gen, device=DEV) for _ in range(3))
    act = torch.randint(0, A, (N, ), generator=gen, device=DEV, dtype=torch.int32)
    r1 = kernels.a2c_loss_fwd_bwd(logits, vals, act, adv, tv, 0.5, 0.01)['losses'].clone()
    seq.append(_norm(big).clone())
    r2 = kernels.a2c_loss_fwd_bwd(logits, vals, act, adv, tv, 0.5, 0.01)['losses'].clone()
    seq.append(_norm(big).clone())
    seq.append(_norm(small).clone())
    assert kernels._flat_ws(big.device, 1) is ws      # really the same workspace throughout
    torch.cuda.synchronize()
    assert ws[:4].view(torch.int32).item() == 0
    assert torch.equal(r1, r2)
    for i, v in enumerate(seq):
        assert torch.equal(v, first if i in (1, 3, 4) else seq[0]), i


# --------------------------------------------------------------------------- adam_step
def _adam_ref(p, g, m, v, norm, lr, b1, b2, eps, step, grad_div, max_norm, clip_mode):
    """float64 torch.optim.Adam step after the clip; returns the new (p, m, v) and their error bounds."""
    lr, b1, b2, eps, max_norm = (_f32(a) for a in (lr, b1, b2, eps, max_norm))
    s = 1.0 / grad_div
    if clip_mode:
        nrm = norm / grad_div
        s *= min(1.0, max_norm / (nrm + 1e-6)) if clip_mode == 1 else max_norm / max(nrm, max_norm)
    gs = g * s
    m1 = b1 * m + (1 - b1) * gs
    v1 = b2 * v + (1 - b2) * gs * gs
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    den = v1.sqrt() / math.sqrt(bc2) + eps
    p1 = p - lr / bc1 * m1 / den
    mag_m = b1 * m.abs() + (1 - b1) * gs.abs()
    kv = 12 if (clip_mode and s * grad_div != 1.0) else 8
    em = 8 * U * mag_m
    ev = 8 * U * b2 * v + kv * U * (1 - b2) * gs * gs
    p32 = p1.float().abs()
    ulp = (torch.nextafter(p32, torch.full_like(p32, math.inf)) - p32).double()
    ep = 2.0 ** -20 * lr / bc1 * mag_m / den + ulp
    return (p1, m1, v1), (ep, em, ev)


def _check_adam(got, ref, bounds, what=''):
    ratios = []
    for name, a, r, b in zip('pmv', got, ref, bounds):
        e = (a.double() - r).abs()
        ratios.append((e / b).max().item())
        assert (e <= b).all(), (what, name, ratios[-1])
    return ratios


ADAM_N = [5, 4099, 2 * GRID_CAP * NT + 77]
# clip mode, max_norm as a multiple of the norm the kernel divides by grad_div (None: no clip), that norm
CLIP_CASES = {
    'none': (0, None, 1.0),
    'torch-below': (1, 2.0, 1.0),
    'torch-above': (1, 0.5, 1.0),
    'torch-1e-3-above': (1, 0.9, 1e-3),
    'torch-1e-3-eps': (1, 1.0005, 1e-3),      # below max_norm, clipped by 0.9995 only through the 1e-6
    'paddle-below': (2, 2.0, 1.0),
    'paddle-above': (2, 0.5, 1.0),
}


@pytest.mark.parametrize('zero_grad', [True, False], ids=['zero', 'keep'])
@pytest.mark.parametrize('grad_div', [1.0, 4.0])
@pytest.mark.parametrize('case', list(CLIP_CASES))
@pytest.mark.parametrize('n', ADAM_N)
def test_adam_step_matches_float64_adam(n, case, grad_div, zero_grad):
    from parl_b200 import kernels
    clip_mode, mult, target = CLIP_CASES[case]
    gen = torch.Generator(device=DEV).manual_seed(n + len(case))
    g = torch.randn(n, generator=gen, device=DEV)
    g *= target * grad_div / g.double().norm().item()            # norm / grad_div lands at `target`
    p = torch.randn(n, generator=gen, device=DEV)
    m = 0.1 * torch.randn(n, generator=gen, device=DEV)
    v = 0.01 * torch.rand(n, generator=gen, device=DEV) ** 2
    norm = _norm(g)
    nv = norm.item()
    max_norm = 0.0 if mult is None else mult * nv / grad_div
    lr, b1, b2, eps, step = 3e-4, 0.9, 0.999, 1e-5, 7
    ref, bounds = _adam_ref(p.double(), g.double(), m.double(), v.double(), nv, lr, b1, b2, eps, step, grad_div,
                            max_norm, clip_mode)
    g0 = g.clone()
    kernels.adam_step(p, g, m, v, lr, b1, b2, eps, step, grad_div=grad_div, grad_norm=norm if clip_mode else None,
                      max_norm=max_norm, clip_mode=clip_mode, zero_grad=zero_grad)
    r = _check_adam((p, m, v), ref, bounds, case)
    print('adam n=%d %s div=%g ratios p %.3g m %.3g v %.3g' % ((n, case, grad_div) + tuple(r)))
    if zero_grad:
        assert torch.equal(g, torch.zeros_like(g)) and not torch.signbit(g).any()
    else:
        assert torch.equal(g, g0)


def test_adam_device_state_matches_host_scalars():
    """step_device / lr_device against the host's step and rate over steps 1..20, the rate changed after step 10.
    The host arguments of the device-state calls are deliberately wrong, so only the device values can be used."""
    from parl_b200 import kernels
    n = 2 * GRID_CAP * NT + 5
    gen = torch.Generator(device=DEV).manual_seed(20)
    host = [torch.randn(n, generator=gen, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)]
    dev = [t.clone() for t in host]
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    lr_dev = torch.zeros(1, device=DEV)
    for t in range(1, 21):
        lr = 1e-3 if t <= 10 else 2.5e-4
        g = torch.randn(n, generator=gen, device=DEV)
        g2 = g.clone()
        norm = _norm(g)
        kernels.adam_step(host[0], g, host[1], host[2], lr, 0.9, 0.999, 1e-8, t, grad_norm=norm, max_norm=40.0,
                          clip_mode=1)
        step_dev.fill_(t)
        lr_dev.fill_(lr)
        kernels.adam_step(dev[0], g2, dev[1], dev[2], 1.0, 0.9, 0.999, 1e-8, 1, grad_norm=norm, max_norm=40.0,
                          clip_mode=1, lr_device=lr_dev, step_device=step_dev)
        for a, b, name in zip(host, dev, 'pmv'):
            assert torch.equal(a, b), (t, name, (a - b).abs().max().item())


# --------------------------------------------------------------------------- FlatAdam
SHAPES = [(3, 5), (7, ), (2, 3, 3), (1, ), (13, )]


def _flat_params(seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=gen, device=DEV)) for s in SHAPES]


def _pad_mask(opt):
    mask = torch.ones(opt.flat.numel(), dtype=torch.bool, device=DEV)
    off = 0
    for p in opt.params:
        mask[off:off + p.numel()] = False
        off += (p.numel() + 3) // 4 * 4
    assert mask.any()
    return mask


@pytest.mark.parametrize('clip', ['torch', 'paddle'])
def test_flat_adam_five_steps_against_float64_adam(clip):
    from parl_b200.engine.optim import FlatAdam
    params = _flat_params(1)
    ref = [p.detach().double().clone().requires_grad_() for p in params]
    lr, max_norm = 3e-3, 1.0
    opt = FlatAdam(params, lr=lr, betas=(0.9, 0.999), eps=1e-8, clip=clip, max_norm=max_norm)
    ropt = torch.optim.Adam(ref, lr=lr, betas=(0.9, 0.999), eps=1e-8, foreach=False)
    pad = _pad_mask(opt)
    gen = torch.Generator(device=DEV).manual_seed(2)
    for t in range(1, 6):
        scale = 0.05 if t % 2 else 3.0                # the global norm alternates below and above max_norm
        grads = [scale * torch.randn(p.shape, generator=gen, device=DEV) for p in params]
        for p, gr in zip(params, grads):
            p.grad.copy_(gr)
        before = [opt.flat.double(), opt.grad.double(), opt.exp_avg.double(), opt.exp_avg_sq.double()]
        opt.step()
        nv = opt.norm.item()
        gref = math.sqrt(sum((gr.double() ** 2).sum().item() for gr in grads))
        assert abs(nv / gref - 1) <= _gamma(1 + 18) + U              # 64 floats: one float4 pass per thread
        got, bnd = _adam_ref(before[0], before[1], before[2], before[3], nv, lr, 0.9, 0.999, 1e-8, t, 1.0, max_norm,
                             opt.clip_mode)
        _check_adam((opt.flat, opt.exp_avg, opt.exp_avg_sq), got, bnd, (clip, t))
        for tns in (opt.flat, opt.grad, opt.exp_avg, opt.exp_avg_sq):
            assert torch.equal(tns[pad], torch.zeros_like(tns[pad])) and not torch.signbit(tns[pad]).any()
        assert torch.equal(opt.grad, torch.zeros_like(opt.grad))
        # the whole run against float64 torch.optim.Adam with the reference clip
        for r, gr in zip(ref, grads):
            r.grad = gr.double()
        if clip == 'torch':
            torch.nn.utils.clip_grad_norm_(ref, max_norm)
        else:
            total = math.sqrt(sum((r.grad ** 2).sum().item() for r in ref))
            for r in ref:
                r.grad.mul_(max_norm / max(total, max_norm))
        ropt.step()
        for p, r in zip(params, ref):
            pd = p.detach().double()
            p32 = p.detach().abs()
            ulp = (torch.nextafter(p32, torch.full_like(p32, math.inf)) - p32).double()
            assert ((pd - r.detach()).abs() <= 6 * ulp + lr * 2.0 ** -12).all(), (clip, t)
            st = ropt.state[r]
            for mine, theirs in ((opt.exp_avg, st['exp_avg']), (opt.exp_avg_sq, st['exp_avg_sq'])):
                off = (p.data.data_ptr() - opt.flat.data_ptr()) // 4
                got_s = mine[off:off + p.numel()].double().view(p.shape)
                assert ((got_s - theirs).abs() <= 2.0 ** -16 * theirs.abs().max()).all(), (clip, t)
    assert opt.step_count == 5


def test_flat_adam_load_state_dict_restores_device_step():
    from parl_b200.engine.optim import FlatAdam
    a_params = _flat_params(4)
    a = FlatAdam(a_params, lr=1e-3, clip='torch', max_norm=0.5).enable_device_state()
    gen = torch.Generator(device=DEV).manual_seed(5)
    for _ in range(3):
        a.grad.copy_(torch.randn(a.grad.shape, generator=gen, device=DEV) * (~_pad_mask(a)))
        a.step()
    sd = a.state_dict()
    b_params = [torch.nn.Parameter(p.detach().clone()) for p in a_params]
    b = FlatAdam(b_params, lr=0.1, clip='torch', max_norm=0.5).enable_device_state()
    b.load_state_dict(sd)
    assert b.step_count == 3 and b.step_dev.item() == 3 and b.lr_dev.item() == np.float32(1e-3)
    g = torch.randn(a.grad.shape, generator=gen, device=DEV) * (~_pad_mask(a))
    a.grad.copy_(g)
    b.grad.copy_(g)
    a.step()
    b.step()
    assert b.step_dev.item() == a.step_dev.item() == 4
    for x, y in ((a.flat, b.flat), (a.exp_avg, b.exp_avg), (a.exp_avg_sq, b.exp_avg_sq)):
        assert torch.equal(x, y)


# --------------------------------------------------------------------------- PPO minibatch: graph replay
def test_ppo_minibatch_graph_replay_equals_eager():
    """Two engines from the same seed, one eager and one replaying its captured minibatch graph (calls 2 and later),
    fed the same rows and learning rates: losses, parameters, Adam moments and the device step stay bit-identical."""
    from parl_b200.engine.ppo import PPOEngine
    engs = []
    for use_graph in (False, True):
        torch.manual_seed(5)
        engs.append(PPOEngine(num_envs=64, step_nums=32, num_minibatches=4, update_epochs=2, seed=9, device=DEV,
                              p_done=0.05, max_episode_steps=20, num_updates=10, use_graph=use_graph))
    for e in engs:
        e.rollout()
        e.compute_returns()
    eager, graph = engs
    assert torch.equal(eager.obs, graph.obs) and torch.equal(eager.advantages, graph.advantages)
    gen = torch.Generator().manual_seed(6)
    for call in range(8):
        idx = torch.randperm(eager.N, generator=gen)[:eager.M].to(device=DEV, dtype=torch.int32)
        lr = 3e-4 * (1.0 - 0.1 * call)
        la = eager.learn_minibatch(idx, lr).clone()
        lb = graph.learn_minibatch(idx, lr).clone()
        torch.cuda.synchronize()
        assert torch.equal(la, lb), (call, la, lb)
        for (name, p), (_, q) in zip(eager.model.named_parameters(), graph.model.named_parameters()):
            assert torch.equal(p, q), (call, name)
        oa, ob = eager.alg.optimizer, graph.alg.optimizer
        assert torch.equal(oa.exp_avg, ob.exp_avg) and torch.equal(oa.exp_avg_sq, ob.exp_avg_sq), call
        assert torch.equal(oa.step_dev, ob.step_dev) and oa.step_dev.item() == call + 1, call
        assert oa.step_count == ob.step_count == call + 1
    assert eager._graph is None and graph._graph is not None
