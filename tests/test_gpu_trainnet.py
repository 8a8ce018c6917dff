"""GPU parity: the hand-written learner network (AtariTrainNet: wgmma forward, dgrad, wgrad) against torch
autograd through the same model (bf16 autocast), and the engine's native learn() against its autograd learn()."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


@pytest.mark.parametrize('fc_backend', ['native', 'library'])
def test_train_net_forward_backward_matches_autograd(fc_backend):
    from parl_b200 import kernels as K
    from parl_b200.engine.nets import AtariActorCritic
    from parl_b200.engine.train_net import AtariTrainNet
    torch.manual_seed(0)
    N, A = 160, 18
    model = AtariActorCritic(A).to(DEV)
    with torch.no_grad():            # non-zero biases so that every path is exercised
        for p in model.parameters():
            if p.dim() == 1:
                p.normal_(0, 0.1)
    for p in model.parameters():
        p.grad = torch.zeros_like(p)
    net = AtariTrainNet(model, N, DEV, fc_backend=fc_backend)
    obs = torch.randint(0, 255, (N, 4, 84, 84), dtype=torch.uint8, device=DEV)
    K.obs_stack_gather(obs, None, 0, 1, net.x0, scale=1.0 / 255.0, s2d=True)
    logits, values = net.forward_from_x0()
    d_logits = torch.randn(N, A, device=DEV) * 0.1
    d_values = torch.randn(N, device=DEV) * 0.1
    net.backward(d_logits, d_values)
    torch.cuda.synchronize()
    got = {n: p.grad.clone() for n, p in model.named_parameters()}
    # references: (1) autograd through the torch model (bf16 autocast) on the same space-to-depth input,
    # (2) the float32 reference-form network on the uint8 NCHW observations
    for p in model.parameters():
        p.grad = None
    rl, rv = model.policy_and_value(net.x0)
    torch.autograd.backward([rl, rv], [d_logits, d_values])
    assert _rel(logits, rl) < 2e-2 and _rel(values.view(-1), rv) < 2e-2
    tb = {n: p.grad.clone() for n, p in model.named_parameters()}
    m32 = AtariActorCritic(A, compute_dtype=torch.float32).to(DEV)
    m32.load_state_dict(model.state_dict())
    l32, v32 = m32.policy_and_value(obs)
    torch.autograd.backward([l32, v32], [d_logits, d_values])
    assert _rel(logits, l32) < 2e-2
    # bf16 activations flip a fraction of ReLU masks, which costs both bf16 implementations a few percent of
    # gradient direction against float32 (measured: torch autocast 6-10 %, ours 5-8 %).  The bar: our gradients
    # are as close to the float32 reference as torch's own bf16 path is, and close to that path itself.
    for (n, p), (_, q) in zip(model.named_parameters(), m32.named_parameters()):
        r_ours, r_torch = _rel(got[n], q.grad), _rel(tb[n], q.grad)
        assert r_ours < 1.15 * r_torch + 0.01, (n, r_ours, r_torch)
        assert _rel(got[n], tb[n]) < 0.15, n


def test_engine_native_learn_matches_autograd_learn():
    from parl_b200.engine.impala import ImpalaEngine
    B, T = 32, 8
    outs = []
    for native in (True, False):
        torch.manual_seed(5)
        eng = ImpalaEngine(num_envs=B, sample_batch_steps=T, act_dim=18, seed=11, device=DEV, use_graph=False,
                           learn_chunk_rows=4, learner_kernels=native, actor_kernels=False)
        eng.rollout()
        losses = eng.learn(1e-3, -0.01)
        torch.cuda.synchronize()
        outs.append((losses[:5].cpu().numpy(), torch.cat([p.detach().reshape(-1) for p in eng.model.parameters()]).cpu()))
    np.testing.assert_allclose(outs[0][0][:4], outs[1][0][:4], rtol=2e-2)
    # one Adam step from identical weights: parameter DELTAS must agree in direction and size
    torch.manual_seed(5)
    from parl_b200.engine.nets import AtariActorCritic
    w0 = torch.cat([p.detach().reshape(-1) for p in AtariActorCritic(18).parameters()])
    d0, d1 = outs[0][1] - w0, outs[1][1] - w0
    cos = torch.dot(d0, d1) / (d0.norm() * d1.norm())
    assert cos > 0.97, cos


def test_pipelined_engine_is_deterministic_and_matches_host_contract():
    """Two-stream double-buffered step(): finite losses, bit-identical across two runs with the same seed, env
    streams identical to the sequential engine; step_host() hands the reference-layout sample dict to the host."""
    from parl_b200.engine.impala import ImpalaEngine
    B, T = 32, 8

    def run(pipeline, n):
        torch.manual_seed(3)
        eng = ImpalaEngine(num_envs=B, sample_batch_steps=T, act_dim=18, seed=21, device=DEV, use_graph=True,
                           pipeline=pipeline)
        out = [eng.step(1e-3, -0.01)[:5].clone() for _ in range(n)]
        torch.cuda.synchronize()
        return eng, torch.stack(out).cpu()
    e1, l1 = run(True, 5)
    e2, l2 = run(True, 5)
    assert torch.isfinite(l1).all() and torch.equal(l1, l2)
    # the env side does not depend on the policy lag: rewards/dones of rollout 0 equal the sequential engine's
    e3, _ = run(False, 1)
    e4, _ = run(True, 1)
    assert torch.equal(e3._sets[0]['rewards'], e4._sets[0]['rewards']) and torch.equal(e3._sets[0]['dones'], e4._sets[0]['dones'])
    # host contract through the pipelined path
    torch.manual_seed(3)
    eng = ImpalaEngine(num_envs=B, sample_batch_steps=T, act_dim=18, seed=21, device=DEV, pipeline=True)
    hosts = [eng.make_host_sample_buffers() for _ in range(2)]
    for _ in range(3):
        losses = eng.step_host(hosts, 1e-3, -0.01)
    torch.cuda.synchronize()
    assert torch.isfinite(losses[:5]).all()
    h = hosts[0]
    assert h['obs'].shape == (B * T, 4, 84, 84) and h['obs'].dtype == torch.uint8
    assert h['actions'].dtype == torch.int64 and h['dones'].dtype == torch.bool
    assert h['behaviour_logits'].shape == (B * T, 18) and int(h['actions'].max()) < 18
    # env-major order (index b*T + t): column 0 of the time-major device buffer is the first T host rows
    s0 = eng._sets[0]
    got = h['rewards'].view(B, T)
    want = s0['rewards'].cpu().t()
    # hosts[0] was last written by rollout 2 (set 0): the device buffer of set 0 still holds that rollout
    assert torch.equal(got, want)


def test_one_launch_operand_refresh_matches_per_operand_copies():
    """engine/packing.py: the index-permutation gather (rl_gather_cast) rebuilds every operand copy exactly as the
    permute + copy expressions do, for the learner's and the actor's net, before and after a weight change."""
    from parl_b200.algorithms import IMPALA
    from parl_b200.engine.actor_net import AtariActorNet
    from parl_b200.engine.nets import AtariActorCritic
    from parl_b200.engine.train_net import AtariTrainNet
    torch.manual_seed(3)
    model = AtariActorCritic(18).to(DEV)
    alg = IMPALA(model, sample_batch_steps=4, gamma=0.99, vf_loss_coeff=0.5, clip_rho_threshold=1.0,
                 clip_pg_rho_threshold=1.0)
    flat = alg.optimizer.flat
    names = ['w1', 'w2', 'w3', 'wfc', 'wpi', 'wv', 'b1', 'b2', 'b3', 'bfc', 'bpi', 'bv']
    pairs = [(AtariTrainNet(model, 128, DEV, flat=flat), AtariTrainNet(model, 128, DEV), names + ['wfcT', 'whT', 'w3T', 'w2T']),
             (AtariActorNet(model, 128, DEV, flat=flat), AtariActorNet(model, 128, DEV), names)]
    for fast, ref, ns in pairs:
        assert fast.ops.flat is not None and ref.ops.flat is None
    for rnd in range(2):
        for fast, ref, ns in pairs:
            fast.pack(), ref.pack()
            torch.cuda.synchronize()
            for n in ns:
                a, b = getattr(fast, n), getattr(ref, n)
                assert a.dtype == b.dtype and torch.equal(a, b), (rnd, n)
                assert a.float().abs().sum().item() > 0 or n.startswith('b'), n
        with torch.no_grad():
            flat.add_(torch.randn_like(flat) * 0.01)          # "a learner update"
