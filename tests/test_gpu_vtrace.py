"""GPU parity: V-trace returns (a1) and the fused IMPALA loss kernel (a1+a2+a3) through the C ABI
against the oracle, the reference's known-answer vectors, and size-independent properties."""
import numpy as np
import pytest
import torch

from oracle import vtrace as ovt

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device('cuda:0')


def _cuda(x):
    return torch.as_tensor(np.ascontiguousarray(x)).to(_dev())


@pytest.mark.parametrize('B', [1, 4])
def test_vtrace_returns_reference_kat(golden, B):
    from parl_b200 import kernels
    g = golden('vtrace_kat')
    k = {n: g['B%d_%s' % (B, n)] for n in ('blp', 'tlp', 'discounts', 'rewards', 'values', 'bootstrap_value')}
    vs, pg = kernels.vtrace_from_importance_weights(*[_cuda(k[n]) for n in
                                                      ('blp', 'tlp', 'discounts', 'rewards', 'values',
                                                       'bootstrap_value')], 3.7, 2.2)
    # same tolerance as the reference test (vtrace_test_paddle.py:140-144)
    np.testing.assert_almost_equal(g['B%d_vs' % B], vs.cpu().numpy(), 5)
    np.testing.assert_almost_equal(g['B%d_pg_advantages' % B], pg.cpu().numpy(), 5)


@pytest.mark.parametrize('T,B', [(5, 3), (49, 512), (200, 33)])
def test_vtrace_returns_vs_oracle(T, B):
    from parl_b200 import kernels
    rng = np.random.RandomState(T * 1000 + B)
    blp = -np.abs(rng.randn(T, B)).astype(np.float32)
    tlp = (blp + 0.5 * rng.randn(T, B)).astype(np.float32)
    disc = ((rng.rand(T, B) > 0.1) * 0.99).astype(np.float32)
    rew = rng.randn(T, B).astype(np.float32)
    val = rng.randn(T, B).astype(np.float32)
    boot = rng.randn(B).astype(np.float32)
    for cr, cp in ((1.0, 1.0), (None, None), (3.7, 2.2)):
        vs, pg = kernels.vtrace_from_importance_weights(_cuda(blp), _cuda(tlp), _cuda(disc), _cuda(rew), _cuda(val),
                                                        _cuda(boot), cr, cp)
        ovs, opg = ovt.from_importance_weights(blp, tlp, disc, rew, val, boot, cr, cp)
        np.testing.assert_allclose(vs.cpu().numpy(), ovs, rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(pg.cpu().numpy(), opg, rtol=1e-5, atol=1e-5)


def make_rollout(T, B, A, seed, p_done=0.1, gaussian_rewards=False):
    """Synthetic rollout of SURVEY.md §8(d): logits ~ 2N(0,1), behaviour = logits + N(0,.5)."""
    rng = np.random.RandomState(seed)
    tl = (2 * rng.randn(T, B, A)).astype(np.float32)
    bl = (tl + 0.5 * rng.randn(T, B, A)).astype(np.float32)
    p = np.exp(bl - bl.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    acts = (p.cumsum(-1) < rng.rand(T, B, 1)).sum(-1).clip(0, A - 1).astype(np.int64)
    rew = rng.randn(T, B).astype(np.float32) if gaussian_rewards else (rng.rand(T, B) < 0.5).astype(np.float32)
    dones = rng.rand(T, B) < p_done
    vals = rng.randn(T, B).astype(np.float32)
    return tl, bl, acts, rew, dones, vals


def _check_loss(T, B, A, seed, layout, act_dtype=torch.int64, clip=(1.0, 1.0), coeffs=(0.5, -0.01), **kw):
    from parl_b200 import kernels
    tl, bl, acts, rew, dones, vals = make_rollout(T, B, A, seed, **kw)
    o = ovt.impala_loss_time_major(tl, bl, acts, rew, dones, vals, 0.99, coeffs[0], coeffs[1], clip[0], clip[1])

    def lay(x):  # oracle arrays are time-major; build the device layout
        return np.ascontiguousarray(np.swapaxes(x, 0, 1)) if layout == kernels.ENV_MAJOR else x
    r = kernels.vtrace_loss_fwd_bwd(
        _cuda(lay(tl)).reshape(T * B, A), _cuda(lay(bl)).reshape(T * B, A), _cuda(lay(acts)).reshape(-1).to(act_dtype),
        _cuda(lay(rew)).reshape(-1), _cuda(lay(dones)).reshape(-1), _cuda(lay(vals)).reshape(-1), T, B, 0.99,
        coeffs[0], coeffs[1], clip[0], clip[1], layout=layout, want_returns=True)
    torch.cuda.synchronize()
    losses = r['losses'].cpu().numpy()
    for i, k in enumerate(('total_loss', 'pi_loss', 'vf_loss', 'entropy', 'kl')):
        np.testing.assert_allclose(losses[i], o[k], rtol=1e-4, atol=1e-4, err_msg=k)
    np.testing.assert_allclose(r['vs'].cpu().numpy(), o['vs'], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(r['pg_advantages'].cpu().numpy(), o['pg_advantages'], rtol=1e-4, atol=1e-4)
    dl = r['d_logits'].cpu().numpy()
    dv = r['d_values'].cpu().numpy()
    if layout == kernels.ENV_MAJOR:
        dl = np.swapaxes(dl.reshape(B, T, A), 0, 1)
        dv = np.swapaxes(dv.reshape(B, T), 0, 1)
    else:
        dl, dv = dl.reshape(T, B, A), dv.reshape(T, B)
    np.testing.assert_allclose(dl, o['d_logits'], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(dv, o['d_values'], rtol=1e-4, atol=1e-5)
    assert np.all(dl[-1] == 0) and np.all(dv[-1] == 0)          # bootstrap row: no gradient


@pytest.mark.parametrize('T,B,A', [(50, 64, 18), (50, 7, 18), (20, 256, 2), (5, 4, 6), (50, 20, 6), (33, 10, 5),
                                   (17, 9, 19), (130, 12, 18), (2, 1, 3)])
@pytest.mark.parametrize('layout', [0, 1])
def test_vtrace_loss_vs_oracle(T, B, A, layout):
    _check_loss(T, B, A, seed=T + B + A, layout=layout)


def test_vtrace_loss_variants():
    _check_loss(50, 32, 18, 1, 0, act_dtype=torch.int32)
    _check_loss(50, 32, 18, 2, 0, clip=(None, None))
    _check_loss(50, 32, 18, 3, 1, clip=(3.7, 2.2), coeffs=(0.25, -0.05), gaussian_rewards=True)
    _check_loss(50, 32, 18, 4, 0, p_done=1.0)
    _check_loss(50, 32, 18, 5, 0, p_done=0.0)


def test_vtrace_loss_full_size_properties():
    """C3 shape (T=50, B=4096, A=18): oracle on a column subset + column-independence property."""
    from parl_b200 import kernels
    T, B, A = 50, 4096, 18
    tl, bl, acts, rew, dones, vals = make_rollout(T, B, A, 77)
    args = [_cuda(tl).reshape(T * B, A), _cuda(bl).reshape(T * B, A), _cuda(acts).reshape(-1),
            _cuda(rew).reshape(-1), _cuda(dones).reshape(-1), _cuda(vals).reshape(-1)]
    r = kernels.vtrace_loss_fwd_bwd(*args, T, B, 0.99, 0.5, -0.01, want_returns=True)
    torch.cuda.synchronize()
    sub = slice(1000, 1064)
    o = ovt.impala_loss_time_major(tl[:, sub], bl[:, sub], acts[:, sub], rew[:, sub], dones[:, sub], vals[:, sub],
                                   0.99, 0.5, -0.01)
    np.testing.assert_allclose(r['vs'].cpu().numpy()[:, sub], o['vs'], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(r['d_logits'].cpu().numpy().reshape(T, B, A)[:, sub], o['d_logits'], rtol=1e-4, atol=1e-5)
    # additivity: the SUM losses of the full batch equal the sum over two half batches
    halves = []
    for lo, hi in ((0, 2048), (2048, 4096)):
        h = kernels.vtrace_loss_fwd_bwd(
            _cuda(tl[:, lo:hi]).reshape(-1, A), _cuda(bl[:, lo:hi]).reshape(-1, A), _cuda(acts[:, lo:hi]).reshape(-1),
            _cuda(rew[:, lo:hi]).reshape(-1), _cuda(dones[:, lo:hi]).reshape(-1), _cuda(vals[:, lo:hi]).reshape(-1),
            T, 2048, 0.99, 0.5, -0.01)
        halves.append(h['losses'].cpu().numpy())
    full = r['losses'].cpu().numpy()
    np.testing.assert_allclose(full[:4], halves[0][:4] + halves[1][:4], rtol=1e-5)
    np.testing.assert_allclose(full[4], 0.5 * (halves[0][4] + halves[1][4]), rtol=1e-5)
    # determinism: same inputs, bit-identical outputs (fixed-order reduction)
    r2 = kernels.vtrace_loss_fwd_bwd(*args, T, B, 0.99, 0.5, -0.01)
    assert torch.equal(r['losses'][:5], r2['losses'][:5]) and torch.equal(r['d_logits'], r2['d_logits'])


def test_tma_and_cpasync_tile_paths_agree():
    """The TMA tensor-map tile path and the cp.async path of the general (v4) kernel are the same arithmetic, and
    the default v8 kernel (register-resident packed-pair arithmetic, two passes in time, in-warp scan) agrees with
    both to float32 round-off.  v8 takes int32 actions only, so modes 0 and 9 get them (shapes v8 does not take —
    T > 64 — run v4 twice)."""
    from parl_b200 import kernels, _lib
    lib = _lib.load()
    for (T, B, A) in [(50, 512, 18), (50, 7 * 4, 6), (130, 64, 18), (20, 256, 2), (50, 4096, 18), (7, 8, 18),
                      (64, 40, 4), (33, 16, 18)]:
        tl, bl, acts, rew, dones, vals = make_rollout(T, B, A, 11)
        args = [_cuda(tl).reshape(T * B, A), _cuda(bl).reshape(T * B, A), _cuda(acts).reshape(-1),
                _cuda(rew).reshape(-1), _cuda(dones).reshape(-1), _cuda(vals).reshape(-1)]
        args32 = list(args)
        args32[2] = args[2].to(torch.int32)
        try:
            lib.rl_debug_set_vtrace_path(4)
            lib.rl_debug_set_tma(1)
            r0 = kernels.vtrace_loss_fwd_bwd(*args, T, B, 0.99, 0.5, -0.01, want_returns=True)
            torch.cuda.synchronize()
            lib.rl_debug_set_tma(0)
            r1 = kernels.vtrace_loss_fwd_bwd(*args, T, B, 0.99, 0.5, -0.01, want_returns=True)
            torch.cuda.synchronize()
            for k in ('d_logits', 'd_values', 'vs', 'pg_advantages'):
                assert torch.equal(r0[k], r1[k]), (k, T, B, A)
            assert torch.equal(r0['losses'][:5], r1['losses'][:5])
            for mode in (0, 9):
                lib.rl_debug_set_vtrace_path(mode)
                r5 = kernels.vtrace_loss_fwd_bwd(*args32, T, B, 0.99, 0.5, -0.01, want_returns=True)
                torch.cuda.synchronize()
                for k in ('d_logits', 'd_values', 'vs', 'pg_advantages'):
                    assert torch.allclose(r5[k], r1[k], rtol=2e-5, atol=2e-5), (k, T, B, A, mode,
                                                                               (r5[k] - r1[k]).abs().max().item())
                assert torch.allclose(r5['losses'][:5], r1['losses'][:5], rtol=1e-5, atol=1e-4), (T, B, A, mode)
        finally:
            lib.rl_debug_set_tma(0)
            lib.rl_debug_set_vtrace_path(0)
