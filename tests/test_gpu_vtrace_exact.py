"""The fused IMPALA loss K1 (csrc/vtrace_loss.cu: rl_vtrace_loss_fwd_bwd) and the V-trace returns kernel a1
(rl_vtrace_from_importance_weights) pinned against references written here.

K1 has two kernels.  vtrace_loss_v8_kernel runs for time-major, 16-byte-aligned operands with T <= 64, B % 4 == 0,
even A <= 18 and int32 actions (what ImpalaEngine and the benchmark launch); vtrace_loss_kernel (v4) runs everything
else through its TMA, cp.async and env-major tile paths.  Every case records the kernels launched inside the call
with torch.profiler's CUDA activity and asserts the one it claims to test.

Float64 reference with a propagated bound.  `reference` restates K1 in float64 (vectorised over B and A, looping
over T for the recurrence) and carries next to each quantity q a first-order forward-error shadow E(q), built op by op
along the kernel's formulation: the log2 domain, nm = -m log2e rounded to fp32, xs = fma(x, log2e, nm), the sums S,
W, Y and Sy, lg2(S), rho = 2^((la - lma) log2e) (v4: expf), the scan acc_t = delta_t + k_t acc_{t+1} with
k_t = g_t min(rho, 1), the advantages, the gradient p_j (adv - c_e (H + log p_j)) - adv [j == a], and the fp32 loss
chain per thread, warp_sum, per CTA, then fp64 across CTAs.  u = 2^-24, gamma(k) = k u / (1 - k u).  MUFU and
intrinsic error constants (PTX ISA and the CUDA C++ Programming Guide's intrinsic-function table):
  * ex2.approx.ftz.f32: relative error <= 2 ulp (2^-22); a result below 2^-126 flushes to zero (absolute 2^-126);
  * lg2.approx.ftz.f32: absolute error <= 2^-22 for x in [0.5, 2], 2 ulp otherwise; the bound uses
    2^-22 (1 + |lg2 x|), which covers both;
  * __fdividef(1, S): <= 2 ulp (2^-22) for 2^-126 <= S <= 2^126 (S >= 1 here: the max term is 2^~0);
  * expf (v4's rho): <= 2 ulp.
The rounding of nm shifts every xs of a row by the same c, |c| <= u |m| log2e.  On the target side it cancels
exactly (log p_j = xs_j - lg2 S, and the gradient is invariant too), so it is left out there.  On the behaviour side
lma = (y_a - my) - ln2 lg2(Sy) mixes the two domains and keeps it: lma, log Sy and the KL carry an absolute u |my|.
The +-1000 logit offsets make that term dominate.
Asserted: |got - ref| <= KAPPA[family] * E, one kappa per output family (returns = vs and pg_advantages, d_values,
d_logits, losses).  Row T - 1 of d_logits and d_values (the bootstrap row) must be exactly 0.
KAPPA is 1 for every family.  Worst measured |got - ref| / E on an H100 80GB HBM3 (400 W power limit), over every
bounded case: returns 0.695, d_values 0.682, d_logits 0.676, losses 0.176.  The three per-element maxima come from
the +-1000-offset cases, where the behaviour side's u |my| term is most of the error.

Exact identities: v8 modes 0/8/9 (programmatic dependent launch)/10/11 (L2 promotion) and repeat calls; v4's TMA,
cp.async, env-major and int64-action paths (the same per-element arithmetic and the same thread-to-element map,
(t, b) = (tid >> 2, tid & 3) per chunk, in both layouts, so the per-thread and per-CTA loss sums are the same too);
column permutations and sub-batches.  a1 against a float32 numpy restatement in the kernel's op order, bit for bit.
Rejections through the C ABI with correctly sized buffers."""
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
EX2 = 2.0 ** -22              # ex2.approx.ftz.f32, relative (2 ulp)
LG2 = 2.0 ** -22              # lg2.approx.ftz.f32, absolute (times 1 + |result|)
DIV = 2.0 ** -22              # __fdividef, relative (2 ulp); also expf
FTZ = 2.0 ** -126             # flush-to-zero of a subnormal result
LOG2E, LN2 = 1.0 / np.log(2.0), np.log(2.0)
V8, V4 = 'vtrace_loss_v8_kernel', 'vtrace_loss_kernel'
KAPPA = dict(returns=1.0, d_values=1.0, d_logits=1.0, losses=1.0)
WORST = {}
PROOF = dict(profiler=0, fallback=0, none=0)     # how each kernel claim was established
SCAN_ROUNDINGS = 16           # roundings a scan tree / chunk carry adds on top of one fma per row (bounded by M_t)


def _g(k):
    return k * U / (1 - k * U)


def _tc(T, A):
    """Rows per v4 chunk, restated from the host rule in rl_vtrace_loss_fwd_bwd."""
    tc = max(30500 // (4 * (2 * A + 2) * 4), 1)
    tc = min(tc, 224 // 4)
    tc = T if tc >= T else tc & ~3
    return max(tc, 1)


@pytest.fixture(scope='module', autouse=True)
def _report_worst():
    yield
    print('\nworst |got - ref| / bound: ' +
          ', '.join('%s %.3g (%s)' % (k, r, tag) for k, (r, tag) in sorted(WORST.items())))
    print('kernel claims: %(profiler)d by profiler, %(fallback)d by the mode-8 / mode-4 fallback, %(none)d unproven'
          % PROOF)


@pytest.fixture
def k1_path():
    """Setter of the K1 triage switches (rl_debug_set_vtrace_path, rl_debug_set_tma); both are back at 0 afterwards."""
    from parl_b200 import _lib
    lib = _lib.load()

    def set_path(mode=0, tma_off=False):
        assert lib.rl_debug_set_vtrace_path(mode) == 0
        assert lib.rl_debug_set_tma(1 if tma_off else 0) == 0
    try:
        yield set_path
    finally:
        lib.rl_debug_set_tma(0)
        lib.rl_debug_set_vtrace_path(0)


def _launched(fn):
    """(fn(), names of the CUDA kernels launched inside it); names is empty when the profiler saw no CUDA activity."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return out, [n for n in names if 'memcpy' not in n.lower() and 'memset' not in n.lower()]


# ------------------------------------------------------------------------------------------------ cases

# value regimes, spread over the matrix (defaults: 2 N(0,1) target logits, behaviour = target + 0.5 N truncated to
# +-1.5 so every log-ratio lies in +-3, actions drawn from the behaviour policy, binary rewards, dones with p = 0.1)
REGIMES = {
    'prod': dict(),
    'hi': dict(offset=1000.0, clip=(0.5, 2.0), dones='seam', rew='gauss', ec=0.05, vf=1.0),
    'lo': dict(offset=-1000.0, clip=(3.7, 2.2), dones='ends', gamma=1.0, ec=0.0),
    'onehot': dict(logits='onehot', clip=None, dones='alt', rew='gauss1e3', vf=1.0),
    'uniform': dict(logits='uniform', clip=(0.5, 2.0), gamma=0.0, dones='none', ec=0.05),
    'onpolicy': dict(logits='onpolicy', dones='all', rew='gauss', ec=-0.01),
    'clip': dict(clip=(0.5, 2.0), dones='seam', rew='gauss1e3', gamma=1.0, vf=1.0, ec=0.0),
    'noclip': dict(clip=None, dones='none', rew='gauss', ec=0.05, gamma=0.99),
}
RNAMES = list(REGIMES)


def make_case(T, B, A, regime='prod', seed=0):
    r = dict(logits='normal', offset=0.0, clip=(1.0, 1.0), gamma=0.99, dones='p10', rew='binary', ec=-0.01, vf=0.5)
    r.update(REGIMES[regime])
    rng = np.random.RandomState(seed * 7919 + T * 131 + B * 17 + A)
    if r['logits'] == 'onehot':
        tl = np.full((T, B, A), -60.0)
        np.put_along_axis(tl, rng.randint(A, size=(T, B, 1)), 60.0, -1)
    elif r['logits'] == 'uniform':
        tl = np.repeat(2 * rng.randn(T, B, 1), A, -1)
    else:
        tl = 2 * rng.randn(T, B, A)
    bl = tl if r['logits'] == 'onpolicy' else tl + np.clip(0.5 * rng.randn(T, B, A), -1.5, 1.5)
    if r['logits'] == 'onehot':
        acts = rng.randint(A, size=(T, B))
    else:
        p = np.exp(bl - bl.max(-1, keepdims=True))
        p /= p.sum(-1, keepdims=True)
        acts = (p.cumsum(-1) < rng.rand(T, B, 1)).sum(-1).clip(0, A - 1)
    R0 = T - min(T, 32)
    d = np.zeros((T, B), bool)
    if r['dones'] == 'p10':
        d = rng.rand(T, B) < 0.1
    elif r['dones'] == 'all':
        d[:] = True
    elif r['dones'] == 'seam':                    # the rows either side of v8's boundary between its two passes
        d[[max(R0 - 1, 0), R0]] = True
    elif r['dones'] == 'ends':
        d[[0, T - 2]] = True
    elif r['dones'] == 'alt':
        d[::2] = True
    rew = {'binary': (rng.rand(T, B) < 0.5) * 1.0, 'gauss': rng.randn(T, B),
           'gauss1e3': 1e3 * rng.randn(T, B)}[r['rew']]
    clip = r['clip'] if r['clip'] is not None else (None, None)
    return dict(regime=regime, tl=(tl + r['offset']).astype(np.float32), bl=(bl + r['offset']).astype(np.float32),
                acts=acts.astype(np.int32), rew=rew.astype(np.float32), dones=d,
                vals=rng.randn(T, B).astype(np.float32),
                gamma=float(np.float32(r['gamma'])), cr=clip[0], cp=clip[1], vf=float(np.float32(r['vf'])),
                ec=float(np.float32(r['ec'])), T=T, B=B, A=A)


def _offset_copy(t, k):
    """A contiguous copy of t that starts k elements into its allocation (a misaligned base pointer)."""
    buf = torch.zeros(t.numel() + k, dtype=t.dtype, device=DEV)
    v = buf[k:].view(t.shape)
    v.copy_(t)
    return v


def _inputs(c, layout=0, act64=False, misalign=None):
    T, B, A = c['T'], c['B'], c['A']

    def lay(x):
        return np.ascontiguousarray(np.swapaxes(x, 0, 1)) if layout == 1 else x
    tl = torch.from_numpy(lay(c['tl'])).to(DEV).reshape(T * B, A)
    bl = torch.from_numpy(lay(c['bl'])).to(DEV).reshape(T * B, A)
    acts = torch.from_numpy(lay(c['acts'])).to(DEV).reshape(-1).to(torch.int64 if act64 else torch.int32)
    rew = torch.from_numpy(lay(c['rew'])).to(DEV).reshape(-1)
    dones = torch.from_numpy(lay(c['dones']).astype(np.uint8)).to(DEV).reshape(-1)
    vals = torch.from_numpy(lay(c['vals'])).to(DEV).reshape(-1)
    if misalign == 'logits':
        tl = _offset_copy(tl, 1)
    elif misalign == 'values':
        vals = _offset_copy(vals, 1)
    elif misalign == 'dones':
        dones = _offset_copy(dones, 1)
    return [tl, bl, acts, rew, dones, vals]


def _call(c, args, layout=0):
    from parl_b200 import kernels
    return kernels.vtrace_loss_fwd_bwd(*args, c['T'], c['B'], c['gamma'], c['vf'], c['ec'], c['cr'], c['cp'],
                                       layout=layout, want_returns=True)


def _host(r, c, layout=0):
    """Kernel outputs as float64 numpy, time-major."""
    T, B, A = c['T'], c['B'], c['A']
    dl = r['d_logits'].double().cpu().numpy()
    dv = r['d_values'].double().cpu().numpy()
    if layout == 1:
        dl, dv = np.swapaxes(dl.reshape(B, T, A), 0, 1), np.swapaxes(dv.reshape(B, T), 0, 1)
    return dict(dl=dl.reshape(T, B, A), dv=dv.reshape(T, B), vs=r['vs'].double().cpu().numpy(),
                pg=r['pg_advantages'].double().cpu().numpy(), losses=r['losses'][:5].double().cpu().numpy())


def _bits(r):
    return {k: r[k].cpu().clone() for k in ('d_logits', 'd_values', 'vs', 'pg_advantages')} | \
        {'losses': r['losses'][:5].cpu().clone()}


def _same_bits(a, b, keys=None):
    for k in keys or a:
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k


# ------------------------------------------------------------------------------------------------ reference

def reference(c, kernel=V8):
    """float64 K1 and its forward-error shadow: name -> (ref, E), every array time-major."""
    T, B, A = c['T'], c['B'], c['A']
    f64 = np.float64
    x, y = c['tl'].astype(f64), c['bl'].astype(f64)
    a = c['acts'].astype(np.int64)[..., None]

    def side(z):
        m = z.max(-1, keepdims=True)
        zs = (z - m) * LOG2E                                  # xs without the common shift of the rounded nm
        e = np.exp2(zs)
        Ezs = 2 * U * np.abs(zs)                              # fma rounding + log2e rounded to fp32
        Ee = e * (LN2 * Ezs + EX2) + FTZ
        S = e.sum(-1)
        ES = Ee.sum(-1) + _g(A) * S
        return m[..., 0], zs, e, Ezs, Ee, S, ES

    m, xs, e, Exs, Ee, S, ES = side(x)
    my, ys, ey, Eys, Eey, Sy, ESy = side(y)
    l2S = np.log2(S)
    El2S = LOG2E * ES / S + LG2 * (1 + np.abs(l2S))
    inv = 1.0 / S
    rinv = ES / S + DIV
    lp = (xs - l2S[..., None]) * LN2                          # log p_j
    p = np.exp(lp)
    W = (e * xs).sum(-1)
    EW = (np.abs(xs) * Ee + e * Exs).sum(-1) + _g(A) * (e * np.abs(xs)).sum(-1)
    Winv = W * inv
    EWinv = EW * inv + np.abs(Winv) * (rinv + U)
    Hn = (p * lp).sum(-1)                                     # sum_j p_j log p_j
    EHn = LN2 * (EWinv + El2S + U * np.abs(Winv - l2S)) + 2 * U * np.abs(Hn)
    H, EH = -Hn, EHn
    xs_a = np.take_along_axis(xs, a, -1)[..., 0]
    la = np.take_along_axis(lp, a, -1)[..., 0]
    Ela = LN2 * (np.take_along_axis(Exs, a, -1)[..., 0] + El2S + U * np.abs(xs_a - l2S)) + 2 * U * np.abs(la)
    l2Sy = np.log2(Sy)
    logSy = LN2 * l2Sy
    ElogSy = LN2 * (LOG2E * ESy / Sy + LG2 * (1 + np.abs(l2Sy))) + 2 * U * np.abs(logSy) + U * np.abs(my)
    y_a = np.take_along_axis(y, a, -1)[..., 0]
    lma = (y_a - my) - logSy
    Elma = ElogSy + U * np.abs(y_a - my) + U * np.abs(lma)
    Yinv = (e * y).sum(-1) * inv
    EY = (np.abs(y) * Ee).sum(-1) + _g(A) * (e * np.abs(y)).sum(-1)
    EYinv = EY * inv + np.abs(Yinv) * (rinv + U)
    lq = y - (my + logSy)[..., None]
    KL = (p * (lp - lq)).sum(-1)
    EKL = EHn + EYinv + ElogSy + U * (np.abs(Hn - Yinv) + np.abs(Hn - Yinv + my) + np.abs(KL))

    rho = np.exp(la - lma)
    Erho = rho * (Ela + Elma + 3 * U * np.abs(la - lma) + EX2) + FTZ
    rhoc = rho if c['cr'] is None else np.minimum(rho, np.float32(c['cr']))
    rpg = rho if c['cp'] is None else np.minimum(rho, np.float32(c['cp']))
    g = np.where(c['dones'], 0.0, c['gamma'])
    r, v = c['rew'].astype(f64), c['vals'].astype(f64)
    L = slice(0, T - 1)                                       # loss rows; row T - 1 is the bootstrap
    vn = v[1:]
    td = r[L] + g[L] * vn - v[L]
    Etd = U * (np.abs(g[L] * vn) + np.abs(r[L] + g[L] * vn) + np.abs(td))
    delta = rhoc[L] * td
    Edelta = Erho[L] * np.abs(td) + rhoc[L] * Etd + U * np.abs(delta)
    k = g[L] * np.minimum(rho[L], 1.0)
    Ek = g[L] * Erho[L] + U * k
    acc = np.zeros((T, B))
    M = np.zeros((T, B))                                      # sum_s (prod k) |delta_s| >= |acc_t|
    Eacc = np.zeros((T, B))
    for t in range(T - 2, -1, -1):
        acc[t] = delta[t] + k[t] * acc[t + 1]
        M[t] = np.abs(delta[t]) + k[t] * M[t + 1]
        Eacc[t] = Edelta[t] + k[t] * Eacc[t + 1] + Ek[t] * M[t + 1] + 2 * U * M[t]
    Eacc += SCAN_ROUNDINGS * U * M
    vs = acc[L] + v[L]
    Evs = Eacc[L] + U * np.abs(vs)
    vs_n = acc[1:] + vn
    Evs_n = Eacc[1:] + U * np.abs(vs_n)
    inner = r[L] + g[L] * vs_n - v[L]
    Einner = g[L] * Evs_n + U * (np.abs(g[L] * vs_n) + np.abs(r[L] + g[L] * vs_n) + np.abs(inner))
    adv = rpg[L] * inner
    Eadv = Erho[L] * np.abs(inner) + rpg[L] * Einner + U * np.abs(adv)
    dv = v[L] - vs
    Edv = Evs + U * np.abs(dv)
    vf, ce = c['vf'], c['ec']
    dval = np.zeros((T, B))
    Edval = np.zeros((T, B))
    dval[L] = vf * dv
    Edval[L] = vf * Edv + U * np.abs(dval[L])

    # d_logits: d_j = e_j fma(c1, xs_j, c0), c0 = fma(c_e ln2, lg2 S, adv - c_e H) / S, c1 = -c_e ln2 / S
    inner2 = adv - ce * H[L]
    Einner2 = Eadv + abs(ce) * EH[L] + U * (np.abs(ce * H[L]) + np.abs(inner2))
    pre = ce * LN2 * l2S[L] + inner2
    Epre = abs(ce) * LN2 * El2S[L] + 3 * U * abs(ce) * LN2 * np.abs(l2S[L]) + Einner2 + U * np.abs(pre)
    c0 = pre * inv[L]
    Ec0 = Epre * inv[L] + np.abs(c0) * (rinv[L] + U)
    c1 = -ce * LN2 * inv[L]
    rc1 = rinv[L] + 3 * U
    Z = c1[..., None] * xs[L] + c0[..., None]
    EZ = (np.abs(c1)[..., None] * Exs[L] + np.abs(c1[..., None] * xs[L]) * rc1[..., None] + Ec0[..., None]
          + U * np.abs(Z))
    dl = np.zeros((T, B, A))
    Edl = np.zeros((T, B, A))
    dl[L] = p[L] * (adv[..., None] - ce * (H[L][..., None] + lp[L]))
    Edl[L] = Ee[L] * np.abs(Z) + e[L] * EZ + U * np.abs(dl[L])
    onehot = np.zeros((T - 1, B, A), bool)
    np.put_along_axis(onehot, a[L], True, -1)
    dl[L] -= onehot * adv[..., None]
    Edl[L] += onehot * (Eadv[..., None] + U * np.abs(dl[L]))

    # losses: fp32 per thread (v8: two passes; v4: one term per chunk), warp_sum (5), per CTA (v8: 4 warps as a
    # 2-level tree; v4: 7 warps in sequence), fp64 across CTAs, one rounding to fp32
    per_thread = 2 if kernel == V8 else -(-T // _tc(T, A))
    depth = per_thread + 5 + (2 if kernel == V8 else 7) + 2

    def chain(terms, Eterms):
        s = terms.sum()
        return s, Eterms.sum() + _g(depth) * np.abs(terms).sum() + U * abs(s)
    pi, Epi = chain(-la[L] * adv, np.abs(adv) * Ela[L] + np.abs(la[L]) * Eadv + U * np.abs(la[L] * adv))
    vfl, Evfl = chain(0.5 * dv * dv, np.abs(dv) * Edv + U * 0.5 * dv * dv)
    ent, Eent = chain(H[L], EH[L])
    kls, Ekls = chain(KL, EKL)
    kl, Ekl = kls / (T * B), Ekls / (T * B) + U * abs(kls / (T * B))
    tot = pi + vfl * vf + ent * ce
    Etot = Epi + vf * Evfl + abs(ce) * Eent + U * (abs(vfl * vf) + abs(pi + vfl * vf) + abs(ent * ce) + abs(tot))
    return dict(vs=(vs, Evs), pg=(adv, Eadv), dv=(dval, Edval), dl=(dl, Edl),
                losses=(np.array([tot, pi, vfl, ent, kl]), np.array([Etot, Epi, Evfl, Eent, Ekl])))


FAMILY = dict(vs='returns', pg='returns', dv='d_values', dl='d_logits', losses='losses')


def check_bound(got, ref, tag=''):
    for name, fam in FAMILY.items():
        want, E = ref[name]
        have = got[name]
        if name in ('dl', 'dv'):
            assert np.all(have[-1] == 0), (tag, name, 'bootstrap row not exactly 0')
            have, want, E = have[:-1], want[:-1], E[:-1]
        err = np.abs(have - want)
        ratio = np.where(E > 0, err / np.where(E > 0, E, 1.0), np.where(err == 0, 0.0, np.inf))
        ratio = np.where(np.isnan(ratio), np.inf, ratio)
        worst = float(ratio.max()) if ratio.size else 0.0
        if worst >= WORST.get(fam, (0.0, ''))[0]:
            WORST[fam] = (worst, tag)
        if worst > KAPPA[fam]:
            i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
            pytest.fail('%s %s: |got - ref| / bound = %.3g at %s (got %r, ref %r, bound %.3g)'
                        % (tag, name, worst, i, have[i], want[i], E[i]))


def assert_kernel(names, claim, got, rerun, loss_rows):
    """The call launched exactly the kernel it claims.  Without profiler activity (and for >= 1000 loss rows): a v8
    claim must equal the mode-8 result bit for bit and differ from the mode-4 one; a v4 claim must equal mode 4."""
    if names:
        ours = [re.search(r'vtrace_loss(_v8)?_kernel', n).group(0) for n in names if 'vtrace_loss' in n]
        assert ours == [claim], names
        PROOF['profiler'] += 1
        return
    if loss_rows < 1000:
        PROOF['none'] += 1
        return
    PROOF['fallback'] += 1
    if claim == V8:
        _same_bits(got, rerun(8))
        m4 = rerun(4)
        assert any(not torch.equal(got[k], m4[k]) for k in got), 'v8 and v4 results identical'
    else:
        _same_bits(got, rerun(4))


def run_case(c, set_path, claim, layout=0, act64=False, misalign=None, mode=0, tma_off=False):
    """Launch under the profiler, assert the kernel, check every output against the float64 bound."""
    args = _inputs(c, layout, act64, misalign)
    set_path(mode, tma_off)
    r, names = _launched(lambda: _call(c, args, layout))
    got = _bits(r)

    def rerun(m):
        set_path(m, tma_off)
        out = _bits(_call(c, args, layout))
        set_path(mode, tma_off)
        return out
    assert_kernel(names, claim, got, rerun, (c['T'] - 1) * c['B'])
    check_bound(_host(r, c, layout), reference(c, claim), '%s T=%d B=%d A=%d %s' % (claim, c['T'], c['B'], c['A'],
                                                                                 c['regime']))
    return got, args


# ------------------------------------------------------------------------------------------------ v8 matrix

V8_CASES = ([(T, 64, 18) for T in (2, 3, 8, 31, 32, 33, 40, 50, 63, 64)] +
            [(50, 512, A) for A in range(2, 19, 2)] + [(8, 4, A) for A in range(2, 19, 2)] +
            [(50, 4096, 18), (50, 512, 18), (50, 4096, 4), (50, 4096, 6)] +
            [(8, 4100, 18), (8, 8192, 6)])                 # 1025 and 2048 CTAs: a second pass of the last-CTA loop
V8_MATRIX = [(T, B, A, RNAMES[i % len(RNAMES)]) for i, (T, B, A) in enumerate(V8_CASES)]


@pytest.mark.parametrize('T,B,A,regime', V8_MATRIX, ids=['T%d-B%d-A%d-%s' % v for v in V8_MATRIX])
def test_v8_within_float64_bound(T, B, A, regime, k1_path):
    run_case(make_case(T, B, A, regime), k1_path, V8)


# ------------------------------------------------------------------------------------------------ identities

def test_v8_modes_and_repeats_bit_identical(k1_path):
    c = make_case(50, 512, 18, 'hi', seed=1)
    args = _inputs(c)
    k1_path(8)
    ref = _bits(_call(c, args))
    for mode in (0, 8, 9, 10, 11, 0):
        k1_path(mode)
        r, names = _launched(lambda: _call(c, args))
        got = _bits(r)
        assert_kernel(names, V8, got, lambda m: (k1_path(m), _bits(_call(c, args)))[1], (c['T'] - 1) * c['B'])
        _same_bits(got, ref)
    # back-to-back launches with programmatic dependent launch on one stream, sharing the loss workspace
    cases = [make_case(*s, seed=2) for s in ((50, 4096, 18, 'prod'), (20, 256, 6, 'lo'), (64, 1024, 4, 'clip'))]
    argss = [_inputs(cc) for cc in cases]
    k1_path(8)
    refs = [_bits(_call(cc, aa)) for cc, aa in zip(cases, argss)]
    k1_path(9)
    outs = [_call(cc, aa) for cc, aa in zip(cases, argss) for _ in range(2)]
    torch.cuda.synchronize()
    for i, o in enumerate(outs):
        _same_bits(_bits(o), refs[i // 2])


V4_PATH_SHAPES = [(130, 12, 18), (97, 8, 18), (50, 30, 6), (61, 12, 11), (33, 6, 2)]


@pytest.mark.parametrize('T,B,A', V4_PATH_SHAPES, ids=['T%d-B%d-A%d' % s for s in V4_PATH_SHAPES])
def test_v4_tile_paths_bit_identical(T, B, A, k1_path):
    """Time-major TMA (int32 actions under mode 4), time-major cp.async, env-major and int64 actions: every output,
    losses included, bit for bit.  (97, 8, 18) runs chunks of 48 rows, so its last chunk holds only the bootstrap
    row; B = 30 and 6 leave a ragged last CTA."""
    assert _tc(97, 18) == 48
    c = make_case(T, B, A, RNAMES[(T + A) % len(RNAMES)], seed=3)
    base, _ = run_case(c, k1_path, V4, mode=4)
    variants = [dict(mode=4, tma_off=True), dict(layout=1), dict(act64=True)]
    for kw in variants:
        args = _inputs(c, kw.get('layout', 0), kw.get('act64', False))
        k1_path(kw.get('mode', 0), kw.get('tma_off', False))
        r, names = _launched(lambda: _call(c, args, kw.get('layout', 0)))
        if names:
            assert_kernel(names, V4, None, None, 0)
        got = _bits(r)
        if kw.get('layout', 0) == 1:
            for k, shape in (('d_logits', (B, T, A)), ('d_values', (B, T))):
                got[k] = got[k].reshape(shape).transpose(0, 1).contiguous().reshape(base[k].shape)
        _same_bits(got, base)


@pytest.mark.parametrize('claim', [V8, V4])
def test_column_permutation(claim, k1_path):
    T, B, A = 50, 512, 18
    c = make_case(T, B, A, 'noclip', seed=4)
    mode = 0 if claim == V8 else 4
    base, _ = run_case(c, k1_path, claim, mode=mode)
    perm = np.random.RandomState(5).permutation(B)
    cp = dict(c)
    for k in ('tl', 'bl', 'acts', 'rew', 'dones', 'vals'):
        cp[k] = np.ascontiguousarray(c[k][:, perm])
    got, _ = run_case(cp, k1_path, claim, mode=mode)
    pt = torch.from_numpy(perm)
    _same_bits({k: got[k].reshape(T - (k in ('vs', 'pg_advantages')), B, -1) for k in got if k != 'losses'},
               {k: base[k].reshape(T - (k in ('vs', 'pg_advantages')), B, -1)[:, pt] for k in base if k != 'losses'})


def test_v8_sub_batch_independent(k1_path):
    T, B, A = 40, 1024, 18
    c = make_case(T, B, A, 'prod', seed=6)
    full, _ = run_case(c, k1_path, V8)
    half = dict(c, B=B // 2)
    for k in ('tl', 'bl', 'acts', 'rew', 'dones', 'vals'):
        half[k] = np.ascontiguousarray(c[k][:, :B // 2])
    got, _ = run_case(half, k1_path, V8)
    for k in ('d_logits', 'd_values', 'vs', 'pg_advantages'):
        n = T - (k in ('vs', 'pg_advantages'))
        assert torch.equal(got[k].reshape(n, B // 2, -1).view(torch.int32),
                           full[k].reshape(n, B, -1)[:, :B // 2].view(torch.int32)), k


# ------------------------------------------------------------------------------------------------ v4 and fallbacks

V4_CASES = [
    ('A1-offset', (20, 64, 1, 'hi'), {}),                        # generic instantiation; log-probs carry |m| u
    ('A11', (40, 36, 11, 'prod'), {}),
    ('A19', (17, 9, 19, 'clip'), {}),
    ('A64', (30, 16, 64, 'lo'), {}),
    ('A256-TC1', (7, 8, 256, 'noclip'), {}),                     # one row per chunk: seven chunks
    ('A1000-TC1', (5, 8, 1000, 'onehot'), {}),
    ('misaligned-logits', (50, 64, 18, 'prod'), dict(misalign='logits')),   # scalar cp.async
    ('env-major-chunks', (130, 12, 18, 'uniform'), dict(layout=1)),
    ('env-major-97', (97, 8, 18, 'onpolicy'), dict(layout=1)),
    ('ctas898', (8, 3590, 6, 'clip'), {}),                       # > 896 CTAs: second pass of v4's last-CTA loop
    # int32 time-major inputs that fail exactly one v8 condition
    ('no-v8-B%4', (50, 62, 18, 'prod'), {}),
    ('no-v8-T65', (65, 64, 18, 'hi'), {}),
    ('no-v8-A20', (50, 64, 20, 'lo'), {}),
    ('no-v8-A-odd', (50, 64, 5, 'noclip'), {}),
    ('no-v8-int64', (50, 64, 18, 'clip'), dict(act64=True)),
    ('no-v8-values+4B', (50, 64, 18, 'uniform'), dict(misalign='values')),
    ('no-v8-dones+1B', (50, 64, 18, 'onehot'), dict(misalign='dones')),
]


@pytest.mark.parametrize('shape,kw', [v[1:] for v in V4_CASES], ids=[v[0] for v in V4_CASES])
def test_v4_within_float64_bound(shape, kw, k1_path):
    T, B, A, regime = shape
    if A >= 238:
        assert _tc(T, A) == 1
    c = make_case(T, B, A, regime, seed=7)
    got, args = run_case(c, k1_path, V4, **kw)
    if kw.get('layout', 0) == 0:
        k1_path(4)
        _same_bits(got, _bits(_call(c, args)))


# ------------------------------------------------------------------------------------------------ a1

def a1_f32(blp, tlp, disc, rew, val, boot, cr, cp):
    """vtrace_returns_kernel in float32 numpy, its op order, with rho = float32(exp(float64(tlp - blp)))."""
    f = np.float32
    d = (tlp - blp).astype(f)
    rho = np.exp(d.astype(np.float64)).astype(f)
    rhoc = rho if cr is None else np.minimum(rho, f(cr))
    rpg = rho if cp is None else np.minimum(rho, f(cp))
    cs = np.minimum(rho, f(1.0))
    T, B = rew.shape
    vs, pg = np.zeros((T, B), f), np.zeros((T, B), f)
    acc = np.zeros(B, f)
    v_next, vs_next = boot.astype(f), boot.astype(f)
    for t in range(T - 1, -1, -1):
        delta = rhoc[t] * ((rew[t] + disc[t] * v_next) - val[t])
        acc = delta + (disc[t] * cs[t]) * acc
        vs[t] = acc + val[t]
        pg[t] = rpg[t] * ((rew[t] + disc[t] * vs_next) - val[t])
        vs_next, v_next = vs[t], val[t]
    return vs, pg, d


def _near_midpoint(d):
    """float64 exp(d) within 2^-50 (relative) of a float32 rounding midpoint: the one place a device exp may round
    the other way."""
    e = np.exp(d.astype(np.float64))
    f = e.astype(np.float32)
    lo = np.where(f.astype(np.float64) <= e, f, np.nextafter(f, np.float32(-np.inf)))
    mid = (lo.astype(np.float64) + np.nextafter(lo, np.float32(np.inf)).astype(np.float64)) / 2
    return np.abs(e - mid) <= 2.0 ** -50 * e


def _a1_inputs(golden):
    g = golden('vtrace_kat')
    out = [('kat-B%d' % B, [g['B%d_%s' % (B, n)].astype(np.float32) for n in
                            ('blp', 'tlp', 'discounts', 'rewards', 'values', 'bootstrap_value')]) for B in (1, 4)]
    for T, B in ((49, 512), (200, 33)):
        rng = np.random.RandomState(T * 1000 + B)
        blp = -np.abs(rng.randn(T, B)).astype(np.float32)
        tlp = (blp + 0.5 * rng.randn(T, B)).astype(np.float32)
        disc = ((rng.rand(T, B) > 0.1) * 0.99).astype(np.float32)
        out.append(('T%d-B%d' % (T, B), [blp, tlp, disc, rng.randn(T, B).astype(np.float32),
                                         rng.randn(T, B).astype(np.float32), rng.randn(B).astype(np.float32)]))
    return out


def test_a1_bit_exact(golden):
    from parl_b200 import kernels
    near_total = 0
    for name, x in _a1_inputs(golden):
        for cr, cp in ((1.0, 1.0), (None, None), (3.7, 2.2)):
            vs, pg = kernels.vtrace_from_importance_weights(*[torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
                                                              for a in x], cr, cp)
            want_vs, want_pg, d = a1_f32(*x, cr, cp)
            near = _near_midpoint(d)
            near_total += int(near.sum())
            # an element next to a midpoint may flip rho by 1 ulp; it reaches its own row of pg and its column's
            # vs at that row and earlier
            free = near | (np.flip(np.cumsum(np.flip(near, 0), 0), 0) > 0)
            for got, want in ((vs.cpu().numpy(), want_vs), (pg.cpu().numpy(), want_pg)):
                same = got.view(np.int32) == want.view(np.int32)
                assert np.all(same | free), (name, cr, cp, int((~same).sum()))
                ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
                assert np.all(ulp[free] <= 1), (name, cr, cp)
    print('\na1: %d rho values within 2^-50 of a float32 rounding midpoint' % near_total)


# ------------------------------------------------------------------------------------------------ rejections

REJECT = [('T1', dict(T=1), -1, 'bad shape'), ('A0', dict(A=0), -1, 'bad shape'),
          ('A1025', dict(A=1025), -1, 'bad shape'), ('layout2', dict(layout=2), -1, 'bad layout'),
          ('workspace', dict(ws_short=True), -5, 'workspace too small')]


@pytest.mark.parametrize('kw,code,msg', [v[1:] for v in REJECT], ids=[v[0] for v in REJECT])
def test_rejections_before_launch(kw, code, msg):
    """Every buffer is sized for the shape passed, so a missing check would still stay inside its buffers."""
    from parl_b200 import _lib
    lib = _lib.load()
    T, B, A, layout = kw.get('T', 8), 16, kw.get('A', 6), kw.get('layout', 0)
    n, na = T * B, T * B * max(A, 1)
    nan = float('nan')
    tl, bl = torch.randn(na, device=DEV), torch.randn(na, device=DEV)
    acts = torch.zeros(n, dtype=torch.int32, device=DEV)
    rew, vals = torch.randn(n, device=DEV), torch.randn(n, device=DEV)
    dones = torch.zeros(n, dtype=torch.uint8, device=DEV)
    losses = torch.full((8, ), nan, device=DEV)
    dl, dv = torch.full((na, ), nan, device=DEV), torch.full((n, ), nan, device=DEV)
    vs, pg = torch.full((n, ), nan, device=DEV), torch.full((n, ), nan, device=DEV)
    need = int(lib.rl_loss_workspace_bytes(B))
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    P = _lib.ptr

    def call():
        return lib.rl_vtrace_loss_fwd_bwd(P(tl), P(bl), P(acts), 0, P(rew), P(dones), P(vals), T, B, A, layout,
                                          0.99, 1.0, 1.0, 0.5, -0.01, P(losses), P(dl), P(dv), P(vs), P(pg), P(ws),
                                          need - 1 if kw.get('ws_short') else ws.numel(), _lib.stream())
    rc, names = _launched(call)
    assert rc == code, (rc, lib.rl_last_error())
    assert msg in lib.rl_last_error().decode()
    assert not any('vtrace' in nm for nm in names), names
    for t in (losses, dl, dv, vs, pg):
        assert torch.isnan(t).all()
    assert int(ws.count_nonzero()) == 0
