"""Micro-benchmarks of individual kernels (CUDA events, rotating >L2 buffers).
    python tools/bench_kernels.py [vtrace|env|losses|conv|all]     (conv is not part of all)
"""
import json
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from parl_b200 import kernels as K  # noqa


def time_fn(fn, iters=50, warmup=5, graph=False):
    """Seconds per call of fn(i).  graph=True: the `iters` calls are captured into ONE CUDA graph and the replay is
    timed, so the figure is the GPU time of back-to-back launches, not the host's launch rate (a K1 call costs
    ~10 us of Python + ctypes, more than the kernel once it is fast)."""
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(iters):
                fn(i)
        g.replay()
        torch.cuda.synchronize()
        best = None
        for _ in range(3):
            st.record()
            g.replay()
            en.record()
            torch.cuda.synchronize()
            t = st.elapsed_time(en) / iters * 1e-3
            best = t if best is None else min(best, t)
        return best
    st.record()
    for i in range(iters):
        fn(i)
    en.record()
    torch.cuda.synchronize()
    return st.elapsed_time(en) / iters * 1e-3


def bench_vtrace(T=50, B=4096, A=18, nbuf=8, iters=64, graph=True):
    dev = 'cuda:0'
    bufs = []
    for i in range(nbuf):
        g = torch.Generator(device=dev).manual_seed(i)
        tl = 2 * torch.randn(T * B, A, device=dev, generator=g)
        bl = tl + 0.5 * torch.randn(T * B, A, device=dev, generator=g)
        acts = torch.randint(0, A, (T * B,), device=dev, dtype=torch.int32, generator=g)
        rew = (torch.rand(T * B, device=dev, generator=g) < 0.5).float()
        dones = (torch.rand(T * B, device=dev, generator=g) < 0.1).to(torch.uint8)
        vals = torch.randn(T * B, device=dev, generator=g)
        out = dict(d_logits=torch.empty_like(tl), d_values=torch.empty_like(vals),
                   losses=torch.empty(8, device=dev))
        bufs.append((tl, bl, acts, rew, dones, vals, out))

    def run(i):
        tl, bl, acts, rew, dones, vals, out = bufs[i % nbuf]
        K.vtrace_loss_fwd_bwd(tl, bl, acts, rew, dones, vals, T, B, 0.99, 0.5, -0.01, out=out)
    sec = time_fn(run, iters=iters, warmup=max(5, nbuf), graph=graph)
    alg_bytes = (T - 1) * B * (12 * A + 17) + 4 * B
    return dict(kernel='vtrace_loss_fwd_bwd', T=T, B=B, A=A, us=sec * 1e6, timing='graph' if graph else 'eager',
                alg_bytes=alg_bytes,
                gbps=alg_bytes / sec / 1e9, footprint_mb=nbuf * alg_bytes / 1e6)


def bench_env(B=4096, HW=84 * 84, nplanes=16, iters=64):
    dev = 'cuda:0'
    planes = torch.zeros(nplanes, B, HW, dtype=torch.uint8, device=dev)
    rew = torch.zeros(B, device=dev)
    done = torch.zeros(B, dtype=torch.uint8, device=dev)
    age = torch.zeros(B, dtype=torch.uint8, device=dev)
    st = K.EpisodeStats(B, dev)
    logits = torch.randn(B, 18, device=dev)
    acts = torch.zeros(B, dtype=torch.int32, device=dev)

    def run(i):
        K.env_atari_synth_step(planes[i % nplanes], rew, done, age, age, st, 1, i, logits=logits, actions_out=acts)
    sec = time_fn(run, iters=iters)
    alg = B * HW
    return dict(kernel='env_atari_synth_step', B=B, us=sec * 1e6, alg_bytes=alg, gbps=alg / sec / 1e9,
                env_steps_per_s=B / sec)


def bench_a2c(N=256 * 20, A=2, nbuf=32):
    """K2 at configs[1]: 256 CartPole envs x 20 steps per update; algorithmic bytes 8A+17 per row (SURVEY 8d)."""
    dev = 'cuda:0'
    g = torch.Generator(device=dev).manual_seed(0)
    bufs = [(torch.randn(N, A, device=dev, generator=g), torch.randn(N, device=dev, generator=g),
             torch.randint(0, A, (N,), device=dev, dtype=torch.int32, generator=g),
             torch.randn(N, device=dev, generator=g), torch.randn(N, device=dev, generator=g)) for _ in range(nbuf)]
    sec = time_fn(lambda i: K.a2c_loss_fwd_bwd(*bufs[i % nbuf], 0.5, -0.01))
    alg = N * (8 * A + 17)
    return dict(kernel='a2c_loss_fwd_bwd', N=N, A=A, us=sec * 1e6, alg_bytes=alg, gbps=alg / sec / 1e9)


def bench_gae(T=2048, B=2048, segments=False, iters=20):
    """K3 at configs[3]: 2048 envs x 2048 steps; 17 B per (t,b) (read r, V, done; write adv, ret)."""
    dev = 'cuda:0'
    g = torch.Generator(device=dev).manual_seed(1)
    r, v = torch.randn(T, B, device=dev, generator=g), torch.randn(T, B, device=dev, generator=g)
    d = (torch.rand(T, B, device=dev, generator=g) < 0.01)
    lv = torch.randn(B, device=dev, generator=g)
    if segments:
        sec = time_fn(lambda i: K.gae_scan_segments(r, v, d.to(torch.uint8), lv, 0.99, 0.95), iters=iters)
    else:
        df, ld = d.float(), torch.zeros(B, device=dev)
        sec = time_fn(lambda i: K.gae_scan(r, v, df, lv, ld, 0.99, 0.95), iters=iters)
    alg = T * B * 17
    return dict(kernel='gae_scan_segments' if segments else 'gae_scan', T=T, B=B, us=sec * 1e6, alg_bytes=alg,
                gbps=alg / sec / 1e9)


def bench_ppo(N=2048 * 64, D=6, iters=30):
    """K3 loss at configs[3]: Gaussian minibatch (obs 17, act 6); 12D+24 B per row."""
    dev = 'cuda:0'
    g = torch.Generator(device=dev).manual_seed(2)
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    vals, act, bv, br, blp, adv = rn(N), rn(N, D), rn(N), rn(N), rn(N), rn(N)
    mean, logstd = rn(N, D), torch.zeros(D, device=dev)
    sec = time_fn(lambda i: K.ppo_loss_fwd_bwd(vals, act, bv, br, blp, adv, mean=mean, logstd=logstd), iters=iters)
    alg = N * (12 * D + 24)
    return dict(kernel='ppo_loss_fwd_bwd(gaussian)+adv_stats', N=N, D=D, us=sec * 1e6, alg_bytes=alg,
                gbps=alg / sec / 1e9)


def bench_td(M=4096, A=18, double_q=True):
    """K4: TD loss of a replay batch; (8..12)A+17 B per sample."""
    dev = 'cuda:0'
    g = torch.Generator(device=dev).manual_seed(3)
    q, qt, qo = (torch.randn(M, A, device=dev, generator=g) for _ in range(3))
    a = torch.randint(0, A, (M,), device=dev, dtype=torch.int32, generator=g)
    r, term = torch.randn(M, device=dev, generator=g), (torch.rand(M, device=dev, generator=g) < 0.05).float()
    sec = time_fn(lambda i: K.td_loss_fwd_bwd(q, qt, a, r, term, 0.99, q_online_next=qo if double_q else None))
    alg = M * ((12 if double_q else 8) * A + 17)
    return dict(kernel='td_loss_fwd_bwd', M=M, A=A, double_q=double_q, us=sec * 1e6, alg_bytes=alg,
                gbps=alg / sec / 1e9)


def bench_per(capacity=1 << 20, batch=4096):
    """C5: priority sample + update on a 1M-leaf fp64 sum tree (latency-bound: tree depth 20)."""
    dev = 'cuda:0'
    tree = K.DeviceSumTree(capacity, dev)
    tree.store(0, capacity, 0.6, 0.01)
    pri = torch.rand(batch, device=dev)
    out = {}
    sec = time_fn(lambda i: out.__setitem__('s', tree.sample(batch, 0.4, float(capacity), seed=7, draw=i)))
    sec_u = time_fn(lambda i: tree.update(out['s'][0], pri, 0.6, 0.01))
    return dict(kernel='per_sample / per_update', capacity=capacity, batch=batch, sample_us=sec * 1e6,
                update_us=sec_u * 1e6, samples_per_s=batch / sec)


def bench_replay_gather(cap=1 << 17, lanes=8, batch=4096, ctx=4, HW=7056):
    """C5: 5-frame window gather from the frame ring; 35 280 B read + 35 280 B written per sample."""
    dev = 'cuda:0'
    frames = torch.randint(0, 255, (cap, HW), device=dev, dtype=torch.uint8)
    over = (torch.rand(cap, device=dev) < 0.05).to(torch.uint8)
    g = torch.Generator(device=dev).manual_seed(5)
    idx = [torch.randint(0, cap - 16 * lanes, (batch, ), device=dev, dtype=torch.int32, generator=g) for _ in range(8)]
    out = torch.empty((batch, ctx + 1, HW), dtype=torch.uint8, device=dev)
    sec = time_fn(lambda i: K.replay_gather_frames(frames, over, idx[i % 8], cap // lanes, ctx, lanes=lanes, out=out))
    alg = batch * (ctx + 1) * HW * 2
    return dict(kernel='replay_gather_frames', batch=batch, lanes=lanes, us=sec * 1e6, alg_bytes=alg,
                gbps=alg / sec / 1e9)


def bench_mlp(N=131072, dims=(17, 64, 64), heads=(6, 1)):
    """K6 (MLP family) at the C4 minibatch: fp32 forward / backward of the MuJoCo actor-critic."""
    dev = 'cuda:0'
    import torch.nn as nn
    torch.manual_seed(0)
    layers = [nn.Linear(dims[i], dims[i + 1]).to(dev) for i in range(len(dims) - 1)]
    hs = [nn.Linear(dims[-1], h).to(dev) for h in heads]
    plan = K.MlpPlan([[(m.weight.detach(), m.bias.detach())] for m in layers] +
                     [[(h.weight.detach(), h.bias.detach()) for h in hs]], K.ACT_TANH)
    x = torch.randn(N, dims[0], device=dev)
    out = torch.empty(N, sum(heads), device=dev)
    d = torch.randn_like(out)
    grads = [(torch.empty_like(m.weight), torch.empty_like(m.bias)) for m in layers + hs]
    sf = time_fn(lambda i: plan.forward(x, out=out), iters=30)
    sb = time_fn(lambda i: plan.backward(x, d, grads=grads), iters=30)
    flop = 2.0 * N * (sum(dims[i] * dims[i + 1] for i in range(len(dims) - 1)) + dims[-1] * sum(heads))
    return dict(kernel='mlp_fwd / mlp_bwd', N=N, dims=list(dims), heads=list(heads), fwd_us=sf * 1e6, bwd_us=sb * 1e6,
                fwd_tflops=flop / sf / 1e12, bwd_tflops=3 * flop / sb / 1e12,
                fwd_gbps=N * (dims[0] + sum(heads)) * 4 / sf / 1e9)


# The five window-conv calls of the Atari actor-critic (engine/train_net.py):
#   name, call, input [H,W,C] (and dtype), weight [rows, cols], output shape, out_mode, mask [H,W,C], bytes written per sample
# Algorithmic bytes are what the layer has to move: its input, the ReLU mask of a data gradient, and the valid output
# region it writes.  MMA FLOPs are what the kernel issues: every position of every 128-row tile, dropped ones included.
_CONVS = (
    ('conv1_fwd', 'fwd', (21, 21, 64), torch.uint8, (32, 256), (12, 12, 128), 1, None, 20 * 20 * 32 * 2),
    ('conv2_fwd', 'fwd', (12, 12, 128), torch.bfloat16, (64, 512), (11, 11, 64), 0, None, 11 * 11 * 64 * 2),
    ('conv3_fwd', 'fwd', (11, 11, 64), torch.bfloat16, (64, 576), (9, 9, 64), 0, None, 9 * 9 * 64 * 2),
    ('conv3_dgrad', 'dgrad', (11, 11, 64), torch.bfloat16, (64, 576), (12, 12, 64), 0, (11, 11, 64), 11 * 11 * 64 * 2),
    ('conv2_dgrad', 'dgrad', (12, 12, 64), torch.bfloat16, (128, 256), (21, 21, 32), 2, (12, 12, 128), 20 * 20 * 32 * 2),
)
_HBM_TBS, _BF16_TFLOPS = 3.35, 989.0      # H100 SXM data sheet (dense BF16)


def bench_conv(name, N, nbuf, iters):
    """One window-conv call (shiftconv_fwd_kernel) at batch N, timed with CUDA events over `nbuf` rotating operand sets."""
    _, kind, xs, xdt, ws, os_, out_mode, ms_, out_bytes = next(c for c in _CONVS if c[0] == name)
    dev = 'cuda:0'
    g = torch.Generator(device=dev).manual_seed(7)
    k = 3 if ws[1] == 576 else 2
    w = (0.05 * torch.randn(ws, device=dev, generator=g)).to(torch.bfloat16)
    bias = 0.1 * torch.randn(ws[0], device=dev, generator=g)
    sets = []
    for _ in range(nbuf):
        if xdt == torch.uint8:
            x = torch.randint(0, 256, (N, ) + xs, device=dev, dtype=torch.uint8, generator=g)
        else:
            x = torch.randn((N, ) + xs, device=dev, generator=g).to(torch.bfloat16)
        mask = torch.randn((N, ) + ms_, device=dev, generator=g).to(torch.bfloat16) if ms_ else None
        sets.append((x, mask, torch.zeros((N, ) + os_, device=dev, dtype=torch.bfloat16)))

    def run(i):
        x, mask, out = sets[i % nbuf]
        if kind == 'fwd':
            K.conv2d_s1_nhwc_bf16_fwd(x, w, bias, k, k, relu=True, out=out, out_mode=out_mode)
        else:
            K.conv2d_s1_nhwc_bf16_dgrad(x, w, k, k, out, act_mask=mask, out_mode=out_mode)
    sec = time_fn(run, iters=iters, warmup=max(3, nbuf))
    in_bytes = xs[0] * xs[1] * xs[2] * (1 if xdt == torch.uint8 else 2)
    mask_bytes = ms_[0] * ms_[1] * ms_[2] * 2 if ms_ else 0
    alg_bytes = N * (in_bytes + mask_bytes + out_bytes)
    tiles = -(-N * xs[0] * xs[1] // 128)
    mma_flop = 2.0 * tiles * 128 * ws[0] * ws[1]        # M = positions, N = output channels, K = taps x input channels
    t_hbm, t_mma = alg_bytes / (_HBM_TBS * 1e12), mma_flop / (_BF16_TFLOPS * 1e12)
    return dict(kernel=name, N=N, ms=sec * 1e3, alg_bytes=alg_bytes, mma_flop=mma_flop,
                bound='hbm' if t_hbm >= t_mma else 'mma', bound_ms=max(t_hbm, t_mma) * 1e3,
                share=max(t_hbm, t_mma) / sec, peaks='H100 SXM data sheet: 3.35 TB/s, 989 TFLOP/s dense BF16')


if __name__ == '__main__':
    which = sys.argv[1] if len(sys.argv) > 1 else 'all'
    if which == 'conv':
        # learner batch: 50 steps x 4096 envs (operands far larger than the L2);  actor batch: 4096, rotating operand
        # sets so that no call finds its input in the 50 MB L2
        for name in [c[0] for c in _CONVS]:
            print(json.dumps(bench_conv(name, 50 * 4096, nbuf=1, iters=10)))
            torch.cuda.empty_cache()
        for name in [c[0] for c in _CONVS]:
            print(json.dumps(bench_conv(name, 4096, nbuf=4, iters=100)))
    if which == 'vtrace_cpasync':
        from parl_b200 import _lib
        _lib.load().rl_debug_set_tma(1)
        r = bench_vtrace()
        r['path'] = 'cp.async'
        print(json.dumps(r))
    if which == 'vtrace_c3':
        print(json.dumps(bench_vtrace()))
    if which in ('vtrace', 'all'):
        print(json.dumps(bench_vtrace()))
        print(json.dumps(bench_vtrace(B=65536, nbuf=2, iters=16)))
        print(json.dumps(bench_vtrace(B=512, nbuf=64)))
    if which in ('env', 'all'):
        print(json.dumps(bench_env()))
        print(json.dumps(bench_env(B=512)))
    if which in ('losses', 'all'):
        # K2-K4 at the BASELINE.json configs[1], [3], [4] shapes (not yet captured under ncu: next round)
        for fn in (bench_a2c, bench_gae, lambda: bench_gae(T=20, B=256, segments=True), bench_ppo, bench_td, bench_per,
                   bench_replay_gather, bench_mlp):
            try:
                print(json.dumps(fn()))
            except Exception as e:      # a tool, not a test: report and carry on
                print(json.dumps(dict(error=repr(e))))
