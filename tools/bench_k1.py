"""K1 (rl_vtrace_loss_fwd_bwd) timing matrix: kernel path x shape, two timing methods.
    python tools/bench_k1.py
 a) 'rot':   64 back-to-back launches over 8 rotating buffer sets (8 x 47 MB > the 50 MB L2 of an H100), captured in one CUDA graph,
             one event pair around the replay (the eager Python loop next to it: host-launch-rate bound)
 b) 'flush': one event pair per launch, a 256 MB fill between launches evicts L2
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from parl_b200 import kernels as K, _lib  # noqa
from tools.bench_kernels import bench_vtrace  # noqa


def flushed(T, B, A, n=12):
    dev = 'cuda:0'
    tl = 2 * torch.randn(T * B, A, device=dev)
    bl = tl + 0.5 * torch.randn(T * B, A, device=dev)
    acts = torch.randint(0, A, (T * B,), device=dev, dtype=torch.int32)
    rew = (torch.rand(T * B, device=dev) < 0.5).float()
    dones = (torch.rand(T * B, device=dev) < 0.1).to(torch.uint8)
    vals = torch.randn(T * B, device=dev)
    out = dict(d_logits=torch.empty_like(tl), d_values=torch.empty_like(vals), losses=torch.empty(8, device=dev))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    ev = []
    for i in range(n):
        flush.fill_(i)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        K.vtrace_loss_fwd_bwd(tl, bl, acts, rew, dones, vals, T, B, 0.99, 0.5, -0.01, out=out)
        b.record()
        ev.append((a, b))
    torch.cuda.synchronize()
    ms = sorted(x.elapsed_time(y) for x, y in ev[2:])
    return sum(ms) / len(ms) * 1e3


if __name__ == '__main__':
    lib = _lib.load()
    # HBM peak: MEASURED_PEAKS.json at the repository root when present, else the H100 SXM data sheet (not measured)
    peaks = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'MEASURED_PEAKS.json')
    peak = float(json.load(open(peaks))['hbm_gbs']) if os.path.exists(peaks) else 3350.0
    for (T, B, A) in [(50, 4096, 18), (50, 512, 18), (50, 65536, 18)]:
        for mode in (0, 4, 9):
            lib.rl_debug_set_vtrace_path(mode)
            nbuf = 8 if B <= 4096 else 2
            r = bench_vtrace(T, B, A, nbuf=nbuf)
            r_eager = bench_vtrace(T, B, A, nbuf=nbuf, graph=False)
            us_f = flushed(T, B, A)
            r.update(mode=mode, frac_rot=r['gbps'] / peak, us_eager_loop=r_eager['us'], us_flushed=us_f,
                     frac_flushed=r['alg_bytes'] / us_f / 1e3 / peak)
            print(json.dumps(r))
    lib.rl_debug_set_vtrace_path(0)
