"""One learner update bracketed by cudaProfilerStart/Stop, for ncu --profile-from-start off:
    ncu --set full --clock-control none --import-source on --profile-from-start off \
        -k regex:"shiftconv|wgrad_window" -o learn python tools/profile_learn.py [envs]
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from parl_b200.engine.impala import ImpalaEngine  # noqa

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
dev = torch.device('cuda', 0)
torch.manual_seed(0)
eng = ImpalaEngine(num_envs=B, sample_batch_steps=50, act_dim=18, seed=1, device=dev, use_graph=False)
for _ in range(2):
    eng.rollout()
    eng.learn(1e-3, -0.01)
eng.rollout()
torch.cuda.synchronize()
torch.cuda.profiler.start()
eng.learn(1e-3, -0.01)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print('done')
