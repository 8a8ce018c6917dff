"""FlatAdam — the learner's optimiser on ONE flat fp32 parameter buffer.

All parameters of the model are re-homed as views into a single contiguous buffer (and their
``.grad`` as views into a second one), so the whole update — global-norm clip + Adam + grad
zeroing — is two kernel launches (rl_grad_global_norm, rl_adam_step) with no host sync, and a
multi-GPU learner all-reduces exactly one tensor.  Semantics follow the reference learners:
  clip='paddle' : paddle.nn.ClipGradByGlobalNorm  (parl/algorithms/paddle/impala/impala.py:113-117)
  clip='torch'  : torch.nn.utils.clip_grad_norm_  (parl/algorithms/torch/a2c.py:66, ppo.py:145)
  clip=None     : plain Adam                      (parl/algorithms/torch/dqn.py:68-71)
"""
import torch

from .. import kernels

_CLIP = {None: 0, 'none': 0, 'torch': 1, 'paddle': 2}


class FlatAdam(object):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, clip=None, max_norm=0.0):
        self.params = [p for p in params if p.requires_grad]
        assert len(self.params) > 0
        dev = self.params[0].device
        if dev.type != 'cuda':
            raise RuntimeError('FlatAdam runs on the H100 only: move the model to CUDA first (no CPU fallback)')
        offs, total = [], 0
        for p in self.params:
            assert p.dtype == torch.float32 and p.device == dev
            offs.append(total)
            total += (p.numel() + 3) // 4 * 4            # keep every view 16-byte aligned
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(total, dtype=torch.float32, device=dev)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)
        self.norm = torch.zeros(1, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for p, o in zip(self.params, offs):
                n = p.numel()
                self.flat[o:o + n].copy_(p.detach().reshape(-1))
                p.data = self.flat[o:o + n].view(p.shape)
                p.grad = self.grad[o:o + n].view(p.shape)
        self.lr, self.betas, self.eps = lr, betas, eps
        self.clip_mode, self.max_norm = _CLIP[clip], max_norm
        self.step_count = 0
        self.step_dev = self.lr_dev = None          # device-resident update count / learning rate (graph replay)

    def enable_device_state(self):
        """Keep the update count and the learning rate on the device so that a captured CUDA graph of the whole
        update (forward, loss, backward, clip, Adam) can be replayed: ``step()`` then increments the device counter
        and the Adam kernel reads both scalars from memory.  Set the rate with ``set_lr`` (outside the graph)."""
        if self.step_dev is None:
            dev = self.flat.device
            self.step_dev = torch.full((1, ), self.step_count, dtype=torch.int32, device=dev)
            self.lr_dev = torch.full((1, ), float(self.lr), dtype=torch.float32, device=dev)
        return self

    def set_lr(self, lr):
        self.lr = float(lr)
        if self.lr_dev is not None:
            self.lr_dev.fill_(self.lr)

    def zero_grad(self):
        self.grad.zero_()

    def step(self, lr=None, grad_div=1.0):
        if lr is not None and self.lr_dev is None:
            self.lr = lr
        self.step_count += 1
        if self.step_dev is not None:
            self.step_dev.add_(1)
        if self.clip_mode:
            kernels.grad_global_norm(self.grad, self.norm)
        kernels.adam_step(self.flat, self.grad, self.exp_avg, self.exp_avg_sq, self.lr, self.betas[0], self.betas[1],
                          self.eps, self.step_count, grad_div=grad_div, grad_norm=self.norm if self.clip_mode else None,
                          max_norm=self.max_norm, clip_mode=self.clip_mode, zero_grad=True, lr_device=self.lr_dev,
                          step_device=self.step_dev)

    def state_dict(self):
        return dict(exp_avg=self.exp_avg, exp_avg_sq=self.exp_avg_sq, step=self.step_count, lr=self.lr)

    def load_state_dict(self, sd):
        self.exp_avg.copy_(sd['exp_avg'])
        self.exp_avg_sq.copy_(sd['exp_avg_sq'])
        self.step_count, self.lr = int(sd['step']), float(sd['lr'])
        if self.step_dev is not None:
            self.step_dev.fill_(self.step_count)
            self.lr_dev.fill_(self.lr)
