"""``RolloutStorage`` in HBM — interface of benchmark/torch/ppo/storage.py:18-76 (append / compute_returns /
sample_batch) with the (T,B) buffers resident on the H100: ``compute_returns`` is one launch of rl_gae_scan (the
reference's backward numpy loop, bit for bit in float32), ``sample_batch(idx)`` gathers the minibatch rows on the
device (rl_gather_rows) and returns device tensors that ``PPO.learn`` takes as they are (numpy with ``as_numpy``)."""
import numpy as np
import torch

from .. import kernels

__all__ = ['RolloutStorage']


def _shape(space):
    return tuple(space.shape) if hasattr(space, 'shape') else ((int(space), ) if int(space) > 0 else ())


class RolloutStorage(object):
    def __init__(self, step_nums, env_num, obs_space, act_space, device=None):
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError('parl_b200.RolloutStorage lives in HBM: no CUDA device visible (no CPU fallback)')
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = dev = torch.device(device)
        self.step_nums, self.env_num = int(step_nums), int(env_num)
        self.obs_shape, self.act_shape = _shape(obs_space), _shape(act_space)
        T, B, f32 = self.step_nums, self.env_num, torch.float32
        self.obs = torch.zeros((T, B) + self.obs_shape, dtype=f32, device=dev)
        self.actions = torch.zeros((T, B) + self.act_shape, dtype=f32, device=dev)
        self.logprobs = torch.zeros((T, B), dtype=f32, device=dev)
        self.rewards = torch.zeros((T, B), dtype=f32, device=dev)
        self.dones = torch.zeros((T, B), dtype=f32, device=dev)
        self.values = torch.zeros((T, B), dtype=f32, device=dev)
        self.cur_step = 0
        self.advantages = self.returns = None

    def _put(self, dst, x):
        dst.copy_(torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).to(dst.dtype).reshape(dst.shape),
                  non_blocking=True)

    def append(self, obs, action, logprob, reward, done, value):
        t = self.cur_step
        self._put(self.obs[t], obs), self._put(self.actions[t], action), self._put(self.logprobs[t], logprob)
        self._put(self.rewards[t], reward), self._put(self.dones[t], done), self._put(self.values[t], value)
        self.cur_step = (t + 1) % self.step_nums

    def compute_returns(self, value, done, gamma=0.99, gae_lambda=0.95):
        dev, f32 = self.device, torch.float32
        last_v = torch.as_tensor(np.asarray(value) if not torch.is_tensor(value) else value).to(dev, f32).reshape(-1)
        last_d = torch.as_tensor(np.asarray(done) if not torch.is_tensor(done) else done).to(dev, f32).reshape(-1)
        self.advantages, self.returns = kernels.gae_scan(self.rewards, self.values, self.dones, last_v.contiguous(),
                                                         last_d.contiguous(), gamma, gae_lambda)
        return self.advantages, self.returns

    def sample_batch(self, idx, as_numpy=False):
        """-> (obs, actions, logprobs, advantages, returns, values) rows ``idx`` of the flattened (T*B) rollout."""
        N = self.step_nums * self.env_num
        idx = torch.as_tensor(np.asarray(idx) if not torch.is_tensor(idx) else idx).to(self.device, torch.int32)
        idx = idx.contiguous()
        row = lambda x, shp: kernels.gather_rows(x.reshape(N, -1), idx).reshape((idx.numel(), ) + shp)
        out = (row(self.obs, self.obs_shape), row(self.actions, self.act_shape), row(self.logprobs, ()),
               row(self.advantages, ()), row(self.returns, ()), row(self.values, ()))
        return tuple(o.cpu().numpy() for o in out) if as_numpy else out
