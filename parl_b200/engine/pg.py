"""REINFORCE on one H100 — the on-device replacement of benchmark/torch/QuickStart/train.py:28-76 (BASELINE
configs[0]: CartPole policy gradient; the reference runs ONE env in one CPU process, here B envs run in lock-step).

    rollout  ONE launch (rl_rollout_mlp): T steps of CartPole physics + policy forward + exact categorical sampling
    returns  reward-to-go inside every episode segment (calc_reward_to_go with gamma = 1.0, train.py:47-50) =
             rl_gae_scan_segments with values 0, gamma 1, lambda 1 and bootstrap 0 (fp64 scan)
    learn    rl_mlp_fwd -> softmax -> rl_pg_loss_fwd_bwd (mean(-log p_a * G), policy_gradient.py:54-75) ->
             softmax backward -> rl_mlp_bwd -> Adam
"""
import torch

from .. import kernels
from ..algorithms import PolicyGradient
from .nets import CartPolePolicy


class PolicyGradientEngine(object):
    def __init__(self, num_envs=256, rollout_steps=200, lr=1e-3, gamma=1.0, seed=0, device=None, env_offset=0,
                 max_episode_steps=200, model=None):
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = dev = torch.device(device)
        self.B, self.T, self.gamma = int(num_envs), int(rollout_steps), float(gamma)
        self.seed, self.env_offset, self.max_episode_steps = int(seed), int(env_offset), int(max_episode_steps)
        self.model = (model if model is not None else CartPolePolicy(4, 2)).to(dev)
        self.alg = PolicyGradient(self.model, lr=float(lr))
        layers, act = self.model.native_layers()
        self.plan = kernels.MlpPlan(layers, act)
        B, T, f32 = self.B, self.T, torch.float32
        self.stats = kernels.EpisodeStats(B, dev)
        self.obs_cur = torch.zeros((B, 4), dtype=f32, device=dev)
        self.obs = torch.empty((T, B, 4), dtype=f32, device=dev)
        self.actions = torch.empty((T, B), dtype=torch.int32, device=dev)
        self.rewards = torch.empty((T, B), dtype=f32, device=dev)
        self.dones = torch.empty((T, B), dtype=torch.uint8, device=dev)
        self.zeros_tb = torch.zeros((T, B), dtype=f32, device=dev)
        self.zeros_b = torch.zeros(B, dtype=f32, device=dev)
        self.logits = torch.empty((T * B, 2), dtype=f32, device=dev)
        self.env_steps = self.sample_steps = 0
        kernels.env_cartpole_step(torch.zeros((B, 4), dtype=f32, device=dev), self.obs_cur, None, None, None, self.stats,
                                  self.seed, 0, max_episode_steps=self.max_episode_steps, env_offset=self.env_offset,
                                  reset=True)

    def rollout(self):
        self.plan.rollout(kernels.ENV_CARTPOLE, kernels.POLICY_CATEGORICAL, self.T, self.obs_cur, self.stats, self.seed,
                          self.env_steps, self.obs, self.actions, self.rewards, self.dones, has_value=False,
                          env_offset=self.env_offset, max_episode_steps=self.max_episode_steps)
        self.env_steps += self.T
        self.sample_steps += self.T * self.B

    def learn(self):
        T, B = self.T, self.B
        togo, _ = kernels.gae_scan_segments(self.rewards, self.zeros_tb, self.dones, self.zeros_b, self.gamma, 1.0)
        x = self.obs.view(T * B, 4)
        self.plan.forward(x, out=self.logits)
        prob = torch.softmax(self.logits, dim=1)
        res = kernels.pg_loss_fwd_bwd(prob, self.actions.view(-1), togo.view(-1))
        dp = res['d_prob']
        d_logits = prob * (dp - (dp * prob).sum(1, keepdim=True))
        self.plan.backward(x, d_logits.contiguous())
        if getattr(self.alg, 'grad_sync', None) is not None:
            self.alg.grad_sync(self.alg.optimizer.grad)
        self.alg.optimizer.step()
        return res['losses']

    def step(self):
        self.rollout()
        return self.learn()

    def get_metrics(self):
        tot = self.stats.totals.tolist()
        n = max(tot[0], 1.0)
        return dict(sample_steps=self.sample_steps, episodes=int(tot[0]), mean_episode_rewards=tot[1] / n,
                    mean_episode_steps=tot[2] / n)
