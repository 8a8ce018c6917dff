"""A2C on one H100 — the on-device replacement of benchmark/torch/a2c/{train.py:33-177, actor.py:30-123}
(BASELINE configs[1]: 256 vectorised CartPole envs, fused GAE + policy-gradient kernels).

    rollout  ONE launch (rl_rollout_mlp): T lock-step steps of all B envs — actor-critic forward, exact categorical
             sampling, CartPole physics with auto-reset, episode statistics — trajectory written time-major
             into (T,B) HBM buffers, values[T] = bootstrap value of the observation after the last step
    returns  rl_gae_scan_segments: calc_gae per episode segment in fp64 (parl/utils/rl_utils.py:21-51 as used by
             actor.py:82-102: next_value = 0 after a done, V(next_obs) at the rollout end)
    learn    rl_mlp_fwd over the T*B observations -> rl_a2c_loss_fwd_bwd (SUM losses + gradients, a2c.py:40-60)
             -> rl_mlp_bwd (recompute, no saved activations) -> clip_grad_norm_(40) + Adam (FlatAdam)
The ``parl.algorithms.A2C`` object (``self.alg``) holds the model and optimiser, so ``get_weights`` /
``set_weights`` / ``Agent.save`` keep working; multi-GPU: ``alg.grad_sync`` all-reduces (SUM) the flat gradient.
"""
import torch

from .. import kernels
from ..algorithms import A2C
from .nets import CartPoleActorCritic


class A2CEngine(object):
    def __init__(self, num_envs=256, sample_batch_steps=20, gamma=0.99, lam=1.0, vf_loss_coeff=0.5, learning_rate=0.001,
                 seed=0, device=None, env_offset=0, max_episode_steps=200, model=None):
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = dev = torch.device(device)
        self.B, self.T = int(num_envs), int(sample_batch_steps)
        self.gamma, self.lam = float(gamma), float(lam)
        self.seed, self.env_offset, self.max_episode_steps = int(seed), int(env_offset), int(max_episode_steps)
        self.model = (model if model is not None else CartPoleActorCritic(4, 2)).to(dev)
        self.alg = A2C(self.model, dict(vf_loss_coeff=vf_loss_coeff, learning_rate=learning_rate))
        layers, act = self.model.native_layers()           # after the optimiser re-homed the parameters
        self.plan = kernels.MlpPlan(layers, act)
        self.A = self.plan.out_dim - 1
        B, T, f32 = self.B, self.T, torch.float32
        self.stats = kernels.EpisodeStats(B, dev)
        self.obs_cur = torch.zeros((B, 4), dtype=f32, device=dev)
        self.obs = torch.empty((T, B, 4), dtype=f32, device=dev)
        self.actions = torch.empty((T, B), dtype=torch.int32, device=dev)
        self.rewards = torch.empty((T, B), dtype=f32, device=dev)
        self.dones = torch.empty((T, B), dtype=torch.uint8, device=dev)
        self.values = torch.empty((T + 1, B), dtype=f32, device=dev)
        self.logits = torch.empty((T * B, self.A), dtype=f32, device=dev)
        self.v_learn = torch.empty((T * B, 1), dtype=f32, device=dev)
        self.env_steps = 0
        self.sample_steps = 0
        self.reset()

    def reset(self):
        scratch = torch.zeros((self.B, 4), dtype=torch.float32, device=self.device)
        kernels.env_cartpole_step(scratch, self.obs_cur, None, None, None, self.stats, self.seed, 0,
                                  max_episode_steps=self.max_episode_steps, env_offset=self.env_offset, reset=True)
        self.env_steps = 0

    def rollout(self):
        """T lock-step steps of all envs (Actor.sample, actor.py:59-110) — one kernel launch."""
        self.plan.rollout(kernels.ENV_CARTPOLE, kernels.POLICY_CATEGORICAL, self.T, self.obs_cur, self.stats, self.seed,
                          self.env_steps, self.obs, self.actions, self.rewards, self.dones, val_out=self.values,
                          has_value=True, env_offset=self.env_offset, max_episode_steps=self.max_episode_steps)
        self.env_steps += self.T
        self.sample_steps += self.T * self.B

    def learn(self, learning_rate=0.001, entropy_coeff=-0.01):
        T, B = self.T, self.B
        adv, tgt = kernels.gae_scan_segments(self.rewards, self.values[:T], self.dones, self.values[T], self.gamma,
                                             self.lam)
        x = self.obs.view(T * B, 4)
        self.plan.forward(x, out=self.logits, out2=self.v_learn, split=self.A)
        res = kernels.a2c_loss_fwd_bwd(self.logits, self.v_learn.view(-1), self.actions.view(-1), adv.view(-1),
                                       tgt.view(-1), self.alg.vf_loss_coeff, entropy_coeff)
        self.plan.backward(x, res['d_logits'], d_out2=res['d_values'].view(-1, 1), split=self.A)
        if self.alg.grad_sync is not None:
            self.alg.grad_sync(self.alg.optimizer.grad)
        self.alg.optimizer.step(lr=learning_rate)
        return res['losses']

    def step(self, learning_rate=0.001, entropy_coeff=-0.01):
        self.rollout()
        return self.learn(learning_rate, entropy_coeff)

    def get_metrics(self):
        tot = self.stats.totals.tolist()
        n = max(tot[0], 1.0)
        return dict(sample_steps=self.sample_steps, episodes=int(tot[0]), mean_episode_rewards=tot[1] / n,
                    mean_episode_steps=tot[2] / n)
