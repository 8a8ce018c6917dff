"""PPO on one H100 — the on-device replacement of benchmark/torch/ppo/{train.py:45-126, agent.py:21-96,
storage.py:18-76, env_utils.py:28-117} (BASELINE configs[3]: MuJoCo-shaped continuous control, obs 17 / act 6,
2048 envs x 2048 steps, 32 minibatches x 10 epochs, clipped-surrogate kernel).

    rollout  ONE launch (rl_rollout_mlp): T lock-step steps — MuJoCo-model forward (shared tanh trunk, mean + value
             heads), diagonal-Gaussian sampling + log-prob, synthetic env step with auto-reset — into the
             RolloutStorage-shaped (T,B) HBM buffers; values[T] = bootstrap value (train.py:104-105)
    returns  rl_gae_scan: RolloutStorage.compute_returns bit for bit (storage.py:45-64); ``dones[t]`` is the done
             flag that PRECEDES observation t, exactly as train.py:97-98 appends it
    update   per epoch a device permutation, per minibatch rl_gather_rows -> rl_mlp_fwd -> rl_adv_stats (+ optional
             (sum, sum^2, n) all-reduce) -> rl_ppo_loss_fwd_bwd (Gaussian) -> rl_mlp_bwd -> clip 0.5 + Adam(eps 1e-5)
Multi-GPU: env columns shard across ranks; ``alg.grad_sync`` all-reduces the flat gradient (then / world, the
losses are means), ``alg.adv_stats_sync`` makes the advantage normalisation global (ppo.py:115-117).
"""
import torch

from .. import kernels
from ..algorithms import PPO
from ..utils.scheduler import LinearDecayScheduler
from .nets import MujocoModel


class PPOEngine(object):
    def __init__(self, num_envs=2048, step_nums=2048, obs_dim=17, act_dim=6, num_minibatches=32, update_epochs=10,
                 gamma=0.99, gae_lambda=0.95, clip_param=0.2, value_loss_coef=0.5, entropy_coef=0.0, initial_lr=3e-4,
                 lr_decay=True, num_updates=1000, seed=0, device=None, env_offset=0, p_done=0.01, max_episode_steps=1000,
                 model=None, vec_normalize=False, use_graph=True):
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = dev = torch.device(device)
        self.B, self.T, self.D, self.AD = int(num_envs), int(step_nums), int(obs_dim), int(act_dim)
        self.num_minibatches, self.update_epochs = int(num_minibatches), int(update_epochs)
        self.gamma, self.gae_lambda = float(gamma), float(gae_lambda)
        self.seed, self.env_offset = int(seed), int(env_offset)
        self.p_done, self.max_episode_steps = float(p_done), int(max_episode_steps)
        self.model = (model if model is not None else MujocoModel(obs_dim, act_dim)).to(dev)
        self.alg = PPO(self.model, clip_param=float(clip_param), value_loss_coef=float(value_loss_coef),
                       entropy_coef=float(entropy_coef), initial_lr=float(initial_lr), continuous_action=True)
        layers, act = self.model.native_layers()
        self.plan = kernels.MlpPlan(layers, act)
        assert self.plan.out_dim == self.AD + 1
        self.lr_scheduler = LinearDecayScheduler(float(initial_lr), int(num_updates)) if lr_decay else None
        B, T, f32 = self.B, self.T, torch.float32
        N = self.N = T * B
        assert N % self.num_minibatches == 0
        self.M = N // self.num_minibatches
        self.stats = kernels.EpisodeStats(B, dev)
        # wrap_rms(env, gamma): a VecNormalizeEnv per env (benchmark/torch/ppo/env_utils.py:121-133), on the device
        self.vn = kernels.VecNormalize(B, self.D, dev, gamma=self.gamma) if vec_normalize else None
        self.obs_cur = torch.zeros((B, self.D), dtype=f32, device=dev)
        self.obs = torch.empty((T, B, self.D), dtype=f32, device=dev)
        self.actions = torch.empty((T, B, self.AD), dtype=f32, device=dev)
        self.logprobs = torch.empty((T, B), dtype=f32, device=dev)
        self.rewards = torch.empty((T, B), dtype=f32, device=dev)
        self.step_dones = torch.empty((T, B), dtype=torch.uint8, device=dev)       # done produced BY step t
        self.dones = torch.zeros((T, B), dtype=f32, device=dev)                    # storage.dones: done BEFORE obs t
        self.last_done = torch.zeros(B, dtype=f32, device=dev)
        self.values = torch.empty((T + 1, B), dtype=f32, device=dev)
        self.mean_mb = torch.empty((self.M, self.AD), dtype=f32, device=dev)
        self.val_mb = torch.empty((self.M, 1), dtype=f32, device=dev)
        self.idx_buf = torch.zeros(self.M, dtype=torch.int32, device=dev)
        self.alg.optimizer.enable_device_state()
        self.use_graph = bool(use_graph)
        self._graph, self._eager_calls, self._mb_losses = None, 0, None
        self.advantages = torch.empty((T, B), dtype=f32, device=dev)
        self.returns = torch.empty((T, B), dtype=f32, device=dev)
        self.env_steps = 0
        self.sample_steps = 0
        self.grad_world = 1            # multi-GPU: divide the all-reduced gradient by the world size (mean losses)
        self.reset()

    def reset(self):
        kernels.env_mujoco_synth_step(self.obs_cur, None, None, self.stats, self.seed, 0, env_offset=self.env_offset,
                                      reset=True)
        if self.vn is not None:
            self.vn.reset(self.obs_cur)
        self.env_steps = 0
        self.last_done.zero_()

    def _logstd(self):
        return self.model.fc_pi_std.detach().reshape(-1)

    def rollout(self):
        T = self.T
        self.plan.rollout(kernels.ENV_MUJOCO_SYNTH, kernels.POLICY_GAUSSIAN, T, self.obs_cur, self.stats, self.seed,
                          self.env_steps, self.obs, self.actions, self.rewards, self.step_dones,
                          logp_out=self.logprobs, val_out=self.values, logstd=self._logstd(), has_value=True,
                          env_offset=self.env_offset, p_done=self.p_done, max_episode_steps=self.max_episode_steps,
                          vecnorm=self.vn)
        # storage.append(obs, action, logprob, reward, done, value) stores the done flag carried INTO step t
        self.dones[0].copy_(self.last_done)
        if T > 1:
            self.dones[1:].copy_(self.step_dones[:T - 1])
        self.last_done.copy_(self.step_dones[T - 1])
        self.env_steps += T
        self.sample_steps += T * self.B

    def compute_returns(self):
        """RolloutStorage.compute_returns(value, done) with value = V(obs after the last step), done = last done."""
        kernels.gae_scan(self.rewards, self.values[:self.T], self.dones, self.values[self.T], self.last_done,
                         self.gamma, self.gae_lambda, out=(self.advantages, self.returns))
        return self.advantages, self.returns

    def _minibatch_body(self):
        """PPO.learn (parl/algorithms/torch/ppo.py:79-149) on the rows ``self.idx_buf`` of the flattened rollout;
        every scalar that changes between calls (learning rate, Adam step count) lives on the device, so the whole
        body — 6 gathers, forward, advantage statistics, loss, backward, clip, Adam — is one CUDA graph."""
        alg, N, idx = self.alg, self.N, self.idx_buf
        obs = kernels.gather_rows(self.obs.view(N, self.D), idx)
        act = kernels.gather_rows(self.actions.view(N, self.AD), idx)
        gv = lambda x: kernels.gather_rows(x.reshape(N, 1), idx).view(-1)
        bv, br, blp, badv = gv(self.values[:self.T]), gv(self.returns), gv(self.logprobs), gv(self.advantages)
        self.plan.forward(obs, out=self.mean_mb, out2=self.val_mb, split=self.AD)
        stats = None
        if alg.norm_adv:
            stats = alg.adv_stats_sync(badv) if alg.adv_stats_sync is not None else kernels.adv_stats(badv)
        res = kernels.ppo_loss_fwd_bwd(self.val_mb.view(-1), act, bv, br, blp, badv, mean=self.mean_mb,
                                       logstd=self._logstd().contiguous(), clip_param=alg.clip_param,
                                       value_loss_coef=alg.value_loss_coef, entropy_coef=alg.entropy_coef,
                                       use_clipped_value_loss=alg.use_clipped_value_loss, norm_adv=alg.norm_adv,
                                       stats=stats)
        self.plan.backward(obs, res['d_mean'], d_out2=res['d_values'].view(-1, 1), split=self.AD)
        self.model.fc_pi_std.grad.copy_(res['d_logstd'].view_as(self.model.fc_pi_std))
        if alg.grad_sync is not None:
            alg.grad_sync(alg.optimizer.grad)
        alg.optimizer.step(grad_div=float(self.grad_world))
        self._mb_losses = res['losses']

    def learn_minibatch(self, idx, lr):
        """One PPO minibatch update on the rows ``idx``; returns the device losses {value, action, entropy, total}.
        The first call runs eagerly, the second captures the CUDA graph, later calls replay it."""
        opt = self.alg.optimizer
        if lr is not None:
            opt.set_lr(lr)
        self.idx_buf.copy_(idx)
        if not self.use_graph or self._eager_calls == 0:
            self._eager_calls += 1
            self._minibatch_body()
            return self._mb_losses
        if self._graph is None:
            count = opt.step_count
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._minibatch_body()
            opt.step_count = count                      # capture is not execution
            self._graph = g
        self._graph.replay()
        opt.step_count += 1
        return self._mb_losses

    def learn(self):
        """PPOAgent.learn (benchmark/torch/ppo/agent.py:54-96): update_epochs shuffles x num_minibatches steps."""
        lr = self.lr_scheduler.step(step_num=1) if self.lr_scheduler is not None else None
        acc = torch.zeros(4, dtype=torch.float32, device=self.device)
        for _ in range(self.update_epochs):
            perm = torch.randperm(self.N, device=self.device, dtype=torch.int32)
            for mb in range(self.num_minibatches):
                acc += self.learn_minibatch(perm[mb * self.M:(mb + 1) * self.M], lr)
        return acc / float(self.update_epochs * self.num_minibatches), lr

    def step(self):
        self.rollout()
        self.compute_returns()
        return self.learn()

    def get_ob_rms(self, env_index=0):
        """(mean, var, count) of one env's observation statistics — what ParallelEnv.eval_ob_rms hands to the
        evaluation env (benchmark/torch/ppo/env_utils.py:100-103, train.py:117-120)."""
        if self.vn is None:
            return None
        return (self.vn.ob_mean[env_index].cpu().numpy(), self.vn.ob_var[env_index].cpu().numpy(),
                float(self.vn.ob_count[env_index].item()))

    def get_metrics(self):
        tot = self.stats.totals.tolist()
        n = max(tot[0], 1.0)
        return dict(sample_steps=self.sample_steps, episodes=int(tot[0]), mean_episode_rewards=tot[1] / n,
                    mean_episode_steps=tot[2] / n)
