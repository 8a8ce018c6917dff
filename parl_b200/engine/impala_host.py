"""The IMPALA example's Actor and Agent on the H100, behind the reference's host contract — drop-in replacements
of examples/IMPALA/actor.py:27-105 and examples/IMPALA/atari_agent.py:21-74 for the Learner loop of
examples/IMPALA/train.py:34-252:

    Actor = parl.remote_class(wait=False)(DeviceImpalaActor)      # train.py:30, actor.py:26
    actor = Actor(config)
    actor.set_weights(agent.get_weights())                        # train.py:171  numpy weight dict
    batch = actor.sample().get()                                  # train.py:173  dict of numpy arrays, env-major
    agent.learn(batch['obs'], batch['actions'], batch['behaviour_logits'], batch['rewards'], batch['dones'],
                lr, entropy_coeff)                                # train.py:134-137

``DeviceImpalaActor`` hosts ``config['env_num']`` lock-stepped synthetic Atari envs and the policy network on the GPU
(one remote actor = one device actor pool instead of one CPU job with 5 envs); ``sample()`` runs the T-step rollout
on the actor's own CUDA stream and copies the sample dict — keys / dtypes / env-major order of actor.py:79-91 — into
pinned host memory (two alternating buffer sets: the dict handed out stays valid until the sample after next).
``AtariAgent.learn`` uploads the numpy arrays and runs IMPALA.learn with the network on the wgmma kernels.
"""
import os
import time

import numpy as np
import torch

from ..core import Agent
from .impala import ImpalaEngine

__all__ = ['DeviceImpalaActor', 'AtariAgent', 'default_config']

default_config = dict(env_num=4096, sample_batch_steps=50, act_dim=18, env_dim=84, gamma=0.99, vf_loss_coeff=0.5,
                      clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0, seed=0, env_offset=0, p_done=0.1)


def _engine(config, role, device):
    c = dict(default_config)
    c.update(config or {})
    return ImpalaEngine(num_envs=c['env_num'], sample_batch_steps=c['sample_batch_steps'], act_dim=c['act_dim'],
                        frame_hw=(c['env_dim'], c['env_dim']), seed=c['seed'], device=device,
                        env_offset=c['env_offset'], gamma=c['gamma'], vf_loss_coeff=c['vf_loss_coeff'],
                        clip_rho_threshold=c['clip_rho_threshold'], clip_pg_rho_threshold=c['clip_pg_rho_threshold'],
                        p_done=c['p_done'], role=role)


def _actor_groups(config):
    """Number of env-column groups the actor pool is split into (see DeviceImpalaActor): config['actor_groups'] or
    $PARL_B200_ACTOR_GROUPS, else the largest of 4 / 2 / 1 that divides env_num and leaves >= 512 envs per group."""
    B = int(config['env_num'])
    g = config.get('actor_groups') or os.environ.get('PARL_B200_ACTOR_GROUPS')
    if g:
        g = int(g)
        assert g >= 1 and B % g == 0, 'actor_groups must divide env_num'
        return g
    for g in (4, 2):
        if B % g == 0 and B // g >= 512:
            return g
    return 1


class DeviceImpalaActor(object):
    """Actor(config) with sample() / set_weights(weights) / get_metrics() (examples/IMPALA/actor.py:54-105).

    The pool is split into G groups of env columns (G engines with env_offset = first column: the Philox streams are
    keyed by the global env index, so the env side is the same as one pool's).  sample() rolls the groups out one
    after the other on the actor stream while a copy stream gathers and downloads the group before: rows
    [g*B/G*T, (g+1)*B/G*T) of the env-major sample dict are one contiguous block per group.  Only the first group's
    rollout is exposed in front of the PCIe copy (4 ms instead of 12 + 3 ms at 4096 envs)."""

    def __init__(self, config=None, device=None):
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)              # the hosting worker thread launches on this GPU
        self.config = dict(default_config)
        self.config.update(config or {})
        self.stream = torch.cuda.Stream(device=self.device)
        self.copy_stream = torch.cuda.Stream(device=self.device)
        G = self.groups = _actor_groups(self.config)
        B, T = int(self.config['env_num']), int(self.config['sample_batch_steps'])
        Bg = B // G
        with torch.cuda.stream(self.stream):
            self.pools = []
            for g in range(G):
                c = dict(self.config)
                c['env_num'], c['env_offset'] = Bg, int(self.config['env_offset']) + g * Bg
                self.pools.append(_engine(c, 'actor', self.device))
            if G > 1:                                   # one set of weights for all groups until set_weights arrives
                w0 = self.pools[0].get_weights()
                for q in self.pools[1:]:
                    q.set_weights(w0)
            self.hosts = [self._make_host_buffers(B * T) for _ in range(2)]
        self.pool = self.pools[0]
        n = Bg * T
        self._views = [[{k: v[g * n:(g + 1) * n] for k, v in h.items()} for g in range(G)] for h in self.hosts]
        self._ev = [torch.cuda.Event() for _ in range(G)]
        self.stream.synchronize()
        self._n = 0
        self._metrics_read = [0] * G

    def _make_host_buffers(self, N):
        """Pinned host arrays with the keys / dtypes / env-major order of Actor.sample() (actor.py:54-91)."""
        p0 = self.pools[0]
        pin = dict(pin_memory=True)
        return dict(obs=torch.empty((N, 4, p0.h, p0.w), dtype=torch.uint8, **pin),
                    actions=torch.empty(N, dtype=torch.int64, **pin),
                    behaviour_logits=torch.empty((N, p0.A), dtype=torch.float32, **pin),
                    rewards=torch.empty(N, dtype=torch.float32, **pin),
                    dones=torch.empty(N, dtype=torch.bool, **pin))

    def sample(self):
        t_begin = time.time()
        which = self._n % 2
        host = self.hosts[which]
        self._n += 1
        torch.cuda.set_device(self.device)
        with torch.cuda.stream(self.stream):
            for g, pool in enumerate(self.pools):
                pool.rollout()
                self._ev[g].record(self.stream)
                with torch.cuda.stream(self.copy_stream):
                    self.copy_stream.wait_event(self._ev[g])
                    pool._sample_dict_to_host(self._views[which][g])
        self.copy_stream.synchronize()                  # every group is on the host; the pools are free again
        self.last_sample_s = time.time() - t_begin      # host wall clock of this call (rollouts + download)
        return {k: v.numpy() for k, v in host.items()}

    def set_weights(self, weights):
        torch.cuda.set_device(self.device)
        with torch.cuda.stream(self.stream):
            p0 = self.pools[0]
            p0.set_weights(weights)                     # numpy dict -> device (the only host->device copy)
            for q in self.pools[1:]:                    # the other groups take theirs device-to-device
                f0, fq = p0._flat_master(), q._flat_master()
                with torch.no_grad():
                    if f0 is not None and fq is not None and f0.numel() == fq.numel():
                        fq.copy_(f0)
                    else:
                        for a, b in zip(q.model.parameters(), p0.model.parameters()):
                            a.copy_(b)
                    for a, b in zip(q.model.buffers(), p0.model.buffers()):
                        a.copy_(b)
                q.repack()
        self.stream.synchronize()

    def get_metrics(self):
        """{'episode_rewards': [...], 'episode_steps': [...]} of the episodes finished since the last call
        (actor.py:93-102: MonitorEnv.next_episode_results of every env)."""
        rets, lens = [], []
        for g, pool in enumerate(self.pools):
            st = pool.stats
            head = int(st.ring_head.item())
            cap = st.ring_cap
            lo = max(self._metrics_read[g], head - cap)
            idx = [i % cap for i in range(lo, head)]
            self._metrics_read[g] = head
            if idx:
                rets += st.ring_ret.cpu()[idx].tolist()
                lens += st.ring_len.cpu()[idx].tolist()
        return {'episode_rewards': rets, 'episode_steps': lens}


class AtariAgent(Agent):
    """Learner-side agent (examples/IMPALA/atari_agent.py:21-74): ``learn`` takes the numpy batch of the Learner's
    reader thread (train.py:102-121) — obs float32 OR uint8 [B*T,4,H,W] (values 0..255), actions int64,
    behaviour_logits float32, rewards float32, dones bool, env-major — plus lr and entropy_coeff; returns
    (total_loss, pi_loss, vf_loss, entropy, kl) as Python floats like atari_agent.py:66-74."""

    def __init__(self, config=None, device=None):
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        self.engine = _engine(config, 'learner', self.device)
        super(AtariAgent, self).__init__(self.engine.alg)
        self._host = None

    def set_weights(self, params):
        self.engine.set_weights(params)

    def restore(self, save_path, model=None, map_location=None):
        super(AtariAgent, self).restore(save_path, model, map_location)
        self.engine.repack()

    @staticmethod
    def _as_tensor(a, dtype):
        t = torch.from_numpy(np.ascontiguousarray(a)) if isinstance(a, np.ndarray) else a
        return t if t.dtype == dtype else t.to(dtype)

    def learn(self, obs_np, actions_np, behaviour_logits_np, rewards_np, dones_np, lr, entropy_coeff):
        # the reference uploads float32 observations (4x the bytes, atari_agent.py:58); uint8 is accepted as is
        obs = obs_np if not isinstance(obs_np, np.ndarray) or obs_np.dtype == np.uint8 else obs_np.astype(np.uint8)
        host = dict(obs=self._as_tensor(obs, torch.uint8), actions=self._as_tensor(actions_np, torch.int64),
                    behaviour_logits=self._as_tensor(behaviour_logits_np, torch.float32),
                    rewards=self._as_tensor(rewards_np, torch.float32), dones=self._as_tensor(dones_np, torch.bool))
        losses = self.engine.learn_from_host(host, float(lr), float(entropy_coeff))
        total, pi, vf, ent, kl = losses[:5].tolist()
        return total, pi, vf, ent, kl
