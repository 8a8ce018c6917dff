"""CPU restatement of the reference IMPALA actor-learner loop (TEST INFRASTRUCTURE / CPU baseline).

Follows examples/IMPALA/train.py:34-252 (Learner: per-actor sampling threads feeding a bounded
sample queue, a learn thread that concatenates samples to train batches, Adam + global-norm clip 40,
stale parameter broadcast every `params_broadcast_interval` pulls), examples/IMPALA/actor.py:27-105
(Actor.sample: 50 steps x 5 envs, env-major merge), examples/IMPALA/atari_agent.py:35-42 (batch-5
CPU inference + np.random.choice per row), parl/env/vector_env.py:41-63 (auto-reset) and
parl/env/atari_wrappers.py (wrapper chain).  Env-steps/s is counted exactly as the reference logs it:
`sample_total_steps += obs.shape[0]` when the learner side consumes a sample (train.py:93), divided by
elapsed wall time (train.py:227,243).

Two env flavours (SURVEY.md Appendix C):
  'lean'      a direct 84x84 uint8 synthetic frame env (parl/tests/gym.py:163-169 distributions, agent-level
              done p = 0.1) behind FrameStack(4,'NCHW') — the most favourable case for the CPU side and the
              distribution the device env reproduces;
  'deepmind'  the mock PongNoFrameskip-v4 of parl/tests/gym.py:138-175 (210x160x3 frames) through the whole
              wrap_deepmind(dim=84,'NCHW') chain of parl/env/atari_wrappers.py:356-385 (Monitor, NoopReset,
              MaxAndSkip(4), EpisodicLife, WarpFrame via cv2, ClipReward, FrameStack) restated in one class.

Actors are OS processes (one per core, single-threaded torch, as the reference's xparl jobs are:
parl/core/torch/agent.py:26, parl/remote/job.py:17) forked ONCE per cluster; they ship their sample dict
back by pickle over a pipe (standing in for cloudpickle + ZeroMQ, parl/remote/communication.py:59-130).
The learner is torch eager float32 on one CUDA device when one is present (BASELINE.md section 3: "learner on
one H100 via torch eager"), else on the CPU threads the actors leave.  paddle is absent, so the network is the
torch twin of the C3 model and V-trace is the reference's Python loop over T (vtrace.py:116-122) in torch.
Used only by bench.py (cpu_baseline / --impl reference) and tests.
"""
import multiprocessing as mp
import os
import queue
import threading
import time

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


class LeanAtariEnv(object):
    """84x84 uint8 frames ~ U{0..254}, reward {0,1}, done p=.1, FrameStack(4, 'NCHW')."""

    def __init__(self, hw=(84, 84), p_done=0.1):
        self.hw, self.p_done = hw, p_done
        self.frames = None

    def _frame(self):
        return np.random.randint(0, 255, self.hw, dtype=np.uint8)

    def reset(self):
        f = self._frame()
        self.frames = [f] * 4
        return np.stack(self.frames)

    def step(self, action):
        f = self._frame()
        reward = float(np.random.choice([0.0, 1.0]))
        done = bool(np.random.choice([True, False], p=[self.p_done, 1 - self.p_done]))
        self.frames = self.frames[1:] + [f]
        return np.stack(self.frames), reward, done, {}


class DeepmindMockPongEnv(object):
    """Mock PongNoFrameskip-v4 (parl/tests/gym.py:138-175) behind wrap_deepmind(dim=84, obs_format='NCHW')
    (parl/env/atari_wrappers.py:356-385), the whole chain restated in one class:
      raw step     : 210x160x3 uint8 ~ randint(0,255), reward choice{0,1}, done p=.1          (gym.py:163-169)
      NoopReset    : on reset, 1..30 raw no-op steps (raw reset again when one of them ends)   (:114-130)
      MaxAndSkip(4): up to 4 raw steps per agent step, reward summed, max over the last two    (:218-243)
      EpisodicLife : done when the (random) lives counter drops; real reset only after a real
                     game over, else one no-op step                                             (:178-215)
      WarpFrame    : cv2 RGB->gray + INTER_AREA resize to 84x84                                 (:246-267)
      ClipReward   : sign                                                                       (:136-151)
      FrameStack(4): last four warped frames, NCHW                                              (:270-307)
    The mock's action meanings are all 'NOOP' so FireResetEnv is not in the chain (:376-377)."""

    def __init__(self, dim=84):
        import cv2
        self.cv2 = cv2
        self.dim = dim
        self.lives = 0
        self.was_real_done = True
        self.obs_buffer = np.zeros((2, 210, 160, 3), dtype=np.uint8)
        self.frames = None

    # raw mock env
    @staticmethod
    def _raw_frame():
        return np.random.randint(0, 255, (210, 160, 3), dtype=np.uint8)

    def _raw_step(self):
        return (self._raw_frame(), np.random.choice([0.0, 1.0]),
                bool(np.random.choice([True, False], p=[0.1, 0.9])))

    @staticmethod
    def _lives():
        return np.random.randint(0, 5)

    def _noop_reset(self):
        self._raw_frame()                                   # env.reset()
        noops = np.random.randint(1, 31)
        obs = None
        for _ in range(noops):
            obs, _, done = self._raw_step()
            if done:
                obs = self._raw_frame()
        return obs

    def _skip_step(self):
        total, done = 0.0, None
        for i in range(4):
            obs, r, done = self._raw_step()
            if i == 2:
                self.obs_buffer[0] = obs
            if i == 3:
                self.obs_buffer[1] = obs
            total += r
            if done:
                break
        return self.obs_buffer.max(axis=0), total, done

    def _warp(self, frame):
        g = self.cv2.cvtColor(frame, self.cv2.COLOR_RGB2GRAY)
        return self.cv2.resize(g, (self.dim, self.dim), interpolation=self.cv2.INTER_AREA)

    def reset(self):
        if self.was_real_done:
            obs = self._noop_reset()
        else:
            obs, _, _ = self._skip_step()
        self.lives = self._lives()
        f = self._warp(obs)
        self.frames = [f] * 4
        return np.array(self.frames)

    def step(self, action):
        obs, r, done = self._skip_step()
        self.was_real_done = done
        lives = self._lives()
        if lives < self.lives and lives > 0:
            done = True
        self.lives = lives
        self.frames = self.frames[1:] + [self._warp(obs)]
        return np.array(self.frames), float(np.sign(r)), done, {}


ENV_FLAVOURS = dict(lean=LeanAtariEnv, deepmind=DeepmindMockPongEnv)


class CpuAtariModel(nn.Module):
    """torch twin of benchmark/torch/a2c/atari_model.py:23-96 (the 84x84 actor-critic)."""

    def __init__(self, act_dim):
        super().__init__()
        self.conv1 = nn.Conv2d(4, 32, 8, 4, 1)
        self.conv2 = nn.Conv2d(32, 64, 4, 2, 2)
        self.conv3 = nn.Conv2d(64, 64, 3, 1, 0)
        self.fc = nn.Linear(64 * 9 * 9, 512)
        self.fc_pi = nn.Linear(512, act_dim)
        self.fc_v = nn.Linear(512, 1)

    def trunk(self, x):
        x = x / 255.0
        x = F.relu(self.conv1(x))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        return F.relu(self.fc(x.flatten(1)))

    def policy(self, x):
        return self.fc_pi(self.trunk(x))

    def value(self, x):
        return self.fc_v(self.trunk(x)).squeeze(1)


def actor_sample(model, envs, obs_batch, T):
    """Actor.sample (examples/IMPALA/actor.py:54-91)."""
    n = len(envs)
    data = [dict(obs=[], actions=[], behaviour_logits=[], rewards=[], dones=[]) for _ in range(n)]
    for _ in range(T):
        with torch.no_grad():
            logits = model.policy(torch.from_numpy(np.stack(obs_batch)).float())
            probs = F.softmax(logits, -1).numpy().astype(np.float64)
        probs /= probs.sum(-1, keepdims=True)
        actions = np.array([np.random.choice(len(p), 1, p=p)[0] for p in probs])     # atari_agent.py:39-40
        nxt = []
        for e in range(n):                                                            # vector_env.py:53-63
            o, r, d, _ = envs[e].step(actions[e])
            if d:
                o = envs[e].reset()
            nxt.append(o)
            data[e]['obs'].append(obs_batch[e])
            data[e]['actions'].append(actions[e])
            data[e]['behaviour_logits'].append(logits[e].numpy())
            data[e]['rewards'].append(r)
            data[e]['dones'].append(d)
        obs_batch = nxt
    out = {k: np.stack([x for e in range(n) for x in data[e][k]]) for k in data[0]}   # env-major merge :79-89
    return out, obs_batch


def _actor_proc(conn, act_dim, env_num, T, seed, flavour):
    torch.set_num_threads(1)
    np.random.seed(seed)
    torch.manual_seed(seed)
    model = CpuAtariModel(act_dim)
    envs = [ENV_FLAVOURS[flavour]() for _ in range(env_num)]
    obs = [e.reset() for e in envs]
    while True:
        msg = conn.recv()
        if msg is None:
            return
        model.load_state_dict({k: torch.from_numpy(v) for k, v in msg.items()})       # set_weights (train.py:171)
        sample, obs = actor_sample(model, envs, obs, T)
        conn.send(sample)                                                             # pickle over a pipe


def vtrace_torch(behaviour_logp, target_logp, discounts, rewards, values, bootstrap, clip_rho=1.0, clip_pg_rho=1.0):
    """from_importance_weights as the reference runs it: a Python loop over T of small tensor ops on the
    learner's device (parl/algorithms/paddle/impala/vtrace.py:99-139)."""
    with torch.no_grad():
        rhos = torch.exp(target_logp - behaviour_logp)
        clipped = torch.clamp(rhos, max=clip_rho)
        cs = torch.clamp(rhos, max=1.0)
        values_t1 = torch.cat([values[1:], bootstrap[None]], 0)
        deltas = clipped * (rewards + discounts * values_t1 - values)
        acc = torch.zeros_like(bootstrap)
        out = []
        for t in range(values.shape[0] - 1, -1, -1):
            acc = deltas[t] + discounts[t] * cs[t] * acc
            out.append(acc)
        vs = torch.stack(out[::-1]) + values
        vs_t1 = torch.cat([vs[1:], bootstrap[None]], 0)
        pg = torch.clamp(rhos, max=clip_pg_rho) * (rewards + discounts * vs_t1 - values)
    return vs, pg


def impala_learn(model, optimizer, batch, T, gamma=0.99, vf_coeff=0.5, ent_coeff=-0.01, lr=1e-3, device='cpu'):
    """IMPALA.learn (parl/algorithms/paddle/impala/impala.py:134-215) in torch float32 on `device`; the float32
    observation batch is what the reference uploads (examples/IMPALA/train.py:106, atari_agent.py:58)."""
    dev = torch.device(device)
    obs = torch.from_numpy(batch['obs'].astype('float32')).to(dev)
    actions = torch.from_numpy(batch['actions'].astype(np.int64)).to(dev)
    bl = torch.from_numpy(batch['behaviour_logits'].astype(np.float32)).to(dev)
    values = model.value(obs)                                                         # two passes, as the reference
    tl = model.policy(obs)
    A = tl.shape[-1]
    t_lsm, b_lsm = F.log_softmax(tl, -1), F.log_softmax(bl, -1)
    onehot = F.one_hot(actions, A).float()
    tlp, blp = (t_lsm * onehot).sum(-1), (b_lsm * onehot).sum(-1)
    p = t_lsm.exp()
    entropy = -(p * t_lsm).sum(-1)
    kl = (p * (t_lsm - b_lsm)).sum(-1).mean()
    B = obs.shape[0] // T

    def tm(x):
        return x.reshape(B, T).transpose(0, 1)
    tlp_, blp_, ent_, v_ = tm(tlp), tm(blp), tm(entropy), tm(values)
    rew = tm(torch.from_numpy(batch['rewards'].astype(np.float32)).to(dev))
    dones = tm(torch.from_numpy(batch['dones'].astype(bool)).to(dev))
    boot = v_[-1]
    disc = (~dones[:-1]).float() * gamma
    vs, pg = vtrace_torch(blp_[:-1].detach(), tlp_[:-1].detach(), disc, rew[:-1], v_[:-1].detach(), boot.detach())
    pi_loss = -(tlp_[:-1] * pg).sum()
    vf_loss = 0.5 * ((v_[:-1] - vs) ** 2).sum()
    total = pi_loss + vf_coeff * vf_loss + ent_coeff * ent_[:-1].sum()
    for g in optimizer.param_groups:
        g['lr'] = lr
    optimizer.zero_grad()
    total.backward()
    gn = torch.sqrt(sum((q.grad ** 2).sum() for q in model.parameters()))
    scale = 40.0 / max(float(gn), 40.0)                                               # ClipGradByGlobalNorm(40)
    for q in model.parameters():
        q.grad.mul_(scale)
    optimizer.step()
    return total.item(), kl.item()


class CpuImpalaCluster(object):
    """One long-lived actor pool + learner (examples/IMPALA/train.py Learner), measured over wall-clock windows.

    Construct it BEFORE the parent touches CUDA (the actors are forked); `window(seconds)` returns
    sample_total_steps / elapsed over that window; `close()` terminates the pool at once."""

    def __init__(self, n_actors=None, env_num=5, T=50, act_dim=18, train_batch_size=1000, seed=0, flavour='lean',
                 learner_device='auto', sample_queue_max_size=8, params_broadcast_interval=5, receiver_threads=8):
        self.cores = os.cpu_count() or 1
        self.n_actors = n_actors if n_actors is not None else max(1, self.cores - 2)
        self.env_num, self.T, self.act_dim, self.train_batch_size = env_num, T, act_dim, train_batch_size
        self.flavour = flavour
        self.params_broadcast_interval = params_broadcast_interval
        ctx = mp.get_context('fork')
        self.conns, self.procs = [], []
        for i in range(self.n_actors):
            a, b = ctx.Pipe()
            p = ctx.Process(target=_actor_proc, args=(b, act_dim, env_num, T, seed + 1 + i, flavour), daemon=True)
            p.start()
            b.close()
            self.conns.append(a)
            self.procs.append(p)
        # ---- learner (after the fork: CUDA is initialised only now)
        if learner_device == 'auto':
            learner_device = 'cuda' if torch.cuda.is_available() else 'cpu'
        self.learner_device = learner_device
        if learner_device == 'cpu':
            self.learner_threads = max(1, self.cores - self.n_actors)
            torch.set_num_threads(self.learner_threads)
        else:
            self.learner_threads = 1
        torch.manual_seed(seed)
        self.model = CpuAtariModel(act_dim).to(learner_device)
        self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3)
        self.sample_q = queue.Queue(maxsize=sample_queue_max_size)
        self.lock = threading.Lock()
        self.cache_params = self._weights()
        self.params_updated = False
        self.cache_params_sent_cnt = 0
        self.sample_total_steps = 0
        self.learn_steps, self.learn_time = 0, 0.0
        self.stop = False
        self.threads = [threading.Thread(target=self._learn_loop, daemon=True)]
        nrecv = max(1, min(receiver_threads, self.n_actors))
        for r in range(nrecv):
            self.threads.append(threading.Thread(target=self._remote_loop, args=(self.conns[r::nrecv], ), daemon=True))
        for th in self.threads:
            th.start()

    def _weights(self):
        return {k: v.detach().cpu().numpy() for k, v in self.model.state_dict().items()}

    def _learn_loop(self):                            # Learner._reader + run_learn (train.py:90-145)
        pending = []
        while not self.stop:
            try:
                s = self.sample_q.get(timeout=0.05)
            except queue.Empty:
                continue
            self.sample_total_steps += s['obs'].shape[0]                               # train.py:93
            pending.append(s)
            if sum(x['obs'].shape[0] for x in pending) >= self.train_batch_size:
                batch = {k: np.concatenate([x[k] for x in pending]) for k in pending[0]}
                pending = []
                t1 = time.time()
                impala_learn(self.model, self.opt, batch, self.T, device=self.learner_device)
                self.learn_time += time.time() - t1
                self.learn_steps += 1
                self.params_updated = True

    def _remote_loop(self, conns):                    # run_remote_sample (train.py:165-194), several actors per thread
        import multiprocessing.connection as mpc
        for c in conns:
            c.send(self.cache_params)
        while not self.stop:
            ready = mpc.wait(conns, timeout=0.05)
            for c in ready:
                try:
                    sample = c.recv()
                except (EOFError, OSError):
                    return
                while not self.stop:
                    try:
                        self.sample_q.put(sample, timeout=0.05)
                        break
                    except queue.Full:
                        continue
                with self.lock:
                    if self.params_updated and self.cache_params_sent_cnt >= self.params_broadcast_interval:
                        self.params_updated = False
                        self.cache_params = self._weights()
                        self.cache_params_sent_cnt = 0
                    self.cache_params_sent_cnt += 1
                    w = self.cache_params
                if self.stop:
                    return
                try:
                    c.send(w)
                except (BrokenPipeError, OSError):
                    return

    def window(self, seconds):
        """Env-steps/s over the next `seconds` of wall clock (sample_total_steps / elapsed, train.py:227,243)."""
        s0, l0, lt0, t0 = self.sample_total_steps, self.learn_steps, self.learn_time, time.time()
        time.sleep(seconds)
        el = time.time() - t0
        ls = self.learn_steps - l0
        return dict(env_steps_per_s=(self.sample_total_steps - s0) / el, elapsed_s=el,
                    sample_steps=self.sample_total_steps - s0, learn_steps=ls,
                    learn_ms_per_batch=(1e3 * (self.learn_time - lt0) / ls) if ls else None)

    def info(self):
        return dict(actors=self.n_actors, env_num=self.env_num, cores=self.cores, flavour=self.flavour,
                    learner_device=self.learner_device, learner_threads=self.learner_threads,
                    train_batch_size=self.train_batch_size, T=self.T)

    def close(self):
        self.stop = True
        for p in self.procs:                          # actors are mid-rollout: do not wait for them
            try:
                p.terminate()
            except Exception:
                pass
        for p in self.procs:
            p.join(timeout=5)
            if p.is_alive():
                p.kill()
        for c in self.conns:
            try:
                c.close()
            except Exception:
                pass
        for th in self.threads:
            th.join(timeout=5)


def run_cpu_impala(seconds=15.0, warmup_seconds=3.0, **kw):
    """One-shot helper: build a cluster, warm up, measure one window, tear down."""
    cl = CpuImpalaCluster(**kw)
    try:
        cl.window(warmup_seconds)
        res = cl.window(seconds)
        res.update(cl.info())
        return res
    finally:
        cl.close()
