"""DQN / DDQN with an HBM-resident (prioritised) Atari frame replay on one H100 — the on-device replacement of
benchmark/torch/dqn/{train.py:50-174, replay_memory.py:22-113, agent.py:57-104} with the proportional PER of
benchmark/fluid/Prioritized_DQN/{proportional_per.py:18-157, per_alg.py:48-69} (BASELINE configs[4]: 1 M-transition
HBM replay, priority sample + TD loss, sharded over the GPUs).

Replay layout (``DeviceAtariReplay``): single uint8 frames [cap_q, lanes, H*W] — ``lanes`` interleaved transition
streams, one per lock-stepped env, so the plane of stream position q is a dense [lanes, H*W] block that the env
kernel writes IN PLACE (appending costs no copy); action / reward / is_over [cap_q, lanes].  The 4-frame context and
the next frame are gathered at sample time (rl_replay_gather_frames, episode-boundary zeroing as
replay_memory.py:59-85), 5 x 7 056 B per sample.  The sum-tree (fp64, reference heap indexing) has one leaf per row.

One engine step = ``update_freq`` lock-step env steps of all lanes (epsilon-greedy on Q of the stacked observation)
followed by one learner update: rl_per_sample (stratified) -> frame gather -> Q / target-Q forward ->
rl_td_loss_fwd_bwd with importance weights -> backward -> Adam -> rl_per_update with |td|.
Multi-GPU (SURVEY.md 8e): every rank owns memory_size/world transitions and its own tree, samples batch/world rows,
all-reduces the flat gradient; the importance weights need the GLOBAL minimum priority: one 1-double all-reduce(MIN).
"""
import torch

from .. import kernels
from ..algorithms import DQN, DDQN
from .nets import AtariQModel


class DeviceAtariReplay(object):
    """benchmark/torch/dqn/replay_memory.py:22-113 in HBM for ``lanes`` lock-stepped env streams."""

    def __init__(self, max_size, frame_hw=(84, 84), context_len=4, lanes=1, device=None):
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError('DeviceAtariReplay lives in HBM: no CUDA device visible (no CPU fallback)')
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = dev = torch.device(device)
        self.lanes, self.context_len = int(lanes), int(context_len)
        self.cap_q = int(max_size) // self.lanes               # stream positions per lane
        assert self.cap_q > 2 * (self.context_len + 2), 'replay too small for its context length'
        self.max_size = self.cap_q * self.lanes
        self.hw = int(frame_hw[0]) * int(frame_hw[1])
        self.frame_hw = tuple(frame_hw)
        self.frames = torch.zeros((self.cap_q, self.lanes, self.hw), dtype=torch.uint8, device=dev)
        self.action = torch.zeros((self.cap_q, self.lanes), dtype=torch.int32, device=dev)
        self.reward = torch.zeros((self.cap_q, self.lanes), dtype=torch.float32, device=dev)
        # "over" everywhere before the first write: the context of the first frames of a lane is zero-filled
        self.is_over = torch.ones((self.cap_q, self.lanes), dtype=torch.uint8, device=dev)
        self.pos = 0                   # stream position holding the CURRENT observation of every lane
        self.filled = 0                # completed positions (transitions with action / reward / next frame)
        self._lane_ids = torch.arange(self.lanes, dtype=torch.int32, device=dev)

    def size(self):
        return self.filled * self.lanes

    __len__ = size

    # ---- write side ------------------------------------------------------------------------------------
    def current_plane(self):
        """[lanes, H*W] view: the current observation frame of every lane."""
        return self.frames[self.pos]

    def next_plane(self):
        """[lanes, H*W] view the env step writes the next frame into (old data at that position is dropped)."""
        return self.frames[(self.pos + 1) % self.cap_q]

    def commit(self, action):
        """Finish the transition at the current position (reward / is_over were written in place by the env kernel,
        the next frame too) and move on: rpm.append(Experience(obs, action, reward, isOver)), train.py:66."""
        self.action[self.pos].copy_(action)
        self.pos = (self.pos + 1) % self.cap_q
        self.filled = min(self.filled + 1, self.cap_q - 1)

    def recent_obs(self, out=None):
        """Current stacked observation of every lane, [lanes, ctx, H, W] uint8: rpm.recent_obs() + [obs]
        (train.py:58-60) — earlier frames of a previous episode are zero."""
        ctx = self.context_len
        start = ((self.pos - (ctx - 1)) % self.cap_q) * self.lanes + self._lane_ids
        o = kernels.replay_gather_frames(self.frames.view(-1, self.hw), self.is_over.view(-1), start.contiguous(),
                                         self.cap_q, ctx, lanes=self.lanes, n_out=ctx, out=out)
        return o.view(self.lanes, ctx, *self.frame_hw)

    # ---- read side -------------------------------------------------------------------------------------
    def valid_rows(self, rows):
        """Rows (= q*lanes + lane) whose 5-frame window is intact: not yet overwritten / not straddling the write
        head (the reference's index offset ``curr_pos + randint(size - ctx - 1)``, replay_memory.py:99-101)."""
        q = rows // self.lanes
        age = (self.pos - 1 - q) % self.cap_q                  # 0 = most recently completed position
        return age < (self.filled - self.context_len)

    def sample_uniform_rows(self, n, generator=None):
        """replay_memory.py:97-103 per lane: uniformly random valid rows."""
        age = torch.randint(0, max(self.filled - self.context_len, 1), (n, ), device=self.device, generator=generator)
        lane = torch.randint(0, self.lanes, (n, ), device=self.device, generator=generator)
        q = (self.pos - 1 - age) % self.cap_q
        return (q * self.lanes + lane).to(torch.int32)

    def gather(self, rows):
        """rows -> (obs [n,ctx,H,W] u8, action [n] i32, reward [n] f32, next_obs [n,ctx,H,W] u8, terminal [n] f32)."""
        ctx, L = self.context_len, self.lanes
        rows = rows.to(torch.int32)
        q, lane = rows // L, rows % L
        start = (((q - (ctx - 1)) % self.cap_q) * L + lane).to(torch.int32).contiguous()
        f = kernels.replay_gather_frames(self.frames.view(-1, self.hw), self.is_over.view(-1), start, self.cap_q, ctx,
                                         lanes=L)
        f = f.view(rows.numel(), ctx + 1, *self.frame_hw)
        ri = rows.contiguous()
        act = kernels.gather_rows(self.action.view(-1, 1), ri).view(-1)
        rew = kernels.gather_rows(self.reward.view(-1, 1), ri).view(-1)
        term = self.is_over.view(-1)[rows.long()].float()
        return f[:, :ctx], act, rew, f[:, 1:], term


class DQNEngine(object):
    def __init__(self, memory_size=1000000, num_envs=256, batch_size=32, act_dim=18, context_len=4, gamma=0.99,
                 lr=3e-4, update_freq=4, prioritized=True, alpha=0.6, beta=0.5, beta_step=1e-4, per_eps=0.01,
                 double_q=False, dueling=False, e_greed=0.1, seed=0, device=None, env_offset=0, p_done=0.1,
                 frame_hw=(84, 84), model=None, compute_dtype=torch.bfloat16):
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = dev = torch.device(device)
        self.B, self.batch_size, self.A = int(num_envs), int(batch_size), int(act_dim)
        self.update_freq, self.e_greed = int(update_freq), float(e_greed)
        self.prioritized, self.alpha, self.beta, self.beta_step, self.per_eps = (bool(prioritized), float(alpha),
                                                                                 float(beta), float(beta_step),
                                                                                 float(per_eps))
        self.seed, self.env_offset, self.p_done = int(seed), int(env_offset), float(p_done)
        self.rpm = DeviceAtariReplay(memory_size, frame_hw, context_len, lanes=self.B, device=dev)
        self.model = (model if model is not None else AtariQModel(act_dim, dueling=dueling)).to(dev)
        self.model = self.model.to(memory_format=torch.channels_last)
        self.alg = (DDQN if double_q else DQN)(self.model, gamma=float(gamma), lr=float(lr))
        self.compute_dtype = compute_dtype
        self.tree = kernels.DeviceSumTree(self.rpm.max_size, dev) if self.prioritized else None
        self.stats = kernels.EpisodeStats(self.B, dev)
        self.ages = torch.zeros((2, self.B), dtype=torch.uint8, device=dev)      # the env kernel's frame-age rows
        self.env_steps = 0
        self.learn_steps = 0
        self.sample_steps = 0
        self.min_sync = None           # multi-GPU: callable(state double[2]) doing all_reduce(MIN) on state[0:1]
        self._gen = torch.Generator(device=dev)
        self._gen.manual_seed(self.seed + 12345 + self.env_offset)
        self.reset()

    def reset(self):
        kernels.env_atari_synth_step(self.rpm.current_plane(), None, None, None, self.ages[0], self.stats, self.seed, 0,
                                     env_offset=self.env_offset, reset=True)
        self.env_steps = 0

    # ------------------------------------------------------------------ actor side
    def _q(self, obs_u8):
        with torch.no_grad(), torch.autocast('cuda', dtype=self.compute_dtype,
                                             enabled=self.compute_dtype != torch.float32):
            return self.model(obs_u8).float()

    def env_step(self):
        """One lock-step step of all lanes: epsilon-greedy action (benchmark/torch/dqn/agent.py:57-65) on the stacked
        observation, env step writing reward / is_over / next frame straight into the replay ring."""
        rpm = self.rpm
        q = self._q(rpm.recent_obs())
        greedy = q.argmax(1).to(torch.int32)
        rnd = torch.randint(0, self.A, (self.B, ), device=self.device, generator=self._gen, dtype=torch.int32)
        explore = torch.rand(self.B, device=self.device, generator=self._gen) < self.e_greed
        action = torch.where(explore, rnd, greedy)
        pos = rpm.pos
        kernels.env_atari_synth_step(rpm.next_plane(), rpm.reward[pos], rpm.is_over[pos], self.ages[0], self.ages[1],
                                     self.stats, self.seed, self.env_steps, p_done=self.p_done,
                                     env_offset=self.env_offset)
        self.ages[0].copy_(self.ages[1])
        rpm.reward[pos].clamp_(-1.0, 1.0)                                   # agent.py:104 reward clipping
        rpm.commit(action)
        if self.tree is not None:
            # the transition just completed enters with the running max priority (proportional_per.py:104-110);
            # the rows whose window the write head now cuts (ctx positions ahead) can no longer be sampled
            self.tree.store(pos * self.B, self.B, self.alpha, self.per_eps)
        self.env_steps += 1
        self.sample_steps += self.B

    # ------------------------------------------------------------------ learner side
    def learn(self):
        rpm, n = self.rpm, self.batch_size
        if self.tree is not None:
            if self.min_sync is not None:
                self.min_sync(self.tree.state)
            tidx, rows, w = self.tree.sample(n, self.beta, float(max(rpm.size(), 1)), seed=self.seed + self.env_offset,
                                             draw=self.learn_steps)
            ok = rpm.valid_rows(rows)
            w = w * ok.float()                       # a window cut by the write head contributes nothing
            rows = torch.where(ok, rows, rows[ok.float().argmax()].expand_as(rows))
            self.beta = min(1.0, self.beta + self.beta_step)
        else:
            rows, w, tidx = rpm.sample_uniform_rows(n, self._gen), None, None
        obs, act, rew, nobs, term = rpm.gather(rows)
        with torch.autocast('cuda', dtype=self.compute_dtype, enabled=self.compute_dtype != torch.float32):
            out = self.alg.learn(obs, act, rew, nobs, term, sample_weight=w)
        self.learn_steps += 1
        if w is not None:
            loss, td_abs = out
            self.tree.update(tidx, td_abs, self.alpha, self.per_eps)        # proportional_per.py:112-118
            return loss
        return out

    def step(self):
        for _ in range(self.update_freq):
            self.env_step()
        return self.learn()

    def warmup(self, n_positions):
        """Fill the ring with ``n_positions`` lock-step steps (train.py:131-137 warm-up to MEMORY_WARMUP_SIZE)."""
        for _ in range(int(n_positions)):
            self.env_step()

    def get_metrics(self):
        tot = self.stats.totals.tolist()
        n = max(tot[0], 1.0)
        return dict(sample_steps=self.sample_steps, episodes=int(tot[0]), mean_episode_rewards=tot[1] / n,
                    mean_episode_steps=tot[2] / n, replay_size=self.rpm.size(), learn_steps=self.learn_steps)
