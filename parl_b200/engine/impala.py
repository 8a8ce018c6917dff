"""The IMPALA actor-learner loop on one H100 (one process per GPU): the on-device replacement of
examples/IMPALA/{train.py:34-252, actor.py:27-105} + the xparl RPC data path
(parl/remote/remote_wrapper.py:178-227).

Rollout buffers live in HBM, time-major:
    planes  [T+4, B, H*W] uint8   frame ring (obs t = planes t..t+3 via ages[t]); plane t+4 is
                                  written by env step t, planes T..T+3 are carried to 0..3
    ages    [T+1, B]      uint8
    beh_logits [T,B,A] f32, actions [T,B] i32, rewards [T,B] f32, dones [T,B] u8
Per step t: policy forward on obs_t -> logits straight into beh_logits[t] -> ONE kernel samples the
actions and steps all B envs (rl_env_atari_synth_step).  The whole T-step rollout is captured in a
CUDA graph (step counter resident on the device) and replayed.  ``learn`` runs the network over all
T*B observations, the fused V-trace loss kernel, backward, (NCCL all-reduce of the flat gradient),
clip + Adam.
"""
import copy
import os

import torch

from .. import kernels
from ..algorithms import IMPALA
from .nets import AtariActorCritic
from .actor_net import AtariActorNet
from .train_net import AtariTrainNet


def host_slab_plan(B, T, samples=16384):
    """(number of slabs, env columns per slab) for uploading a [B*T] env-major batch slab by slab, or None when the
    batch is too small to be worth it (or samples <= 0: the one-shot path).  A slab is a whole number of env columns
    (V-trace scans a column over all T rows), all slabs are equal, about ``samples`` samples each (16 384 = 327 columns
    at T = 50: ~7 ms of H2D, ~2 ms of compute)."""
    if samples <= 0:
        return None
    target = max(1, samples // T)
    if B < 2 * target:
        return None
    n = -(-B // target)
    while B % n:
        n += 1
    return n, B // n


class ImpalaEngine(object):
    def __init__(self, num_envs=4096, sample_batch_steps=50, act_dim=18, frame_hw=(84, 84), seed=0, device=None,
                 env_offset=0, gamma=0.99, vf_loss_coeff=0.5, clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0,
                 p_done=0.1, model=None, learn_chunk_rows=5, use_graph=True, actor_kernels='auto',
                 learner_kernels='auto', pipeline=False, role='both', actor_sms=None, learner_sms=None,
                 obs_dtype=None):
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        assert role in ('both', 'actor', 'learner')
        # role 'actor': only the actor pool (envs, rollout buffers, packed actor network) — what a remote Actor hosts;
        # role 'learner': only the learner (train network, loss buffers) — what the Learner's Agent hosts.  The two
        # halves then talk through the reference's host contract (numpy sample dicts, numpy weight dicts).
        self.role = role
        # pipelined engines: CTA caps of the persistent network kernels of the two streams (None = one CTA per SM).
        # With both at the SM count the actor's and the learner's whole-GPU grids serialise; capped, they co-reside.
        env_a, env_l = os.environ.get('PARL_B200_ACTOR_SMS'), os.environ.get('PARL_B200_LEARNER_SMS')
        self.actor_sms = int(env_a) if env_a else (actor_sms or 0)
        self.learner_sms = int(env_l) if env_l else (learner_sms or 0)
        if pipeline and actor_sms is None and learner_sms is None and not env_a and not env_l and int(num_envs) <= 768:
            # small per-GPU pools (the 8-GPU share of the 4096-actor workload): both streams' kernels are short and
            # latency-bound, so the 132 SMs of an H100 are split between them and their kernels co-reside instead of
            # serialising whole-GPU grids.  (57, 75) rescales the split measured on a 148-SM GPU to 132 SMs; it has
            # not been measured on H100 (the actor_sms / learner_sms arguments override it)
            self.actor_sms, self.learner_sms = 57, 75
        if role != 'both':
            assert not pipeline, 'actor-only / learner-only engines are driven through the host contract'
        self.B, self.T, self.A = int(num_envs), int(sample_batch_steps), int(act_dim)
        self.h, self.w = frame_hw
        self.hw = self.h * self.w
        self.seed, self.env_offset, self.p_done = int(seed), int(env_offset), p_done
        dev = self.device
        B, T, A = self.B, self.T, self.A
        # rollout buffer sets: one, or two when actor and learner are pipelined (double buffering)
        self.pipeline = bool(pipeline)
        self._sets = []
        for _ in range(0 if role == 'learner' else (2 if self.pipeline else 1)):
            self._sets.append(dict(
                planes=torch.zeros((T + 4, B, self.hw), dtype=torch.uint8, device=dev),
                ages=torch.zeros((T + 1, B), dtype=torch.uint8, device=dev),
                beh_logits=torch.zeros((T, B, A), dtype=torch.float32, device=dev),
                actions=torch.zeros((T, B), dtype=torch.int32, device=dev),
                rewards=torch.zeros((T, B), dtype=torch.float32, device=dev),
                dones=torch.zeros((T, B), dtype=torch.uint8, device=dev)))
        if self._sets:
            self._bind(0)
        self.stats = kernels.EpisodeStats(B, dev)
        self.s2d = (self.h, self.w) == (84, 84)              # conv1 space-to-depth input [N,21,21,64]
        # 'uint8' (default): the observation plane stays uint8 (half the bytes, 5.8 GB less per buffer set) and the
        # conv1 kernels widen it to bf16 in shared memory; 'bf16': the gather pre-scales to bf16.
        if obs_dtype is None:
            obs_dtype = os.environ.get('PARL_B200_OBS_DTYPE', 'uint8')
        obs_shape = (21, 21, 64) if self.s2d else (self.h, self.w, 4)
        # per-step policy input, pre-scaled bf16 (space-to-depth blocks on 84x84 frames, else NHWC) or uint8 blocks
        self.obs_dtype = torch.uint8 if (self.s2d and obs_dtype in ('uint8', 'u8', torch.uint8)) else torch.bfloat16
        self.obs_step = torch.empty((B, ) + obs_shape, dtype=self.obs_dtype, device=dev)
        self.fuse_step_gather = os.environ.get('PARL_B200_FUSE_STEP_GATHER', '1') != '0'

        self.step_dev = torch.zeros(T, dtype=torch.int32, device=dev)      # global env-step index of row t
        self.step_dev.copy_(torch.arange(T, dtype=torch.int32))
        self.model = model if model is not None else AtariActorCritic(A)
        self.model.to(dev)
        self.alg = IMPALA(self.model, sample_batch_steps=T, gamma=gamma, vf_loss_coeff=vf_loss_coeff,
                          clip_rho_threshold=clip_rho_threshold, clip_pg_rho_threshold=clip_pg_rho_threshold)
        self.learn_chunk_rows = int(learn_chunk_rows)
        native_ok = (self.h, self.w) == (84, 84) and isinstance(self.model, AtariActorCritic)
        use_native_learner = role != 'actor' and (learner_kernels is True or (learner_kernels == 'auto' and native_ok))
        # learner forward+backward on hand-written wgmma kernels (no autograd) when the model is the Atari net
        self.train_net = AtariTrainNet(self.model, T * B, dev, obs_dtype=self.obs_dtype if self.s2d else torch.bfloat16,
                                       flat=self._flat_master()) \
            if use_native_learner else None
        # learner inputs: one pre-scaled bf16 NHWC buffer per chunk (each is saved by autograd for conv1's
        # weight gradient, so chunks must not share storage): T*B*56 KB in total
        self.obs_chunks = [] if (self.train_net is not None or role == 'actor') else [
            torch.empty((min(self.learn_chunk_rows, T - t0) * B, ) + obs_shape, dtype=torch.bfloat16, device=dev)
            for t0 in range(0, T, self.learn_chunk_rows)]
        if role != 'actor':
            self.tgt_logits = torch.empty((T, B, A), dtype=torch.float32, device=dev)
            self.values = torch.empty((T, B), dtype=torch.float32, device=dev)
            self.loss_out = dict(losses=torch.zeros(8, device=dev), d_logits=torch.empty((T * B, A), device=dev),
                                 d_values=torch.empty(T * B, device=dev))
        # actor-side policy forward: hand-written wgmma conv/GEMM kernels when the model is the Atari
        # actor-critic on 84x84 frames ('auto'), else the user's torch Model
        use_native = role != 'learner' and (actor_kernels is True or (actor_kernels == 'auto' and self.s2d and
                                                                     isinstance(self.model, AtariActorCritic)))
        self.actor_net = AtariActorNet(self.model, B, dev, flat=self._flat_master()) if use_native else None
        # Shared observation plane: the actor's per-step conv1 input (space-to-depth uint8, 28 KB per env step) is
        # written straight into row t of a (T,B) plane of the rollout buffer set and the learner's conv1 forward /
        # weight gradient read it from there — the learner never re-gathers the frame ring.  5.8 GB per set at
        # T*B = 204 800: HBM is spent (180 GB) to save one full pass over the observations per update.
        # Pipelined engines whose actor runs the user's torch Model (no native actor net): the actor stream must not
        # read the fp32 master weights while the learner stream's Adam step overwrites them (ADVICE r1), so the
        # rollout runs on a SNAPSHOT copy of the model that is refreshed on the actor stream before each rollout.
        self._actor_model = copy.deepcopy(self.model) if (self.pipeline and self.actor_net is None) else None
        if self._actor_model is not None:
            for q in self._actor_model.parameters():
                q.requires_grad_(False)
        self.share_obs = self.actor_net is not None and self.train_net is not None
        if self.share_obs:
            for st in self._sets:
                st['x0'] = torch.empty((T, B) + obs_shape, dtype=self.obs_dtype, device=dev)
            self._bind(self._cur_set)
        self.sample_steps = 0
        self.use_graph = use_graph
        self._graphs = [None] * len(self._sets)
        self._graph_launches = 0
        self._k = 0
        if self.pipeline:
            self.actor_stream = torch.cuda.Stream(device=dev)
            self._roll_done = [torch.cuda.Event() for _ in range(2)]
            self._learn_done = [None, None]
            self._ev_pack = torch.cuda.Event()
        if role != 'learner':
            self.reset()

    def _flat_master(self):
        """The optimizer's flat fp32 parameter buffer (operand copies are refreshed from it in one launch)."""
        opt = getattr(self.alg, 'optimizer', None)
        return getattr(opt, 'flat', None)

    def _bind(self, i):
        """Make buffer set i the one the attribute names (planes, ages, beh_logits, ...) refer to."""
        self._cur_set = i
        for k, v in self._sets[i].items():
            setattr(self, k, v)

    # ------------------------------------------------------------------ env side
    def reset(self):
        # the reset frame goes where the carry at the start of the next rollout picks it up
        T = self.T
        last = self._sets[-1]               # rollout 0 goes into set 0 and carries from the last set's tail
        kernels.env_atari_synth_step(last['planes'][T + 3], None, None, None, last['ages'][T], self.stats, self.seed, 0,
                                     env_offset=self.env_offset, reset=True)
        self.step_dev.copy_(torch.arange(T, dtype=torch.int32) - T)

    def _rollout_body(self):
        T = self.T
        prev = self._sets[(self._cur_set - 1) % len(self._sets)]      # the set the previous rollout filled
        with torch.no_grad():
            # carry the previous rollout's last observation (4 planes + age row) to the front; done HERE and
            # not at the end of the previous rollout so that learn() still sees rows 0..3 intact
            self.planes[0:4].copy_(prev['planes'][T:T + 4])
            self.ages[0].copy_(prev['ages'][T])
            self.step_dev.add_(T)
            # per env step: [obs gather ->] policy forward -> env step.  On 84x84 uint8 observations the env step of
            # row t also produces obs(t+1) (rl_env_atari_synth_step_gather): one launch less per step
            fuse = self.s2d and self.obs_dtype == torch.uint8 and self.fuse_step_gather
            for t in range(T):
                obs_t = self.x0[t] if self.share_obs else self.obs_step
                if t == 0 or not fuse:
                    kernels.obs_stack_gather(self.planes, self.ages, t, 1, obs_t, scale=1.0 / 255.0, s2d=self.s2d)
                if self.actor_net is not None:
                    self.actor_net.policy(obs_t, self.beh_logits[t])
                else:
                    pol = self._actor_model if self._actor_model is not None else self.model
                    self.beh_logits[t].copy_(pol.policy(obs_t))
                if fuse and t + 1 < T:
                    obs_n = self.x0[t + 1] if self.share_obs else self.obs_step
                    kernels.env_atari_synth_step_gather(self.planes, t, self.rewards[t], self.dones[t], self.ages[t],
                                                        self.ages[t + 1], self.stats, self.seed, obs_n, p_done=self.p_done,
                                                        env_offset=self.env_offset, logits=self.beh_logits[t],
                                                        actions_out=self.actions[t], step_dev=self.step_dev[t:])
                else:
                    kernels.env_atari_synth_step(self.planes[t + 4], self.rewards[t], self.dones[t], self.ages[t],
                                                 self.ages[t + 1], self.stats, self.seed, 0, p_done=self.p_done,
                                                 env_offset=self.env_offset, logits=self.beh_logits[t],
                                                 actions_out=self.actions[t], step_dev=self.step_dev[t:])

    def _run_rollout(self, i):
        """Rollout into buffer set i on the current stream (graph replay after the first, eager, run)."""
        self._bind(i)
        if self.actor_sms or self.learner_sms:
            kernels.set_sm_limit(self.actor_sms)          # read at launch: baked into the rollout graph at capture
            try:
                self._run_rollout_inner(i)
            finally:
                kernels.set_sm_limit(self.learner_sms)    # the learner's eager launches that follow
            return
        self._run_rollout_inner(i)

    def _run_rollout_inner(self, i):
        if self.use_graph:
            if self._graphs[i] is None:
                self._rollout_body()                      # eager once (allocator / autotune warm-up), then capture
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                before = kernels.launch_count()
                with torch.cuda.graph(g):
                    self._rollout_body()
                self._graph_launches = kernels.launch_count() - before
                kernels.add_graph_launches(-self._graph_launches)      # capture is not execution
                self._graphs[i] = g
            else:
                self._graphs[i].replay()
                kernels.add_graph_launches(self._graph_launches)
        else:
            self._rollout_body()
        self.sample_steps += self.T * self.B

    def rollout(self):
        """T lock-step env steps for all B envs (the device analogue of Actor.sample())."""
        assert not self.pipeline, 'pipelined engines are driven by step()'
        self._run_rollout(0)

    def step(self, learning_rate=0.001, entropy_coeff=-0.01):
        """One actor-learner iteration.  Sequential engines: rollout then learn.  Pipelined engines (SURVEY.md
        8f-1, the device analogue of the reference's sample queue + stale parameter broadcast,
        examples/IMPALA/train.py:37-38,182-194): rollout k+1 runs on the actor stream into the other buffer
        set, with the weights of update k-1, WHILE the learner stream trains on rollout k."""
        if not self.pipeline:
            self.rollout()
            return self.learn(learning_rate, entropy_coeff)
        cur_stream = torch.cuda.current_stream()
        k = self._k
        if k == 0:                                        # prologue: rollout 0
            self.actor_stream.wait_stream(cur_stream)
            with torch.cuda.stream(self.actor_stream):
                self._run_rollout(0)
                self._roll_done[0].record(self.actor_stream)
        cur, nxt = k % 2, (k + 1) % 2
        with torch.cuda.stream(self.actor_stream):
            if self._learn_done[nxt] is not None:          # update k-1 finished: its weights are final, set nxt is free
                self.actor_stream.wait_event(self._learn_done[nxt])
            self._snapshot_actor_weights()
            self._ev_pack.record(self.actor_stream)
            self._run_rollout(nxt)
            self._roll_done[nxt].record(self.actor_stream)
        cur_stream.wait_event(self._ev_pack)              # the actor has taken its copy of the weights
        cur_stream.wait_event(self._roll_done[cur])
        self._bind(cur)
        losses = self.learn(learning_rate, entropy_coeff)
        ev = torch.cuda.Event()
        ev.record(cur_stream)
        self._learn_done[cur] = ev
        self._k += 1
        return losses

    def _snapshot_actor_weights(self):
        """Actor-side copy of the current weights, taken on the actor stream (bf16 operand copies of the native
        actor net, or the snapshot model of a torch actor)."""
        if self.actor_net is not None:
            self.actor_net.pack()
        elif self._actor_model is not None:
            with torch.no_grad():
                for q, p in zip(self._actor_model.parameters(), self.model.parameters()):
                    q.copy_(p)
                for q, p in zip(self._actor_model.buffers(), self.model.buffers()):
                    q.copy_(p)

    # ------------------------------------------------------------------ weights / checkpoints
    def repack(self):
        """Refresh every packed operand copy from the fp32 master weights.  Call after ANY external change of the
        model's parameters (set_weights, load_state_dict, Agent.restore, sync_weights_to into this model)."""
        if self.train_net is not None:
            self.train_net.pack()
        st = getattr(self, '_host_slab_state', None)
        if st is not None:
            st['net'].pack()
        self._snapshot_actor_weights()

    def get_weights(self):
        return self.alg.get_weights()

    def set_weights(self, weights):
        self.alg.set_weights(weights)
        self.repack()

    def save(self, path):
        """Model weights + optimiser moments + step counters (torch.save)."""
        d = os.path.dirname(path)
        if d and not os.path.exists(d):
            os.makedirs(d)
        torch.save(dict(model=self.model.state_dict(), optimizer=self.alg.optimizer.state_dict(),
                        sample_steps=self.sample_steps), path)

    def restore(self, path, map_location=None):
        ck = torch.load(path, map_location=map_location)
        self.model.load_state_dict(ck['model'])
        self.alg.optimizer.load_state_dict(ck['optimizer'])
        self.sample_steps = int(ck.get('sample_steps', 0))
        self.repack()

    # ------------------------------------------------------------------ learner side
    def learn(self, learning_rate=0.001, entropy_coeff=-0.01):
        """One IMPALA update on the (T,B) rollout in HBM (impala.py:134-215 semantics)."""
        T, B, A = self.T, self.B, self.A
        if self.train_net is not None:
            return self._learn_native(learning_rate, entropy_coeff)
        rows = self.learn_chunk_rows
        outs = []
        for ci, t0 in enumerate(range(0, T, rows)):
            n = min(rows, T - t0)
            obs = self.obs_chunks[ci]
            kernels.obs_stack_gather(self.planes, self.ages, t0, n, obs, scale=1.0 / 255.0, s2d=self.s2d)
            logits, values = self.model.policy_and_value(obs)
            self.tgt_logits[t0:t0 + n].copy_(logits.detach().view(n, B, A))
            self.values[t0:t0 + n].copy_(values.detach().view(n, B))
            outs.append((logits, values, t0, n))
        ev = getattr(self, 'k1_events', None)
        if ev is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        res = kernels.vtrace_loss_fwd_bwd(self.tgt_logits.view(T * B, A), self.beh_logits.view(T * B, A),
                                          self.actions.view(-1), self.rewards.view(-1), self.dones.view(-1),
                                          self.values.view(-1), T, B, self.alg.gamma, self.alg.vf_loss_coeff,
                                          entropy_coeff, self.alg.clip_rho_threshold, self.alg.clip_pg_rho_threshold,
                                          layout=kernels.TIME_MAJOR, out=self.loss_out)
        if ev is not None:
            e1.record()
            ev.append((e0, e1))
        dl = res['d_logits'].view(T, B, A)
        dv = res['d_values'].view(T, B)
        tensors, grads = [], []
        for logits, values, t0, n in outs:
            tensors += [logits, values]
            grads += [dl[t0:t0 + n].reshape(n * B, A), dv[t0:t0 + n].reshape(n * B)]
        torch.autograd.backward(tensors, grads)
        if self.alg.grad_sync is not None:
            self.alg.grad_sync(self.alg.optimizer.grad)
        self.alg.optimizer.step(lr=learning_rate)
        if self.actor_net is not None and not self.pipeline:
            self.actor_net.pack()              # refresh the actor's bf16 operand copies (weights never leave HBM)
        return res['losses'].clone()

    def _learn_native(self, learning_rate, entropy_coeff):
        """learn() with the network forward/backward on the hand-written kernels (AtariTrainNet), launched eagerly."""
        res = self._learn_fwd_bwd(entropy_coeff)
        if self.alg.grad_sync is not None:
            self.alg.grad_sync(self.alg.optimizer.grad)
        self._learn_apply(learning_rate)
        return res['losses'].clone()

    def _learn_fwd_bwd(self, entropy_coeff):
        """Forward, fused V-trace loss, backward: fills the flat gradient buffer."""
        T, B, A = self.T, self.B, self.A
        net = self.train_net
        if self.share_obs:
            logits, values = net.forward_from_x0(self.x0.view(T * B, 21, 21, 64))
        else:
            logits, values = net.forward(self.planes, self.ages, T)
        ev = getattr(self, 'k1_events', None)
        if ev is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        res = kernels.vtrace_loss_fwd_bwd(logits, self.beh_logits.view(T * B, A), self.actions.view(-1),
                                          self.rewards.view(-1), self.dones.view(-1), values.view(-1), T, B,
                                          self.alg.gamma, self.alg.vf_loss_coeff, entropy_coeff,
                                          self.alg.clip_rho_threshold, self.alg.clip_pg_rho_threshold,
                                          layout=kernels.TIME_MAJOR, out=self.loss_out)
        if ev is not None:
            e1.record()
            ev.append((e0, e1))
        self.tgt_logits, self.values = logits.view(T, B, A), values.view(T, B)
        net.backward(res['d_logits'], res['d_values'])
        return res

    def _learn_apply(self, learning_rate):
        """Clip + Adam on the (all-reduced) flat gradient, then refresh the kernels' operand copies."""
        opt = self.alg.optimizer
        if opt.lr_dev is not None:
            if learning_rate is not None and float(learning_rate) != opt.lr:
                opt.set_lr(learning_rate)                 # device-resident rate
            opt.step()
        else:
            opt.step(lr=learning_rate)
        self.train_net.pack()
        if self.actor_net is not None and not self.pipeline:
            self.actor_net.pack()

    # ------------------------------------------------------------------ reference-facing host contract
    def make_host_sample_buffers(self):
        """Pinned host arrays with the keys / dtypes / env-major order of Actor.sample()
        (examples/IMPALA/actor.py:54-91): obs [B*T,4,H,W] uint8, actions int64, behaviour_logits f32,
        rewards f32, dones bool."""
        N = self.B * self.T
        pin = dict(pin_memory=True)
        return dict(obs=torch.empty((N, 4, self.h, self.w), dtype=torch.uint8, **pin),
                    actions=torch.empty(N, dtype=torch.int64, **pin),
                    behaviour_logits=torch.empty((N, self.A), dtype=torch.float32, **pin),
                    rewards=torch.empty(N, dtype=torch.float32, **pin),
                    dones=torch.empty(N, dtype=torch.bool, **pin))

    def _sample_dict_to_host(self, host):
        """Enqueue the device->host copies of the current buffer set as the reference's env-major sample dict."""
        T, B = self.T, self.B
        em = lambda x: x.transpose(0, 1).contiguous()
        obs_dev = getattr(self, '_obs_em', None)
        if obs_dev is None:
            obs_dev = self._obs_em = torch.empty((B * T, 4, self.h, self.w), dtype=torch.uint8, device=self.device)
        kernels.obs_stack_gather(self.planes, self.ages, 0, T, obs_dev, layout=kernels.ENV_MAJOR)
        host['obs'].copy_(obs_dev, non_blocking=True)
        host['actions'].copy_(em(self.actions).view(-1).long(), non_blocking=True)
        host['behaviour_logits'].copy_(em(self.beh_logits).view(B * T, self.A), non_blocking=True)
        host['rewards'].copy_(em(self.rewards).view(-1), non_blocking=True)
        host['dones'].copy_(em(self.dones).view(-1).bool(), non_blocking=True)

    def sample_to_host(self, host):
        """rollout() + device->host copy of the sample dict in the reference's env-major layout."""
        self.rollout()
        self._sample_dict_to_host(host)
        torch.cuda.current_stream().synchronize()
        return host

    def step_host(self, hosts, learning_rate=0.001, entropy_coeff=-0.01):
        """Pipelined iteration THROUGH HOST MEMORY (the reference-facing contract, examples/IMPALA/train.py:165-194):
        the actor stream produces rollout k+1 and copies its numpy-layout sample dict to pinned host buffers
        hosts[(k+1)%2] while the learner stream uploads hosts[k%2] and trains on it."""
        assert self.pipeline and len(hosts) == 2
        cur_stream = torch.cuda.current_stream()
        k = self._k
        if not hasattr(self, '_host_ready'):
            self._host_ready = [torch.cuda.Event() for _ in range(2)]
        if k == 0:
            self.actor_stream.wait_stream(cur_stream)
            with torch.cuda.stream(self.actor_stream):
                self._run_rollout(0)
                self._sample_dict_to_host(hosts[0])
                self._host_ready[0].record(self.actor_stream)
        cur, nxt = k % 2, (k + 1) % 2
        with torch.cuda.stream(self.actor_stream):
            if self._learn_done[nxt] is not None:
                self.actor_stream.wait_event(self._learn_done[nxt])
            self._snapshot_actor_weights()
            self._ev_pack.record(self.actor_stream)
            self._run_rollout(nxt)
            self._sample_dict_to_host(hosts[nxt])
            self._host_ready[nxt].record(self.actor_stream)
        cur_stream.wait_event(self._ev_pack)
        cur_stream.wait_event(self._host_ready[cur])
        losses = self.learn_from_host(hosts[cur], learning_rate, entropy_coeff)
        ev = torch.cuda.Event()
        ev.record(cur_stream)
        self._learn_done[cur] = ev
        self._k += 1
        return losses

    def learn_from_host(self, host, learning_rate, entropy_coeff):
        """Agent.learn(numpy...) contract (examples/IMPALA/atari_agent.py:44-74): host arrays -> H2D ->
        IMPALA.learn in the reference's env-major order, processed in column slabs."""
        T, B, A = self.T, self.B, self.A
        dev = self.device
        acts = host['actions'].to(dev, non_blocking=True)
        bl = host['behaviour_logits'].to(dev, non_blocking=True)
        rew = host['rewards'].to(dev, non_blocking=True)
        dones = host['dones'].to(dev, non_blocking=True)
        if self.train_net is not None and self._host_slab_plan() is not None:
            return self._learn_from_host_slabs(host, acts, bl, rew, dones, learning_rate, entropy_coeff)
        if self.train_net is not None:
            # native learner: stacked uint8 observations -> conv1's space-to-depth input -> wgmma forward/backward
            net = self.train_net
            slab = 16384
            for s0 in range(0, B * T, slab):
                n = min(slab, B * T - s0)
                obs = host['obs'][s0:s0 + n].to(dev, non_blocking=True)
                kernels.obs_stack_gather(obs, None, 0, 1, net.x0[s0:s0 + n], scale=1.0 / 255.0, s2d=True)
            logits, values = net.forward_from_x0()
            res = kernels.vtrace_loss_fwd_bwd(logits, bl, acts, rew, dones, values.view(-1), T, B, self.alg.gamma,
                                              self.alg.vf_loss_coeff, entropy_coeff, self.alg.clip_rho_threshold,
                                              self.alg.clip_pg_rho_threshold, layout=kernels.ENV_MAJOR, out=self.loss_out)
            net.backward(res['d_logits'], res['d_values'])
        else:
            slab = max(1, (self.learn_chunk_rows * B) // T)          # env columns per forward slab
            tgt = torch.empty((B * T, A), dtype=torch.float32, device=dev)
            val = torch.empty(B * T, dtype=torch.float32, device=dev)
            outs = []
            for b0 in range(0, B, slab):
                nb = min(slab, B - b0)
                obs = host['obs'][b0 * T:(b0 + nb) * T].to(dev, non_blocking=True)
                logits, values = self.model.policy_and_value(obs)
                tgt[b0 * T:(b0 + nb) * T].copy_(logits.detach())
                val[b0 * T:(b0 + nb) * T].copy_(values.detach())
                outs.append((logits, values, b0 * T, nb * T))
            res = kernels.vtrace_loss_fwd_bwd(tgt, bl, acts, rew, dones, val, T, B, self.alg.gamma,
                                              self.alg.vf_loss_coeff, entropy_coeff, self.alg.clip_rho_threshold,
                                              self.alg.clip_pg_rho_threshold, layout=kernels.ENV_MAJOR, out=self.loss_out)
            tensors, grads = [], []
            for logits, values, o, n in outs:
                tensors += [logits, values]
                grads += [res['d_logits'][o:o + n], res['d_values'][o:o + n]]
            torch.autograd.backward(tensors, grads)
        if self.alg.grad_sync is not None:
            self.alg.grad_sync(self.alg.optimizer.grad)
        self.alg.optimizer.step(lr=learning_rate)
        if self.train_net is not None:
            self.train_net.pack()
        if self.actor_net is not None and not self.pipeline:
            self.actor_net.pack()
        return res['losses'].clone()

    def _host_slab_plan(self):
        """(number of slabs, env columns per slab) of the slab-pipelined host learner, or None: see host_slab_plan."""
        samples = getattr(self, 'host_slab_samples', None)
        if samples is None:
            samples = int(os.environ.get('PARL_B200_HOST_SLAB_SAMPLES', '16384'))
        return host_slab_plan(self.B, self.T, samples)

    def _learn_from_host_slabs(self, host, acts, bl, rew, dones, learning_rate, entropy_coeff):
        """learn_from_host with the H2D copy of the observations PIPELINED against the learner's compute: the batch
        is cut into equal slabs of whole env columns; a copy stream uploads slab i+1 into one of two staging buffers
        while the compute stream runs gather -> forward -> V-trace loss -> backward on slab i (a slab-sized
        AtariTrainNet) and adds its parameter gradient into an accumulator.  IMPALA's loss is a SUM over samples
        (impala.py:67-79), so per-slab gradients add up to the whole-batch gradient (fp32 summation order differs from
        the one-shot path: round-off only); one optimizer step per call, as before.  With 5.8 GB of observations per
        4096x50 batch the PCIe copy (~104 ms) was serialised in front of ~25 ms of compute; now only the last slab's
        compute is exposed."""
        T, B, A = self.T, self.B, self.A
        dev = self.device
        nsl, cols = self._host_slab_plan()
        ns = cols * T
        st = getattr(self, '_host_slab_state', None)
        if st is None or st['ns'] != ns:
            grad = self.alg.optimizer.grad
            st = self._host_slab_state = dict(
                ns=ns,
                net=AtariTrainNet(self.model, ns, dev, obs_dtype=self.obs_dtype if self.s2d else torch.bfloat16,
                                  flat=self._flat_master()),
                obs=[torch.empty((ns, 4, self.h, self.w), dtype=torch.uint8, device=dev) for _ in range(2)],
                copy_stream=torch.cuda.Stream(device=dev),
                ev_h2d=[torch.cuda.Event() for _ in range(2)], ev_free=[torch.cuda.Event() for _ in range(2)],
                acc=torch.empty_like(grad), losses=torch.zeros((nsl, 8), dtype=torch.float32, device=dev),
                d_logits=torch.empty((ns, A), dtype=torch.float32, device=dev),
                d_values=torch.empty(ns, dtype=torch.float32, device=dev))
        net, cs = st['net'], st['copy_stream']
        cur = torch.cuda.current_stream()
        cs.wait_stream(cur)                       # the staging buffers are free once the previous call's work is done
        grad = self.alg.optimizer.grad
        for i in range(nsl):
            s0, j = i * ns, i % 2
            with torch.cuda.stream(cs):
                if i >= 2:
                    cs.wait_event(st['ev_free'][j])
                st['obs'][j].copy_(host['obs'][s0:s0 + ns], non_blocking=True)
                st['ev_h2d'][j].record(cs)
            cur.wait_event(st['ev_h2d'][j])
            kernels.obs_stack_gather(st['obs'][j], None, 0, 1, net.x0, scale=1.0 / 255.0, s2d=True)
            st['ev_free'][j].record(cur)          # the staging buffer is consumed once the gather has run
            logits, values = net.forward_from_x0()
            res = kernels.vtrace_loss_fwd_bwd(logits, bl[s0:s0 + ns], acts[s0:s0 + ns], rew[s0:s0 + ns], dones[s0:s0 + ns],
                                              values.view(-1), T, cols, self.alg.gamma, self.alg.vf_loss_coeff,
                                              entropy_coeff, self.alg.clip_rho_threshold, self.alg.clip_pg_rho_threshold,
                                              layout=kernels.ENV_MAJOR,
                                              out=dict(losses=st['losses'][i], d_logits=st['d_logits'],
                                                       d_values=st['d_values']))
            net.backward(res['d_logits'], res['d_values'])
            if i == 0:
                st['acc'].copy_(grad)
            else:
                st['acc'].add_(grad)
        grad.copy_(st['acc'])
        if self.alg.grad_sync is not None:
            self.alg.grad_sync(grad)
        self.alg.optimizer.step(lr=learning_rate)
        net.pack()
        self.train_net.pack()
        if self.actor_net is not None and not self.pipeline:
            self.actor_net.pack()
        losses = st['losses'].sum(0)
        losses[4] = losses[4] / nsl               # KL is a mean over samples; the slabs are equal
        return losses

    # ------------------------------------------------------------------ metrics (Actor.get_metrics analogue)
    def get_metrics(self):
        tot = self.stats.totals.tolist()
        n = max(tot[0], 1.0)
        return dict(sample_steps=self.sample_steps, episodes=int(tot[0]), mean_episode_rewards=tot[1] / n,
                    mean_episode_steps=tot[2] / n)
