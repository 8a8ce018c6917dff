"""Actor-side inference of the Atari actor-critic entirely on hand-written wgmma kernels
(rl_conv2d_s1_nhwc_bf16_fwd x3 in TMA-window form + rl_gemm_bf16_tn x2): the policy forward the reference runs on CPU, batch 5,
inside every remote actor (examples/IMPALA/actor.py:60-62, atari_agent.py:35-42) — here once per time
step for the whole pool, reading the space-to-depth observation written by rl_obs_stack_gather and writing
the logits straight into the (T,B,A) rollout buffer.

The bf16 operand copies of the parameters are re-packed from the fp32 master weights after every learner
update (``pack``): conv kernels in (r,s,c)-ordered [Cout, K] form, conv1 in its space-to-depth form, the
fc weight with (H,W,C)-ordered columns.
"""
import os

import torch

from .. import kernels
from .packing import PackedOperands


class AtariActorNet(object):
    def __init__(self, model, batch, device, window_form=True, flat=None):
        self.model = model
        self.B = int(batch)
        dev = self.device = torch.device(device)
        bf = torch.bfloat16
        self.window_form = window_form
        # fc + policy head in one call (rl_gemm_bf16_tn_heads): the head (N2 = 18) is a warp-level mma.sync kernel
        # instead of a tensor-core GEMM tile whose run time would be all prologue at that width
        self.fuse_heads = os.environ.get('PARL_B200_FUSE_HEADS', '1') != '0'
        # window form: conv1 writes conv2's zero-padded 2x2-block input [B,12,12,128] (border stays zero)
        self.a1 = (torch.zeros((self.B, 12, 12, 128), dtype=bf, device=dev) if window_form else
                   torch.empty((self.B, 20, 20, 32), dtype=bf, device=dev))
        self.a2 = torch.empty((self.B, 11, 11, 64), dtype=bf, device=dev)
        self.a3 = torch.empty((self.B, 9, 9, 64), dtype=bf, device=dev)
        self.h = torch.empty((self.B, 512), dtype=bf, device=dev)
        A = model.fc_pi.weight.shape[0]
        self.A = A
        f32 = torch.float32
        self.ops = PackedOperands(dev)
        for name, shape, dt in (('w1', (32, 256), bf), ('w2', (64, 512), bf), ('w3', (64, 576), bf),
                                ('wfc', (512, 5184), bf), ('wpi', (A, 512), bf), ('wv', (1, 512), bf),
                                ('b1', (32, ), f32), ('b2', (64, ), f32), ('b3', (64, ), f32), ('bfc', (512, ), f32),
                                ('bpi', (A, ), f32), ('bv', (1, ), f32)):
            self.ops.declare(name, shape, dt)
        self.ops.materialize(self)
        if flat is not None:
            self.ops.bind_flat(flat, model, self._sources)
        self.pack()

    def _sources(self, P, full):
        """The operand copies as tensor expressions over the parameters (see engine/packing.py)."""
        # conv1 8x8/4 -> 2x2/1 on 4x4 pixel blocks: W1[o,c,4a+dy,4b+dx] -> [o, (a,b), (dy,dx,c)]
        w1 = P('conv1.weight').view(32, 4, 2, 4, 2, 4).permute(0, 2, 4, 3, 5, 1).reshape(32, 256)    # (o, a, b, dy, dx, c)
        if self.window_form:
            # conv2 4x4/2/p2 -> 2x2/1 on 2x2 pixel blocks: W2[o,c,2a+dy,2b+dx] -> [o, (a,b), (dy,dx,c)]
            w2 = P('conv2.weight').view(64, 32, 2, 2, 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(64, 512)
        else:
            w2 = P('conv2.weight').permute(0, 2, 3, 1).reshape(64, 512)                             # (o, r, s, c)
        return [('w1', w1), ('w2', w2), ('w3', P('conv3.weight').permute(0, 2, 3, 1).reshape(64, 576)),
                ('wfc', P('fc.weight').view(512, 64, 9, 9).permute(0, 2, 3, 1).reshape(512, 5184)),
                ('wpi', P('fc_pi.weight')), ('wv', P('fc_v.weight')), ('b1', P('conv1.bias')), ('b2', P('conv2.bias')),
                ('b3', P('conv3.bias')), ('bfc', P('fc.bias')), ('bpi', P('fc_pi.bias')), ('bv', P('fc_v.bias'))]

    @torch.no_grad()
    def pack(self):
        """fp32 master weights -> bf16 kernel operands, in place (safe between CUDA-graph replays): one gather launch
        per dtype when the parameters live in the optimizer's flat buffer, else one copy per operand."""
        self.ops.refresh(self.model, self._sources)

    def policy(self, obs_s2d, logits_out):
        """obs_s2d [B,21,21,64] uint8 (bytes; conv1 scales by 1/255 while widening) or bf16 (already scaled)
        -> logits_out [B,A] float32."""
        K = kernels
        if self.window_form:
            K.conv2d_s1_nhwc_bf16_fwd(obs_s2d, self.w1, self.b1, 2, 2, relu=True, out=self.a1, out_mode=1)
            K.conv2d_s1_nhwc_bf16_fwd(self.a1, self.w2, self.b2, 2, 2, relu=True, out=self.a2)
            K.conv2d_s1_nhwc_bf16_fwd(self.a2, self.w3, self.b3, 3, 3, relu=True, out=self.a3)
        else:
            K.conv2d_nhwc_bf16_fwd(obs_s2d, self.w1, self.b1, 2, 2, 1, 0, relu=True, out=self.a1)
            K.conv2d_nhwc_bf16_fwd(self.a1, self.w2, self.b2, 4, 4, 2, 2, relu=True, out=self.a2)
            K.conv2d_nhwc_bf16_fwd(self.a2, self.w3, self.b3, 3, 3, 1, 0, relu=True, out=self.a3)
        if self.fuse_heads:
            K.gemm_bf16_tn_heads(self.a3.view(self.B, 5184), self.wfc, self.bfc, self.h, self.wpi, self.bpi, logits_out)
        else:
            K.gemm_bf16_tn(self.a3.view(self.B, 5184), self.wfc, self.bfc, relu=True, out=self.h)
            K.gemm_bf16_tn(self.h, self.wpi, self.bpi, relu=False, out=logits_out)
        return logits_out

    def value(self, values_out):
        """Value head on the trunk features of the last ``policy`` call -> values_out [B,1] float32."""
        return kernels.gemm_bf16_tn(self.h, self.wv, self.bv, relu=False, out=values_out)
