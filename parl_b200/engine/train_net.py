"""Learner-side forward AND backward of the Atari actor-critic on hand-written wgmma kernels — no autograd,
no cuDNN on the convolution path.

Layers (a13: benchmark/torch/a2c/atari_model.py:23-96), all stride-1 in TMA-window form after space-to-depth:
    x0 [N,21,21,64] bf16 pre-scaled by 1/255 (or uint8 bytes, widened inside the conv1 kernels) --conv1' 2x2--> a1 (padded 2x2-block layout [N,12,12,128]) --conv2' 2x2--> a2 [N,11,11,64]
       --conv3 3x3--> a3 [N,9,9,64] == [N,5184] --fc--> h [N,512] --heads--> logits [N,A], values [N]
Backward (after the fused loss kernel delivered d_logits / d_values):
    heads/fc data gradients : rl_gemm_bf16_tn_masked (ReLU masks fused in the epilogue)
    conv data gradients     : rl_conv2d_s1_nhwc_bf16_dgrad (same windows, flipped taps, ReLU mask fused)
    conv weight gradients   : rl_conv2d_s1_nhwc_bf16_wgrad (positions as the GEMM K dimension, register-resident accumulators)
    bias gradients          : from the weight-gradient pass (one extra wgmma.mma per K step against ones); fc: rl_colsum_bf16
    fc / head weight gradients: two plain library GEMMs (torch.matmul -> cuBLAS), the only library calls left
Activations for the whole learner batch stay resident in HBM (about 120 KB per sample in bf16).
Gradients are written into the parameters' ``.grad`` views of the FlatAdam buffer in the reference layouts.
"""
import torch

from .. import kernels as K
from .packing import PackedOperands


class AtariTrainNet(object):
    def __init__(self, model, n_samples, device, fc_backend='auto', obs_dtype=torch.bfloat16, flat=None):
        self.model = model
        assert obs_dtype in (torch.uint8, torch.bfloat16)
        self.obs_dtype = obs_dtype          # bfloat16: pre-scaled operand (default); uint8: conv1 reads bytes (u8in kernels)
        N = self.N = int(n_samples)
        dev = self.device = torch.device(device)
        bf, f32 = torch.bfloat16, torch.float32
        A = self.A = model.fc_pi.weight.shape[0]
        z = lambda *s: torch.zeros(s, dtype=bf, device=dev)
        e = lambda *s: torch.empty(s, dtype=bf, device=dev)
        # activations
        # x0 (conv1's space-to-depth input) is allocated on first use: the on-device engine hands in the rollout
        # buffer's own observation plane (written by the actor at step t) instead, see ImpalaEngine.share_obs
        self._x0 = self._x0_in = None
        self.a1, self.a2, self.a3 = z(N, 12, 12, 128), e(N, 11, 11, 64), e(N, 9, 9, 64)
        self.h = e(N, 512)
        self.logits = torch.empty((N, A), dtype=f32, device=dev)
        self.values = torch.empty((N, 1), dtype=f32, device=dev)
        # gradients of activations (grids are zero where no valid output exists and are never written there)
        self.dheads, self.dh = z(N, 32), e(N, 512)
        self.da3g, self.da2g, self.da1g = z(N, 11, 11, 64), z(N, 12, 12, 64), z(N, 21, 21, 32)
        # operand copies of the weights (carved from two arenas, refreshed by one gather launch per dtype: packing.py)
        self.ops = PackedOperands(dev)
        for name, shape, dt in (('w1', (32, 256), bf), ('w2', (64, 512), bf), ('w3', (64, 576), bf),
                                ('wfc', (512, 5184), bf), ('wpi', (A, 512), bf), ('wv', (1, 512), bf),
                                ('wfcT', (5184, 512), bf), ('whT', (512, 32), bf), ('w3T', (64, 576), bf),
                                ('w2T', (128, 256), bf), ('b1', (32, ), f32), ('b2', (64, ), f32), ('b3', (64, ), f32),
                                ('bfc', (512, ), f32), ('bpi', (A, ), f32), ('bv', (1, ), f32)):
            self.ops.declare(name, shape, dt)
        self.ops.materialize(self)
        if flat is not None:
            self.ops.bind_flat(flat, model, self._sources)
        # weight-gradient scratch (KRSC, float32)
        self.dw1 = torch.empty((32, 256), dtype=f32, device=dev)
        self.dw2 = torch.empty((64, 512), dtype=f32, device=dev)
        self.dw3 = torch.empty((64, 576), dtype=f32, device=dev)
        self.dbs = [torch.empty(n, dtype=f32, device=dev) for n in (512, 64, 64, 32)]     # bias-gradient scratch
        # the two big fc contractions (K=5184 / N=5184 over all samples) go to the library GEMM by default at large
        # batches, with our fused epilogue kernels around it
        self.fc_library = fc_backend == 'library' or (fc_backend == 'auto' and N > 16384)
        self.da3c = e(N, 5184) if self.fc_library else None
        self.pack()

    @property
    def x0(self):
        if self._x0 is None:
            self._x0 = torch.empty((self.N, 21, 21, 64), dtype=self.obs_dtype, device=self.device)
        return self._x0

    def _sources(self, P, full):
        """The operand copies as tensor expressions over the parameters (see engine/packing.py)."""
        A = self.A
        w2p = P('conv2.weight').view(64, 32, 2, 2, 2, 2).permute(0, 2, 4, 3, 5, 1)        # (o, a, b, dy, dx, c)
        wfc = P('fc.weight').view(512, 64, 9, 9).permute(0, 2, 3, 1).reshape(512, 5184)   # columns in (h,w,c) order
        whT = full((512, 32))
        whT[:, :A] = P('fc_pi.weight').t()
        whT[:, A:A + 1] = P('fc_v.weight').t()
        return [('w1', P('conv1.weight').view(32, 4, 2, 4, 2, 4).permute(0, 2, 4, 3, 5, 1).reshape(32, 256)),
                ('w2', w2p.reshape(64, 512)),
                ('w2T', w2p.permute(3, 4, 5, 1, 2, 0).reshape(128, 256)),                 # [(dy,dx,c)][(a,b,o)]
                ('w3', P('conv3.weight').permute(0, 2, 3, 1).reshape(64, 576)),           # (o, r, s, c)
                ('w3T', P('conv3.weight').permute(1, 2, 3, 0).reshape(64, 576)),          # [c][(r,s,o)]
                ('wfc', wfc), ('wfcT', wfc.t()), ('wpi', P('fc_pi.weight')), ('wv', P('fc_v.weight')), ('whT', whT),
                ('b1', P('conv1.bias')), ('b2', P('conv2.bias')), ('b3', P('conv3.bias')), ('bfc', P('fc.bias')),
                ('bpi', P('fc_pi.bias')), ('bv', P('fc_v.bias'))]

    @torch.no_grad()
    def pack(self):
        self.ops.refresh(self.model, self._sources)

    # ------------------------------------------------------------------ forward
    def forward(self, planes, ages, t_count, layout=K.TIME_MAJOR):
        """Observations of rows [0, t_count) of the frame ring -> self.logits [N,A], self.values [N,1]."""
        N = self.N
        K.obs_stack_gather(planes, ages, 0, t_count, self.x0, layout=layout, scale=1.0 / 255.0, s2d=True)
        return self.forward_from_x0()

    def forward_from_x0(self, x0=None):
        """x0 [N,21,21,64] uint8 or pre-scaled bf16 (default: this net's own buffer); kept by reference for conv1's
        weight gradient."""
        N = self.N
        x0 = self._x0_in = self.x0 if x0 is None else x0
        K.conv2d_s1_nhwc_bf16_fwd(x0, self.w1, self.b1, 2, 2, relu=True, out=self.a1, out_mode=1)
        K.conv2d_s1_nhwc_bf16_fwd(self.a1, self.w2, self.b2, 2, 2, relu=True, out=self.a2)
        K.conv2d_s1_nhwc_bf16_fwd(self.a2, self.w3, self.b3, 3, 3, relu=True, out=self.a3)
        if self.fc_library:
            torch.matmul(self.a3.view(N, 5184), self.wfcT, out=self.h)
            K.bias_act_bf16(self.h, self.bfc, relu=True)
        else:
            K.gemm_bf16_tn(self.a3.view(N, 5184), self.wfc, self.bfc, relu=True, out=self.h)
        K.gemm_bf16_tn(self.h, self.wpi, self.bpi, relu=False, out=self.logits)
        K.gemm_bf16_tn(self.h, self.wv, self.bv, relu=False, out=self.values)
        return self.logits, self.values

    # ------------------------------------------------------------------ backward
    def _bias_grad(self, grid, scratch, param):
        """param.grad = column sums of a gradient grid (a side stream was tried in round 1: the column sums then
        merely share HBM bandwidth with the tensor-core kernels, no net gain)."""
        param.grad.copy_(K.colsum_bf16(grid, out=scratch))

    @torch.no_grad()
    def backward(self, d_logits, d_values):
        """d_logits [N,A] f32, d_values [N] f32 -> fills ``p.grad`` of every model parameter."""
        N, A, m = self.N, self.A, self.model
        self.dheads[:, :A].copy_(d_logits)
        self.dheads[:, A].copy_(d_values.reshape(-1))
        # heads
        dwh = self.dheads[:, :A + 1].t().float() @ self.h.float() if N <= 4096 else \
            (self.dheads[:, :A + 1].t() @ self.h).float()
        m.fc_pi.weight.grad.copy_(dwh[:A])
        m.fc_v.weight.grad.copy_(dwh[A:A + 1])
        m.fc_pi.bias.grad.copy_(d_logits.sum(0))          # head bias gradients straight from the fp32 loss gradients
        m.fc_v.bias.grad.copy_(d_values.sum().reshape(1))
        K.gemm_bf16_tn_masked(self.dheads, self.whT, self.h, self.dh)                       # dh = (dheads.Wh) * (h>0)
        # fc
        a3f = self.a3.view(N, 5184)
        dwfc = (self.dh.t() @ a3f).float()                                                   # [512, 5184] (h,w,c) cols
        m.fc.weight.grad.copy_(dwfc.view(512, 9, 9, 64).permute(0, 3, 1, 2).reshape(512, 5184))
        self._bias_grad(self.dh, self.dbs[0], m.fc.bias)
        if self.fc_library:
            torch.matmul(self.dh, self.wfc, out=self.da3c)                                   # [N, 5184] compact
            K.mask_scatter_grid_bf16(self.da3c, self.a3, self.da3g, N, 9, 9, 11, 11, 64)    # ReLU mask + 11x11 grid
        else:
            da3 = self.da3g.view(N, 121 * 64)
            for y in range(9):   # image row y of the 9x9 output = 576 contiguous columns of the 11x11 gradient grid
                K.gemm_bf16_tn_masked(self.dh, self.wfcT[y * 576:(y + 1) * 576], a3f[:, y * 576:(y + 1) * 576],
                                      da3[:, y * 704:y * 704 + 576])
        # conv3
        K.conv2d_s1_nhwc_bf16_wgrad(self.da3g, self.a2, 3, 3, dw_krsc=self.dw3, db=self.dbs[1])
        m.conv3.weight.grad.copy_(self.dw3.view(64, 3, 3, 64).permute(0, 3, 1, 2))
        m.conv3.bias.grad.copy_(self.dbs[1])
        K.conv2d_s1_nhwc_bf16_dgrad(self.da3g, self.w3T, 3, 3, self.da2g, act_mask=self.a2)   # onto the 12x12 grid
        # conv2 (2x2 block form)
        K.conv2d_s1_nhwc_bf16_wgrad(self.da2g, self.a1, 2, 2, dw_krsc=self.dw2, db=self.dbs[2])
        m.conv2.weight.grad.copy_(self.dw2.view(64, 2, 2, 2, 2, 32).permute(0, 5, 1, 3, 2, 4).reshape(64, 32, 4, 4))
        m.conv2.bias.grad.copy_(self.dbs[2])
        K.conv2d_s1_nhwc_bf16_dgrad(self.da2g, self.w2T, 2, 2, self.da1g, act_mask=self.a1, out_mode=2)
        # conv1 (4x4 block form): 64-byte gradient rows -> role-swapped weight-gradient kernel (SWIZZLE_64B operand)
        K.conv2d_s1_nhwc_bf16_wgrad(self.da1g, self._x0_in, 2, 2, dw_krsc=self.dw1, db=self.dbs[3])
        m.conv1.weight.grad.copy_(self.dw1.view(32, 2, 2, 4, 4, 4).permute(0, 5, 1, 3, 2, 4).reshape(32, 4, 8, 8))
        m.conv1.bias.grad.copy_(self.dbs[3])
