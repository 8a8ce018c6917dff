"""Operand copies of the network kernels and their one-launch refresh.

The wgmma kernels read the weights in their own layouts (bf16 KRSC filters, space-to-depth and transposed forms,
(H,W,C)-ordered fc columns, float32 biases).  Every element of every copy is ONE element of the optimizer's flat
float32 master buffer (``FlatAdam.flat``; zero for padding), so after a learner update all of them are rebuilt by one
``rl_gather_cast`` launch per dtype from a precomputed index permutation — instead of ~26 permute + copy launches, which
is a fixed cost per update that weighs on the small per-GPU batches of the 8-GPU strong-scaling run.

The index permutation is not derived by hand: the net describes its copies ONCE as tensor expressions over the
parameters (``sources(P, full)``), and the same expressions are evaluated on int32 index tensors.  Models whose
parameters are not views of one flat buffer (stand-alone nets in the tests) use the expressions directly
(``dst.copy_(src)``)."""
import torch

from .. import kernels as K

_ALIGN = 128          # elements: every carved operand starts on a 256-byte (bf16) / 512-byte (f32) boundary


class PackedOperands(object):
    def __init__(self, device):
        self.device = torch.device(device)
        self._specs = []
        self.arenas, self.slots = {}, {}
        self.flat = None
        self.idx = {}

    def declare(self, name, shape, dtype):
        self._specs.append((name, tuple(int(s) for s in shape), dtype))

    def materialize(self, owner):
        """Allocate one zeroed arena per dtype and set ``owner.<name>`` to its view."""
        for dtype in (torch.bfloat16, torch.float32):
            off = 0
            for name, shape, dt in self._specs:
                if dt != dtype:
                    continue
                n = 1
                for s in shape:
                    n *= s
                self.slots[name] = (dtype, off, n, shape)
                off += (n + _ALIGN - 1) // _ALIGN * _ALIGN
            self.arenas[dtype] = torch.zeros(max(off, _ALIGN), dtype=dtype, device=self.device)
        for name, (dtype, off, n, shape) in self.slots.items():
            setattr(owner, name, self.arenas[dtype][off:off + n].view(shape))

    # ---------------------------------------------------------------- refresh
    @torch.no_grad()
    def refresh(self, model, sources):
        """``sources(P, full)`` -> [(name, tensor expression over the parameters)]; P(name) is the parameter (or its
        index tensor), full(shape) a zero (or -1) tensor of the matching kind for partially filled copies."""
        if self.flat is not None:
            # the index permutation addresses the flat buffer: a model whose parameters were re-homed since (model.to(),
            # a new optimizer) would silently be refreshed from stale memory
            if self._probe.data_ptr() != self._probe_ptr:
                raise RuntimeError('parl_b200: the model parameters no longer live in the flat buffer the operand refresh '
                                   'was bound to (rebuild the net / engine after re-homing the parameters)')
            for dtype, idx in self.idx.items():
                K.gather_cast(self.flat, idx, self.arenas[dtype])
            return
        params = dict(model.named_parameters())
        exprs = sources(lambda n: params[n], lambda shape: torch.zeros(shape, dtype=torch.float32, device=self.device))
        for name, src in exprs:
            dtype, off, n, shape = self.slots[name]
            self.arenas[dtype][off:off + n].view(shape).copy_(src)

    @torch.no_grad()
    def bind_flat(self, flat, model, sources):
        """Switch to the one-launch refresh: requires every parameter to be a contiguous view of ``flat``."""
        base, total = flat.data_ptr(), flat.numel()
        index = {}
        for name, p in model.named_parameters():
            off = (p.data_ptr() - base) // 4
            if p.dtype != torch.float32 or not p.is_contiguous() or (p.data_ptr() - base) % 4 or off < 0 or \
                    off + p.numel() > total:
                return False
            index[name] = (torch.arange(p.numel(), dtype=torch.int32, device=self.device) + int(off)).view(p.shape)
        exprs = sources(lambda n: index[n], lambda shape: torch.full(shape, -1, dtype=torch.int32, device=self.device))
        idx = dict((dt, torch.full((a.numel(), ), -1, dtype=torch.int32, device=self.device)) for dt, a in self.arenas.items())
        for name, src in exprs:
            dtype, off, n, shape = self.slots[name]
            assert tuple(src.shape) == shape, (name, tuple(src.shape), shape)
            idx[dtype][off:off + n] = src.reshape(-1)
        self.idx, self.flat = idx, flat
        self._probe = next(iter(model.parameters()))
        self._probe_ptr = self._probe.data_ptr()
        return True
