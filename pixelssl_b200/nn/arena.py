"""Flat HBM parameter arena + the fused optimiser/EMA step + the data-parallel wrapper.

Reference mechanism being replaced: ``nn.DataParallel`` (nn/func.py:58-59) re-broadcasting 176 MB
of parameters every forward, ``torch.optim.SGD`` + a 320-tensor Python EMA loop
(ssl_mt.py:359-363).  Here: every parameter is a view into ONE contiguous fp32 buffer (same for
gradients and momentum), SGD+EMA is one kernel per learning-rate group, and multi-GPU is one
process per GPU with a single NCCL all-reduce of the flat gradient buffer."""
import torch
import torch.nn as nn

from .. import ops


# False: models built now stay single-process even when torch.distributed is initialised (no BN statistics exchange,
# no gradient all-reduce) - used by bench.py's ddp_check to run the big-batch yardstick on one rank
DISTRIBUTED = True


class ParamArena:
    def __init__(self, module):
        params = [p for p in module.parameters()]
        self.params = params
        dev = params[0].device
        total = sum(p.numel() for p in params)
        # segments aligned to 8 elements: 32 bytes in fp32 (128-bit accesses), 16 bytes in the arena-wide fp16 pairs
        # (TMA descriptors over a slice need a 16-byte aligned base)
        offs, cur = [], 0
        for p in params:
            offs.append(cur)
            cur += (p.numel() + 7) // 8 * 8
        self.numel = cur
        self.offsets = offs
        self.data = torch.zeros(cur, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(cur, dtype=torch.float32, device=dev)
        self.mom = None
        self.steps = 0
        self._index = {}
        with torch.no_grad():
            for p, o in zip(params, offs):
                n = p.numel()
                view = self._view_like(self.data, o, p)
                view.copy_(p.data)
                p.data = view
                p.grad = self._view_like(self.grad, o, p)
                self._index[id(p)] = (o, n)
        # conv weights (4-D, stored [Cout][kh*kw][Cin]): table for the batched transpose / tf32 split of a step
        rows, tiles = [], 0
        self._conv_at = {}
        for p, o in zip(params, offs):
            if p.dim() == 4 and p.is_contiguous(memory_format=torch.channels_last):
                co, ci, kh, kw = p.shape
                rows.append([o, o, co, kh * kw, ci, tiles])
                self._conv_at[o] = (co, kh * kw, ci)
                tiles += ((ci + 31) // 32) * ((co + 31) // 32) * kh * kw
        self._conv_table = torch.tensor(rows, dtype=torch.int64, device=dev) if rows else None
        self._conv_tiles = tiles
        self._derived = {}            # name -> flat tensor; valid for self._derived_key
        self._derived_key = None
        self.distributed = DISTRIBUTED
        ops.register_param_arena(self)

    def derived(self, name):
        """Per-step derived copies of the whole arena, produced with ONE launch each and cached until the parameters
        change: 't' = every conv weight transposed to [Cin][taps][Cout] (dgrad operand), 'hi'/'lo' = tf32 split of
        the arena, 't_hi'/'t_lo' = split of the transposed arena.  Views are taken by element offset."""
        key = (ops.step_epoch(), self.data._version)
        if key != self._derived_key:
            self._derived_key, self._derived_valid = key, set()
        if name in self._derived_valid:
            return self._derived[name]
        if name not in self._derived:
            self._derived[name] = torch.zeros_like(self.data)
        if name == 't':
            if self._conv_table is None:
                raise ValueError('arena holds no convolution weights')
            ops.transpose_weights_batched(self.data, self._derived['t'], self._conv_table, self._conv_tiles)
        elif name in ('hi', 'lo'):
            for other in ('hi', 'lo'):
                if other not in self._derived:
                    self._derived[other] = torch.zeros_like(self.data)
            ops.split_tf32_into(self.data, self._derived['hi'], self._derived['lo'])
            self._derived_valid.update(('hi', 'lo'))
        elif name in ('t_hi', 't_lo'):
            src = self.derived('t')
            for other in ('t_hi', 't_lo'):
                if other not in self._derived:
                    self._derived[other] = torch.zeros_like(self.data)
            ops.split_tf32_into(src, self._derived['t_hi'], self._derived['t_lo'])
            self._derived_valid.update(('t_hi', 't_lo'))
        elif name in ('h16', 'h16_t'):
            # fp16 pairs (hi plane, lo plane) of the whole arena / of the transposed arena, one launch each
            src = self.data if name == 'h16' else self.derived('t')
            if self._derived[name].dtype != torch.float16:
                self._derived[name] = torch.zeros((2, self.numel), dtype=torch.float16, device=self.data.device)
            ops.call('pxl_h16_split', ops._p(src), ops._p(self._derived[name][0]), ops._p(self._derived[name][1]),
                     self.numel, float(ops.H16_W_SCALE), ops._p(None), 0, ops._stream())
        else:
            raise KeyError(name)
        self._derived_valid.add(name)
        return self._derived[name]

    def locate(self, t):
        """Element offset of tensor ``t`` inside this arena's parameter buffer, or None."""
        d = t.data_ptr() - self.data.data_ptr()
        if d < 0 or d >= 4 * self.numel or d % 4:
            return None
        return d // 4

    @staticmethod
    def _view_like(flat, off, p):
        """A view of flat[off:off+numel] with p's shape AND p's physical layout."""
        n = p.numel()
        seg = flat[off:off + n]
        if p.dim() == 4 and p.is_contiguous(memory_format=torch.channels_last) and not p.is_contiguous():
            o, i, h, w = p.shape
            return seg.view(o, h, w, i).permute(0, 3, 1, 2)
        return seg.view(p.shape)

    def zero_grad(self):
        ops.new_step()
        self.grad.zero_()
        for p, o in zip(self.params, self.offsets):
            if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + 4 * o:
                p.grad = self._view_like(self.grad, o, p)

    def segments(self, group_params):
        """Merge the arena ranges of ``group_params`` into maximal contiguous [start, end) runs."""
        spans = sorted(self._index[id(p)] for p in group_params)
        runs = []
        for o, n in spans:
            end = o + (n + 7) // 8 * 8
            if runs and runs[-1][1] == o:
                runs[-1][1] = end
            else:
                runs.append([o, end])
        return [(a, min(b, self.numel)) for a, b in runs]

    def all_reduce_grads(self, group=None):
        import torch.distributed as dist
        if self.distributed and dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            if dist.get_backend(group) == 'nccl':
                dist.all_reduce(self.grad, op=dist.ReduceOp.AVG, group=group)     # the 1/world scaling rides in the reduction
            else:
                dist.all_reduce(self.grad, group=group)
                self.grad.div_(dist.get_world_size(group))

    def sgd_step(self, optimizer, teacher=None, ema_d=0.0):
        """torch.optim.SGD.step() semantics (momentum, weight decay, dampening 0, no nesterov) read
        from ``optimizer.param_groups`` (so LR schedulers keep working), fused with the teacher
        EMA (ssl_mt.py:359-363) when ``teacher`` (a ParamArena with identical layout) is given."""
        if self.mom is None:
            self.mom = torch.zeros_like(self.data)
        first = self.steps == 0
        for g in optimizer.param_groups:
            if g.get('nesterov', False) or g.get('dampening', 0) != 0 or g.get('maximize', False):
                raise NotImplementedError('fused SGD supports dampening=0, nesterov=False only')
            mom = g.get('momentum', 0.0)
            for a, b in self.segments(g['params']):
                ops.sgd_ema_(self.data[a:b], self.grad[a:b], self.mom[a:b],
                             teacher.data[a:b] if teacher is not None else None,
                             g['lr'], mom, g.get('weight_decay', 0.0), ema_d, first or mom == 0)
        if first:
            for g in optimizer.param_groups:
                if g.get('momentum', 0.0) != 0:
                    for p in g['params']:
                        o, n = self._index[id(p)]
                        optimizer.state[p]['momentum_buffer'] = self._view_like(self.mom, o, p)
        self.steps += 1
        ops.new_step()           # parameters changed under torch's feet: drop cached tf32 splits

    def adam_step(self, optimizer):
        """torch.optim.Adam.step() semantics (no amsgrad) on the flat arena: the FC discriminator /
        flaw detector optimiser (ssl_adv.py:101-102, ssl_gct.py:153-154)."""
        if getattr(self, 'exp_avg', None) is None:
            self.exp_avg = torch.zeros_like(self.data)
            self.exp_avg_sq = torch.zeros_like(self.data)
        self.steps += 1
        for g in optimizer.param_groups:
            if g.get('amsgrad', False) or g.get('maximize', False):
                raise NotImplementedError('fused Adam supports amsgrad=False only')
            b1, b2 = g['betas']
            for a, b in self.segments(g['params']):
                ops.adam_(self.data[a:b], self.grad[a:b], self.exp_avg[a:b], self.exp_avg_sq[a:b], g['lr'], b1, b2,
                          g['eps'], g.get('weight_decay', 0.0), self.steps)
            for p in g['params']:
                st = optimizer.state[p]
                if 'exp_avg' not in st:
                    o, n = self._index[id(p)]
                    st['exp_avg'] = self._view_like(self.exp_avg, o, p)
                    st['exp_avg_sq'] = self._view_like(self.exp_avg_sq, o, p)
                st['step'] = torch.tensor(float(self.steps))
        ops.new_step()

    def invalidate(self):
        """Parameters were written behind the arena's back (load_state_dict, param.copy_): drop every derived copy
        (transposes, tf32 splits, fp16 pairs) and per-tensor split caches."""
        self._derived_key = None
        ops.new_step()

    def adopt_optimizer_state(self, optimizer):
        """After ``optimizer.load_state_dict`` (resume): pull the loaded SGD momentum buffers / Adam moments and
        step count into the flat arena and point the optimizer state back at the arena views, so that the fused
        update continues exactly where the checkpoint left off (torch.optim semantics on resume)."""
        found_sgd = False
        adam_step = None
        for g in optimizer.param_groups:
            for p in g['params']:
                st = optimizer.state.get(p, {})
                o, n = self._index[id(p)]
                buf = st.get('momentum_buffer')
                if buf is not None:
                    if self.mom is None:
                        self.mom = torch.zeros_like(self.data)
                    view = self._view_like(self.mom, o, p)
                    view.copy_(buf)
                    st['momentum_buffer'] = view
                    found_sgd = True
                if 'exp_avg' in st and 'exp_avg_sq' in st:
                    if getattr(self, 'exp_avg', None) is None:
                        self.exp_avg = torch.zeros_like(self.data)
                        self.exp_avg_sq = torch.zeros_like(self.data)
                    for key, flat in (('exp_avg', self.exp_avg), ('exp_avg_sq', self.exp_avg_sq)):
                        view = self._view_like(flat, o, p)
                        if st[key].data_ptr() != view.data_ptr():
                            view.copy_(st[key])
                        st[key] = view
                    step = st.get('step', 0)
                    step = int(step.item()) if torch.is_tensor(step) else int(step)
                    adam_step = step if adam_step is None else max(adam_step, step)
        if adam_step is not None:
            self.steps = adam_step          # bias correction continues from the checkpoint's step count
        elif found_sgd:
            self.steps = max(self.steps, 1)
        self.invalidate()


class EngineParallel(nn.Module):
    """Stands where ``nn.DataParallel`` stood (nn/func.py:58): holds the task model as ``.module``.
    One process drives one GPU; with torch.distributed initialised (world_size > 1) parameters are
    broadcast from rank 0 at construction, BN layers share statistics over NCCL and
    ``arena.all_reduce_grads()`` averages gradients."""

    def __init__(self, module):
        super().__init__()
        self.module = module
        self.arena = None

    def cuda(self, device=None):
        super().cuda(device)
        self.arena = ParamArena(self.module)
        self._setup_distributed()
        return self

    def _setup_distributed(self):
        import torch.distributed as dist
        if DISTRIBUTED and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.broadcast(self.arena.data, src=0)
            for b in self.module.buffers():
                dist.broadcast(b, src=0)
            from .modules import BatchNorm2d
            for m in self.module.modules():
                if isinstance(m, BatchNorm2d) or hasattr(m, 'num_BN'):       # BatchNorm2d and IBNorm
                    m.sync_group = dist.group.WORLD
            _ensure_peer_exchange(dist.group.WORLD)

    def forward(self, *inputs, **kwargs):
        return self.module(*inputs, **kwargs)

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        if self.arena is not None:
            self.arena.invalidate()       # the copies into the parameter views bypass the arena's version counter
        return out



_peer_exchange_state = {}


def _ensure_peer_exchange(group):
    """BN statistics travel over NVLink peer memory (nn/peer.py) when every rank drives a CUDA device of this node
    and PXL_PEER_BN != 0; otherwise the per-layer NCCL all-reduce stays.  Set up once per process group."""
    import os
    import torch.distributed as dist
    from .. import ops
    if id(group) in _peer_exchange_state:
        return _peer_exchange_state[id(group)]
    px = None
    want = os.environ.get('PXL_PEER_BN', '1') != '0' and torch.cuda.is_available() and dist.get_backend(group) == 'nccl'
    flags = [None] * dist.get_world_size(group)
    dist.all_gather_object(flags, bool(want), group=group)
    if all(flags) and dist.get_world_size(group) <= 8:
        from .peer import PeerExchange
        px = PeerExchange(group)
        ops.register_peer_exchange(group, px)
    _peer_exchange_state[id(group)] = px
    return px
