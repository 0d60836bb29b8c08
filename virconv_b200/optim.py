"""The parameter update of the adam_onecycle / adam_cosin training step on the library's two kernels (vc_optim_step).

The reference's loop ends every iteration with (tools/train_utils/train_utils.py:50-52)

    clip_grad_norm_(model.parameters(), GRAD_NORM_CLIP)
    optimizer.step()            # OptimWrapper (fastai_optim.py:132-149) over Adam(betas=(mom, 0.99)): one p.data.mul_ per tensor
    optimizer.zero_grad()       # for the true weight decay, then torch.optim.Adam

`FusedAdamOneCycle` does the same arithmetic for every tensor in two launches, with no host read:

    opt = FusedAdamOneCycle.from_model(model, wd=0.01)          # the groups build_optimizer makes (optimization/__init__.py:19-32)
    sched = OneCycle(opt, total_steps, lr_max, moms, div_factor, pct_start)     # the reference's scheduler, unchanged
    for it, batch in enumerate(loader):
        sched.step(it)                                          # sets opt.lr / opt.mom
        loss_fn(model(batch)).backward()
        opt.step(max_norm=10.0)                                 # clip + decay + Adam; the gradients are left as they are
        opt.zero_grad()

or, inside a captured step, `graph.GraphedStep(model, loss_fn, optimizer=opt, max_grad_norm=10.0)`.

What differs from the reference, on purpose: a step whose total gradient norm is not finite (or, in a captured step, whose
replay raised an overflow or error flag) is SKIPPED — parameters, Adam state and the step count stay as they were, and
`skipped_steps()` grows — where the reference multiplies every gradient by NaN.  One step count serves all tensors (torch
keeps one per tensor; they agree whenever a tensor either always or never receives a gradient, as VirConv's do).

Multi-GPU order: backward, `parallel.allreduce_gradients(params)`, then the eager `step()`; the captured step refuses a
world size above one because the all-reduce has to sit between its backward and its update.
"""
from __future__ import annotations

import weakref

import numpy as np
import torch
import torch.nn as nn

from . import _lib, ops

CHUNK = 4096                    # VC_OPTIM_CHUNK
MAX_GUARDS = 8                  # VC_OPTIM_MAX_GUARDS
_SEG_WORDS = 5                  # vc_optim_seg: p, g, m, v, n
_CHUNK_DT = np.dtype([('seg', '<i4'), ('len', '<i4'), ('off', '<i8')])       # vc_optim_chunk
BN_TYPES = (nn.BatchNorm1d, nn.BatchNorm2d, nn.BatchNorm3d, nn.SyncBatchNorm)

_LIVE = weakref.WeakSet()
_UNSET = object()


def live_optimizers():
    """The fused optimizers alive in this process (reference_env's clip_grad_norm_ looks its parameters up here)."""
    return list(_LIVE)


def chunk_list(numels, chunk=CHUNK):
    """The chunk list of tensors with `numels` elements: each tensor cut into pieces of at most `chunk` elements."""
    assert chunk > 0 and chunk % 4 == 0, chunk
    rows = [(i, min(chunk, n - off), off) for i, n in enumerate(numels) for off in range(0, int(n), chunk)]
    return np.array(rows, dtype=_CHUNK_DT)


def leaf_param_groups(model):
    """The two parameter groups the reference builds for adam_onecycle / adam_cosin: the model flattened to its leaf modules
    (the ones without children) in depth-first order, the trainable parameters of the non-BatchNorm leaves first, those of the
    BatchNorm leaves second.  A parameter a module WITH children owns directly is in neither (the flattening never visits
    it); -> ([non-BN, BN], those left-out trainable parameters)."""
    groups, seen = ([], []), set()
    for mod in model.modules():
        if next(mod.children(), None) is not None:
            continue
        for p in mod.parameters(recurse=False):
            if p.requires_grad and id(p) not in seen:
                seen.add(id(p))
                groups[1 if isinstance(mod, BN_TYPES) else 0].append(p)
    rest = [p for p in model.parameters() if p.requires_grad and id(p) not in seen]
    return [groups[0], groups[1]], rest


def pack_state_dict(param_groups, t, entries):
    """torch.optim.Adam's state_dict: param_groups with their tensors numbered in order, state[i] = {step, exp_avg,
    exp_avg_sq} for the tensors of `entries` ({position: (exp_avg, exp_avg_sq)}), all at step `t` (none before the first)."""
    groups, k = [], 0
    for g in param_groups:
        n = len(g['params'])
        groups.append(dict(g, params=list(range(k, k + n))))
        k += n
    state = {i: {'step': torch.tensor(float(t)), 'exp_avg': m, 'exp_avg_sq': v} for i, (m, v) in entries.items() if t > 0}
    return {'state': state, 'param_groups': groups}


def unpack_state_dict(sd, group_sizes):
    """-> (t, {position: (exp_avg, exp_avg_sq)}, the first group's hyper-parameters) of a torch.optim.Adam state_dict whose
    groups hold `group_sizes` tensors.  One step count serves every tensor here: a checkpoint whose tensors disagree raises."""
    groups = sd['param_groups']
    if [len(g['params']) for g in groups] != list(group_sizes):
        raise ValueError('the checkpoint has parameter groups of %s tensors, this optimizer of %s'
                         % ([len(g['params']) for g in groups], list(group_sizes)))
    ids = [i for g in groups for i in g['params']]
    entries, steps = {}, set()
    for pos, i in enumerate(ids):
        st = sd['state'].get(i)
        if st is not None:
            entries[pos] = (st['exp_avg'], st['exp_avg_sq'])
            steps.add(int(float(st['step'])))
    if len(steps) > 1:
        raise ValueError('the checkpoint\'s tensors have different step counts %s; one count serves all tensors here' % sorted(steps))
    return (steps.pop() if steps else 0), entries, groups[0]


_LOADED = set()


def _load_kernels(dev):
    """Launch both kernels once per device over an empty chunk list and scratch blocks, so that a captured step is never
    their first launch (the first launch loads the kernel, which a stream under capture may refuse)."""
    if dev in _LOADED:
        return
    lib = _lib.load()
    blk = torch.zeros(32, dtype=torch.float64, device=dev)             # hyper [0:5], counters [8:10], status [16:24]
    ws = torch.zeros(lib.vc_optim_ws_bytes(0), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.vc_optim_step(None, 0, None, 0, -1.0, None, 0, blk.data_ptr(), blk[8:].data_ptr(), blk[16:].data_ptr(), 0,
                                     ws.data_ptr(), ws.numel(), ops._stream()), 'vc_optim_step')
    _LOADED.add(dev)


class _Binding:
    """One device segment table of an optimizer and what fills it: the gradient addresses go through `slots` pinned copies of
    the table, each guarded by an event, and reach the device by an asynchronous copy only when an address changed."""

    def __init__(self, opt, guards, slots):
        self.opt = opt
        n = len(opt.all_params)
        self.host = torch.zeros((slots, max(n, 1), _SEG_WORDS), dtype=torch.int64).pin_memory()
        self.host_np = self.host.numpy()
        self.host_np[:, :n] = opt._seg_rows[None]
        self.dev = torch.zeros((max(n, 1), _SEG_WORDS), dtype=torch.int64, device=opt.device)
        self.events, self.slot, self.staged = [None] * slots, 0, None
        self.guards = [g for g in guards]                  # (kept alive: the kernels read them)
        words = []
        for g in self.guards:
            if not (g.is_cuda and g.dtype == torch.int32 and g.is_contiguous()):
                raise ValueError('a guard is a contiguous CUDA int32 tensor, got %s %s' % (g.device, g.dtype))
            words += [g.data_ptr() + 4 * i for i in range(g.numel())]
        if len(words) > MAX_GUARDS:
            raise ValueError('at most %d guard words, got %d' % (MAX_GUARDS, len(words)))
        self.n_guards, self.guard_ptrs = len(words), _lib.host_ptrs(words)

    def set_grads(self, grads):
        """grads: one tensor or None per entry of opt.all_params."""
        opt = self.opt
        ptrs = tuple(0 if g is None else g.data_ptr() for g in grads)
        if ptrs == self.staged:
            return
        for g, p in zip(grads, opt.all_params):
            if g is not None and not (g.is_cuda and g.dtype == torch.float32 and g.is_contiguous() and g.numel() == p.numel()
                                      and g.device == opt.device):
                raise ValueError('a gradient is a contiguous fp32 tensor of its parameter\'s size on %s, got %s %s %s'
                                 % (opt.device, g.device, g.dtype, tuple(g.shape)))
        slot = self.slot
        self.slot = (slot + 1) % len(self.events)
        ev = self.events[slot]
        if ev is not None and not ev.query():
            ev.synchronize()                               # (a whole ring back: only when the GPU is far behind)
        n = len(ptrs)
        self.host_np[slot, :n, 1] = np.array(ptrs, dtype=np.uint64).view(np.int64) if n else 0
        self.dev.copy_(self.host[slot], non_blocking=True)
        if not torch.cuda.is_current_stream_capturing():
            # (under capture the copy becomes a node of the graph, re-reading this slot on every replay: a captured step's
            #  binding has one slot and stages once)
            ev = torch.cuda.Event()
            ev.record()
            self.events[slot] = ev
        self.staged = ptrs
        for i, a in enumerate(ptrs[:len(opt.params)]):
            if a:
                opt._seen[i] = True

    def launch(self, max_norm):
        opt = self.opt
        _lib.check(_lib.load().vc_optim_step(self.dev.data_ptr(), len(opt.all_params), opt._chunks.data_ptr(), opt._n_chunks,
                                             -1.0 if max_norm is None else float(max_norm), self.guard_ptrs, self.n_guards,
                                             opt._hyper.data_ptr(), opt._counters.data_ptr(), opt._status.data_ptr(),
                                             opt.max_ctas, opt._ws.data_ptr(), opt._ws.numel(), ops._stream()), 'vc_optim_step')


class FusedAdamOneCycle:
    """Adam with true weight decay and gradient-norm clipping over fp32 CUDA parameters, presenting what the reference's
    loop and schedulers touch on OptimWrapper: `lr`, `mom`, `beta`, `wd`, `param_groups`, `step`, `zero_grad`, `state_dict`,
    `load_state_dict`.

    params: a list of parameters (one group) or [non-BatchNorm parameters, BatchNorm parameters] (the reference's two
    groups); parameters with requires_grad=False are left out.  norm_only: tensors whose gradients count in the total norm
    (clip_grad_norm_ runs over model.parameters()) but which this optimizer does not update.  guards: device int32 tensors
    the eager step() reads; a non-zero word makes that step a skipped one.  max_ctas: cap of both grids (0: one CTA per
    chunk); the result does not depend on it.

    `state[p]['exp_avg']` / `['exp_avg_sq']` are views of two flat fp32 buffers the optimizer owns."""

    HYPER_SLOTS = 8

    def __init__(self, params, lr=3e-3, wd=0.0, betas=(0.9, 0.99), eps=1e-8, norm_only=(), guards=(), max_ctas=0):
        params = list(params)
        groups = [list(g) for g in params] if params and isinstance(params[0], (list, tuple)) else [params, []]
        if len(groups) != 2:
            raise ValueError('one parameter list, or the two groups [non-BatchNorm, BatchNorm]; got %d groups' % len(groups))
        self.groups = [[p for p in g if p.requires_grad] for g in groups]
        self.params = self.groups[0] + self.groups[1]
        self.norm_only = [p for p in norm_only if p.requires_grad]
        self.all_params = self.params + self.norm_only
        if not self.params:
            raise ValueError('no trainable parameter')
        if len({id(p) for p in self.all_params}) != len(self.all_params):
            raise ValueError('a parameter appears twice')
        self.device = self.params[0].device
        for p in self.all_params:
            if not (p.is_cuda and p.dtype == torch.float32 and p.device == self.device and p.is_contiguous()):
                raise ValueError('FusedAdamOneCycle updates contiguous fp32 CUDA parameters on one device; got %s %s %s'
                                 % (p.device, p.dtype, tuple(p.shape)))
        self.max_ctas = int(max_ctas)
        lib = _lib.load()
        dev = self.device
        _load_kernels(dev)
        # m and v: two flat buffers, every tensor's slice starting on a 16-byte boundary
        numels = [p.numel() for p in self.params]
        starts = np.concatenate([[0], np.cumsum([(n + 3) // 4 * 4 for n in numels])]).astype(np.int64)
        self.exp_avg_flat = torch.zeros(int(starts[-1]), dtype=torch.float32, device=dev)
        self.exp_avg_sq_flat = torch.zeros(int(starts[-1]), dtype=torch.float32, device=dev)
        self.state = {}
        for p, s, n in zip(self.params, starts, numels):
            self.state[p] = {'exp_avg': self.exp_avg_flat[s:s + n].view_as(p), 'exp_avg_sq': self.exp_avg_sq_flat[s:s + n].view_as(p)}
        self._seen = [False] * len(self.params)            # tensors that have had a gradient: the ones with Adam state
        rows = [(p.data_ptr(), 0, self.state[p]['exp_avg'].data_ptr(), self.state[p]['exp_avg_sq'].data_ptr(), p.numel())
                for p in self.params] + [(0, 0, 0, 0, p.numel()) for p in self.norm_only]
        self._seg_rows = np.array(rows, dtype=np.uint64).view(np.int64).reshape(len(rows), _SEG_WORDS)
        chunks = chunk_list([p.numel() for p in self.all_params])
        self._n_chunks = int(chunks.shape[0])
        self._chunks = torch.from_numpy(chunks.view(np.uint8).reshape(-1).copy()).to(dev)
        self._ws = torch.zeros(lib.vc_optim_ws_bytes(self._n_chunks), dtype=torch.uint8, device=dev)
        self._status = torch.zeros(8, dtype=torch.float64, device=dev)          # vc_optim_status, 64 bytes
        self._counters = torch.zeros(2, dtype=torch.int64, device=dev)          # applied (t), skipped
        self._hyper = torch.zeros(5, dtype=torch.float64, device=dev)
        self._hyper_host = torch.zeros((self.HYPER_SLOTS, 5), dtype=torch.float64).pin_memory()
        self._hyper_ev, self._hyper_slot, self._hyper_dirty = [None] * self.HYPER_SLOTS, 0, True
        self._lr, self._mom, self._beta, self._eps, self._wd = float(lr), float(betas[0]), float(betas[1]), float(eps), float(wd)
        self._pending_max_norm = None
        self._eager = _Binding(self, guards, 4)
        self._param_ids = frozenset(id(p) for p in self.all_params)
        _LIVE.add(self)

    @classmethod
    def from_model(cls, model, wd, lr=3e-3, betas=(0.9, 0.99), **kwargs):
        """The optimizer build_optimizer makes for OPTIMIZER adam_onecycle / adam_cosin (wd = WEIGHT_DECAY, true_wd, bn_wd)."""
        groups, rest = leaf_param_groups(model)
        return cls(groups, lr=lr, wd=wd, betas=betas, norm_only=rest, **kwargs)

    # ---- hyper-parameters (OptimWrapper's properties) ------------------------------------------------------------
    def _set(self, name, val):
        if isinstance(val, (list, tuple)):
            val = val[-1]
        val = float(val)
        if val != getattr(self, name):
            setattr(self, name, val)
            self._hyper_dirty = True

    lr = property(lambda self: self._lr, lambda self, v: self._set('_lr', v))
    mom = property(lambda self: self._mom, lambda self, v: self._set('_mom', v))
    beta = property(lambda self: self._beta, lambda self, v: None if v is None else self._set('_beta', v))
    wd = property(lambda self: self._wd, lambda self, v: self._set('_wd', v))

    @property
    def param_groups(self):
        """torch.optim.Adam's groups as OptimWrapper leaves them (weight_decay 0: the decay is applied outside Adam)."""
        return [dict(params=g, lr=self._lr, betas=(self._mom, self._beta), eps=self._eps, weight_decay=0, amsgrad=False,
                     maximize=False, foreach=None, capturable=False, differentiable=False, fused=None) for g in self.groups]

    def stage_hyper(self):
        """Send lr / mom / beta / eps / wd to the device if one changed: one asynchronous copy from a pinned ring slot."""
        if not self._hyper_dirty:
            return
        slot = self._hyper_slot
        self._hyper_slot = (slot + 1) % self.HYPER_SLOTS
        ev = self._hyper_ev[slot]
        if ev is not None and not ev.query():
            ev.synchronize()
        self._hyper_host[slot].copy_(torch.tensor([self._lr, self._mom, self._beta, self._eps, self._wd], dtype=torch.float64))
        self._hyper.copy_(self._hyper_host[slot], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._hyper_ev[slot] = ev
        self._hyper_dirty = False

    # ---- the step -------------------------------------------------------------------------------------------------
    def owns(self, ids):
        """The ids of `ids` (id(parameter)) this optimizer updates or counts in its norm."""
        return self._param_ids & ids

    def clip_grad_norm(self, max_norm):
        """Record `max_norm` for the next step() (what clip_grad_norm_ before optimizer.step() means); nothing runs."""
        self._pending_max_norm = float(max_norm)

    def bind(self, guards=()):
        """A segment table of its own for a captured step: -> binding with set_grads(grads per all_params) and
        launch(max_norm).  guards: device int32 tensors; a non-zero word makes the step a skipped one."""
        return _Binding(self, guards, 1)

    def step(self, max_norm=_UNSET):
        """Clip to `max_norm` (None: no clipping; not given: what clip_grad_norm recorded, else None), decay, Adam — over
        every parameter's current .grad, which is left unmodified.  No host read, two launches."""
        if max_norm is _UNSET:
            max_norm = self._pending_max_norm
        self._pending_max_norm = None
        self._eager.set_grads([p.grad for p in self.all_params])
        self.stage_hyper()
        self._eager.launch(max_norm)

    def zero_grad(self, set_to_none=True):
        for p in self.all_params:
            if set_to_none:
                p.grad = None
            elif p.grad is not None:
                p.grad.zero_()

    @property
    def last_total_norm(self):
        """Device float64 scalar: the total gradient norm of the last step (clip_grad_norm_'s return value)."""
        return self._status[0]

    def applied_steps(self):
        """Steps applied so far (Adam's t).  Reads the device."""
        return int(self._counters[0].item())

    def skipped_steps(self):
        """Steps skipped by the guard so far.  Reads the device."""
        return int(self._counters[1].item())

    # ---- checkpoints: torch.optim.Adam's layout, as the reference's checkpoint_state stores it ---------------------
    def state_dict(self):
        t = self.applied_steps()
        # (copies: a checkpoint is a snapshot, and torch's load_state_dict keeps tensors that already have the right type)
        entries = {i: (self.state[p]['exp_avg'].clone(), self.state[p]['exp_avg_sq'].clone())
                   for i, p in enumerate(self.params) if self._seen[i]}
        return pack_state_dict(self.param_groups, t, entries)

    def load_state_dict(self, sd):
        t, entries, g0 = unpack_state_dict(sd, [len(g) for g in self.groups])
        self.exp_avg_flat.zero_()
        self.exp_avg_sq_flat.zero_()
        self._seen = [i in entries for i in range(len(self.params))]
        for i, (m, v) in entries.items():
            self.state[self.params[i]]['exp_avg'].copy_(m)
            self.state[self.params[i]]['exp_avg_sq'].copy_(v)
        self._counters[0] = t
        self.lr, self.mom, self.beta = g0['lr'], g0['betas'][0], g0['betas'][1]
        self._set('_eps', g0['eps'])
