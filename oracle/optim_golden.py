"""Record what the reference's OWN optimizer path computes — `build_optimizer` / `build_scheduler` (tools/train_utils/
optimization/__init__.py: OptimWrapper.create over Adam, OneCycle) with torch's `clip_grad_norm_`, driven as
train_one_epoch drives them (train_utils.py:31, 50-52) — as tests/golden/optim_ref.npz.  Needs the reference's sources; the
fixture it writes is committed, so the tests need neither.  Everything runs on the CPU in float32, as the model trains.

The module tree (`golden_tree`) has what the group construction has to get right: conv-like and linear leaves, BatchNorm
leaves, a parent module that owns a parameter directly (the leaf flattening never visits it, so no group holds it, while
clip_grad_norm_ over model.parameters() still counts its gradient), a frozen leaf, and a leaf that never receives a
gradient (decayed by OptimWrapper.step, skipped by Adam).  The gradients are a seeded sequence (`golden_grads`), scaled so
that some steps clip at MAX_NORM and some do not.

    python -m oracle.optim_golden REFERENCE_ROOT [OUT_DIR]
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.nn as nn

SEED = 47
STEPS = 40
MAX_NORM = 10.0
CHECKPOINTS = (1, 10, 25, 40)
CFG = dict(OPTIMIZER='adam_onecycle', LR=0.01, WEIGHT_DECAY=0.01, MOMENTUM=0.9, MOMS=[0.95, 0.85], PCT_START=0.4, DIV_FACTOR=10,
           DECAY_STEP_LIST=[35, 45], LR_DECAY=0.1, LR_CLIP=0.0000001, LR_WARMUP=False, WARMUP_EPOCH=1, GRAD_NORM_CLIP=MAX_NORM)


class _Block(nn.Module):
    def __init__(self):
        super().__init__()
        self.scale = nn.Parameter(torch.ones(5))          # owned by a module with children
        self.fc = nn.Linear(8, 16)
        self.bn = nn.BatchNorm1d(16)


class _Tree(nn.Module):
    def __init__(self):
        super().__init__()
        self.stem = nn.Sequential(nn.Conv2d(3, 8, 3, bias=False), nn.BatchNorm2d(8), nn.ReLU())
        self.block = _Block()
        self.odd = nn.Linear(5, 7)
        self.frozen = nn.Linear(4, 4, bias=False)
        self.unused = nn.Linear(3, 5)                      # never receives a gradient
        self.head = nn.Linear(16, 1)
        self.frozen.weight.requires_grad = False


def golden_tree():
    from oracle.testing import fill_module
    m = _Tree()
    fill_module(m, SEED)
    return m


def grad_names(model):
    """The parameters that receive a gradient every step."""
    return [n for n, p in model.named_parameters() if p.requires_grad and not n.startswith('unused.')]


def golden_grads(model, step):
    """{name: float32 gradient} of iteration `step` (0-based): standard normal times 2.0 on every third step (total norm
    about 45: clipped at 10) and times 0.1 otherwise (about 2.3: not clipped)."""
    rng = np.random.default_rng([SEED, step])
    scale = 2.0 if step % 3 == 0 else 0.1
    shapes = {n: tuple(p.shape) for n, p in model.named_parameters()}
    return {n: (rng.standard_normal(shapes[n]) * scale).astype(np.float32) for n in grad_names(model)}


def make(reference_root):
    import virconv_b200.reference_env as renv
    renv.install(reference_root=reference_root)
    tools = os.path.join(reference_root, 'tools')
    if tools not in sys.path:
        sys.path.append(tools)
    from train_utils.optimization import build_optimizer, build_scheduler
    from torch.nn.utils import clip_grad_norm_
    cfg = renv.EasyDict(CFG)
    model = golden_tree()
    named = dict(model.named_parameters())
    name_of = {id(p): n for n, p in named.items()}
    opt = build_optimizer(model, cfg)
    sched, _ = build_scheduler(opt, total_iters_each_epoch=STEPS, total_epochs=1, last_epoch=-1, optim_cfg=cfg)
    out = {'group0': np.array([name_of[id(p)] for p in opt.param_groups[0]['params']]),
           'group1': np.array([name_of[id(p)] for p in opt.param_groups[1]['params']])}
    for n, p in named.items():
        out['init.' + n] = p.detach().numpy().copy()
    lr, mom, norm = [], [], []
    for it in range(STEPS):
        sched.step(it)
        lr.append(float(opt.lr))
        mom.append(float(opt.mom))
        for n, g in golden_grads(model, it).items():
            named[n].grad = torch.from_numpy(g.copy())
        norm.append(float(clip_grad_norm_(model.parameters(), cfg.GRAD_NORM_CLIP)))
        opt.step()
        opt.zero_grad()
        if it + 1 in CHECKPOINTS:
            for n, p in named.items():
                out['p.%d.%s' % (it + 1, n)] = p.detach().numpy().copy()
                st = opt.state.get(p)
                if st:
                    out['m.%d.%s' % (it + 1, n)] = st['exp_avg'].numpy().copy()
                    out['v.%d.%s' % (it + 1, n)] = st['exp_avg_sq'].numpy().copy()
    sd = opt.state_dict()
    out.update(lr=np.array(lr), mom=np.array(mom), total_norm=np.array(norm),
               sd_state_keys=np.array(sorted(sd['state']), dtype=np.int64),
               sd_steps=np.array([float(sd['state'][k]['step']) for k in sorted(sd['state'])]),
               sd_group0=np.array(sd['param_groups'][0]['params'], dtype=np.int64),
               sd_group1=np.array(sd['param_groups'][1]['params'], dtype=np.int64),
               sd_state_fields=np.array(sorted(sd['state'][sorted(sd['state'])[0]])),
               sd_betas=np.array(sd['param_groups'][0]['betas']), sd_weight_decay=np.array(sd['param_groups'][0]['weight_decay']))
    assert any(n > MAX_NORM for n in norm) and any(n < MAX_NORM for n in norm)
    return out


def main(argv):
    root = argv[1]
    out_dir = argv[2] if len(argv) > 2 else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')
    data = make(root)
    path = os.path.join(out_dir, 'optim_ref.npz')
    np.savez_compressed(path, **data)
    print('%s: %d arrays, %d bytes' % (path, len(data), os.path.getsize(path)))


if __name__ == '__main__':
    main(sys.argv)
