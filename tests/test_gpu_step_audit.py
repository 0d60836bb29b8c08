"""The plan executor's bf16 (or fp32) runs, every layer audited against float64: the training step (BatchNorm from the batch
statistics), the frozen-BatchNorm step of fine-tuning (model.train(False), forward and backward from the running
statistics) and the test-time forward (running statistics, no backward) of VirConv-L and of VirConv-T over the ROT_NUM = 3
copies packed along x, eager and replayed from graph.GraphedForward.

After one forward (+ backward), each layer's float64 reference is fed that layer's own operands as the run left them in its
arena (executor._Run.slot / layer_forward / layer_backward), so every check is of one kernel in isolation and errors do not
compound from layer to layer.  With exact operands only the fp32 accumulation order is left, so the tolerances are tight
enough to see one 128-row tile lost or counted twice; a sensitivity check inside the test proves that for every layer's
weight gradient at its own size.

Checked per layer: the conv output x, the BN statistics, y and its bf16 shadow, the running buffers, d_gamma / d_beta, the
BN backward's dx (bf16), the weight gradient (with the kernel's own operands: bf16 input shadow and dxb for the tensor-core
wgrad, fp32 input and dx for the fp32 one) and, per feature slot, the final input gradient as the float64 sum of its
consumers' contributions (dgrads, concat column routing, layer-discard scatter, the published loss gradient).

With running statistics the BN state comes from _adversarial_bn (running statistics of a real batch, rescaled and shifted;
negative gamma; a channel with running_var = 0), and two more sensitivity checks per layer prove that y's bound sees a tail
that takes the batch statistics of x, or ignores the sign of gamma."""
import copy
import math
import time

import numpy as np
import pytest
import torch

from oracle import audit
from oracle import xbatch as oxb
from oracle.gather2d import representatives
from oracle.testing import fill_module, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG_T = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
TILE = 128
TOL = dict(x=1e-4, mean=1e-5, invstd=1e-5, y=1e-5, running=1e-6, dgamma=1e-4, dbeta=1e-4, wgrad=3e-5, slot=1e-4, sums=1e-5,
           loss=1e-6, pub=1e-6)
FP32_REL = 2.0 ** -22         # the bound of an fp32 result (fp32 mode): a few ulps, plus 1e-6 of the largest element
TC_DGRAD = ('conv_dgrad_tc', 'conv_dgrad_scatter_tc', 'conv_dgrad_gather2d_tc')
OP_CBR, OP_CAT, OP_DISCARD = 4, 5, 6
SENS = 100                    # a sensitivity reference must miss y's bound by this factor at least


def _rows(t):
    """valid rows of a run view: the device count in static mode, else all"""
    return int(t.num_rows.item()) if hasattr(t, 'num_rows') else t.shape[0]


class _Audit:
    """worst measured value of every check, printed at the end of a case"""

    def __init__(self, case):
        self.case, self.worst = case, {}

    def note(self, name, value, limit, where):
        v = float(value)
        self.worst[name] = max(self.worst.get(name, 0.0), v)
        assert v <= limit, (self.case, name, where, v, limit)

    def least(self, name, value, floor, where):
        v = float(value)
        self.worst[name] = min(self.worst.get(name, math.inf), v)
        assert v > floor, (self.case, name, where, v, floor)

    def report(self, t0):
        print('\n[step audit] %s (%.1f s): ' % (self.case, time.time() - t0)
              + ', '.join('%s %.3g' % kv for kv in sorted(self.worst.items())))


def _capture(monkeypatch):
    """Every executor run of the step, with the gradient autograd hands each published tensor (ext_grads) and the int32
    input coordinates it was given (the caller's tensor: a graph's input buffer holds those of the last replay)."""
    from virconv_b200 import executor
    runs, real = [], executor.run_plan

    def run_plan(plan, feats, coords, *a, **kw):
        run, res = real(plan, feats, coords, *a, **kw)
        run.coords0 = coords
        run.pub_grads = {}
        for name, (f, *_) in res.items():
            if f.requires_grad:
                f.register_hook(lambda g, name=name, run=run: run.pub_grads.__setitem__(name, g.detach().clone()))
        runs.append(run)
        return run, res

    monkeypatch.setattr(executor, 'run_plan', run_plan)
    return runs


def _bn_state(model):
    return {id(m): (m.running_mean.clone(), m.running_var.clone(), int(m.num_batches_tracked.item()))
            for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)}


def _step(model, bd, loss_fn, runs, det=False):
    """forward + loss + backward with the conv launches recorded -> (loss, out, timing records, BN buffers before)"""
    from virconv_b200 import executor, ops
    for p in model.parameters():
        p.grad = None
    bn0 = _bn_state(model)
    runs.clear()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    executor.timing_start()
    try:
        out = model(bd)
        loss = loss_fn(out)
        loss.backward()
    finally:
        recs = executor.timing_stop()
        torch.use_deterministic_algorithms(prev)
    torch.cuda.synchronize()
    assert int(ops.tc_error_flag(DEV).item()) == 0
    assert runs and all(r.deterministic_bytes()[0] == det for r in runs)
    return float(loss.detach()), out, recs, bn0


def _forward(model, bd, runs):
    """a test-time forward (torch.no_grad()) with the conv launches recorded -> (out, timing records, BN buffers before)"""
    from virconv_b200 import executor, ops
    bn0 = _bn_state(model)
    runs.clear()
    executor.timing_start()
    try:
        with torch.no_grad():
            out = model(bd)
    finally:
        recs = executor.timing_stop()
    torch.cuda.synchronize()
    assert int(ops.tc_error_flag(DEV).item()) == 0
    return out, recs, bn0


def _adversarial_bn(model, bd, seed):
    """A BatchNorm state that exercises the eval-mode tail, on `model` (on the device): fill_module, then the running
    statistics of one training-mode forward of the batch `bd` (momentum 1, on a copy of the model: a plan caches the
    momentum it was built with), so that y is centred and about half the ReLUs pass; then per channel running_var times
    a factor in [0.5, 2] and running_mean moved by half a standard deviation either way; gamma negated on a third of the
    channels; and on one channel per layer running_var = 0, eps alone under the square root (its gamma scaled by
    sqrt(eps / var), so that channel keeps the scale of its output and the later layers' inputs stay in range)."""
    fill_module(model, seed)
    model.to(DEV)
    tmp = copy.deepcopy(model).train()
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)]
    tmp_bns = [m for m in tmp.modules() if isinstance(m, torch.nn.BatchNorm1d)]
    for m in tmp_bns:
        m.momentum = 1.0
    with torch.no_grad():
        tmp(dict(bd))
    torch.cuda.synchronize()
    rng = np.random.default_rng(seed)
    with torch.no_grad():
        for m, t in zip(bns, tmp_bns):
            c = m.num_features
            var, mean = t.running_var.double().cpu().numpy(), t.running_mean.double().cpu().numpy()
            assert np.all(np.isfinite(var)) and np.all(np.isfinite(mean))
            rv = var * rng.uniform(0.5, 2.0, c)
            rm = mean + rng.choice([-0.5, 0.5], c) * np.sqrt(var)
            g = m.weight.double().cpu().numpy()
            g[rng.choice(c, (c + 1) // 3, replace=False)] *= -1
            dead = int(rng.integers(c))
            g[dead] *= math.sqrt(m.eps / (rv[dead] + m.eps))
            rv[dead] = 0.0
            m.running_var.copy_(torch.from_numpy(rv))
            m.running_mean.copy_(torch.from_numpy(rm))
            m.weight.copy_(torch.from_numpy(g))
    return model


def _dgrad_ref(run, li, lb, w, n_in, n_out, nbr, rb):
    """float64 input-gradient contribution of layer li's dgrad [n_in, c_in], from the operands its kernel read"""
    tc = lb['dgrad'] in TC_DGRAD
    d = (lb['dxb'] if tc else lb['dx'])
    assert d is not None, (li, lb['dgrad'])
    d = d[:n_out].double()
    if lb['sums'] is None:
        return audit.conv_grads(torch.zeros(n_in, w.shape[2], device=DEV), w, nbr, n_out, d)[0], None
    # gather form over [dout; S]: S (the per-pixel sums of dout at each pixel's lowest row) as the kernel read it, and
    # checked itself against float64 sums of dout
    i_in = run.plan.rb_keys[rb][2]
    idx, shape = run.indices(i_in)
    rep = torch.from_numpy(representatives(idx[:n_in].cpu().numpy(), shape)).to(DEV)
    s_ref = torch.zeros_like(d).index_add_(0, rep, d)
    is_rep = rep == torch.arange(n_in, device=DEV)
    s = lb['sums'][:n_in].double()
    err = audit.bound_excess(s[is_rep], s_ref[is_rep]) if tc else rel_err(s[is_rep], s_ref[is_rep]) / TOL['sums']
    K, c = w.shape[1], w.shape[1] // 2
    din = d @ w[:, c, :]
    for k in range(K):
        if k == c:
            continue
        j = nbr[K - 1 - k, :n_in].long()
        i = torch.nonzero(is_rep & (j >= 0)).squeeze(1)
        din.index_add_(0, i, s[j[i]] @ w[:, k, :])
    return din, err


def _audit_run(run, bn0, A, static, bn_stats='batch', backward=True):
    """every layer of one run, then (backward) every feature slot's final gradient.  bn_stats: 'batch' (training: BN from
    the statistics of x, running buffers updated) or 'running' (eval / frozen BatchNorm: from the running buffers, which
    stay as they were); backward: a backward ran after the forward."""
    assert bn_stats in ('batch', 'running')
    running = bn_stats == 'running'
    plan = run.plan
    bf16 = run.precision == 'bf16'
    contrib = {}
    kinds = []
    if running:
        assert not plan.discards       # StVD discards layers only in training: the reference's eval forward keeps every row

    def add(slot, rows, val):
        if slot not in contrib:
            contrib[slot] = torch.zeros(rows, plan.f_channels[slot], dtype=torch.float64, device=DEV)
        contrib[slot][:val.shape[0]] += val

    for li, (conv, bn) in enumerate(plan.layers):
        where = (li, plan.layers[li][0].indice_key)
        lf, lb = run.layer_forward(li), run.layer_backward(li)
        X, Y = run.slot(lf['in_slot']), run.slot(lf['out_slot'])
        nbr = run.rulebook(lf['rb'])[0]
        x = lf['x']
        n, n_in = _rows(x), _rows(X['f32'] if X['f32'] is not None else X['bf16'])
        co, ci = conv.out_channels, conv.in_channels
        W = conv.weight.detach().reshape(co, -1, ci).double()
        Wb = conv.weight.detach().reshape(co, -1, ci).bfloat16().double()
        kinds += [(lb['fwd'], li)]
        if backward:
            kinds += [(lb['wgrad'], li)] + ([(lb['dgrad'], li)] if lb['dgrad'] else [])
        # ---- forward
        tc_fwd = lb['fwd'] == 'conv_fwd_tc'
        assert tc_fwd == bf16, where
        inp = X['bf16'] if tc_fwd else X['f32']
        x_ref = audit.conv(inp[:n_in], Wb if tc_fwd else W, nbr, n)
        A.note('x', rel_err(x[:n], x_ref) / TOL['x'], 1, where)
        mean_b, invstd_b, var, var_u = audit.batch_stats(x[:n], bn.eps)
        rm0, rv0, nbt0 = bn0[id(bn)]
        if running:
            mean, invstd = rm0.double(), 1.0 / torch.sqrt(rv0.double() + bn.eps)
        else:
            mean, invstd = mean_b, invstd_b
        st = lf['stats']
        A.note('mean', rel_err(st[2], mean) / TOL['mean'], 1, where)
        A.note('invstd', rel_err(st[3], invstd) / TOL['invstd'], 1, where)
        gamma, beta = bn.weight.detach(), bn.bias.detach()
        y_ref = audit.bn_relu_fwd(x[:n], mean, invstd, gamma, beta)
        # sensitivity (running statistics): a tail that took the batch statistics of x, or |gamma| (the sign of gamma lost
        # where it decides the ReLU), must be far outside y's bound
        sens = {}
        if running:
            sens = {'sens_batch_stats': audit.bn_relu_fwd(x[:n], mean_b, invstd_b, gamma, beta),
                    'sens_abs_gamma': audit.bn_relu_fwd(x[:n], mean, invstd, gamma.abs(), beta)}
        if Y['f32'] is not None:
            A.note('y', rel_err(Y['f32'][:n], y_ref) / TOL['y'], 1, where)
            for name, y_alt in sens.items():
                A.least(name, rel_err(y_alt, y_ref) / TOL['y'], SENS, where)
            if bf16:
                assert torch.equal(Y['bf16'][:n], Y['f32'][:n].bfloat16()), where
        elif bf16:
            A.note('yb', audit.bound_excess(Y['bf16'][:n], y_ref), 1, where)
            for name, y_alt in sens.items():
                A.least(name, audit.bound_excess(y_alt, y_ref), SENS, where)
        if static:
            for t in (Y['f32'], Y['bf16']):
                assert t is None or bool((t[n:] == 0).all()), where
        if running:
            assert torch.equal(bn.running_mean, rm0) and torch.equal(bn.running_var, rv0), where
            assert int(bn.num_batches_tracked.item()) == nbt0, where
        else:
            rm, rv = audit.running_update(rm0, rv0, mean, var_u, bn.momentum)
            A.note('running', max(rel_err(bn.running_mean, rm), rel_err(bn.running_var, rv)) / TOL['running'], 1, where)
            assert int(bn.num_batches_tracked.item()) == nbt0 + 1, where
        if not backward:
            continue
        # ---- backward: BN
        dy = lb['dy']
        if dy is None:        # the caller's own gradient tensor: a published slot no other layer reads
            dy = next(run.pub_grads[nm] for nm, s, _ in plan.published if s == lf['out_slot'])
        dy = dy[:n]
        x64 = x[:n].double()
        active = x64 * st[0].double() + st[1].double() > 0     # the kernel's own ReLU decision: sign of fmaf(x, scale, shift)
        dx_ref, dg_ref, db_ref = audit.bn_relu_bwd(dy, x[:n], st[2], st[3], gamma, beta, not running, active)
        A.note('dgamma', rel_err(bn.weight.grad, dg_ref) / TOL['dgamma'], 1, where)
        A.note('dbeta', rel_err(bn.bias.grad, db_ref) / TOL['dbeta'], 1, where)
        if bf16 and (lb['dxb'] is not None or not running):     # (the frozen-BN step's fp32 wgrad and dgrads read dx only)
            A.note('dxb', audit.bound_excess(lb['dxb'][:n], dx_ref), 1, where)
        if lb['dx'] is not None:
            A.note('dx', audit.bound_excess(lb['dx'][:n], dx_ref, rel=FP32_REL), 1, where)
        if static:
            for t in (lb['dx'], lb['dxb']):
                assert t is None or bool((t[n:] == 0).all()), where
        # ---- weight gradient, with the operands of the kernel that ran
        if lb['wgrad'] == 'conv_wgrad_tc':
            a, d = X['bf16'], lb['dxb']
        else:
            assert lb['wgrad'] == 'conv_wgrad', where
            a, d = X['f32'], lb['dx']
        assert a is not None and d is not None, where
        dw_ref = audit.conv_grads(a[:n_in], W, nbr, n, d[:n], need_din=False)[1]
        dw = conv.weight.grad.reshape(co, -1, ci)
        A.note('wgrad', rel_err(dw, dw_ref) / TOL['wgrad'], 1, where)
        # sensitivity: the reference without its middle 128-row tile must be far outside the tolerance
        t = (n + TILE - 1) // TILE // 2
        d_cut = d[:n].clone()
        d_cut[t * TILE:(t + 1) * TILE] = 0
        dw_cut = audit.conv_grads(a[:n_in], W, nbr, n, d_cut, need_din=False)[1]
        A.least('tile_shift', rel_err(dw_cut, dw_ref), 5 * TOL['wgrad'], where)
        # ---- input gradient contribution
        if lb['dgrad'] is not None:
            din, s_err = _dgrad_ref(run, li, lb, Wb if lb['dgrad'] in TC_DGRAD else W, n_in, n, nbr, lf['rb'])
            if s_err is not None:
                A.note('pixel_sums', s_err, 1, where)
            add(lf['in_slot'], n_in, din)
        else:             # (the network input, or a layer discard of it: no parameter gradient flows there)
            assert lf['in_slot'] in plan.no_grad, where
    if not backward:
        return kinds
    # ---- published gradients (ext_grads) and the routing ops, in reverse plan order
    for name, slot, iset in plan.published:
        g = run.pub_grads.get(name)
        if g is not None:
            add(slot, _rows(run.slot(slot)['f32']), g[:_rows(run.slot(slot)['f32'])].double())
    keeps = dict(zip((op for _, op in sorted(plan.discards)), run.kept_rows()))
    for op in reversed(range(len(plan.rows_i))):
        r = plan.rows_i[op]
        if r[0] == OP_CAT and r[4] in contrib:
            a, b, o = r[2], r[3], r[4]
            ca = plan.f_channels[a]
            add(a, contrib[o].shape[0], contrib[o][:, :ca])
            add(b, contrib[o].shape[0], contrib[o][:, ca:])
        elif r[0] == OP_DISCARD and r[19] in contrib and r[18] != 0:
            keep = keeps[op]
            k = _rows(keep)
            xs = r[18]
            n_x = _rows(run.slot(xs)['f32'])
            v = torch.zeros(n_x, plan.f_channels[xs], dtype=torch.float64, device=DEV)
            v[keep[:k].long()] = contrib[r[19]][:k]
            add(xs, n_x, v)
    # ---- every slot's final gradient
    checked = 0
    for slot in range(1, plan.n_f):
        g = run.slot(slot)['grad']
        if g is None:
            continue
        cat_out = [r for r in plan.rows_i if r[0] == OP_CAT and r[4] == slot]
        if cat_out and run.query(1, cat_out[0][2])[5] == run.query(1, slot)[5]:
            continue          # the concat's buffer is its inputs' gradients (column slices), which are checked as those
        rows = _rows(g)
        ref = contrib.get(slot, torch.zeros(rows, g.shape[1], dtype=torch.float64, device=DEV))
        A.note('slot_grad', rel_err(g[:rows], ref[:rows]) / TOL['slot'], 1, ('slot', slot))
        if static:
            assert bool((g[rows:] == 0).all()), ('slot', slot)
        checked += 1
    assert checked > 0
    return kinds


def _check_kinds(kinds, recs):
    """the kernel each layer's reference assumed is the one the timing records saw launched"""
    assert sorted(kinds) == sorted((k, l) for k, l, _ in recs)


# ------------------------------------------------------------------------------------------------ VirConv-L
def _model(precision):
    from virconv_b200.backbone import VirConvL8x
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision=precision)
    fill_module(m, 666)
    return m.to(DEV).train()


def _batch(ids, training=True):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, training=training)    # the bench's density: 16384 LiDAR + 80000 virtual points, 40000 voxels
    bd = {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(DEV),
          'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib}
    if b.aug_param is not None:                      # (training only)
        bd['aug_param'] = torch.from_numpy(b.aug_param.copy())
    return bd


def _named(out):
    named = dict(out['multi_scale_3d_features'])
    named['out'] = out['encoded_spconv_tensor']
    return named


def _loss(out):
    from virconv_b200.graph import masked_mean
    return sum(masked_mean(t) for t in _named(out).values())


def _audit_l(model, bd, runs, case, det=False, static=False, min_tiles=0, bn_stats='batch'):
    t0 = time.time()
    A = _Audit(case)
    loss, out, recs, bn0 = _step(model, bd, _loss, runs, det)
    assert len(runs) == 1
    run = runs[0]
    kinds = _audit_run(run, bn0, A, static, bn_stats)
    _check_kinds(kinds, recs)
    # the loss: float64 masked means of the published fp32 features; their gradient is 1 / (rows * c) on the valid rows
    ref = 0.0
    for name, slot, _ in run.plan.published:
        f = run.slot(slot)['f32']
        n = _rows(f)
        ref += float(f[:n].double().mean())
        g = run.pub_grads[name].double()
        A.note('pub_grad', rel_err(g[:n], torch.full_like(g[:n], 1.0 / (n * f.shape[1]))) / TOL['pub'], 1, name)
        assert bool((g[n:] == 0).all()), name
    A.note('loss', abs(loss - ref) / max(1.0, abs(ref)) / TOL['loss'], 1, 'loss')
    n1 = _rows(run.layer_forward(0)['x'])
    assert (n1 + TILE - 1) // TILE >= min_tiles, n1
    A.report(t0)


def test_step_audit_bf16_exact(lib_built, monkeypatch):
    """(a) the bench step: bf16, exact mode, the bench batch (two scenes, ~80 000 voxels)"""
    runs = _capture(monkeypatch)
    _audit_l(_model('bf16'), _batch([0, 1]), runs, 'bf16 exact')


def test_step_audit_bf16_static(lib_built, monkeypatch):
    """(b) static mode run eagerly: capacity-sized inputs with NaN past the count, device row counts; zero tails"""
    from virconv_b200 import executor, ops
    runs = _capture(monkeypatch)
    model = _model('bf16')
    batch = _batch([0, 1])
    with torch.no_grad():
        model(dict(batch))
    caps = executor.measured_caps(executor.last_run(model), 1.3, 256)
    n = batch['voxel_features'].shape[0]
    cap0 = (int(n * 1.25) + 255) // 256 * 256
    vf = torch.full((cap0, batch['voxel_features'].shape[1]), float('nan'), device=DEV)
    vc = torch.full((cap0, 4), -1.0, device=DEV)
    vf[:n] = batch['voxel_features']
    vc[:n] = batch['voxel_coords']
    spec = executor.StaticSpec(torch.tensor([n], dtype=torch.int32, device=DEV), caps, torch.zeros(1, dtype=torch.int32, device=DEV))
    bd = {'voxel_features': vf, 'voxel_coords': vc, 'batch_size': 2, 'calib': batch['calib'], 'aug_param': batch['aug_param'],
          'virconv_static': spec, 'virconv_proj': ops.projection_params(batch['calib'], batch['aug_param'], 2, DEV)}
    _audit_l(model, bd, runs, 'bf16 static', static=True)
    assert int(spec.overflow.item()) == 0


def test_step_audit_bf16_deterministic(lib_built, monkeypatch):
    """(c) the bench step under torch.use_deterministic_algorithms: tile-ordered BN sums, chunked wgrad, gather-form dgrad"""
    runs = _capture(monkeypatch)
    _audit_l(_model('bf16'), _batch([0, 1]), runs, 'bf16 deterministic', det=True)


def test_step_audit_bf16_eight_scenes(lib_built, monkeypatch):
    """(d) eight scenes at the bench's density: >= 2 500 layer-1 tiles, so the dynamic tile scheduler's look-ahead runs at
    its full depth and every CTA of the persistent kernels takes many tiles"""
    runs = _capture(monkeypatch)
    _audit_l(_model('bf16'), _batch(list(range(8))), runs, 'bf16 eight scenes', min_tiles=2500)


def test_step_audit_fp32_exact(lib_built, monkeypatch):
    """(e) fp32 precision: the fp32 kernels, the same audit with fp32 results in place of bf16 roundings"""
    runs = _capture(monkeypatch)
    _audit_l(_model('fp32'), _batch([0, 1]), runs, 'fp32 exact')


# ------------------------------------------------------------------------------------------------ VirConv-L, running statistics
def _running_model(precision):
    """VirConv-L in eval mode with the adversarial BN state (running statistics of scenes 2 and 3)"""
    from virconv_b200.backbone import VirConvL8x
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision=precision)
    return _adversarial_bn(m, _batch([2, 3]), 666).eval()


@pytest.mark.parametrize('precision', ['bf16', 'fp32'])
def test_eval_audit_exact(lib_built, monkeypatch, precision):
    """(g) the test-time forward of VirConv-L, exact mode, on the bench batch: BN from the running statistics"""
    runs = _capture(monkeypatch)
    t0 = time.time()
    A = _Audit('eval %s exact' % precision)
    model = _running_model(precision)
    out, recs, bn0 = _forward(model, _batch([0, 1], training=False), runs)
    assert len(runs) == 1 and runs[0].static is None and not runs[0].training
    _check_kinds(_audit_run(runs[0], bn0, A, False, 'running', backward=False), recs)
    A.report(t0)


def test_eval_audit_bf16_static_graph(lib_built, monkeypatch):
    """(h) the same forward replayed from graph.GraphedForward (static mode, capacity-sized buffers, device row counts): the
    captured run's arena audited after one replay, zero tails.  (Which kernels a layer runs is checked by the eager cases:
    no timing records inside a capture.)"""
    from virconv_b200.graph import GraphedForward
    runs = _capture(monkeypatch)
    t0 = time.time()
    A = _Audit('eval bf16 static graph')
    model = _running_model('bf16')
    bn0 = _bn_state(model)
    fwd = GraphedForward(model, margin=1.3, grain=256)
    fwd(_batch([0, 1], training=False))
    torch.cuda.synchronize()
    assert fwd.recaptures == 1 and int(fwd.ovf_host.max()) == 0
    run = runs[-1]                    # the captured run: its arena belongs to the graph and holds the replay's results
    assert run.static is not None and not run.training
    kinds = _audit_run(run, bn0, A, True, 'running', backward=False)
    assert all(k == 'conv_fwd_tc' for k, _ in kinds)
    A.report(t0)


@pytest.mark.parametrize('precision', ['bf16', 'fp32'])
def test_step_audit_frozen_bn(lib_built, monkeypatch, precision):
    """(i) the fine-tuning step with frozen BatchNorm (model.train(False), forward and backward): the tensor-core forward
    with the eval tail, the fp32 weight gradient and dgrads (bf16), the eval branch of the BN backward"""
    runs = _capture(monkeypatch)
    _audit_l(_running_model(precision), _batch([0, 1], training=False), runs, 'frozen-BN %s' % precision,
             bn_stats='running')


# ------------------------------------------------------------------------------------------------ VirConv-T
def test_step_audit_virconv_t(lib_built, monkeypatch):
    """(f) one VirConv-T step as bench.py --model T runs it: two plans (LiDAR and virtual-point streams), StVD layer discards
    drawn on the device"""
    from virconv_b200 import scenes
    from virconv_b200.backbone import VirConv8x
    runs = _capture(monkeypatch)
    t0 = time.time()
    A = _Audit('VirConv-T bf16')
    m = VirConv8x(CFG_T, 8, [1408, 1600, 80], discard_mode='paper', discard_rng='device', precision='bf16')
    fill_module(m, 667)
    m.to(DEV).train()
    b = scenes.make_batch_mm([0, 1], 16384, 80000, 16000, training=True)
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param),
              stvd_seed=torch.tensor([1234], dtype=torch.int64, device=DEV))

    def tensors(out):
        ts = [out['encoded_spconv_tensor']]
        for grp in ('multi_scale_3d_features', 'multi_scale_3d_features_mm'):
            ts += [t for t in out[grp].values() if t is not None]
        return ts

    loss, out, recs, bn0 = _step(m, bd, lambda o: sum(t.features.mean() for t in tensors(o)), runs)
    assert len(runs) == 2 and any(r.plan.discards for r in runs)
    kinds = []
    for run in runs:
        for _, op in run.plan.discards:
            assert 0 < run.query(5, op)[1] < run.query(5, op)[3], op       # each discard dropped rows
        kinds += _audit_run(run, bn0, A, False)
    _check_kinds(kinds, recs)
    ref = sum(float(t.features.detach().double().mean()) for t in tensors(out))
    A.note('loss', abs(loss - ref) / max(1.0, abs(ref)) / TOL['loss'], 1, 'loss')
    A.report(t0)


def _named_t(out, s):
    """the LiDAR stream's split tensors of copy `s`, as VirConv8x's eval forward publishes them"""
    named = {k: out['multi_scale_3d_features' + s][k] for k in ('x_conv3', 'x_conv4')}
    named['out'] = out['encoded_spconv_tensor' + s]
    return named


@pytest.mark.parametrize('mode', ['exact', 'graph'])
def test_eval_audit_virconv_t_rot3(lib_built, monkeypatch, mode):
    """(j) bench.py's eval_rot3 workload: VirConv-T's test-time forward (bf16) over ROT_NUM = 3 copies of 40 000 voxels each.
    The LiDAR plan runs once over the copies packed along x into [81, 1600, 4 * 1408], the virtual-point plan once per copy;
    every layer of every run audited with the running statistics.  The packed input is oracle.xbatch.pack of the copies, and
    each copy's published x_conv3, x_conv4 and out are, bit for bit, oracle.xbatch.split of the packed run's slots.  exact:
    the eager forward; graph: one replay of graph.GraphedForward (static mode, zero tails)."""
    from virconv_b200 import parallel, scenes
    from virconv_b200.backbone import VirConv8x
    from virconv_b200.graph import GraphedForward
    runs = _capture(monkeypatch)
    t0 = time.time()
    A = _Audit('eval VirConv-T rot3 %s' % mode)
    m = VirConv8x(CFG_T, 8, [1408, 1600, 80], precision='bf16')
    tb = scenes.make_batch_mm([2, 3], 16384, 80000, 40000, training=True)
    sbd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in tb.arrays.items()}
    sbd.update(batch_size=tb.batch_size, calib=tb.calib, aug_param=torch.from_numpy(tb.aug_param.copy()))
    _adversarial_bn(m, sbd, 667).eval()
    R = 3
    b = scenes.make_batch_mm(parallel.shard_scene_ids(100, 0, 1, 2), 16384, 80000, 40000, training=False, rot_num=R)
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, transform_param=torch.from_numpy(b.transform_param.copy()))
    sfx = [''] + [str(i) for i in range(1, R)]
    static = mode == 'graph'
    if static:
        bn0 = _bn_state(m)
        fwd = GraphedForward(m, margin=1.3, grain=256)
        out = fwd(bd)
        torch.cuda.synchronize()
        assert fwd.recaptures == 1 and int(fwd.ovf_host.max()) == 0
        runs = runs[-(1 + R):]            # the captured runs, audited after the replay
    else:
        out, recs, bn0 = _forward(m, dict(bd), runs)
    assert len(runs) == 1 + R and all((r.static is not None) == static and not r.training for r in runs)
    lidar = runs[0]
    assert lidar.plan is m._plan_lidar() and all(r.plan is m._plan_mm() for r in runs[1:])
    kinds = []
    for run in runs:
        kinds += _audit_run(run, bn0, A, static, 'running', backward=False)
    if static:
        assert all(k == 'conv_fwd_tc' for k, _ in kinds)
    else:
        _check_kinds(kinds, recs)
    # the packed input: copy after copy, x moved by i * W
    W = m.sparse_shape[2]
    assert lidar.query(2, 0)[3:6] == [m.sparse_shape[0], m.sparse_shape[1], 4 * W]
    pf, pc, n = oxb.pack([bd['voxel_features' + s].cpu().numpy() for s in sfx],
                         [bd['voxel_coords' + s].int().cpu().numpy() for s in sfx],
                         [bd['voxel_features' + s].shape[0] for s in sfx], W)
    X0 = lidar.slot(0)['f32']
    assert _rows(X0) == n
    assert torch.equal(X0[:n].cpu(), torch.from_numpy(pf[:n])) and torch.equal(lidar.coords0[:n].cpu(), torch.from_numpy(pc[:n]))
    # each copy's published tensors: the oracle's split of the packed run's slots
    slots = {name: (slot, iset) for name, slot, iset in lidar.plan.published}
    for name in ('x_conv3', 'x_conv4', 'out'):
        slot, iset = slots[name]
        f = lidar.slot(slot)['f32']
        k = _rows(f)
        idx, shape = lidar.indices(iset)
        parts = oxb.split(f[:k].cpu().numpy(), idx[:k].cpu().numpy(), k, shape[2], R)
        assert sum(p[2] for p in parts) > 0, name
        for s, (wf, wi, wn) in zip(sfx, parts):
            t = _named_t(out, s)[name]
            rows = int(t.num_rows.item()) if static else t.features.shape[0]
            assert rows == wn, (name, s, rows, wn)
            assert list(t.spatial_shape) == [shape[0], shape[1], shape[2] // 4], (name, s)
            assert torch.equal(t.features[:rows].cpu(), torch.from_numpy(wf[:wn])), (name, s)
            assert torch.equal(t.indices[:rows].int().cpu(), torch.from_numpy(wi[:wn])), (name, s)
    A.report(t0)
