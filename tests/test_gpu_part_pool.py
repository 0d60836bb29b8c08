"""GPU tests of the part-score RoI pooling (rules R1-R4 of csrc/part_pool.cu): forward and part-map gradient against the
reference's own float64 results (tests/golden/part_pool_ref.npz) and, at VirConv-T's full size, against
oracle/part_pool.py; bit-identical repeats on dirty memory with torch's deterministic flag on and off; CUDA-graph
capture of forward + backward; the drop-in `obtain_conf_preds`; the argument checks."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import part_pool as o
from oracle import part_pool_golden as g

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-4      # of the largest magnitude: the sample coordinates round in fp32
CASES = ('A', 'B', 'C', 'D')


def golden():
    return np.load(os.path.join(os.path.dirname(__file__), 'golden', 'part_pool_ref.npz'))


def _mb():
    sys.path.insert(0, os.path.join(ROOT, 'profiles'))
    import microbench_part_pool as mb
    return mb


@pytest.fixture()
def det_flag():
    saved = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(saved)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _run(parts, rois, grad, S, offsets, scale):
    from virconv_b200.part_pool import part_pool
    p = parts.detach().clone().requires_grad_()
    out = part_pool(p, rois, S, offsets, scale)
    (d,) = torch.autograd.grad(out, [p], grad.view(-1, 1))
    return out.detach(), d


@pytest.mark.parametrize('case', CASES)
def test_matches_reference_golden(lib_built, case):
    z = golden()
    S, off, scale, _ = g.geom_of(z, case)
    dev = torch.device('cuda')
    t = {k: torch.from_numpy(z[f'{case}.{k}']).to(dev) for k in ('parts', 'rois', 'g')}
    out, d = _run(t['parts'], t['rois'], t['g'], S, off, scale)
    assert out.shape == (t['rois'].shape[0] * t['rois'].shape[1], 1)
    assert _rel(out.cpu(), z[f'{case}.out']) < TOL
    assert _rel(d.cpu(), z[f'{case}.dparts']) < TOL
    assert np.array_equal(d.cpu().numpy() != 0, z[f'{case}.dparts'] != 0)      # zero exactly where no tap lands
    assert _rel(out.cpu(), z[f'f32.{case}.out']) < TOL and _rel(d.cpu(), z[f'f32.{case}.dparts']) < TOL


@pytest.mark.parametrize('N', [160, 50])
def test_full_size_matches_oracle(lib_built, N):
    mb = _mb()
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(N)
    parts = torch.randn(mb.MAP, device=dev, generator=gen)
    rois = mb.kitti_rois(2, N, 7 + N, dev)
    grad = torch.randn(2 * N, device=dev, generator=gen)
    out, d = _run(parts, rois, grad, mb.S, mb.OFFSETS, mb.SCALE)
    pn, rn, gn = parts.cpu().numpy(), rois.cpu().numpy(), grad.cpu().numpy()
    assert _rel(out.cpu(), o.forward(pn, rn, mb.S, mb.OFFSETS, mb.SCALE)) < TOL
    assert _rel(d.cpu(), o.backward(rn, gn, pn.shape, mb.S, mb.OFFSETS, mb.SCALE)) < TOL
    # and against the reference's control flow over torch on the same GPU (its rotation is a matmul: fp32, not TF32)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        p = parts.clone().requires_grad_()
        ref = mb.reference_arm(p, rois)
        (dref,) = torch.autograd.grad(ref, [p], grad.view(-1, 1))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    assert _rel(out.cpu(), ref.detach().cpu()) < TOL and _rel(d.cpu(), dref.cpu()) < TOL


def _collide_rois(dev):
    r = _mb().kitti_rois(2, 160, 5, dev)
    r[:, :] = r[:, :1].clone()                      # every RoI of a scene the same box: every tap collides
    r[1, :, 0:2] = torch.tensor([35.2, 0.0], device=dev)
    return r


def test_bit_identical_repeats(lib_built, det_flag):
    mb = _mb()
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(3)
    parts = torch.randn(mb.MAP, device=dev, generator=gen)
    grad = torch.randn(2 * 160, device=dev, generator=gen)
    for rois in (mb.kitti_rois(2, 160, 11, dev), _collide_rois(dev)):
        first = None
        for flag in (False, True, False, True):
            torch.use_deterministic_algorithms(flag)
            for _ in range(2):
                junk = torch.full((64 << 20,), float('nan'), device=dev)        # leaves dirty blocks in the cache
                del junk
                out, d = _run(parts, rois, grad, mb.S, mb.OFFSETS, mb.SCALE)
                if first is None:
                    first = (out, d)
                    assert torch.isfinite(d).all() and (d != 0).any()
                else:
                    assert torch.equal(out, first[0]) and torch.equal(d, first[1])


def test_deterministic_flag_forward_backward(lib_built, det_flag):
    from virconv_b200.part_pool import part_pool
    mb = _mb()
    dev = torch.device('cuda')
    torch.use_deterministic_algorithms(True)
    parts = torch.randn(mb.MAP, device=dev, requires_grad=True)
    rois = mb.kitti_rois(2, 160, 13, dev)
    out = part_pool(parts, rois, mb.S, mb.OFFSETS, mb.SCALE)
    (out * torch.arange(out.numel(), device=dev).view(-1, 1)).sum().backward()
    assert parts.grad is not None and parts.grad.shape == parts.shape


def test_cuda_graph_replays_equal_eager(lib_built):
    from virconv_b200.part_pool import part_pool
    mb = _mb()
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(21)
    parts = torch.randn(mb.MAP, device=dev, generator=gen).requires_grad_()
    rois = mb.kitti_rois(2, 160, 17, dev)
    grad = torch.randn(2 * 160, 1, device=dev, generator=gen)

    def step():     # detached outputs: no autograd graph (and no grad accumulator of `parts`) outlives a step
        out = part_pool(parts, rois, mb.S, mb.OFFSETS, mb.SCALE)
        (d,) = torch.autograd.grad(out, [parts], grad)
        return out.detach(), d

    eager = [t.clone() for t in step()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for _ in range(3):
        for t in outs:
            t.fill_(float('nan'))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(outs[0], eager[0]) and torch.equal(outs[1], eager[1])


def test_drop_in_method(lib_built, monkeypatch):
    from virconv_b200 import part_pool as pp
    mb = _mb()
    dev = torch.device('cuda')
    head = types.SimpleNamespace(grid_offsets=[0.0, 40.0], featmap_stride=0.4)
    parts = torch.randn(mb.MAP, device=dev)
    rois = mb.kitti_rois(2, 50, 19, dev)
    got = pp.obtain_conf_preds(head, parts, rois)
    assert got.shape == (100, 1)
    assert torch.equal(got, pp.part_pool(parts, rois, 7, (0.0, 40.0), 1 / 0.4))
    assert _rel(got.cpu(), o.forward(parts.cpu().numpy(), rois.cpu().numpy(), 7, (0.0, 40.0), 1 / 0.4)) < TOL
    empty = pp.obtain_conf_preds(head, parts, rois[:, :0])
    assert empty.shape == (0,) and empty.dtype == torch.float32 and empty.is_cuda
    calls = []
    monkeypatch.setattr(pp, '_reference_obtain_conf_preds', lambda s, a, b: calls.append(b) or 'ref')
    r = rois.clone().requires_grad_()
    assert pp.obtain_conf_preds(head, parts, r) == 'ref' and calls[0] is r
    with pytest.raises(ValueError, match='49 channels'):
        pp.obtain_conf_preds(head, parts[:, :36], rois)


def test_argument_checks(lib_built):
    from virconv_b200.part_pool import MAX_ROIS, part_pool
    dev = torch.device('cuda')
    parts = torch.zeros(2, 49, 20, 16, device=dev)
    rois = torch.zeros(2, 10, 7, device=dev)
    part_pool(parts, rois, 7, (0.0, 40.0), 2.5)
    bad = [(parts.double(), rois, 7), (parts, rois.double(), 7), (parts[:, :36], rois, 7), (parts, rois[..., :6], 7),
           (parts, rois[:1], 7), (parts, torch.zeros(2, MAX_ROIS + 1, 7, device=dev), 7), (parts, rois, 1),
           (torch.zeros(2, 289, 4, 4, device=dev), rois, 17)]
    for p, r, s in bad:
        with pytest.raises(ValueError, match='obtain_conf_preds'):
            part_pool(p, r, s, (0.0, 40.0), 2.5)
    # a non-contiguous part map and RoIs with extra columns
    wide = torch.zeros(2, 10, 9, device=dev)
    t = torch.randn(2, 20, 16, 49, device=dev).permute(0, 3, 1, 2)
    out = part_pool(t, wide, 7, (0.0, 40.0), 2.5)
    assert torch.equal(out, part_pool(t.contiguous(), wide[..., :7].contiguous(), 7, (0.0, 40.0), 2.5))
