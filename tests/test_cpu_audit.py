"""CPU tests of the float64 references the step audit (test_gpu_step_audit.py) holds every layer to: BatchNorm1d + ReLU
forward / backward from given statistics against torch.nn.BatchNorm1d under float64 autograd, the bf16 bound against
torch's round-to-nearest-even, and the conv's autograd gradients against the sums they stand for."""
import numpy as np
import pytest
import torch

from oracle import audit


@pytest.mark.parametrize('training,adversarial', [(True, False), (False, False), (False, True), (True, True)],
                         ids=['True', 'False', 'eval-adversarial', 'train-adversarial'])
def test_bn_relu_matches_torch_batchnorm(training, adversarial):
    """adversarial: the BatchNorm state of the step audit's running-statistics cases — gamma negative on every third
    channel, running statistics of the scale of x with the mean shifted by half a standard deviation, and one channel with
    running_var = 0 (eps alone under the square root)"""
    torch.manual_seed(0)
    n, c, eps, mom = 300, 16, 1e-3, 0.01
    x = (torch.randn(n, c, dtype=torch.float64) * torch.linspace(0.2, 3.0, c, dtype=torch.float64)
         + torch.linspace(-1, 1, c, dtype=torch.float64))
    bn = torch.nn.BatchNorm1d(c, eps=eps, momentum=mom).double()
    with torch.no_grad():
        bn.weight.copy_(torch.linspace(0.5, 1.5, c))
        bn.bias.copy_(torch.linspace(-0.3, 0.3, c))
        bn.running_mean.copy_(torch.linspace(-0.1, 0.1, c))
        bn.running_var.copy_(torch.linspace(0.5, 1.5, c))
        if adversarial:
            bn.weight[::3] *= -1
            sd = x.std(0)
            bn.running_mean.copy_(x.mean(0) + 0.5 * sd * torch.where(torch.arange(c) % 2 == 0, 1.0, -1.0).double())
            bn.running_var.copy_(sd ** 2 * torch.linspace(0.5, 2.0, c, dtype=torch.float64))
            bn.running_var[5] = 0.0
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    bn.train(training)
    xt = x.clone().requires_grad_(True)
    y = torch.relu(bn(xt))
    dy = torch.randn(n, c, dtype=torch.float64)
    y.backward(dy)

    mean, invstd, var, var_u = audit.batch_stats(x, eps)
    if not training:
        mean, invstd = rm0, 1.0 / torch.sqrt(rv0 + eps)
    else:
        rm, rv = audit.running_update(rm0, rv0, mean, var_u, mom)
        assert torch.allclose(rm, bn.running_mean, rtol=1e-14, atol=1e-14)
        assert torch.allclose(rv, bn.running_var, rtol=1e-14, atol=1e-14)
    yr = audit.bn_relu_fwd(x, mean, invstd, bn.weight.detach(), bn.bias.detach())
    assert torch.allclose(yr, y.detach(), rtol=1e-12, atol=1e-12)
    dx, dg, db = audit.bn_relu_bwd(dy, x, mean, invstd, bn.weight.detach(), bn.bias.detach(), training)
    assert torch.allclose(dx, xt.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(dg, bn.weight.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(db, bn.bias.grad, rtol=1e-10, atol=1e-12)
    # an explicit mask equal to the float64 one gives the same result
    m = audit.relu_mask(x, mean, invstd, bn.weight.detach(), bn.bias.detach())
    assert torch.equal(audit.bn_relu_bwd(dy, x, mean, invstd, bn.weight.detach(), bn.bias.detach(), training, m)[0], dx)


def test_bf16_bound_accepts_rounding_and_rejects_one_ulp_more():
    torch.manual_seed(1)
    r = torch.cat([torch.randn(5000, dtype=torch.float64) * 10.0 ** torch.randint(-3, 3, (5000,)).double(),
                   torch.tensor([0.0, 1e-12, -1e-12], dtype=torch.float64)])
    got = r.float().bfloat16()
    assert audit.bound_excess(got, r) <= 1.0                  # round to nearest: half an ulp < 2^-8 |r|
    # a result two bf16 ulps off (a lost or doubled term of that size) does not pass
    big = r.abs() > 1e-3 * r.abs().max()
    ulp = torch.ldexp(torch.ones_like(r), torch.frexp(r)[1] - 8)
    off = got.double() + torch.where(big, 2 * ulp * torch.sign(r), torch.zeros_like(r))
    assert audit.bound_excess(off, r) > 1.0
    assert audit.bound_excess(r, r) == 0.0
    # rel = 0: a plain absolute bound relative to the largest element
    assert audit.bound_excess(r + 0.5e-6 * r.abs().max(), r, rel=0.0) == pytest.approx(0.5)


def test_conv_grads_are_the_rulebook_sums():
    rng = np.random.default_rng(2)
    n_in, n_out, K, ci, co = 40, 30, 5, 3, 4
    nbr = rng.integers(-1, n_in, (K, n_out)).astype(np.int32)
    inp = torch.from_numpy(rng.normal(size=(n_in, ci)))
    w = torch.from_numpy(rng.normal(size=(co, K, ci)))
    dout = torch.from_numpy(rng.normal(size=(n_out, co)))
    out = audit.conv(inp, w, torch.from_numpy(nbr), n_out)
    din, dw = audit.conv_grads(inp, w, torch.from_numpy(nbr), n_out, dout)
    want_out = np.zeros((n_out, co))
    want_din = np.zeros((n_in, ci))
    want_dw = np.zeros((co, K, ci))
    for k in range(K):
        for o in range(n_out):
            i = nbr[k, o]
            if i < 0:
                continue
            want_out[o] += w[:, k, :].numpy() @ inp[i].numpy()
            want_din[i] += dout[o].numpy() @ w[:, k, :].numpy()
            want_dw[:, k, :] += np.outer(dout[o].numpy(), inp[i].numpy())
    assert np.allclose(out.numpy(), want_out, rtol=1e-12, atol=1e-12)
    assert np.allclose(din.numpy(), want_din, rtol=1e-12, atol=1e-12)
    assert np.allclose(dw.numpy(), want_dw, rtol=1e-12, atol=1e-12)
    assert audit.conv_grads(inp, w, torch.from_numpy(nbr), n_out, dout, need_din=False)[0] is None
