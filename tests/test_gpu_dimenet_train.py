"""DimeNet++ training on the device (nb200_dimenet_train_grads through DimeNetEnergyFn): parameter gradients of energy and force losses against
float64 autograd of the oracle with create_graph=True, at the config's sizes and at the benchmark batch, the training-mode outputs against
eval mode, and a few Adam steps."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from test_dimenet_emu import _fixture, _models  # noqa: E402
from test_dimenet_train_emu import _check, _oracle_grads, _seeds  # noqa: E402

pytestmark = pytest.mark.gpu


class D:
    def __init__(self, z, pos, batch):
        self.z, self.pos, self.batch = z, pos, batch


def _data(z, pos, batch):
    return D(torch.as_tensor(z).long().cuda(), torch.as_tensor(pos).float().cuda(), torch.as_tensor(batch).long().cuda())


def _device_grads(net, data, c, v):
    net.train()
    net.zero_grad(set_to_none=True)
    e, f = net(data)
    loss = e.new_zeros(())
    if c is not None:
        loss = loss + (c.float().cuda() * e).sum()
    if v is not None:
        loss = loss + (v.float().cuda() * f).sum()
    loss.backward()
    return {k: (p.grad if p.grad is not None else torch.zeros_like(p)).double().cpu() for k, p in net.named_parameters()}


@pytest.mark.parametrize("with_forces", [False, True])
def test_gpu_gradients_against_oracle(with_forces):
    net, ora = _models(num_blocks=6, latent=50)
    net = net.cuda()
    z, pos, batch = _fixture([0, 1, 2])
    c, v = _seeds(3, len(z), 7)
    v = v if with_forces else None
    _check(_device_grads(net, _data(z, pos, batch), c, v), _oracle_grads(ora, z, pos, batch, c, v), 221)


def test_gpu_force_only_gradients():
    net, ora = _models(num_blocks=6, latent=50)
    net = net.cuda()
    z, pos, batch = _fixture([4, 8])
    _, v = _seeds(2, len(z), 8)
    _check(_device_grads(net, _data(z, pos, batch), None, v), _oracle_grads(ora, z, pos, batch, None, v), 221, zero_ok={"regr_or_cls_nn.6.bias"})


def test_gpu_benchmark_batch_masked_seeds():
    """256 synthetic molecules, c and v nonzero on 4 of them: the full-batch gradients equal the oracle's on those 4 molecules alone."""
    from nabladft_b200.synth import synth_batch

    s = synth_batch(0, 256)
    ptr = s["mol_ptr"]
    batch = np.repeat(np.arange(256), np.diff(ptr))
    chosen = [0, 97, 180, 255]
    c_all = torch.zeros(256, dtype=torch.float64)
    v_all = torch.zeros(len(s["z"]), 3, dtype=torch.float64)
    c4, _ = _seeds(4, 1, 9)
    gen = torch.Generator().manual_seed(10)
    zs, ps, bs, vs = [], [], [], []
    for k, m in enumerate(chosen):
        a, b = ptr[m], ptr[m + 1]
        c_all[m] = c4[k]
        v_all[a:b] = torch.randn(b - a, 3, generator=gen, dtype=torch.float64)
        zs.append(s["z"][a:b]); ps.append(s["pos"][a:b]); bs.append(np.full(b - a, k)); vs.append(v_all[a:b])
    net, ora = _models(num_blocks=6, latent=50)
    net = net.cuda()
    got = _device_grads(net, _data(s["z"], s["pos"], batch), c_all, v_all)
    ref = _oracle_grads(ora, np.concatenate(zs), np.concatenate(ps), np.concatenate(bs), c4, torch.cat(vs))
    _check(got, ref, 221)


def test_gpu_training_outputs_equal_eval_outputs():
    net, _ = _models(num_blocks=6, latent=50)
    net = net.cuda()
    data = _data(*_fixture([0, 1, 2, 3]))
    e_eval, f_eval = net.eval()(data)
    net.train()
    e_tr, f_tr = net(data)
    assert e_tr.requires_grad and f_tr.requires_grad
    assert torch.equal(e_tr.detach(), e_eval) and torch.equal(f_tr.detach(), f_eval)


def test_gpu_adam_steps_lower_l1_loss():
    net, ora = _models(num_blocks=6, latent=50)
    net = net.cuda()
    z, pos, batch = _fixture([0, 1, 2, 3, 4, 5])
    data = _data(z, pos, batch)
    e_ref, f_ref, _ = ora(torch.as_tensor(z).long(), torch.as_tensor(pos).double(), torch.as_tensor(batch).long())
    e_t = (e_ref + 0.5).float().cuda()  # targets the untrained model misses
    f_t = (0.9 * f_ref).float().cuda()
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    losses = []
    net.train()
    for _ in range(6):
        opt.zero_grad()
        e, f = net(data)
        loss = (e - e_t).abs().mean() + (f - f_t).abs().mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0], losses
