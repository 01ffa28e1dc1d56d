"""Inception-v3, DenseNet-161 and SqueezeNet 1.0 / 1.1 on CPU: train-mode logits, every parameter gradient and the
running statistics of the fp32 composites against float64 torchvision with the same weights, and the tie rule of torch's
max-pool that the GPU max-pool checks rely on."""
import copy

import pytest
import torch
import torch.nn.functional as F
import torchvision

from distributeddeeplearning_b200 import models, ops


def _train_step_vs_float64(name, size, batch=2, **kw):
    """One train-mode forward / backward of the repo's model (fp32 composite), of torchvision in fp32 and of torchvision
    in float64 on the same weights and input (Inception-v3: main + 0.4 * aux loss).  Returns [(what, repo, fp32
    torchvision, float64 torchvision)] for the logits, every parameter gradient and every running statistic."""
    torch.manual_seed(0)
    m = models.get_model(name, **kw)
    t32 = getattr(torchvision.models, name)(**kw, **({"init_weights": False} if name.startswith("inception") else {}))
    t32.load_state_dict(m.state_dict())
    # PyTorch's CPU convolution loses accuracy in its backward with channels-last weights (torchvision with the same
    # weight layout gives bit-identical gradients, a few % off float64 on some BN parameters): contiguous copies make the
    # composite as accurate as fp32 torchvision
    with torch.no_grad():
        for p in m.parameters():
            p.data = p.data.contiguous()
    t64 = copy.deepcopy(t32).double()
    x = torch.randn(batch, 3, size, size)
    y = torch.arange(batch) * 7 % 1000
    outs = []
    for net, xent, xx in ((m, ops.softmax_cross_entropy, x), (t32, F.cross_entropy, x), (t64, F.cross_entropy, x.double())):
        net.train()
        o = net(xx)
        o = list(o) if isinstance(o, tuple) else [o]
        sum(w * xent(h, y) for w, h in zip((1.0, 0.4), o)).backward()
        outs.append(o)
    rows = [(f"logits {i}", *(o[i].detach() for o in outs)) for i in range(len(outs[0]))]
    ps = [dict(net.named_parameters()) for net in (m, t32, t64)]
    rows += [(k, *(d[k].grad for d in ps)) for k in ps[2]]
    bs = [dict(net.named_buffers()) for net in (m, t32, t64)]
    rows += [(k, *(d[k] for d in bs)) for k, b in bs[2].items() if b.dtype.is_floating_point]
    return rows


def _rel(a, b):
    return float((a.double() - b).norm() / max(float(b.norm()), 1e-30))


def _check(rows, tol):
    """Each tensor of the repo's model within ``tol`` (relative, in norm) of float64, or within twice the error of fp32
    torchvision where that is larger: a few BN gradients of a randomly initialised net cancel down to where fp32
    rounding alone is a few % of them."""
    assert len(rows) > 0
    for k, a, b, ref in rows:
        assert a is not None and _rel(a, ref) <= max(tol, 2 * _rel(b, ref)), (k, _rel(a, ref), _rel(b, ref))


def test_inception_v3_train_logits_aux_gradients_and_running_stats_equal_float64_torchvision():
    # 299 is the smallest input the aux head takes (its 5x5 conv needs a 17x17 map before its 5/3 average pool)
    rows = _train_step_vs_float64("inception_v3", 299, dropout=0.0)
    assert [r[0] for r in rows[:2]] == ["logits 0", "logits 1"] and any(r[0].endswith("running_var") for r in rows)
    _check(rows, 1e-3)


@pytest.mark.parametrize("name", ["squeezenet1_0", "squeezenet1_1"])
def test_squeezenet_train_gradients_equal_float64_torchvision(name):
    _check(_train_step_vs_float64(name, 96, dropout=0.0), 1e-4)


def test_densenet161_train_gradients_and_running_stats_equal_float64_torchvision():
    rows = _train_step_vs_float64("densenet161", 64)
    assert any(r[0].endswith("running_mean") for r in rows)
    _check(rows, 1e-3)


def test_torch_max_pool_routes_ties_to_the_first_maximum_in_row_major_order():
    """The GPU max-pool checks compare the kernels' arg-max with torch's float64 CPU max-pool on inputs full of ties;
    both must take the first maximum of a window in row-major order (the kernels' strict `>` compare)."""
    x = torch.zeros(1, 1, 6, 6, dtype=torch.float64)
    x[0, 0, 0, 2] = x[0, 0, 1, 0] = x[0, 0, 1, 2] = 1.0           # window (0, 0): three maxima
    x[0, 0, 4, 4] = x[0, 0, 5, 5] = -1.0                          # ceil-mode window (2, 2): 2x2 taps, two at 0
    for ceil in (False, True):
        xr = x.clone().requires_grad_(True)
        y, idx = F.max_pool2d(xr, 3, 2, 0, ceil_mode=ceil, return_indices=True)
        y.backward(torch.ones_like(y))
        assert y.shape[-1] == (3 if ceil else 2)
        assert idx[0, 0, 0, 0] == 2                              # (0, 2) comes before (1, 0) and (1, 2)
        assert idx[0, 0, 1, 1] == 2 * 6 + 2                      # all-zero window (2..4, 2..4): its first tap
        if ceil:
            assert idx[0, 0, 2, 2] == 4 * 6 + 5                  # (4, 5) is the first 0 of rows 4..5, columns 4..5
        assert float(xr.grad[0, 0, 1, 0]) == 0.0 and float(xr.grad[0, 0, 1, 2]) == 0.0 and float(xr.grad[0, 0, 0, 2]) > 0
