"""Training-mode forward (batch-statistics BN) + full backward of ``Darknet`` on the GPU against the REFERENCE model's
own autograd (tests/golden/make_golden.py section 7: reference Darknet in train(), CPU fp32, loss = sum(p * G)/100).

Precision: operands, activations and activation gradients are bf16 (fp32 accumulate / fp32 parameter gradients),
the reference is fp32 end to end -- so the comparison is statistical per parameter tensor: cosine similarity of the
sampled gradient entries and ratio of norms.  Tolerances are stated below; they bound the bf16 path, they are not the
north_star's 1e-4 (unreachable with 8-bit mantissas, DESIGN.md section 5)."""
import os

import numpy as np
import pytest
import torch

from builders import small_train_model
from helpers import GOLDEN, init_darknet_weights

pytestmark = pytest.mark.gpu


def test_train_forward_backward_vs_reference_autograd():
    g = np.load(os.path.join(GOLDEN, "darknet_train_golden.npz"), allow_pickle=True)
    m = small_train_model()
    x = torch.from_numpy(g["x"]).cuda()
    ps = m(x)
    assert isinstance(ps, list) and len(ps) == 3
    for k, p in enumerate(ps):
        want = g["p%d" % k]
        assert tuple(p.shape) == want.shape and p.requires_grad
        err = np.abs(p.detach().cpu().numpy() - want)
        scale = np.abs(want).max()
        # measured: a torch graph with bf16 operand rounding at the same points differs from the fp32 reference by the
        # same 1.5-2.6 % rms (train-mode BN on a random-weight 75-layer net amplifies rounding noise)
        assert err.max() <= 0.2 * scale and np.sqrt((err ** 2).mean()) <= 4e-2 * scale, (k, err.max(), scale)
    loss = sum((p * torch.from_numpy(g["g%d" % k]).cuda()).sum() for k, p in enumerate(ps)) / 100.0
    assert abs(float(loss.detach()) - float(g["loss"])) <= 0.15 * max(1.0, abs(float(g["loss"])))
    loss.backward()
    names = [str(n) for n in g["names"]]
    params = dict(m.named_parameters())
    assert set(names) == set(params)
    cos_all, ratio_all = [], []
    for name, norm, idx, smp in zip(names, g["norms"], g["sample_idx"], g["samples"]):
        grad = params[name].grad
        assert grad is not None, name
        got = grad.reshape(-1)[torch.from_numpy(idx.astype(np.int64)).cuda()].float().cpu().numpy()
        smp = smp.astype(np.float64)
        cos = float((got * smp).sum() / (np.linalg.norm(got) * np.linalg.norm(smp) + 1e-30))
        cos_all.append(cos)
        ratio_all.append(float(grad.float().norm()) / (float(norm) + 1e-30))
    cos_all, ratio_all = np.array(cos_all), np.array(ratio_all)
    big = np.array([n.endswith("Conv2d.weight") for n in names])
    # Gradient direction decorrelates smoothly with depth (0.997 at the heads -> ~0.8 at the stem): every layer's
    # PReLU-derivative mask flips where the 2 % forward noise crosses zero.  Norms are preserved to a few percent.
    # The tight wiring check is test_mini_graph_* below; this one guards the full graph statistically.
    idx = {n: i for i, n in enumerate(names)}
    for head in ("module_list.105.Conv2d.weight", "module_list.93.Conv2d.weight", "module_list.81.Conv2d.weight"):
        assert cos_all[idx[head]] >= 0.985, (head, cos_all[idx[head]])
    assert cos_all[big].min() >= 0.65 and np.median(cos_all[big]) >= 0.75, (cos_all[big].min(), np.median(cos_all[big]))
    # bf16 rounding noise, amplified by 75 layers of train-mode BN, moves the stem layers' gradient norms by several
    # percent against the fp32 reference
    assert np.all(np.abs(ratio_all[big] - 1) <= 0.15), ratio_all[big]
    assert np.median(np.abs(ratio_all[big] - 1)) <= 0.02
    bnp = np.array([("BatchNorm2d" in n) or n.endswith("Conv2d.bias") for n in names])
    # BN vectors of the stem layers are the noisiest quantities of the whole graph against the fp32 reference (few
    # elements, deepest back-propagation path): bf16 rounding moves single entries by > 20 %, the bulk stays within a few
    # percent.  Between identical runs they do not move at all (tests/test_determinism_gpu.py).
    assert np.median(cos_all[bnp]) >= 0.75 and np.all(np.abs(ratio_all[bnp] - 1) <= 0.35)
    assert np.median(np.abs(ratio_all[bnp] - 1)) <= 0.05
    # running statistics followed nn.BatchNorm2d (momentum 0.1, unbiased variance)
    assert np.allclose(m.module_list[0].BatchNorm2d.running_mean.cpu().numpy(), g["rm0"], rtol=2e-2, atol=2e-3)
    assert np.allclose(m.module_list[0].BatchNorm2d.running_var.cpu().numpy(), g["rv0"], rtol=2e-2, atol=2e-3)
    assert np.allclose(m.module_list[75].BatchNorm2d.running_mean.cpu().numpy(), g["rm75"], rtol=5e-2, atol=2e-2)


def test_mini_graph_eval_and_train_vs_reference():
    """19-block graph with every structural feature of yolov3.cfg (stride 2, shortcuts, route alias, upsample, concat
    with a doubly-consumed source, two heads): eval forward, train forward and ALL gradients vs the reference model."""
    import rotate_yolov3_b200 as pkg
    from helpers import mini_cfg
    g = np.load(os.path.join(GOLDEN, "mini_train_golden.npz"))
    m = pkg.Darknet(mini_cfg(64, 48), {"context_factor": 1.0}, arc="default")
    init_darknet_weights(m, seed=77)
    m = m.cuda()
    x = torch.from_numpy(g["x"]).cuda()
    m.eval()
    with torch.no_grad():
        io, pe = m(x)
    for k, p in enumerate(pe):
        want = g["pe%d" % k]
        assert float(np.abs(p.cpu().numpy() - want).max()) <= 2e-2 * np.abs(want).max()
    m.train()
    ps = m(x)
    for k, p in enumerate(ps):
        want = g["p%d" % k]
        err = np.abs(p.detach().cpu().numpy() - want)
        assert err.max() <= 3e-2 * np.abs(want).max() and np.sqrt((err ** 2).mean()) <= 6e-3 * np.abs(want).max()
    loss = sum((p * torch.from_numpy(g["g%d" % k]).cuda()).sum() for k, p in enumerate(ps)) / 10.0
    loss.backward()
    worst = 1.0
    slope_scale = max(abs(float(g["grad:" + n])) for n, _ in m.named_parameters() if n.endswith("activation.weight"))
    for name, prm in m.named_parameters():
        want = torch.from_numpy(g["grad:" + name]).cuda().reshape(-1).double()
        got = prm.grad.reshape(-1).double()
        if name.endswith("activation.weight"):
            # one scalar per block = a sum over the whole activation with heavy cancellation: bounded against the
            # largest slope gradient of the net
            assert abs(float(got) - float(want)) <= 0.3 * slope_scale, (name, float(got), float(want))
            continue
        cos = float((got * want).sum() / (got.norm() * want.norm() + 1e-30))
        ratio = float(got.norm() / (want.norm() + 1e-30))
        worst = min(worst, cos)
        # measured: 0.9999 at the heads, 0.989 at the stem (13 bf16 layers of accumulated rounding noise), norms +-5 %
        tol = 0.95 if "BatchNorm2d" in name else 0.98
        assert cos >= tol and abs(ratio - 1) <= 0.06, (name, cos, ratio)
    assert worst >= 0.95


def test_sgd_step_reduces_a_toy_loss():
    """three SGD steps on a fixed batch with a quadratic loss on the heads: the loss must go down"""
    m = small_train_model()
    opt = torch.optim.SGD(m.parameters(), lr=2e-4, momentum=0.0)
    x = torch.rand(2, 3, 128, 160, device="cuda")
    losses = []
    for _ in range(4):
        opt.zero_grad(set_to_none=True)
        ps = m(x)
        loss = sum((p ** 2).mean() for p in ps)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0], losses


def test_device_prefetcher_hands_out_the_batches_in_order():
    """parallel.DevicePrefetcher: batch i+1 is copied on a side stream while batch i is consumed; values and order kept"""
    from rotate_yolov3_b200.parallel import DevicePrefetcher
    dev = torch.device("cuda", 0)
    pf = DevicePrefetcher(dev)
    hosts = [(torch.full((4, 3, 64, 64), float(i)).pin_memory(), torch.arange(7.0).pin_memory() + i) for i in range(5)]
    pf.put(*hosts[0])
    acc = torch.zeros((), device=dev)
    for i in range(5):
        x, t = pf.get()
        if i + 1 < 5:
            pf.put(*hosts[i + 1])
        assert x.device == dev and float(x.mean()) == float(i) and float(t[0]) == float(i)
        acc = acc + x.sum() * 0 + t.sum()
    assert float(acc) == sum(float(h[1].sum()) for h in hosts)
