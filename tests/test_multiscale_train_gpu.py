"""Training at changing image and batch sizes (train.py --multi-scale, the short last batch of an epoch) from one
activation pool per model: every step of a cached plan gives the bits of a
freshly built plan -- heads, loss and items, every gradient, the BatchNorm running statistics and the parameters after
an SGD step -- a revisited shape builds no plan and allocates nothing, the pool grows only to the largest shape, and a
backward whose activations a forward of another shape overwrote raises.  Weights are random, so stale halos or padding
channels left by a larger shape would show; the poisoned runs fill the whole pool with NaN bytes before every step.
The reference model drops its plans and its pool before every step: a fresh plan in zeroed storage, the parent's
behaviour."""
import gc
import os

import pytest
import torch

import helpers
from builders import STEP_HYP, transfer_mask
from helpers import GOLDEN
from multiscale_cases import (collect, grid_bytes, images, pair, poison_pool, yolov3_small)  # noqa: F401 (collect: fixture)

pytestmark = pytest.mark.gpu
REF = os.path.join(GOLDEN, "reference_cfg")

# normalised [image, class, x, y, w, h, angle]; images 0..2 so that the short batch of 3 keeps every target
TARGETS = [[0, 0, 0.30, 0.40, 0.25, 0.08, 0.5], [1, 0, 0.70, 0.60, 0.30, 0.10, -0.9],
           [2, 0, 0.50, 0.50, 0.20, 0.07, 1.2], [0, 0, 0.20, 0.80, 0.22, 0.09, -0.3]]
# (batch, height, width): a shape, another, the first with a short batch, pool growth (which drops the cached plans),
# a smaller shape laid out in the grown pool, cached revisits
SEQ = [(4, 320, 320), (4, 192, 256), (3, 320, 320), (4, 416, 416), (4, 192, 256), (4, 416, 416), (4, 192, 256)]
LR = 1e-3


def _mini():
    import rotate_yolov3_b200 as pkg
    return pkg.Darknet(helpers.mini_cfg(64, 48), {"context_factor": 1.0}, arc="default")


def _se():
    import rotate_yolov3_b200 as pkg
    old = os.getcwd()
    os.chdir(REF)                   # the SE cfg names its anchor file relative to the reference root
    try:
        return pkg.Darknet("cfg/HRSC+/yolov3_512_se.cfg", {"context_factor": 1.0}, arc="default")
    finally:
        os.chdir(old)


def _m():
    from builders import m_model
    return m_model()


def _targets(b):
    return torch.tensor([t for t in TARGETS if t[0] < b]).cuda()


def _fresh(m):
    """drop every training plan and the pool: the next step builds its plan in zeroed storage"""
    m._tplan = None
    m._pools = {}


def _pool_bytes(m):
    return sum(p.nbytes for p in m._pools.values())


def _train_step(m, x, t, mask=None):
    """forward, compute_loss, backward, SGD; everything a step produces, on the host"""
    from rotate_yolov3_b200.loss import compute_loss
    for p, tr in zip(m.parameters(), mask or [True] * len(list(m.parameters()))):
        p.requires_grad_(bool(tr))
        p.grad = None
    ps = m(x)
    loss, items = compute_loss(ps, t.clone(), m, STEP_HYP)
    loss.backward()
    out = {"p%d" % k: p.detach().cpu() for k, p in enumerate(ps)}
    out["loss"], out["items"] = loss.detach().cpu(), items.detach().cpu()
    with torch.no_grad():
        for n, p in m.named_parameters():
            out["grad:" + n] = p.grad.cpu() if p.grad is not None else None
            if p.grad is not None:
                p.sub_(LR * p.grad)
            p.grad = None
        for n, p in m.named_parameters():
            out["param:" + n] = p.cpu()
        for n, bf in m.named_buffers():
            out["buf:" + n] = bf.cpu()
    del ps, loss, items
    return out


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t      # NaN payloads compared too


def _equal(got, want, what):
    assert got.keys() == want.keys()
    for k in want:
        if want[k] is None:
            assert got[k] is None, (what, k)
        else:
            assert torch.equal(_bits(got[k]), _bits(want[k])), (what, k)


def _run_sequence(make, seed, seq, graph, poison=False, mask_fn=None):
    cand, ref = pair(make, seed)
    cand.use_cuda_graph = ref.use_cuda_graph = graph
    mask = mask_fn(cand) if mask_fn else None
    seen = {}
    for k, (b, h, w) in enumerate(seq):
        x, t = images(b, h, w, k), _targets(b)
        key = (b, h, w, x.device)
        revisit = key in seen
        if poison:
            poison_pool(cand)
        torch.cuda.synchronize()
        m0, g0, pool0 = torch.cuda.memory_allocated(), grid_bytes(cand), _pool_bytes(cand)
        got = _train_step(cand, x, t, mask)
        torch.cuda.synchronize()
        if revisit:
            assert cand._tplan is seen[key], "a revisited shape built a new plan"
            assert torch.cuda.memory_allocated() - m0 == grid_bytes(cand) - g0, \
                "a revisited shape allocated device memory"
        if _pool_bytes(cand) != pool0:          # growth dropped every cached plan
            assert pool0 < _pool_bytes(cand) and list(cand._tplans.values()) == [cand._tplan]
            seen = {}
        seen[key] = cand._tplan
        assert sorted(map(id, cand._tplans.values())) == sorted(map(id, seen.values()))
        _fresh(ref)
        want = _train_step(ref, x, t, mask)
        _equal(got, want, (b, h, w))
    return cand


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("poison", [False, True])
@pytest.mark.parametrize("make", [_mini, yolov3_small], ids=["mini", "yolov3"])
def test_sequence_equals_fresh_plans(make, graph, poison):
    cand = _run_sequence(make, 11, SEQ, graph, poison)
    # the pool holds exactly the largest shape's requirement: what a fresh model needs for that shape alone
    one, _ = pair(make, 11)
    _train_step(one, images(4, 416, 416, 0), _targets(4))
    assert _pool_bytes(cand) == _pool_bytes(one)


@pytest.mark.parametrize("graph", [False, True])
def test_sequence_with_frozen_layers(graph):
    _run_sequence(yolov3_small, 12, SEQ, graph, mask_fn=transfer_mask)


@pytest.mark.parametrize("make", [_se, _m], ids=["se", "yolov3-m"])
def test_se_and_dilated_graphs_at_two_sizes(make):
    seq = [(2, 160, 192), (2, 128, 160), (2, 160, 192), (1, 128, 160)]
    _run_sequence(make, 13, seq, graph=False, poison=True)


def test_backward_after_a_forward_of_another_shape_raises():
    m, _ = pair(_mini, 14)
    pa = m(images(2, 96, 128, 0))
    pb = m(images(2, 64, 64, 1))
    with pytest.raises(RuntimeError):
        sum(p.sum() for p in pa).backward()
    sum(p.sum() for p in pb).backward()          # the latest forward's backward still runs


def test_peak_memory_of_a_size_sequence_is_that_of_its_largest_shape():
    fresh, _ = pair(yolov3_small, 15)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    _train_step(fresh, images(4, 416, 416, 0), _targets(4))
    peak_one = torch.cuda.max_memory_allocated() - base
    need = _pool_bytes(fresh)
    del fresh, _
    m, other = pair(yolov3_small, 15)
    del other
    gc.collect()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    for k, s in enumerate((416, 256, 416, 320)):
        _train_step(m, images(4, s, s, k), _targets(4))
    peak_seq = torch.cuda.max_memory_allocated() - base
    assert peak_seq <= 1.05 * peak_one, (peak_seq, peak_one)
    assert _pool_bytes(m) == need


def test_zero_halo_multi_vs_torch():
    """halo ring and channels [c_real, c_stride) zeroed, every other byte unchanged, on NaN-filled buffers"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import _lib
    # the last job has more units than one pass of the grid-stride loop (128 x 256 threads): ring and interior units
    # of one job are then split across passes
    jobs = [(2, 5, 7, 27, 64), (1, 3, 4, 0, 32), (3, 6, 2, 32, 32), (2, 4, 4, 18, 32), (1, 9, 11, 200, 256),
            (2, 100, 120, 37, 64)]
    bufs = []
    g = torch.Generator(device="cuda").manual_seed(3)
    for b, h, w, c, cs in jobs:
        t = torch.randint(-32768, 32767, (b, h + 2, w + 2, cs), dtype=torch.int16, device="cuda", generator=g)
        t[..., ::3] = -1                                      # 0xFFFF: NaN bit patterns among the random ones
        bufs.append(t)
    want = []
    for t, (b, h, w, c, cs) in zip(bufs, jobs):
        r = t.clone()
        r[:, 0], r[:, -1], r[:, :, 0], r[:, :, -1] = 0, 0, 0, 0
        r[..., c:] = 0
        want.append(r)
    table = (_lib.HaloJob * len(jobs))(*[_lib.HaloJob(t.data_ptr(), b, h, w, c, cs, 0)
                                         for t, (b, h, w, c, cs) in zip(bufs, jobs)])
    dev = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8).cuda()
    _lib.check(pkg._lib.lib.ryolo_zero_halo_multi(_lib.ptr(dev), len(jobs), _lib.stream_ptr(dev.device)), "zero_halo")
    torch.cuda.synchronize()
    for t, r in zip(bufs, want):
        assert torch.equal(t, r)
