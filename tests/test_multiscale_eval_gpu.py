"""Eval at changing image sizes (detect.py --multi-scale alternates two sizes on every image) from one activation pool
per model and batch size: every forward of a cached eval plan gives the bits of a freshly built plan, io and the raw
heads, with CUDA graphs off and on and with the whole pool filled with NaN bytes before every call; a revisit with
unchanged weights builds no plan, packs no weight and allocates nothing; an in-place weight update between calls gives
the outputs of a fresh plan with the new weights."""
import pytest
import torch

from multiscale_cases import (collect, grid_bytes, images, pair, poison_pool, yolov3_small)  # noqa: F401 (collect: fixture)

pytestmark = pytest.mark.gpu


def _fresh(m):
    """drop every eval plan and the pools: the next call builds its plan in zeroed storage"""
    m._plan = None
    m._pools = {}


def _call(m, x):
    with torch.no_grad():
        io, ps = m(x)
        return io.cpu(), [p.cpu() for p in ps]


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("poison", [False, True])
def test_alternating_sizes_equal_fresh_plans(graph, poison, monkeypatch):
    from rotate_yolov3_b200 import layout as L
    cand, ref = pair(yolov3_small, 16)
    cand.eval(), ref.eval()
    cand.use_cuda_graph = ref.use_cuda_graph = graph
    packs = []
    real_pack = L.pack_weights
    monkeypatch.setattr(L, "pack_weights", lambda *a, **k: packs.append(1) or real_pack(*a, **k))
    sizes = [(1, 320, 320), (1, 256, 384)] * 3
    seen = {}
    for k, shape in enumerate(sizes + [None] + sizes[:4]):
        if shape is None:
            with torch.no_grad():          # an in-place weight update between calls (what an optimizer step does)
                for m in (cand, ref):
                    m.module_list[2].Conv2d.weight.mul_(0.5)
                    m.module_list[1].BatchNorm2d.running_var.add_(0.25)
            seen = {}
            continue
        b, h, w = shape
        x = images(b, h, w, k % 2)
        if poison:
            poison_pool(cand)
        torch.cuda.synchronize()
        m0, g0, n0 = torch.cuda.memory_allocated(), grid_bytes(cand), len(packs)
        io, ps = _call(cand, x)
        torch.cuda.synchronize()
        key = (b, h, w)
        if key in seen:
            assert cand._plan is seen[key], "a revisit built a new plan"
            assert len(packs) == n0, "a revisit with unchanged weights packed weights"
            assert torch.cuda.memory_allocated() - m0 == grid_bytes(cand) - g0, "a revisit allocated device memory"
        seen[key] = cand._plan
        _fresh(ref)
        io_r, ps_r = _call(ref, x)
        assert torch.equal(_bits(io), _bits(io_r)), (k, b, h, w)
        for p, q in zip(ps, ps_r):
            assert torch.equal(_bits(p), _bits(q)), (k, b, h, w)
