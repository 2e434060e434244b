"""The matched-row scatter of the loss backward (ryolo_loss_rows_scatter_add, csrc/loss.cu), bit for bit.

Contract: for every cell hit by at least one live row (mask set, indices inside the map), channel k of the head cotangent
becomes the chain fmaf(vals[jn, k], scale, ... fmaf(vals[j1, k], scale, g[cell, k])) over that cell's live rows
j1 < ... < jn; every other element keeps its value.  The reference here restates that chain on the host with exact
rational arithmetic and one round-to-nearest-even to fp32 per fmaf, so the device result must match it in every bit.

Inputs: the real assignment mask of the batch-64 training step (bench.make_targets(64, 100) through
_targets_masked_stacked, three heads of 72 anchors), and synthetic row sets that stress the walk: every row live, every
row on one cell, live rows only at the first and the last row, the rows of one cell spread far apart, rows outside the
map, more channels than a warp has lanes.  Each case also runs three times, the last next to a second stream of matmuls,
and must give the same bits every time."""
import ctypes
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from builders import repeat

pytestmark = pytest.mark.gpu


def _round_f32(x):
    """the fp32 nearest to the rational x, ties to even (x != 0)"""
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1                                    # 2^e <= a < 2^(e + 1)
    q = Fraction(2) ** (max(e, -126) - 23)        # spacing of the fp32 values around a (subnormals below 2^-126)
    r = float(round(a / q) * q)                   # round() of a Fraction rounds half to even
    return -r if x < 0 else r


def _fmaf(a, b, c):
    """fmaf(a, b, c) of fp32 values given as Python floats: a * b + c rounded once"""
    exact = Fraction(a) * Fraction(b) + Fraction(c)
    if exact == 0:
        p_neg = (math.copysign(1.0, a) * math.copysign(1.0, b)) < 0
        if (a == 0 or b == 0) and c == 0 and p_neg and math.copysign(1.0, c) < 0:
            return -0.0
        return 0.0
    return _round_f32(exact)


def _nchw_head(B, na, ny, nx, no, gen, dense_channel=None):
    """a head cotangent stored as the NCHW [B, na*no, ny, nx] buffer the head convolution uses, and its
    [B, na, ny, nx, no] view.  dense_channel: only that channel is non-zero (what obj_bce_bwd leaves), else all random"""
    v = torch.randn(B, na, ny, nx, no, generator=gen)
    if dense_channel is not None:
        keep = torch.zeros(no)
        keep[dense_channel] = 1.0
        v = v * keep
    base = v.permute(0, 1, 4, 2, 3).contiguous().view(B, na * no, ny, nx).cuda()
    return base, base.view(B, na, no, ny, nx).permute(0, 1, 3, 4, 2)


def _scatter(base0, shape, idx, mask, vals, scale):
    from rotate_yolov3_b200 import _lib as L
    B, na, ny, nx, no = shape
    base = base0.clone()
    g = base.view(B, na, no, ny, nx).permute(0, 1, 3, 4, 2)
    strides = (ctypes.c_longlong * 5)(*g.stride())
    cols = [idx[:, k].contiguous().cuda() for k in range(4)]
    m8 = mask.to(torch.uint8).cuda()
    L.check(L.lib.ryolo_loss_rows_scatter_add(L.ptr(g), strides, B, na, ny, nx, no, *[L.ptr(c) for c in cols], L.ptr(m8),
                                              int(idx.shape[0]), L.ptr(vals), L.ptr(scale), L.stream_ptr()), "scatter")
    return (base,)


def _expected(base0, shape, idx, mask, vals, scale):
    """base0 with every hit cell replaced by its row-order fmaf chain"""
    B, na, ny, nx, no = shape
    idx_n = idx.numpy()
    live = mask.numpy().astype(bool) & (idx_n[:, 0] >= 0) & (idx_n[:, 0] < B) & (idx_n[:, 1] >= 0) & (idx_n[:, 1] < na) \
        & (idx_n[:, 2] >= 0) & (idx_n[:, 2] < ny) & (idx_n[:, 3] >= 0) & (idx_n[:, 3] < nx)
    rows = np.nonzero(live)[0]
    exp = base0.clone()
    if len(rows) == 0:
        return exp, 0, 0
    view = exp.view(B, na, no, ny, nx).permute(0, 1, 3, 4, 2)
    cells = {}
    for j in rows:                                       # increasing row order
        cells.setdefault(tuple(int(v) for v in idx_n[j]), []).append(j)
    keys = list(cells)
    ci = torch.tensor(keys, dtype=torch.long)
    start = view[ci[:, 0], ci[:, 1], ci[:, 2], ci[:, 3]].cpu().double().numpy()        # [cells, no]
    v = vals.cpu().double().numpy()
    s = float(scale.cpu()[0])
    out = np.empty_like(start)
    for n, key in enumerate(keys):
        for k in range(no):
            acc = float(start[n, k])
            for j in cells[key]:
                acc = _fmaf(float(v[j, k]), s, acc)
            out[n, k] = acc
    view[ci[:, 0], ci[:, 1], ci[:, 2], ci[:, 3]] = torch.from_numpy(out).float().cuda()
    return exp, len(rows), max(len(r) for r in cells.values())


def _check(shape, idx, mask, vals, scale, gen, dense_channel=None):
    base0, _ = _nchw_head(*shape, gen, dense_channel)
    (got,) = repeat(lambda: _scatter(base0, shape, idx, mask, vals, scale))
    exp, live, most = _expected(base0, shape, idx, mask, vals, scale)
    assert torch.equal(got.view(torch.int32), exp.view(torch.int32))
    return live, most


def _random_cells(shape, n, gen):
    B, na, ny, nx, _ = shape
    return torch.stack([torch.randint(0, s, (n,), generator=gen) for s in (B, na, ny, nx)], 1)


SHAPE = (2, 3, 10, 12, 7)


def _vals(n, no, gen):
    return torch.randn(n, no, generator=gen).cuda()


def test_scatter_bench_assignment_bitwise():
    """the rows, mask and head shapes of the batch-64 training step"""
    import bench
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    from rotate_yolov3_b200.loss import _targets_masked_stacked
    net = pkg.Darknet(cfgs.yolov3_cfg(), dict(bench.TRAIN_HYP), arc="default")
    net.nc, net.hyp = 1, dict(bench.TRAIN_HYP)
    sizes = []
    for li in net.yolo_layers:
        layer = net.module_list[li]
        n = 608 // {0: 32, 1: 16, 2: 8}[len(sizes)]
        layer.create_grids((608, 608), (n, n), "cpu")
        sizes.append((layer.na, n))
    r = _targets_masked_stacked(net, bench.make_targets(64, 100), net.hyp)
    gen = torch.Generator().manual_seed(21)
    scale = torch.tensor([20.35 / (64 * 72 * 76 * 76)], device="cuda")
    assert r["R"] == 72 * 192
    for i, (na, n) in enumerate(sizes):
        shape = (64, na, n, n, 7)
        idx = torch.stack([r[k][i] for k in ("b", "a", "gj", "gi")], 1).cpu()
        mask = r["mask"][i].cpu()
        live, most = _check(shape, idx, mask, _vals(r["R"], 7, gen), scale, gen, dense_channel=5)
        assert live > 0, i


@pytest.mark.parametrize("case", ["all_live", "one_cell", "first_and_last", "far_apart", "out_of_range", "wide"])
def test_scatter_synthetic_bitwise(case):
    gen = torch.Generator().manual_seed(["all_live", "one_cell", "first_and_last", "far_apart", "out_of_range",
                                         "wide"].index(case) + 30)
    shape = SHAPE if case != "wide" else (2, 3, 10, 12, 40)
    R = 5000
    idx = _random_cells(shape, R, gen)
    mask = torch.ones(R, dtype=torch.bool)
    if case == "all_live":
        idx = _random_cells(shape, 64, gen)[torch.randint(0, 64, (R,), generator=gen)]    # ~80 rows per cell
    elif case == "one_cell":
        idx[:] = idx[0]
    elif case == "first_and_last":
        mask[:] = False
        mask[0] = mask[R - 1] = True
        idx[R - 1] = idx[0]
    elif case == "far_apart":
        mask[torch.randperm(R, generator=gen)[:R // 2]] = False
        mask[7] = True
        for j in (1, 999, R // 2, R - 2):
            idx[j], mask[j] = idx[7], True
    elif case == "out_of_range":
        idx = _random_cells(shape, 40, gen)[torch.randint(0, 40, (R,), generator=gen)]
        bad = torch.randperm(R, generator=gen)[:R // 5]
        B, na, ny, nx, _ = shape
        idx[bad[0::6], 3] = nx
        idx[bad[1::6], 2] = -1
        idx[bad[2::6], 0] = B
        idx[bad[3::6], 1] = na
        idx[bad[4::6], 3] = -5
        idx[bad[5::6], 2] = ny
        mask[torch.randperm(R, generator=gen)[:R // 7]] = False
    elif case == "wide":          # 40 channels: two passes of the warp over the keys
        idx = _random_cells(shape, 100, gen)[torch.randint(0, 100, (R,), generator=gen)]
    scale = torch.tensor([0.37], device="cuda")
    live, most = _check(shape, idx, mask, _vals(R, shape[4], gen), scale, gen)
    want_live = {"first_and_last": 2, "one_cell": R, "all_live": R}
    if case in want_live:
        assert live == want_live[case]
    if case == "far_apart":
        assert most >= 5
