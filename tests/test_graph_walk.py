"""The graph walk the eval, training and parity-precision plans share (rotate-yolov3_b200/graph.py), checked on the CPU
against what the module tree states on its own: conv input channels, the blocks a conv's epilogue absorbs, concat
placement and the heads; and the refusals of each plan."""
import pytest
import torch

from builders import REF_CFGS, graph_model
from helpers import SMALL_ANCHORS, cfg_conv

CPU = torch.device("cpu")


@pytest.mark.parametrize("name", ["yolov3", "mini", "micro", "odd", "tiny_trunk"] + REF_CFGS)
def test_walk_matches_the_module_tree(name):
    from rotate_yolov3_b200 import graph as G
    m, h, w = graph_model(name)
    defs = m.module_defs
    g = G.Graph(m, h, w, ("se", "maxpool"), "block type %r")
    convs = [i for i, d in enumerate(defs) if d["type"] == "convolutional"]
    assert sorted(g.convs) == convs
    for i, cv in g.convs.items():
        assert cv.cin == m.module_list[i].Conv2d.weight.shape[1], i
    for j, d in enumerate(defs):
        if d["type"] in ("shortcut", "upsample"):
            by = [cv.i for cv in g.convs.values() if cv.mat == j and (cv.fuse_res if d["type"] == "shortcut" else cv.fuse_up)]
            assert by == [j - 1], (j, by)
    # wire every launch like a plan does, on meta tensors
    bufs = G.Buffers(g, lambda hh, ww, cs: (torch.empty((1, hh + 2, ww + 2, cs), device="meta"), None), 32)
    made = {}
    for t, i in g.ops:
        if t != "convolutional" or not g.convs[i].is_head:
            layer = g.convs[i].mat if t == "convolutional" else i
            assert layer not in made
            made[layer] = bufs.out(layer)[0]
    for i, d in enumerate(defs):
        if d["type"] == "route" and "," in d["layers"]:
            srcs = [int(x) for x in d["layers"].split(",")]
            srcs = [l if l > 0 else i + l for l in srcs]
            group, off = bufs.views[i], 0
            for l in srcs:
                assert l in made, (i, l)
                assert made[l].buf is group.buf and made[l].ch_off == off, (i, l)
                off += made[l].c
            assert off == group.c
    heads = [i for i, cv in g.convs.items() if cv.is_head]
    if m.yolo_layers:
        assert heads == [y - 1 for y in m.yolo_layers]
    else:
        assert heads and heads == [i for i in convs if not hasattr(m.module_list[i], "BatchNorm2d")
                                   and not hasattr(m.module_list[i], "activation")]


def test_odd_grid_stride2_runs_without_space_to_depth():
    from rotate_yolov3_b200.parity_path import ParityPlan
    from rotate_yolov3_b200.train_path import TrainPlan
    m, h, w = graph_model("odd")
    plan = TrainPlan(m, 1, h, w, CPU)
    odd = [b for b in plan.blocks if b.stride == 2 and b.src.h % 2]
    assert [b.i for b in odd] == [6] and not odd[0].s2d and odd[0].dz_up is not None
    assert all(b.s2d for b in plan.blocks if b.stride == 2 and b not in odd)
    for training in (True, False):
        with pytest.raises(NotImplementedError, match="even input sizes"):
            ParityPlan(m, 1, h, w, CPU, training)


def test_plans_refuse_what_they_cannot_run():
    from rotate_yolov3_b200 import graph as G
    from rotate_yolov3_b200.parity_path import ParityPlan
    from rotate_yolov3_b200.train_path import TrainPlan
    se, h, w = graph_model("cfg/HRSC+/yolov3_512_se.cfg")
    for training in (True, False):
        with pytest.raises(NotImplementedError, match="bf16"):
            ParityPlan(se, 1, h, w, CPU, training)
    tiny, h, w = graph_model("tiny_trunk")
    with pytest.raises(NotImplementedError, match="maxpool"):
        TrainPlan(tiny, 1, h, w, CPU)
    import rotate_yolov3_b200 as pkg
    cfg = "[net]\nwidth=32\nheight=32\nchannels=3\n\n" + cfg_conv(32, 3) + cfg_conv(32, 1) + "[route]\nlayers = -2\n\n"
    cfg += "[shortcut]\nfrom=-2\nactivation=linear\n\n" + cfg_conv(21, 1, bn=0, act="linear")
    cfg += "[yolo]\nmask = 0-2\nanchors = %s\nclasses=1\nnum=6\n\n" % SMALL_ANCHORS
    m = pkg.Darknet(cfg, {"context_factor": 1.0}, arc="default")
    with pytest.raises(NotImplementedError, match="shortcut at block 3 does not follow a convolution"):
        G.Graph(m, 32, 32, ("se", "maxpool"), "block type %r")
    with pytest.raises(NotImplementedError, match="shortcut at block 3"):
        TrainPlan(m, 1, 32, 32, CPU)
    with pytest.raises(NotImplementedError, match="shortcut at block 3"):
        ParityPlan(m, 1, 32, 32, CPU, True)


def test_training_refuses_heads_wider_than_the_head_gradient():
    """72 anchors per head: 22 classes give 2016-channel heads (trains), 23 give 2088 (refused at plan build, naming
    the limit, before any buffer or launch; eval still runs them, test_multiclass_f64_gpu.py)"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    from rotate_yolov3_b200.train_path import HEAD_GRAD_MAX_CHANNELS, TrainPlan
    assert HEAD_GRAD_MAX_CHANNELS == 2048
    for nc, ok in ((22, True), (23, False)):
        m = pkg.Darknet(cfgs.yolov3_cfg(width=64, height=64, classes=nc), {"context_factor": 1.0}, arc="default")
        if ok:
            plan = TrainPlan(m, 1, 64, 64, CPU)
            assert [b.cout for b in plan.blocks if b.is_head] == [2016] * 3
        else:
            with pytest.raises(NotImplementedError, match=r"limited to 2048 channels.*\(81, 2088\), \(93, 2088\)"):
                TrainPlan(m, 1, 64, 64, CPU)
