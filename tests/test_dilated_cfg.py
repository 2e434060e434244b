"""The reference's multi-branch dilated graphs on the CPU side (cfg/yolov3-m.cfg, cfg/HRSC/yolov3-m.cfg,
cfg/HRSC+/yolov3_512_matrix.cfg): Darknet builds the reference's module tree, state_dict keys and shapes
(tests/golden/darknet_m_golden.npz, make_golden_m.py), .weights files are byte-identical to the reference's
save_weights, the plans that have no kernel for these graphs refuse them, and the phase decomposition that the eval
plan runs the dilated convs through equals F.conv2d(dilation=...) in float64."""
import hashlib
import json
import re

import pytest
import torch
import torch.nn.functional as F

from builders import DILATIONS, golden_text, m_cfg_text, m_golden, m_model, phase_merge, phase_split
from helpers import init_darknet_weights

M_CFGS = ["cfg/yolov3-m.cfg", "cfg/HRSC/yolov3-m.cfg", "cfg/HRSC+/yolov3_512_matrix.cfg"]


@pytest.mark.parametrize("cfg", M_CFGS)
def test_darknet_builds_the_reference_module_tree(cfg):
    g = m_golden()
    m = m_model(cfg)
    assert repr(m.module_list) == golden_text(g, "tree:" + cfg)
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == json.loads(golden_text(g, "state:" + cfg))
    assert sum(p.numel() for p in m.parameters()) == int(g["n_params:" + cfg])
    assert len(m.yolo_layers) == 16 and all(m.module_list[i].na == 72 for i in m.yolo_layers)
    dconv = [i for i, d in enumerate(m.module_defs) if d["type"] == "d-convolutional"]
    assert len(dconv) == 36 and all(type(m.module_list[i].activation).__name__ == "LeakyReLU" for i in dconv)


def test_checkpoint_round_trip_with_the_reference_keys():
    a = init_darknet_weights(m_model(), seed=3)
    b = m_model()
    b.load_state_dict(a.state_dict())
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)


def test_weights_file_is_byte_identical_to_the_reference(tmp_path):
    from rotate_yolov3_b200.weights_io import load_darknet_weights, save_weights
    g = m_golden()
    m = init_darknet_weights(m_model(), seed=json.loads(golden_text(g, "seeds"))["eval_w"])
    path = str(tmp_path / "m.weights")
    save_weights(m, path)
    with open(path, "rb") as f:
        data = f.read()
    assert len(data) == int(g["weights_bytes"])
    assert hashlib.sha256(data).hexdigest() == golden_text(g, "weights_sha256")
    # the branch blocks' own (unused) conv / BN weights are in the file, like the reference's, and load back
    m2 = m_model()
    load_darknet_weights(m2, path)
    for (k, va), vb in zip(m.state_dict().items(), m2.state_dict().values()):
        if ".BatchNorm2d." in k or ".Conv2d." in k:
            i = int(k.split(".")[1])
            if m.module_defs[i]["type"] == "convolutional":
                assert torch.equal(va, vb), k


def _block(text, i, repl):
    """cfg text with the i-th [..] block's body replaced"""
    parts = re.split(r"(?m)^(?=\[)", text)
    parts[i + 1] = repl
    return "".join(parts)


def test_unsupported_shared_and_dilated_blocks_are_refused():
    import rotate_yolov3_b200 as pkg
    text = m_cfg_text("cfg/yolov3-m.cfg")
    hyp = {"context_factor": 1.0}
    no_owner = ("[d-convolutional]\ndilation=(1,2)\nbatch_normalize=1\nsize=3\nstride=1\npad=1\nfilters=1024\n"
                "activation=leaky\n\n")
    with pytest.raises(NotImplementedError, match="without weight_from"):
        pkg.Darknet(_block(text, 114, no_owner), hyp)
    # weight_from naming a route block (no Conv2d)
    bad = ("[convolutional]\nbatch_normalize=1\nfilters=512\nsize=1\nstride=1\npad=1\nactivation=leaky\n"
           "weight_from = 112\n\n")
    with pytest.raises(NotImplementedError, match="weight_from=112"):
        pkg.Darknet(_block(text, 113, bad), hyp)


def test_training_plan_gradient_slots_and_parity_refusal():
    """the training plan returns a gradient for exactly the parameters the reference's forward uses (golden
    *_has_grad), sums each shared weight's uses in its owner's slot, and runs the odd-grid stride-2 conv (block 108) on
    the zero-insertion path; parity precision refuses the graph"""
    from rotate_yolov3_b200.parity_path import ParityPlan
    from rotate_yolov3_b200.train_path import TrainPlan
    m = m_model()
    has = [bool(h) for h in m_golden()["default_has_grad"]]
    for h, w, grid in ((128, 160, (4, 5)), (416, 416, (13, 13)), (608, 608, (19, 19))):
        tp = TrainPlan(m, 2, h, w, torch.device("cpu"))
        got = [(int(n.split(".")[1]), ".".join(n.split(".")[2:])) in tp.param_slots for n in tp.names]
        assert got == has
        b108 = [b for b in tp.blocks if b.i == 108][0]
        assert (b108.src.h, b108.src.w) == grid and b108.stride == 2 and not b108.s2d
        assert (b108.oh, b108.ow) == (-(-grid[0] // 2), -(-grid[1] // 2))
        by = {b.i: b for b in tp.blocks}
        for b in tp.blocks:
            if b.owner is not None:
                assert b.dw is by[b.owner].dw and b.pw is by[b.owner].pw and b.pwd is by[b.owner].pwd
        # the DDP bucket bounds come from the owners' slots only: every bound is a block with gradients
        assert all(b.arena_end is None for b in tp.blocks if b.owner is not None)
    mp = m_model(precision="parity")
    for training in (True, False):
        with pytest.raises(NotImplementedError, match="weight_from"):
            ParityPlan(mp, 1, 64, 64, torch.device("cpu"), training)


@pytest.mark.parametrize("dil", DILATIONS)
def test_phase_decomposition_equals_the_dilated_conv_f64(dil):
    dh, dw = dil
    g = torch.Generator().manual_seed(dh * 10 + dw)
    wt = torch.randn(6, 5, 3, 3, generator=g, dtype=torch.float64)
    for n in (13, 19, 26, 38, 52, 76):
        for h, w in ((n, n), (n, n + 3)):
            x = torch.randn(2, 5, h, w, generator=g, dtype=torch.float64)
            want = F.conv2d(x, wt, padding=dil, dilation=dil)
            got = phase_merge(F.conv2d(phase_split(x, dh, dw), wt, padding=1), 2, h, w, dh, dw)
            assert torch.allclose(got, want, rtol=1e-12, atol=1e-12), (dil, h, w)


def test_dilate_entry_points_check_their_arguments():
    import rotate_yolov3_b200 as pkg
    lib = pkg._lib.lib
    assert lib.ryolo_dilate_split(None, 64, 1, 13, 13, 64, 1, 2, None, 64, None) == -1
    assert b"bad argument" in lib.ryolo_last_error()
    assert lib.ryolo_dilate_merge(None, 64, 1, 13, 13, 60, 1, 2, None, 0, 0, None, 64, None) == -1
