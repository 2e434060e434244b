"""The reference's squeeze-excitation graphs on the CPU side: cfg/HRSC+/yolov3_512_se.cfg and cfg/ICDAR/yolov3_608_se.cfg
parse like the reference parser (tests/golden/darknet_se_golden.npz, make_golden_se.py), Darknet builds the reference's
module tree and state_dict names, and parity precision refuses [se] blocks (SE runs in bf16 only)."""
import contextlib
import json
import os

import numpy as np
import pytest
import torch

from builders import se_golden
from helpers import GOLDEN

REF = os.path.join(GOLDEN, "reference_cfg")
SE_CFGS = ["cfg/HRSC+/yolov3_512_se.cfg", "cfg/ICDAR/yolov3_608_se.cfg"]
SE_BLOCKS = list(range(13, 42, 4)) + list(range(46, 75, 4)) + [79, 83, 87, 91]


@contextlib.contextmanager
def in_reference_layout():
    """the cfgs name their k-means anchor files relative to the reference root"""
    cwd = os.getcwd()
    os.chdir(REF)
    try:
        yield
    finally:
        os.chdir(cwd)


@pytest.mark.parametrize("cfg", SE_CFGS)
def test_se_cfgs_parse_like_the_reference(cfg):
    from rotate_yolov3_b200.parse_config import parse_model_cfg
    with in_reference_layout():
        ours = parse_model_cfg(cfg)
    want = json.loads(se_golden()["parse:" + cfg].item().decode())
    assert len(ours) == len(want) == 128
    for i, (a, b) in enumerate(zip(ours, want)):
        assert set(a) == set(b), (i, set(a) ^ set(b))
        for k in b:
            if k == "anchors":
                assert np.array_equal(np.asarray(a[k], dtype=np.float64), np.asarray(b[k], dtype=np.float64)), (i, k)
            else:
                assert a[k] == b[k], (i, k, a[k], b[k])
    blocks = ours[1:]
    assert [i for i, b in enumerate(blocks) if b["type"] == "se"] == SE_BLOCKS
    assert [i for i, b in enumerate(blocks) if b["type"] == "yolo"] == [102, 114, 126]
    # every shortcut after an SE skips it: `from=-4` reads the SE's input
    for i in SE_BLOCKS:
        assert blocks[i + 3]["type"] == "shortcut" and int(blocks[i + 3]["from"]) == -4
    assert blocks[106]["layers"].replace(" ", "") == "-1,61" and blocks[118]["layers"].replace(" ", "") == "-1,36"


@pytest.mark.parametrize("cfg", SE_CFGS)
def test_darknet_builds_the_reference_module_tree(cfg):
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200.models import SELayer
    with in_reference_layout():
        m = pkg.Darknet(cfg, {"context_factor": 1.0}, arc="default")
    g = se_golden()
    assert list(m.state_dict().keys()) == [str(n) for n in g["state_names"]]
    assert sum(p.numel() for p in m.parameters()) == int(g["n_params"])
    se = [i for i, mod in enumerate(m.module_list) if isinstance(mod, SELayer)]
    assert se == SE_BLOCKS
    for i in se:
        c = int(m.module_defs[i]["channels"])
        assert tuple(m.module_list[i].fc[0].weight.shape) == (c // 16, c)
        assert tuple(m.module_list[i].fc[2].weight.shape) == (c, c // 16)
    assert "module_list.13.fc.0.weight" in m.state_dict() and "module_list.91.fc.2.weight" in m.state_dict()
    # the SE inputs are all routed (shortcut `from=-4`; blocks 36 and 61 also by the concat routes)
    assert all((i - 1) in m.routes for i in se) and {36, 61} <= set(m.routes)


def test_parity_precision_refuses_se_blocks():
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200.parity_path import ParityPlan
    with in_reference_layout():
        m = pkg.Darknet(SE_CFGS[0], {"context_factor": 1.0}, arc="default", precision="parity")
    for training in (True, False):
        with pytest.raises(NotImplementedError, match="bf16"):
            ParityPlan(m, 1, 64, 64, torch.device("cpu"), training)


def test_se_workspace_query_needs_no_gpu():
    import rotate_yolov3_b200 as pkg
    lib = pkg._lib.lib
    small, big = lib.ryolo_se_workspace_bytes(1, 19, 19, 1024, 64), lib.ryolo_se_workspace_bytes(64, 76, 76, 256, 16)
    assert big > small >= 4 * (2 * 1024 + 64)
    assert lib.ryolo_se_workspace_bytes(0, 76, 76, 256, 16) == 0
    st = lib.ryolo_se_fwd(None, 256, None, 256, 2, 8, 8, 256, None, None, 16, None, None, None, None, 0, None)
    assert st == -1 and b"bad argument" in lib.ryolo_last_error()
