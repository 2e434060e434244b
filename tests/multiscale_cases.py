"""TEST INFRASTRUCTURE: the models, inputs and the garbage-collecting fixture of the multi-scale tests
(test_multiscale_train_gpu.py, test_multiscale_eval_gpu.py).  A test module uses the fixture by importing `collect`."""
import gc

import pytest
import torch

import helpers
from builders import STEP_HYP
from helpers import SMALL_ANCHORS


@pytest.fixture(autouse=True)
def collect():
    """a model and its plans reference each other: collect the previous test's before this one allocates"""
    gc.collect()
    torch.cuda.empty_cache()
    yield
    gc.collect()


def yolov3_small():
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    return pkg.Darknet(cfgs.yolov3_cfg(classes=1, anchors=SMALL_ANCHORS, n_anchors=6), {"context_factor": 1.0},
                       arc="default")


def pair(make, seed):
    """two models with the same weights and buffers"""
    out = []
    for _ in range(2):
        m = make()
        helpers.init_darknet_weights(m, seed=seed)
        m.nc, m.hyp = 1, STEP_HYP
        out.append(m.cuda().train())
    return out


def images(b, h, w, k):
    return torch.rand(b, 3, h, w, generator=torch.Generator().manual_seed(100 + k)).cuda()


def poison_pool(m):
    """fill every pool of the model with NaN bytes and drop its owner"""
    for pool in m._pools.values():
        if pool.storage is not None:
            pool.storage.fill_(0xFF)          # NaN in bf16 and fp32
            pool.owner = None                 # the storage no longer holds any plan's invariants


def grid_bytes(m):
    """device bytes of the YOLO layers' grids, which create_grids re-makes at every change of shape (as before pools)"""
    seen = {}
    for yi in m.yolo_layers:
        for v in vars(m.module_list[yi]).values():
            if isinstance(v, torch.Tensor) and v.is_cuda:
                st = v.untyped_storage()
                seen[st.data_ptr()] = -(-st.nbytes() // 512) * 512
    return sum(seen.values())
