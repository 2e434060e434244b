"""CPU checks of the drop-in boundary: the C-ABI library loads without a GPU and exports every symbol
include/ryolo.h declares; argument errors come back as status codes, never as exceptions across the ABI."""
import ctypes
import os
import re

import pytest

from helpers import REPO


def _declared():
    src = open(os.path.join(REPO, "include", "ryolo.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ryolo_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported_abi_v2():
    import rotate_yolov3_b200 as pkg
    names = _declared()
    assert len(names) >= 10
    for n in names:
        assert hasattr(pkg._lib.lib, n), "libryolo.so does not export %s" % n
        assert n in pkg._lib.SIGNATURES, "ctypes binding missing for %s" % n
    assert set(pkg._lib.SIGNATURES) == set(names)
    assert pkg._lib.lib.ryolo_abi_version() == 2


def test_workspace_queries_need_no_gpu():
    import rotate_yolov3_b200 as pkg
    lib = pkg._lib.lib
    assert lib.ryolo_rnms_workspace_bytes(0) > 0
    w1, w2 = lib.ryolo_rnms_workspace_bytes(1000), lib.ryolo_rnms_workspace_bytes(20000)
    assert w2 > w1 > 1000 * 6 * 4
    assert w2 >= 20000 * 313 * 8  # the suppression mask dominates
    assert lib.ryolo_nms_filter_workspace_bytes(545832) >= (545832 // 256) * 4


def test_bad_arguments_return_status():
    import rotate_yolov3_b200 as pkg
    lib = pkg._lib.lib
    st = lib.ryolo_riou_paired(None, None, 4, 2, 5, 0, None, None)   # stride < 5
    assert st == -1 and b"bad argument" in lib.ryolo_last_error()
    st = lib.ryolo_riou_pairwise(None, 4, 5, None, 4, 5, 7, None, None)  # unknown mode
    assert st == -1
    st = lib.ryolo_rnms(None, -1, 0.5, None, None, None, 0, None)
    assert st == -1


def test_python_boundary_matches_reference_errors():
    """r_nms on a CPU tensor raises RuntimeError like CHECK_CUDA (rotate_polygon_nms.cpp:3,8); an empty CUDA-less
    call path is not reachable without a device, so only the type check is exercised here."""
    import torch
    import rotate_yolov3_b200 as pkg
    with pytest.raises(RuntimeError):
        pkg.r_nms(torch.zeros(4, 6), 0.5)
    with pytest.raises(RuntimeError):
        pkg.r_nms([[0, 0, 1, 1, 0, 1]], 0.5)


def test_no_oracle_in_product():
    """The product must never route through oracle/ (or any CPU fallback)."""
    pkg_dir = os.path.join(REPO, "rotate-yolov3_b200")
    for root, _, files in os.walk(pkg_dir):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(root, f), errors="ignore").read()
                assert "librbox_oracle" not in txt and "oracle/_ref" not in txt.replace("oracle/_ref (", ""), f


def test_no_environment_knobs():
    """Nothing the library or the package computes depends on the environment: no getenv in the CUDA sources, and the
    only environment read in the package is the build's NVCC lookup."""
    pkg_dir = os.path.join(REPO, "rotate-yolov3_b200")
    for root, _, files in os.walk(os.path.join(pkg_dir, "csrc")):
        for f in files:
            assert "getenv(" not in open(os.path.join(root, f), errors="ignore").read(), f
    for root, _, files in os.walk(pkg_dir):
        for f in files:
            if f.endswith(".py"):
                txt = open(os.path.join(root, f)).read()
                if f == "build.py":
                    txt = txt.replace('os.environ.get("NVCC")', "", 1)
                assert not re.search(r"os\.environ|os\.getenv", txt), f
